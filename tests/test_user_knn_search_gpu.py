"""
User-kNN neighbour search on the device (``lk_uknn_search``) against SciPy's ``user_vectors @ x`` with the
reference's self-exclusion and ``>= min_sim`` mask (user.py:189-214), compared on neighbour indices and
f32 similarity bits; and the UserKNNScorer component, whose neighbour lists now come from the device,
against SciPy neighbours fed to the same device aggregation.
"""

import pickle

import numpy as np
import pytest
import torch

from lkpy_b200 import _lib, data, engine
from lkpy_b200.components import Dataset, ItemList, RecQuery
from lkpy_b200.knn_user import UserKNNConfig, UserKNNScorer

pytestmark = pytest.mark.gpu

DEFAULT_MIN_SIM = UserKNNConfig().min_sim  # 1e-6
SMALLEST = float(np.finfo(np.float64).smallest_normal)


def ref_neighbours(V, x: np.ndarray, self_: int, min_sim: float):
    sims = V @ x
    if self_ >= 0:
        sims[self_] = 0
    mask = sims >= min_sim
    return np.flatnonzero(mask).astype(np.int32), sims[mask].astype(np.float32)


def check_csr(indptr, rows, sims, refs):
    indptr, rows, sims = indptr.cpu().numpy(), rows.cpu().numpy(), sims.cpu().numpy()
    assert len(indptr) == len(refs) + 1 and indptr[0] == 0 and len(rows) == indptr[-1] == len(sims)
    for q, (r_rows, r_sims) in enumerate(refs):
        lo, hi = indptr[q], indptr[q + 1]
        assert np.array_equal(rows[lo:hi], r_rows), f"query {q}: neighbour set differs"
        assert np.array_equal(sims[lo:hi].view(np.int32), r_sims.view(np.int32)), f"query {q}: similarity bits differ"
    return int(indptr[-1])


def dense_row(V, u):
    return V[[int(u)], :].toarray()[0]


@pytest.fixture(scope="module", params=["explicit", "implicit"])
def trained(request, ml_small):
    m = UserKNNScorer(feedback=request.param)
    m.train(Dataset(ml_small))
    return m


@pytest.fixture(scope="module")
def state(trained, cuda_lib):
    return engine.UserNeighbourState.create(trained.user_vectors, _lib.require_device())


def test_all_known_users_one_batch(trained, state):
    V = trained.user_vectors
    users = np.arange(V.shape[0])
    indptr, rows, sims = state.neighbours(state.known_queries(users), DEFAULT_MIN_SIM)
    nnz = check_csr(indptr, rows, sims, [ref_neighbours(V, dense_row(V, u), int(u), DEFAULT_MIN_SIM) for u in users])
    assert nnz > 50_000


@pytest.mark.parametrize("which", ["clamp", "0.1", "equal", "f64_vs_f32"])
def test_min_sim_values(trained, state, which):
    V = trained.user_vectors
    users = np.arange(0, V.shape[0], 3)
    sims0 = V @ dense_row(V, users[1])
    sims0[users[1]] = 0
    pos = np.sort(sims0[sims0 > 0.02])
    if which == "clamp":
        min_sim = SMALLEST
    elif which == "0.1":
        min_sim = 0.1
    elif which == "equal":  # inclusive: a neighbour whose sim equals min_sim exactly is kept
        min_sim = float(pos[len(pos) // 2])
    else:  # a sim just above min_sim in f64 whose f32 cast lies below it: kept
        s = next(float(v) for v in pos if float(np.float32(v)) < v)
        min_sim = (float(np.float32(s)) + s) / 2
        assert float(np.float32(s)) < min_sim <= s
    indptr, rows, sims = state.neighbours(state.known_queries(users), min_sim)
    refs = [ref_neighbours(V, dense_row(V, u), int(u), min_sim) for u in users]
    check_csr(indptr, rows, sims, refs)
    if which == "equal":
        assert min_sim in V @ dense_row(V, users[1])
    if which == "f64_vs_f32":
        s1 = sims.cpu().numpy()[int(indptr[1]) : int(indptr[2])]
        assert (s1.astype(np.float64) < min_sim).any()  # kept on the f64 comparison although its f32 weight is smaller


def test_provided_histories(trained, state, ml_small):
    V = trained.user_vectors
    explicit = trained.config.explicit
    n_items = V.shape[1]
    rng = np.random.default_rng(9)
    cases = []  # (item numbers with -1 for unknown ids, ratings, self)
    nums = rng.choice(n_items, 40, replace=False).astype(np.int32)
    cases.append((np.concatenate([nums, nums[:5]]), None, -1))  # duplicates: the last value wins
    cases.append((np.concatenate([nums[:10], [-1, -1]]), None, -1))  # unknown items
    cases.append((np.array([-1, -1, -1], np.int32), None, -1))  # nothing known
    cases.append((np.zeros(0, np.int32), None, -1))  # empty
    u = 17
    lo, hi = np.searchsorted(ml_small.users, [u, u + 1])
    cases.append((ml_small.items[lo:hi].astype(np.int32), ml_small.ratings[lo:hi], u))  # known user + its history
    specs, refs = [], []
    for nums, r, self_ in cases:
        if r is None:
            r = (rng.integers(1, 11, len(nums)) * 0.5).astype(np.float32)
        items, vals, _ = engine.history_query(nums, r if explicit and len(r) else None)
        dense = np.zeros(n_items, dtype=np.float32)
        mask = nums >= 0
        if explicit and len(r):
            dense[nums[mask]] = r[mask] - float(r.mean())
        else:
            dense[nums[mask]] = 1.0
        specs.append((items, vals, None if self_ < 0 else self_))
        refs.append(ref_neighbours(V, dense, self_, DEFAULT_MIN_SIM))
    # mixed with known-user rows (gathered from V on the device)
    specs.insert(2, 5)
    refs.insert(2, ref_neighbours(V, dense_row(V, 5), 5, DEFAULT_MIN_SIM))
    specs.append(600)
    refs.append(ref_neighbours(V, dense_row(V, 600), 600, DEFAULT_MIN_SIM))
    indptr, rows, sims = state.neighbours(state.queries(specs), DEFAULT_MIN_SIM)
    check_csr(indptr, rows, sims, refs)
    counts = np.diff(indptr.cpu().numpy())
    assert counts[0] > 0 and counts[3] == 0 and counts[4] == 0  # all-unknown and empty: no neighbours
    assert counts[5] > 0 and u not in rows.cpu().numpy()[indptr[5] : indptr[6]]  # known user + history: self excluded


def test_synthetic_multi_tile(cuda_lib):
    inter = data.synth_interactions(60_000, 3_000, 1_500_000, seed=3)
    m = UserKNNScorer()
    m.train(Dataset(inter))
    V = m.user_vectors
    st = engine.UserNeighbourState.create(V, _lib.require_device())
    g = st.geom
    tile = g.warps * g.tile_cols
    assert g.n_halves >= 3 and V.shape[0] % tile != 0
    rng = np.random.default_rng(1)
    counts = np.diff(V.indptr)
    users = np.concatenate([np.argsort(-counts)[:8], rng.choice(V.shape[0], 56, replace=False)])
    indptr, rows, sims = st.neighbours(st.known_queries(users), DEFAULT_MIN_SIM)
    refs = [ref_neighbours(V, dense_row(V, u), int(u), DEFAULT_MIN_SIM) for u in users]
    check_csr(indptr, rows, sims, refs)
    last_tile = rows.cpu().numpy() >= (g.n_halves - 1) * tile
    assert last_tile.any()  # neighbours found in the partial last tile too


def test_empty_and_neighbourless_batches(trained, state):
    indptr, rows, sims = state.neighbours(state.known_queries([]), DEFAULT_MIN_SIM)
    assert indptr.cpu().tolist() == [0] and rows.numel() == 0 and sims.numel() == 0
    # unit vectors: no cosine reaches 2
    indptr, rows, _ = state.neighbours(state.known_queries([0, 1, 2]), 2.0)
    assert indptr.cpu().tolist() == [0, 0, 0, 0] and rows.numel() == 0
    none = (np.zeros(0, np.int32), np.zeros(0), None)
    indptr, rows, _ = state.neighbours(state.queries([none, none]), DEFAULT_MIN_SIM)
    assert indptr.cpu().tolist() == [0, 0, 0] and rows.numel() == 0


def test_pool_overflow_is_reported(trained, state):
    V = trained.user_vectors
    qs = state.known_queries([0, 1, 2, 3])
    with pytest.raises(_lib.EngineError, match="overflow"):
        state.neighbours(qs, DEFAULT_MIN_SIM, capacity=3)
    # the state stays usable: the status word is reset by the next search
    indptr, rows, sims = state.neighbours(qs, DEFAULT_MIN_SIM)
    check_csr(indptr, rows, sims, [ref_neighbours(V, dense_row(V, u), u, DEFAULT_MIN_SIM) for u in range(4)])


def _scipy_path_scores(m: UserKNNScorer, queries, targets):
    """The component's result with SciPy neighbours (the host path it replaced) fed to the same device
    aggregation: a restatement of user.py:189-255."""
    st = m._device_state()
    dev = st.sim_cols.device
    V = m.user_vectors
    r_ptr, t_ptr, nbrs, sims, tgts, metas = [0], [0], [], [], [], []
    for q, items in zip(queries, targets):
        q = RecQuery.create(q)
        nb = None
        if len(items) > 0:
            index = m.users.number(q.user_id, missing=None) if q.user_id is not None else None
            x, umean = None, 0.0
            if q.query_items is None:
                if index is not None:
                    x = dense_row(V, index)
                    umean = float(m.user_means[index]) if m.config.explicit else 0.0
            elif len(q.query_items) > 0:
                x = np.zeros(len(m.items), dtype=np.float32)
                nos = q.query_items.numbers(vocabulary=m.items, missing="negative")
                ok = nos >= 0
                if m.config.explicit:
                    urv = np.require(q.query_items.field("rating"), dtype=np.float32)
                    umean = float(urv.mean())
                    x[nos[ok]] = urv[ok] - umean
                else:
                    x[nos[ok]] = 1.0
            if x is not None:
                rr, ss = ref_neighbours(V, x, -1 if index is None else int(index), m.config.min_sim)
                if len(rr):
                    nb = (rr, ss, umean)
        iidx = items.numbers(vocabulary=m.items, missing="negative").astype(np.int32)
        if nb is None:
            metas.append(None)
            r_ptr.append(r_ptr[-1])
            t_ptr.append(t_ptr[-1])
            continue
        ki = iidx >= 0
        nbrs.append(nb[0])
        sims.append(nb[1])
        tgts.append(iidx[ki])
        metas.append((ki, nb[2]))
        r_ptr.append(r_ptr[-1] + len(nb[0]))
        t_ptr.append(t_ptr[-1] + int(ki.sum()))
    t = lambda a, dt: torch.from_numpy(np.asarray(a, dtype=dt)).to(dev)  # noqa: E731
    sc, _ = st.score(
        t(r_ptr, np.int64), t(np.concatenate(nbrs), np.int32), t(np.concatenate(sims), np.float32),
        t(t_ptr, np.int64), t(np.concatenate(tgts), np.int32), m.config.max_nbrs, m.config.min_nbrs,
    )  # fmt: skip
    sc = sc.cpu().numpy()
    out = []
    for i, items in enumerate(targets):
        full = np.full(len(items), np.nan, dtype=np.float32)
        if metas[i] is not None:
            ki, umean = metas[i]
            full[ki] = sc[t_ptr[i] : t_ptr[i + 1]] + np.float32(umean)
        out.append(full)
    return out


def _same_bits(a: np.ndarray, b: np.ndarray) -> bool:
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.int32), b[~np.isnan(b)].view(np.int32))


@pytest.mark.parametrize("explicit", [True, False])
def test_component_matches_scipy_neighbours(cuda_lib, ml_small, explicit):
    m = UserKNNScorer(feedback="explicit" if explicit else "implicit", max_nbrs=12, min_nbrs=2)
    ds = Dataset(ml_small)
    m.train(ds)
    rng = np.random.default_rng(8)
    items = ItemList(item_nums=rng.choice(ml_small.n_items, 300, replace=False).astype(np.int32), vocabulary=ds.items)
    with_unknown = ItemList(item_ids=np.concatenate([items.ids()[:50], [-7, -8]]))
    hist = ds.user_history(40)
    dup_hist = ItemList(
        item_ids=np.concatenate([hist.ids(), hist.ids()[:3], [-99]]),
        rating=np.concatenate([hist.field("rating"), np.float32([1.0, 5.0, 2.5, 4.0])]),
    )
    queries = [ds.users.id(int(u)) for u in rng.choice(ml_small.n_users, 10, replace=False)]
    queries += [
        RecQuery(user_id=None, query_items=hist),  # history, no known user
        RecQuery(user_id=ds.users.id(40), query_items=dup_hist),  # known user + history with duplicates
        RecQuery(user_id="nobody"),  # unknown user
        RecQuery(user_id=None, query_items=ItemList(item_ids=np.array([-1, -2]), rating=np.float32([3, 4]))),
        ds.users.id(3),
    ]
    targets = [items] * len(queries)
    targets[1] = with_unknown
    targets[4] = ItemList(item_ids=np.zeros(0, dtype=items.ids().dtype))  # empty target list: no search
    got = m.score_batch(queries, targets)
    want = _scipy_path_scores(m, queries, targets)
    for g, w in zip(got, want):
        assert _same_bits(np.asarray(g.scores(), dtype=np.float32), w)
    assert np.isnan(got[12].scores()).all() and np.isnan(got[13].scores()).all()
    assert np.isfinite(got[0].scores()).any()
    one = m(queries[2], items)
    assert _same_bits(one.scores(), got[2].scores())

    clone = pickle.loads(pickle.dumps(m))
    assert "_nbr_state" not in clone.__dict__ and "_state" not in clone.__dict__
    again = clone.score_batch(queries, targets)
    for g, a in zip(got, again):
        assert _same_bits(np.asarray(g.scores(), dtype=np.float32), np.asarray(a.scores(), dtype=np.float32))
