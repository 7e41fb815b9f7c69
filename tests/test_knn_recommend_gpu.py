"""
Batched top-n recommendation from the kNN scorers (``lk_knn_recommend_batch``, the ranking mode of the dense
scoring kernel) against the reference's per-query composition, bit for bit:

    cands = all item numbers ascending, minus the query's items when exclude == "query"
    il    = scorer(query, ItemList(item_nums=cands))
    top   = il[argtopn(il.scores, n)]

with the scores from the oracle's ScoreAccumulator emulation (item mode) or the scorer's own ``score_batch``
(user mode, pinned against the oracle elsewhere), the f32 offset, and ``oracle.argtopn``.
"""

import pickle

import numpy as np
import pytest
import scipy.sparse as sps
import torch

import oracle
from lkpy_b200 import _lib, data, engine
from lkpy_b200.components import Dataset, ItemList, RecQuery
from lkpy_b200.knn import ItemKNNScorer
from lkpy_b200.knn_user import UserKNNScorer

pytestmark = pytest.mark.gpu

DENSE_ACTIVE_CAP = 8192  # touched targets a CTA keeps in shared memory (knn_score.cu)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_lib.require_device())


def expected_item(S, means, ri, rv, max_nbrs, min_nbrs, n, exclude):
    """(items, score bits, nbr_counts) of the host composition for one item-kNN query (engine-level history)."""
    n_items = S.shape[0]
    cands = np.arange(n_items, dtype=np.int32)
    if exclude:
        cands = np.setdiff1d(cands, ri[ri >= 0]).astype(np.int32)
    sc, ct = oracle.knn_score(S, ri, rv, cands, max_nbrs, min_nbrs)
    if means is not None:
        sc = sc + means[cands]  # f32 + f32, as ItemKNNScorer.score_batch
    top = oracle.argtopn(sc, n)
    return cands[top], sc[top], ct[top]


def check_rows(idx, val, nbrs, cnt, q, want_items, want_vals, want_nbrs, n):
    c = int(cnt[q])
    assert c == len(want_items), q
    assert np.array_equal(idx[q, :c], want_items), q
    assert np.array_equal(val[q, :c].view(np.int32), want_vals.astype(np.float32).view(np.int32)), q
    if want_nbrs is not None:
        assert np.array_equal(nbrs[q, :c], want_nbrs), q
    # padding
    assert (idx[q, c:] == -1).all() and np.isnan(val[q, c:]).all() and (nbrs[q, c:] == 0).all(), q


def _histories(R, means, users, explicit, rng):
    hists = []
    for u in users:
        s, e = R.indptr[u], R.indptr[u + 1]
        ri = R.indices[s:e].astype(np.int32)
        perm = rng.permutation(len(ri))
        ri = ri[perm].copy()
        rv = R.data[s:e][perm].astype(np.float32)
        if explicit:
            rv = rv - means[ri]
        hists.append((ri, rv))
    return hists


def _recommend(st, hists, explicit, means, max_nbrs, min_nbrs, n, exclude):
    ptr_ = np.cumsum([0] + [len(h[0]) for h in hists]).astype(np.int64)
    ri = _t(np.concatenate([h[0] for h in hists]).astype(np.int32))
    rv = _t(np.concatenate([h[1] for h in hists]).astype(np.float32)) if explicit else None
    ip = _t(ptr_)
    out = st.recommend(
        ip, ri, rv, max_nbrs, min_nbrs, n, item_offset=_t(means) if explicit else None,
        excl_indptr=ip if exclude else None, excl_items=ri if exclude else None,
    )  # fmt: skip
    return [x.cpu().numpy() for x in out]


CASES = [  # explicit, save_nbrs, max_nbrs, min_nbrs, n, exclude
    (True, None, 20, 1, 100, True),
    (True, 20, 20, 1, 10, False),
    (False, None, 128, 1, 1024, True),
    (False, 20, 1, 1, 1, True),
    (True, None, 1, 1, 1024, False),
    (False, None, 20, 2, 10, False),
    (True, 20, 128, 2, 100, True),
    (False, 20, 20, 1, 100, False),
]


@pytest.mark.parametrize("explicit,save_nbrs,max_nbrs,min_nbrs,n,exclude", CASES)
def test_item_recommend_matches_host_composition(cuda_lib, ml_small, explicit, save_nbrs, max_nbrs, min_nbrs, n,
                                                 exclude):  # fmt: skip
    ui, iu, means = data.knn_item_matrices(ml_small, explicit)
    S = oracle.knn_build(ui, iu, 1e-6, save_nbrs)
    R = ml_small.coo().tocsr()
    rng = np.random.default_rng(23)
    heavy = int(np.argmax(np.diff(R.indptr)))
    users = np.concatenate([[heavy], rng.choice(ml_small.n_users, 30, replace=False)])
    hists = _histories(R, means, users, explicit, rng)
    for ri, _ in hists[1:6]:
        if len(ri) > 4:
            ri[1] = -1  # a null history entry (an unknown item after the vocabulary lookup)
    hists.append((np.zeros(0, np.int32), np.zeros(0, np.float32)))  # an empty history
    row_len = np.diff(S.indptr)
    thin = int(np.flatnonzero(row_len > 0)[np.argmin(row_len[row_len > 0])])
    hists.append((np.int32([thin]), np.float32([0.5])))  # few scorable candidates: cnt < n for larger n
    st = engine.KnnScorerState.create(S.shape[0], S.indptr, S.indices, S.data, _lib.require_device())
    if save_nbrs is None and not explicit:
        # the heaviest user's touched list spills out of shared memory, so the spill row is used (the centred
        # explicit model keeps only the positive similarities, and its heaviest user touches fewer targets)
        sc, _ = st.score_all_items(_t(np.int64([0, len(hists[0][0])])), _t(hists[0][0]),
                                   _t(hists[0][1]) if explicit else None, max_nbrs, 1)  # fmt: skip
        assert int((~torch.isnan(sc)).sum()) > DENSE_ACTIVE_CAP
    m = means if explicit else None
    idx, val, nbrs, cnt = _recommend(st, hists, explicit, m, max_nbrs, min_nbrs, n, exclude)
    assert idx.shape == (len(hists), n)
    for q, (ri, rv) in enumerate(hists):
        wi, wv, wc = expected_item(S, m, ri, rv if explicit else None, max_nbrs, min_nbrs, n, exclude)
        check_rows(idx, val, nbrs, cnt, q, wi, wv, wc, n)
    assert cnt[len(hists) - 2] == 0
    if n > row_len[thin] and min_nbrs == 1:  # (with min_nbrs 2 a one-item history scores nothing)
        assert 0 < cnt[-1] < n


@pytest.mark.parametrize("n", [10, 100, 1000])
def test_ties_replay_the_heap(cuda_lib, n):
    """Equal similarities and implicit feedback: every score is an integer, so the cut at n falls inside large tie
    groups and the order of equal scores is the heap's."""
    rng = np.random.default_rng(4)
    n_items = 3000
    S = sps.random(n_items, n_items, density=0.02, format="csr", random_state=5, dtype=np.float32)
    S.data[:] = 0.5
    S.sort_indices()
    st = engine.KnnScorerState.create(n_items, S.indptr, S.indices, S.data, _lib.require_device())
    hists = [(rng.choice(n_items, int(rng.integers(1, 60)), replace=False).astype(np.int32), None) for _ in range(40)]
    hists = [(ri, np.zeros(len(ri), np.float32)) for ri, _ in hists]
    for exclude in (True, False):
        idx, val, nbrs, cnt = _recommend(st, hists, False, None, 20, 1, n, exclude)
        for q, (ri, _) in enumerate(hists):
            wi, wv, wc = expected_item(S, None, ri, None, 20, 1, n, exclude)
            check_rows(idx, val, nbrs, cnt, q, wi, wv, wc, n)
        assert len(np.unique(val[0, : cnt[0]])) < cnt[0]  # there are ties in the output


def test_null_similarity_raises(cuda_lib):
    """A NaN similarity reached by a query is an error (status 2), as in dense scoring."""
    S = sps.csr_array((np.float32([0.5, np.nan]), np.int32([1, 0]), np.int64([0, 1, 2, 2])), shape=(3, 3))
    st = engine.KnnScorerState.create(3, S.indptr, S.indices, S.data, _lib.require_device())
    with pytest.raises(ValueError, match="similarity is null"):
        _recommend(st, [(np.int32([1]), np.float32([0.0]))], False, None, 20, 1, 2, True)
    idx, _, _, cnt = _recommend(st, [(np.int32([0]), np.float32([0.0]))], False, None, 20, 1, 2, False)
    assert cnt.tolist() == [1] and idx[0].tolist() == [1, -1]


def test_many_queries_per_cta_leave_the_slot_map_clean(cuda_lib, ml_small):
    ui, iu, means = data.knn_item_matrices(ml_small, True)
    S = oracle.knn_build(ui, iu, 1e-6, 20)
    R = ml_small.coo().tocsr()
    rng = np.random.default_rng(11)
    base = _histories(R, means, rng.choice(ml_small.n_users, 50, replace=False), True, rng)
    hists = [base[i % len(base)] for i in range(3000)]
    st = engine.KnnScorerState.create(S.shape[0], S.indptr, S.indices, S.data, _lib.require_device())
    assert len(hists) > 4 * int(cuda_lib.lk_knn_score_dense_ctas())
    idx, val, nbrs, cnt = _recommend(st, hists, True, means, 20, 1, 50, True)
    want = [expected_item(S, means, ri, rv, 20, 1, 50, True) for ri, rv in base]
    for q in range(len(hists)):
        check_rows(idx, val, nbrs, cnt, q, *want[q % len(base)], 50)
    # the same state still scores all items exactly: the ranking walk left the slot map at zero
    ptr_ = np.cumsum([0] + [len(h[0]) for h in base[:8]]).astype(np.int64)
    sc, ct = st.score_all_items(_t(ptr_), _t(np.concatenate([h[0] for h in base[:8]])),
                                _t(np.concatenate([h[1] for h in base[:8]])), 20, 1)  # fmt: skip
    sc, ct = sc.cpu().numpy(), ct.cpu().numpy()
    all_items = np.arange(S.shape[0], dtype=np.int32)
    for q, (ri, rv) in enumerate(base[:8]):
        osc, oct_ = oracle.knn_score(S, ri, rv, all_items, 20, 1)
        assert np.array_equal(ct[q], oct_)
        assert np.array_equal(np.isnan(sc[q]), np.isnan(osc))
        ok = ~np.isnan(osc)
        assert np.array_equal(sc[q][ok].view(np.int32), osc[ok].view(np.int32))


@pytest.mark.parametrize("explicit", [True, False])
def test_fused_equals_unfused_device_path(cuda_lib, ml_small, explicit):
    """score_all_items, the offsets and the exclusion mask, the transpose and topn_columns give the same bits."""
    ui, iu, means = data.knn_item_matrices(ml_small, explicit)
    S = oracle.knn_build(ui, iu, 1e-6, None)
    R = ml_small.coo().tocsr()
    rng = np.random.default_rng(2)
    hists = _histories(R, means, rng.choice(ml_small.n_users, 64, replace=False), explicit, rng)
    st = engine.KnnScorerState.create(S.shape[0], S.indptr, S.indices, S.data, _lib.require_device())
    m = means if explicit else None
    n = 100
    idx, val, nbrs, cnt = _recommend(st, hists, explicit, m, 20, 1, n, True)
    ptr_ = np.cumsum([0] + [len(h[0]) for h in hists]).astype(np.int64)
    sc, ct = st.score_all_items(_t(ptr_), _t(np.concatenate([h[0] for h in hists])),
                                _t(np.concatenate([h[1] for h in hists])) if explicit else None, 20, 1)  # fmt: skip
    if explicit:
        sc = sc + _t(means)[None, :]
    for q, (ri, _) in enumerate(hists):
        sc[q, _t(ri[ri >= 0]).long()] = float("nan")
    u_idx, u_val, u_cnt = engine.topn_columns(sc.T.contiguous(), n)
    u_idx, u_val, u_cnt = u_idx.cpu().numpy(), u_val.cpu().numpy(), u_cnt.cpu().numpy()
    ct = ct.cpu().numpy()
    assert np.array_equal(cnt, u_cnt) and np.array_equal(idx, u_idx)
    assert np.array_equal(val.view(np.int32), u_val.view(np.int32))
    for q in range(len(hists)):
        assert np.array_equal(nbrs[q, : cnt[q]], ct[q, idx[q, : cnt[q]]])


# ---------------------------------------------------------------------------
# components
# ---------------------------------------------------------------------------


def _item_cands(m, query, exclude, n_items):
    cands = np.arange(n_items, dtype=np.int32)
    qi = RecQuery.create(query).query_items
    if exclude and qi is not None:
        known = qi.numbers(vocabulary=m.items, missing="negative")
        cands = np.setdiff1d(cands, known[known >= 0]).astype(np.int32)
    return cands


def _host_composition(m, query, n, exclude, n_items, with_counts):
    cands = _item_cands(m, query, exclude, n_items)
    il = m(query, ItemList(item_nums=cands, vocabulary=m.items))
    sc = np.asarray(il.scores(), dtype=np.float32)
    top = oracle.argtopn(sc, n)
    return cands[top], sc[top], (il.field("nbr_counts")[top] if with_counts else None)


def _same(got: ItemList, want):
    wi, wv, wc = want
    assert np.array_equal(got.numbers(), wi)
    assert np.array_equal(got.ids(), got._vocab.ids(wi))
    assert np.array_equal(np.asarray(got.scores(), np.float32).view(np.int32), wv.view(np.int32))
    if wc is not None:
        assert np.array_equal(got.field("nbr_counts"), wc)


@pytest.mark.parametrize("explicit", [True, False])
def test_item_component_recommend_batch(cuda_lib, ml_small, explicit):
    ds = Dataset(ml_small)
    m = ItemKNNScorer(feedback="explicit" if explicit else "implicit", save_nbrs=20)
    m.train(ds)
    hist = ds.user_history(7)
    unknown = ItemList(item_ids=np.concatenate([hist.ids(), [-5]]), rating=np.concatenate([hist.field("rating"), [3.0]]))
    queries = [ds.user_history(u) for u in (0, 1, 40, 300)] + [
        unknown,  # an unknown item in the history
        ItemList(item_ids=hist.ids()[:0], rating=np.zeros(0, np.float32)),  # empty history
        RecQuery(user_id=ds.users.id(3)),  # no history at all
    ]
    n_items = ml_small.n_items
    for exclude in ("query", None):
        got = m.recommend_batch(queries, 25, exclude=exclude)
        assert len(got) == len(queries)
        for q, g in zip(queries, got):
            if RecQuery.create(q).query_items is None or len(RecQuery.create(q).query_items) == 0:
                assert len(g) == 0
                continue
            _same(g, _host_composition(m, q, 25, exclude == "query", n_items, True))
            assert g.field("nbr_counts") is not None
    if explicit:
        with pytest.raises(RuntimeError):
            m.recommend_batch([ItemList(item_ids=hist.ids())], 5)
    # n <= 0 gives empty lists, n beyond the engine's top-n limit is refused, n beyond n_items is clamped
    assert all(len(g) == 0 for g in m.recommend_batch(queries[:2], 0))
    with pytest.raises(ValueError):
        m.recommend_batch(queries[:1], 1025)
    with pytest.raises(ValueError):
        m.recommend_batch(queries[:1], 5, exclude="history")
    # pickling drops the device state; the reloaded scorer recommends the same
    clone = pickle.loads(pickle.dumps(m))
    a, b = m.recommend_batch(queries[:4], 40), clone.recommend_batch(queries[:4], 40)
    for x, y in zip(a, b):
        _same(x, (y.numbers(), np.asarray(y.scores(), np.float32), y.field("nbr_counts")))


@pytest.mark.parametrize("explicit", [True, False])
def test_user_component_recommend_batch(cuda_lib, ml_small, explicit):
    ds = Dataset(ml_small)
    m = UserKNNScorer(feedback="explicit" if explicit else "implicit", max_nbrs=12, min_nbrs=2)
    m.train(ds)
    rng = np.random.default_rng(8)
    hist = ds.user_history(40)
    dup_hist = ItemList(
        item_ids=np.concatenate([hist.ids(), hist.ids()[:3], [-99]]),
        rating=np.concatenate([hist.field("rating"), np.float32([1.0, 5.0, 2.5, 4.0])]),
    )
    queries = [ds.users.id(int(u)) for u in rng.choice(ml_small.n_users, 6, replace=False)]
    queries += [
        RecQuery(user_id=None, query_items=hist),  # history, no known user
        RecQuery(user_id=ds.users.id(40), query_items=dup_hist),  # known user, unknown and repeated items
        RecQuery(user_id="nobody"),  # unknown user without a history
        RecQuery(user_id=None, query_items=ItemList(item_ids=np.array([-1, -2]), rating=np.float32([3, 4]))),
    ]
    n_items = ml_small.n_items
    for exclude in ("query", None):
        for n in (1, 30, 1024):
            got = m.recommend_batch(queries, n, exclude=exclude)
            for q, g in zip(queries, got):
                cands = _item_cands(m, q, exclude == "query", n_items)
                sc = np.asarray(m.score_batch([q], [ItemList(item_nums=cands, vocabulary=m.items)])[0].scores(),
                                np.float32)  # fmt: skip
                top = oracle.argtopn(sc, n)
                _same(g, (cands[top], sc[top], None))
    got = m.recommend_batch(queries, 30)
    assert len(got[8]) == 0 and len(got[9]) == 0  # unknown user; a history without a known item: no neighbour
    assert len(got[0]) == 30
    assert all(len(g) == 0 for g in m.recommend_batch(queries[:2], -1))
    with pytest.raises(ValueError):
        m.recommend_batch(queries[:1], 2000)
    clone = pickle.loads(pickle.dumps(m))
    for x, y in zip(m.recommend_batch(queries, 30), clone.recommend_batch(queries, 30)):
        _same(x, (y.numbers(), np.asarray(y.scores(), np.float32), None))
