"""
kNN scoring at the benchmark's shape (ML-25M-shaped synthetic, 162,541 users x 59,047 items): the dense kernel
of ``knn_score.cu`` in item and user mode, score and rank mode, and the list kernel, against the oracle's
restatements (``oracle.knn_score``, ``oracle.user_score``, ``oracle.argtopn``) bit for bit.

The small fixtures never reach the dense kernel's size thresholds; this shape does:
  * more touched targets than the CTA keeps in shared memory (DENSE_ACTIVE_CAP): the tail spills into the
    query's count row (score mode) or the CTA's spill row (rank mode);
  * histories of several DENSE_HIST_CHUNK chunks, and user-mode neighbour lists of tens of thousands;
  * rank mode's walk over the slot map in 29 chunks of RANK_CHUNK items;
  * the per-CTA rows reused by 16,384 queries of one launch, as ``bench.py`` scores them.
The similarity matrix is built on the device and copied to the host as the oracle's input, so these checks do
not depend on the build (``test_scale_parity.py::test_knn_build_rows_at_ml25m_shape`` checks that).
"""

import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import scipy.sparse as sps
import torch

import oracle
from lkpy_b200 import _lib, data, engine
from lkpy_b200.components import Dataset
from lkpy_b200.knn_user import UserKNNScorer

pytestmark = pytest.mark.gpu

KNN_MIN_SIM, KNN_SAVE, KNN_MAX_NBRS = 1e-6, 20, 20  # bench.py
BATCH = 16_384  # bench.py's --score-batch: users per score_all_items launch
DENSE_ACTIVE_CAP = 8192  # touched targets a CTA keeps in shared memory (knn_score.cu)
DENSE_HIST_CHUNK = 2048  # history entries flattened at a time (knn_score.cu)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_lib.require_device())


def _pmap(fn, args):
    """The oracle calls of a sample, several at a time (ctypes releases the GIL)."""
    with ThreadPoolExecutor(max(1, min(16, os.cpu_count() or 1))) as ex:
        return list(ex.map(fn, args))


def assert_rows_exact(sc, ct, want_sc, want_ct, what):
    """Scores as int32 views, NaN pattern and counts equal."""
    assert np.array_equal(ct, want_ct), what
    nan = np.isnan(want_sc)
    assert np.array_equal(np.isnan(sc), nan), what
    assert np.array_equal(sc[~nan].view(np.int32), want_sc[~nan].view(np.int32)), what


def assert_topn_exact(idx, val, nbrs, cnt, want_items, want_vals, want_nbrs, n, what):
    """One rank-mode row: items, score bits and neighbour counts, then the -1 / NaN / 0 padding."""
    c = int(cnt)
    assert c == len(want_items), what
    assert np.array_equal(idx[:c], want_items), what
    assert np.array_equal(val[:c].view(np.int32), np.asarray(want_vals, np.float32).view(np.int32)), what
    if want_nbrs is not None:
        assert np.array_equal(nbrs[:c], want_nbrs), what
    assert (idx[c:] == -1).all() and np.isnan(val[c:]).all() and (nbrs[c:] == 0).all(), what


def ranked(sc, ct, n, excl=None, item_offset=None, query_offset=None):
    """The host composition of one query's top n over all items: candidates are all items minus ``excl``,
    ``(score + item_offset) + query_offset`` in f32, then ``argtopn``.  Returns (items, scores, counts)."""
    cands = np.arange(len(sc), dtype=np.int32)
    if excl is not None:
        cands = np.setdiff1d(cands, excl[excl >= 0]).astype(np.int32)
    s = sc[cands]
    if item_offset is not None:
        s = (s + item_offset[cands]).astype(np.float32)
    if query_offset is not None:
        s = (s + np.float32(query_offset)).astype(np.float32)
    top = oracle.argtopn(s, n)
    return cands[top], s[top], ct[cands][top]


def touched_targets(S: sps.csr_array, items: np.ndarray) -> int:
    """|union of the similarity rows of ``items``|: the targets a history touches."""
    items = items[items >= 0]
    starts, lens = S.indptr[items], np.diff(S.indptr)[items]
    tot = int(lens.sum())
    if tot == 0:
        return 0
    first = np.repeat(starts - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    mark = np.zeros(S.shape[1], dtype=bool)
    mark[S.indices[first + np.arange(tot)]] = True
    return int(mark.sum())


def most_touched(R, S: sps.csr_array, k: int) -> tuple[np.ndarray, np.ndarray]:
    """The ``k`` users with the most touched targets (ties to the lower user number) and their counts.  Exact:
    users are visited by the bound min(summed row lengths, n_items), and the walk stops below the k-th count."""
    row_len = np.diff(S.indptr)
    c = np.concatenate([[0], np.cumsum(row_len[R.indices], dtype=np.int64)])
    bound = np.minimum(c[R.indptr[1:]] - c[R.indptr[:-1]], S.shape[1])
    users, counts = [], []
    for u in np.argsort(-bound, kind="stable"):
        if len(counts) >= k and bound[u] < np.sort(counts)[-k]:
            break
        users.append(int(u))
        counts.append(touched_targets(S, R.indices[R.indptr[u] : R.indptr[u + 1]]))
    users, counts = np.array(users), np.array(counts)
    top = np.lexsort((users, -counts))[:k]
    return users[top], counts[top]


# ---------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def ml25m():
    return data.synth_interactions_cached(os.environ.get("LK_BENCH_DATA_CACHE"), **data.ML25M_SHAPE)


@pytest.fixture(scope="module")
def ratings(ml25m):
    """users x items ratings (SciPy CSR, rows sorted by item): the histories bench.py scores."""
    R = ml25m.coo().tocsr()
    R.sort_indices()
    return R


def _item_model(ml25m, explicit: bool):
    """The device-built similarity matrix (bench's min_sim and save_nbrs) as a scorer state, its host copy (the
    oracle's input) and the item means."""
    dev = _lib.require_device()
    kui, kiu, means = data.knn_item_matrices(ml25m, explicit)
    plan = engine.KnnBuildPlan.create(engine.DeviceCSR.from_host(kui, dev), engine.DeviceCSR.from_host(kiu, dev))
    cols, vals, cnt = plan.build_topk(KNN_MIN_SIM, KNN_SAVE)
    indptr, c, v = engine.topk_rows_to_csr(cols, vals, cnt)
    del plan, cols, vals, cnt
    S = sps.csr_array((v.cpu().numpy(), c.cpu().numpy(), indptr.cpu().numpy()), shape=(ml25m.n_items,) * 2)
    st = engine.KnnScorerState.create(ml25m.n_items, indptr, c, v, dev)
    torch.cuda.empty_cache()
    return st, S, means


def _item_sample(R, S, means, seed):
    """The query sample, chosen on the host: [(label, history items int32, history values f32 or None)], the
    values centred by the item means (None for implicit).  Every precondition that makes it worth scoring is
    asserted."""
    n_users, n_items = R.shape
    lens = np.diff(R.indptr)
    row_len = np.diff(S.indptr)
    rng = np.random.default_rng(seed)

    longest = np.argsort(-lens, kind="stable")[:8]
    chunks = -(-lens[longest] // DENSE_HIST_CHUNK)
    assert chunks[0] >= 4, f"longest history {lens[longest[0]]} spans fewer than 4 history chunks"
    heavy, touched = most_touched(R, S, 8)
    assert touched[0] > 2 * DENSE_ACTIVE_CAP, touched  # most of the touched list spills
    assert (touched > DENSE_ACTIVE_CAP).all(), touched
    empty = np.flatnonzero(lens == 0)[:2]
    assert len(empty) == 2
    taken = set(longest) | set(heavy) | set(empty)
    pool = np.setdiff1d(np.arange(n_users), np.fromiter(taken, dtype=np.int64))
    rand = rng.choice(pool, 32, replace=False)

    def user(u):
        ri = R.indices[R.indptr[u] : R.indptr[u + 1]].astype(np.int32)
        rv = R.data[R.indptr[u] : R.indptr[u + 1]].astype(np.float32)
        return ri, rv

    vals = np.unique(R.data[: 100_000]).astype(np.float32)  # the rating scale
    hists = [(f"longest/{u}", *user(u)) for u in longest]
    hists += [(f"touched/{u}", *user(u)) for u in heavy]
    hists += [(f"random/{u}", *user(u)) for u in rand]
    hists += [(f"empty/{u}", *user(u)) for u in empty]
    # every item once, in a seeded order: 29 history chunks, the most touched targets possible
    every = rng.permutation(n_items).astype(np.int32)
    hists.append(("every_item", every, rng.choice(vals, n_items)))
    # repeats and null entries across chunk boundaries
    ri0 = user(longest[0])[0]
    rep = np.concatenate([ri0, rng.choice(ri0, 2_500), np.full(300, -1, np.int32)]).astype(np.int32)
    rep = rep[rng.permutation(len(rep))]
    hists.append(("repeats_and_nulls", rep, rng.choice(vals, len(rep))))
    # one item whose similarity row is empty (or the shortest row)
    lone = int(np.argmin(row_len))
    hists.append((f"lone_item/{lone}/row_len={row_len[lone]}", np.array([lone], np.int32), vals[-1:].copy()))

    out = []
    for label, ri, rv in hists:
        if means is None:
            rv = None
        else:
            rv = (rv.astype(np.float32) - means[np.maximum(ri, 0)]).astype(np.float32)
        out.append((label, ri, rv))
    figures = {
        "longest_history": int(lens[longest[0]]), "longest_history_chunks": int(chunks[0]),
        "histories_ge_4_chunks": int((chunks >= 4).sum()),
        "most_touched": touched.tolist(), "every_item_touched": touched_targets(S, every),
        "lone_item_row_len": int(row_len[lone]),
    }  # fmt: skip
    print(f"\n[knn-scale] item sample ({'explicit' if means is not None else 'implicit'}): {figures}")
    return out


def _oracle_rows(S, sample, max_nbrs, min_nbrs):
    all_items = np.arange(S.shape[0], dtype=np.int32)
    return _pmap(lambda h: oracle.knn_score(S, h[1], h[2], all_items, max_nbrs, min_nbrs), sample)


def _batch(ri_list, rv_list):
    """Device CSR of a batch of histories (int64 offsets, int32 items, f32 values or None)."""
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in ri_list])]).astype(np.int64)
    ri = np.concatenate(ri_list).astype(np.int32) if ptr[-1] else np.zeros(0, np.int32)
    rv = None
    if rv_list is not None:
        rv = np.concatenate(rv_list).astype(np.float32) if ptr[-1] else np.zeros(0, np.float32)
    return _t(ptr), _t(ri), (None if rv is None else _t(rv))


@pytest.fixture(scope="module")
def item_explicit(cuda_lib, ml25m, ratings):
    """The explicit model, its sample and the bench batch: the first 16,384 users with the sample's queries at
    evenly spread positions (the first and the last included), history values centred as bench.py centres them."""
    st, S, means = _item_model(ml25m, True)
    sample = _item_sample(ratings, S, means, seed=25)
    pos = np.linspace(0, BATCH - 1, len(sample)).round().astype(np.int64)
    assert pos[0] == 0 and pos[-1] == BATCH - 1 and len(np.unique(pos)) == len(sample)
    R = ratings
    ri_list = [R.indices[R.indptr[u] : R.indptr[u + 1]] for u in range(BATCH)]
    rv_list = [(R.data[R.indptr[u] : R.indptr[u + 1]] - means[ri_list[u]]).astype(np.float32) for u in range(BATCH)]
    for p, (_label, ri, rv) in zip(pos, sample):
        ri_list[p], rv_list[p] = ri, rv
    batch = _batch(ri_list, rv_list)
    want = _oracle_rows(S, sample, KNN_MAX_NBRS, 1)
    # score mode of the whole batch; only the sampled rows leave the device
    sc, ct = st.score_all_items(*batch, KNN_MAX_NBRS, 1)
    p = _t(pos)
    rows = sc[p].cpu().numpy(), ct[p].cpu().numpy()
    del sc, ct
    torch.cuda.empty_cache()
    return {"st": st, "S": S, "means": means, "sample": sample, "pos": pos, "batch": batch, "want": want,
            "rows": rows}  # fmt: skip


# ---------------------------------------------------------------------------------------------------------------
# item mode
# ---------------------------------------------------------------------------------------------------------------


def test_item_score_all_items_bench_batch(item_explicit):
    """score_all_items over bench's 16,384-query launch, explicit, max_nbrs 20, min_nbrs 1."""
    m = item_explicit
    sc, ct = m["rows"]
    for i, (label, _ri, _rv) in enumerate(m["sample"]):
        assert_rows_exact(sc[i], ct[i], *m["want"][i], f"{label} at position {m['pos'][i]}")


def test_item_score_lists_kernel_all_targets(item_explicit, ratings):
    """The list kernel (``score``) with every item as an explicit target, for 64 queries: the sample and
    random users."""
    m = item_explicit
    R, means, n_items = ratings, m["means"], m["S"].shape[0]
    rng = np.random.default_rng(64)
    extra = rng.choice(R.shape[0], 64 - len(m["sample"]), replace=False)
    qs = [(h[1], h[2]) for h in m["sample"]]
    for u in extra:
        ri = R.indices[R.indptr[u] : R.indptr[u + 1]].astype(np.int32)
        qs.append((ri, (R.data[R.indptr[u] : R.indptr[u + 1]] - means[ri]).astype(np.float32)))
    all_items = np.arange(n_items, dtype=np.int32)
    more = _pmap(lambda h: oracle.knn_score(m["S"], h[0], h[1], all_items, KNN_MAX_NBRS, 1), qs[len(m["want"]) :])
    want = m["want"] + more
    ip, ri, rv = _batch([q[0] for q in qs], [q[1] for q in qs])
    tgt_ptr = _t(np.arange(len(qs) + 1, dtype=np.int64) * n_items)
    tgt = _t(np.tile(all_items, len(qs)))
    sc, ct = m["st"].score(ip, ri, rv, tgt_ptr, tgt, KNN_MAX_NBRS, 1)
    sc, ct = sc.cpu().numpy().reshape(len(qs), n_items), ct.cpu().numpy().reshape(len(qs), n_items)
    for i in range(len(qs)):
        assert_rows_exact(sc[i], ct[i], *want[i], f"query {i}")


@pytest.mark.parametrize("n", [100, 1024])
def test_item_recommend_bench_batch(item_explicit, n):
    """Rank mode over the same 16,384-query launch: the item means as the offset, the history excluded; against
    the oracle composition and against argtopn of the batch's own score rows.  Then a score-mode call on the same
    state is still exact: the rank walk left the slot maps clean."""
    m = item_explicit
    st, means, pos = m["st"], m["means"], m["pos"]
    ip, ri, rv = m["batch"]
    idx, val, nbrs, cnt = st.recommend(ip, ri, rv, KNN_MAX_NBRS, 1, n, item_offset=_t(means), excl_indptr=ip,
                                       excl_items=ri)  # fmt: skip
    p = _t(pos)
    idx, val, nbrs, cnt = (x[p].cpu().numpy() for x in (idx, val, nbrs, cnt))
    sc_rows, ct_rows = m["rows"]
    for i, (label, hri, _rv) in enumerate(m["sample"]):
        what = f"{label} at position {pos[i]}, n={n}"
        want = ranked(*m["want"][i], n, excl=hri, item_offset=means)
        assert_topn_exact(idx[i], val[i], nbrs[i], cnt[i], *want, n, what)
        got_rows = ranked(sc_rows[i], ct_rows[i], n, excl=hri, item_offset=means)
        assert_topn_exact(idx[i], val[i], nbrs[i], cnt[i], *got_rows, n, what + " (score-mode rows)")
    del idx, val, nbrs, cnt
    small = m["sample"][:8] + m["sample"][-3:]
    sc, ct = st.score_all_items(*_batch([h[1] for h in small], [h[2] for h in small]), KNN_MAX_NBRS, 1)
    sc, ct = sc.cpu().numpy(), ct.cpu().numpy()
    want = m["want"][:8] + m["want"][-3:]
    for i, h in enumerate(small):
        assert_rows_exact(sc[i], ct[i], *want[i], f"{h[0]} after rank mode")


def test_item_score_all_items_implicit(cuda_lib, ml25m, ratings):
    """The implicit model (similarity sums), the sample alone in one launch, max_nbrs 128, min_nbrs 2."""
    st, S, _ = _item_model(ml25m, False)
    sample = _item_sample(ratings, S, None, seed=26)
    want = _oracle_rows(S, sample, 128, 2)
    sc, ct = st.score_all_items(*_batch([h[1] for h in sample], None), 128, 2)
    sc, ct = sc.cpu().numpy(), ct.cpu().numpy()
    for i, (label, _ri, _rv) in enumerate(sample):
        assert_rows_exact(sc[i], ct[i], *want[i], label)


# ---------------------------------------------------------------------------------------------------------------
# user mode
# ---------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def user_model(cuda_lib, ml25m):
    """UserKNNScorer's training products (user-centred ratings, unit user vectors) and the two scorer states over
    the 162,541 x 59,047 rating matrix: centred values (explicit) and structure only (implicit)."""
    m = UserKNNScorer(feedback="explicit")
    m.train(Dataset(ml25m))
    R = m.user_ratings
    dev = _lib.require_device()
    states = {
        True: engine.KnnScorerState.create(R.shape[1], R.indptr, R.indices, R.values, dev, user_mode=True),
        False: engine.KnnScorerState.create(R.shape[1], R.indptr, R.indices, None, dev, user_mode=True),
    }
    return {"R": R, "V": m.user_vectors, "means": m.user_means, "states": states}


@pytest.fixture(scope="module")
def neighbour_lists(user_model):
    """Ascending random user subsets of 1 to 65,000 users with f32 similarities in (0, 1] (coarse, so equal
    weights meet at the heap boundary), the 64 heaviest users, and one list of all-equal similarities."""
    R = user_model["R"]
    n_users = R.shape[0]
    lens = np.diff(R.indptr)
    rng = np.random.default_rng(81)
    lists = []
    for size in (1, 2_047, 2_048, 2_049, 20_000, 65_000):
        users = np.sort(rng.choice(n_users, size, replace=False)).astype(np.int32)
        lists.append((f"random/{size}", users, (rng.integers(1, 1001, size) / 1000).astype(np.float32)))
    heavy = np.sort(np.argsort(-lens, kind="stable")[:64]).astype(np.int32)
    lists.append(("heaviest/64", heavy, (1.0 - rng.random(64)).astype(np.float32)))
    eq = np.sort(rng.choice(n_users, 5_000, replace=False)).astype(np.int32)
    lists.append(("equal/5000", eq, np.full(len(eq), 0.5, np.float32)))
    contrib = [int(lens[u].sum()) for _l, u, _s in lists]
    heavy_chunks = -(-len(lists[5][1]) // DENSE_HIST_CHUNK)
    assert heavy_chunks >= 30 and max(contrib) > 5_000_000
    print(f"\n[knn-scale] neighbour lists: {[(lab, len(u), c) for (lab, u, _s), c in zip(lists, contrib)]}")
    return lists


@pytest.fixture(scope="module")
def user_oracle(user_model, neighbour_lists):
    """Oracle rows of every neighbour list over all items, per (explicit, max_nbrs, min_nbrs); computed once."""
    R, n_items = user_model["R"], user_model["R"].shape[1]
    all_items = np.arange(n_items, dtype=np.int32)
    cache = {}

    def get(explicit, max_nbrs, min_nbrs):
        key = (explicit, max_nbrs, min_nbrs)
        if key not in cache:
            cache[key] = _pmap(
                lambda ls: oracle.user_score(R, ls[1], ls[2], all_items, max_nbrs, min_nbrs, explicit), neighbour_lists
            )
        return cache[key]

    return get


@pytest.mark.parametrize("explicit", [True, False], ids=["explicit", "implicit"])
@pytest.mark.parametrize("max_nbrs,min_nbrs", [(20, 1), (20, 2), (128, 1), (128, 2)])
def test_user_score_and_recommend(user_model, neighbour_lists, user_oracle, explicit, max_nbrs, min_nbrs):
    """User mode, every list against all items: score mode (score_all_items) and rank mode (n = 100, the query
    offsets added in f32 with explicit feedback, a few items excluded per query)."""
    st = user_model["states"][explicit]
    want = user_oracle(explicit, max_nbrs, min_nbrs)
    batch = _batch([ls[1] for ls in neighbour_lists], [ls[2] for ls in neighbour_lists])
    sc, ct = st.score_all_items(*batch, max_nbrs, min_nbrs)
    sc, ct = sc.cpu().numpy(), ct.cpu().numpy()
    for i, (label, _u, _s) in enumerate(neighbour_lists):
        assert_rows_exact(sc[i], ct[i], *want[i], label)
    del sc, ct

    n_items = user_model["R"].shape[1]
    rng = np.random.default_rng(max_nbrs * 10 + min_nbrs)
    qoff = rng.uniform(2.5, 4.0, len(neighbour_lists)).astype(np.float32) if explicit else None
    excl = [rng.choice(n_items, 50, replace=False).astype(np.int32) for _ in neighbour_lists]
    e_ptr = _t(np.arange(len(excl) + 1, dtype=np.int64) * 50)
    idx, val, nbrs, cnt = st.recommend(*batch, max_nbrs, min_nbrs, 100, query_offset=None if qoff is None else _t(qoff),
                                       excl_indptr=e_ptr, excl_items=_t(np.concatenate(excl)))  # fmt: skip
    idx, val, nbrs, cnt = (x.cpu().numpy() for x in (idx, val, nbrs, cnt))
    for i, (label, _u, _s) in enumerate(neighbour_lists):
        w = ranked(*want[i], 100, excl=excl[i], query_offset=None if qoff is None else qoff[i])
        assert_topn_exact(idx[i], val[i], nbrs[i], cnt[i], *w, 100, label)


def test_user_search_then_score(user_model):
    """End to end: neighbour search for 8 users on the device, then scoring of the lists it returned, compared
    with oracle.user_score on those same lists (the search itself is checked in test_user_knn_search_gpu.py)."""
    R, V = user_model["R"], user_model["V"]
    lens = np.diff(R.indptr)
    rng = np.random.default_rng(8)
    heaviest = np.argsort(-lens, kind="stable")[:2]
    users = np.concatenate([heaviest, rng.choice(np.flatnonzero(lens > 0), 6, replace=False)])
    ns = engine.UserNeighbourState.create(V, _lib.require_device())
    indptr, rows, sims = ns.neighbours(ns.known_queries(users), KNN_MIN_SIM)
    del ns
    ip, nb, sm = indptr.cpu().numpy(), rows.cpu().numpy(), sims.cpu().numpy()
    sizes = np.diff(ip)
    print(f"\n[knn-scale] searched neighbour lists: {sizes.tolist()}")
    assert sizes.max() > 4 * DENSE_HIST_CHUNK
    sc, ct = user_model["states"][True].score_all_items(indptr, rows, sims, 20, 1)
    sc, ct = sc.cpu().numpy(), ct.cpu().numpy()
    all_items = np.arange(R.shape[1], dtype=np.int32)
    want = _pmap(lambda q: oracle.user_score(R, nb[ip[q] : ip[q + 1]], sm[ip[q] : ip[q + 1]], all_items, 20, 1, True),
                 range(len(users)))  # fmt: skip
    for q, u in enumerate(users):
        assert_rows_exact(sc[q], ct[q], *want[q], f"user {u} ({sizes[q]} neighbours)")
