"""
The bias model, bias and popularity ranking, and BiasedSVD's exact stages at the benchmark's shape (ML-25M-shaped
synthetic, 162,541 users x 59,047 items, 25,000,095 ratings), bit for bit against the host statements:

* ``lk_bias_learn`` against ``BiasModel.learn``: the mean's pairwise tree with walkers that recurse below the cut
  at depth 16 and every combine level at work, and entity chains of up to 80,315 (items) and 8,528 (users) adds,
  on ratings where the order of those chains shows in the biases;
* ``lk_offset_score_batch`` in rank mode (``BiasScorer`` / ``PopScorer.recommend_batch``) over 59,047 items for a
  32,768-query call, as ``tools/basic_bench.py`` makes it, against ``bo.bias_scores`` / ``item_scores`` then
  ``bo.ranked``;
* ``BiasedSVDScorer.train``'s residual matrix and ``lk_spmm`` products (item rows of up to 80,315 entries, empty
  user rows, W = 26, 64 and 74) against ``tests/svd_oracle.py``, and its ranking against ``score_matrix`` columns.

The small fixtures of tests/test_basic_gpu.py and tests/test_svd_gpu.py reach none of these lengths.
"""

import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sps
import torch

import basic_oracle as bo
import oracle
import svd_oracle as so
from lkpy_b200 import _lib, basic, data, engine, svd
from lkpy_b200.basic import BiasModel, BiasScorer, PopScorer
from lkpy_b200.components import Dataset, ItemList, RecQuery
from lkpy_b200.data import Interactions
from lkpy_b200.svd import BiasedSVDScorer
from test_basic_gpu import check_ranking, check_same
from test_svd_gpu import SV_TOL

pytestmark = pytest.mark.gpu

HEAVIEST_ITEM, LONGEST_USER = 80_315, 8_528  # ratings of the most rated item and of the most active user
QUERIES = 32_768  # tools/basic_bench.py --users: queries in one recommend_batch call
SVD_SEED, SVD_K = 2025, 64
SPMM_WIDTHS = (26, 64, 74)  # one partial slice; k; k + 10, as the range finder multiplies


def _bits(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


# ---------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def ml25m():
    return data.synth_interactions_cached(os.environ.get("LK_BENCH_DATA_CACHE"), **data.ML25M_SHAPE)


@pytest.fixture(scope="module")
def noisy(ml25m):
    """The bench's users and items, ratings ``+ N(0, 1e-3)`` in f32: the global mean rounds differently from
    the exact sum."""
    rng = np.random.default_rng(25)
    r = (ml25m.ratings + rng.standard_normal(ml25m.nnz) * 1e-3).astype(np.float32)
    return Interactions(ml25m.users, ml25m.items, r, ml25m.n_users, ml25m.n_items)


@pytest.fixture(scope="module")
def cancelling(noisy):
    """The noisy ratings with ``bo.cancelling_ratings``: +-2^36 along 4-cycles through the most rated item, so
    that the partial sums of most entity chains pass through +-2^36 while the biases stay small."""
    r = bo.cancelling_ratings(noisy, np.random.default_rng(30))
    return Interactions(noisy.users, noisy.items, r, noisy.n_users, noisy.n_items)


@pytest.fixture(scope="module")
def shape_facts(ml25m):
    """The lengths that make this shape worth checking, asserted."""
    it = ml25m
    items, users = np.bincount(it.items, minlength=it.n_items), np.bincount(it.users, minlength=it.n_users)
    assert items.max() == HEAVIEST_ITEM and users.max() == LONGEST_USER
    empty = np.flatnonzero(users == 0)
    assert len(empty) > 0
    # every walker of the mean's tree sums more than a leaf (128 values), so pairwise_sum recurses
    sizes = np.array([bo.mean_node(it.nnz, bo.MEAN_DEPTH, p)[1] for p in range(1 << bo.MEAN_DEPTH)])
    assert sizes.sum() == it.nnz and sizes.min() > 128
    return {"item_counts": items, "user_counts": users, "empty_users": empty}


# ---------------------------------------------------------------------------------------------------------------
# the bias learner
# ---------------------------------------------------------------------------------------------------------------

LEARN_CASES = [
    ("bench", np.float32, (5.0, 0.1), ("user", "item")),
    ("bench", np.float64, 0.0, ("item",)),
    ("bench", np.float32, 0.0, ("user",)),
    ("noisy", np.float32, 0.0, ("user", "item")),
    ("noisy", np.float64, (5.0, 0.1), ("user", "item")),
    ("noisy", np.float32, (5.0, 0.1), ("item",)),
    ("cancelling", np.float64, 0.0, ("user", "item")),
    ("cancelling", np.float32, 0.0, ("user", "item")),
    ("cancelling", np.float64, (5.0, 0.1), ("user",)),
]  # fmt: skip


@pytest.mark.parametrize("which,dtype,damping,entities", LEARN_CASES,
                         ids=[f"{w}-{np.dtype(t).name}-{d}-{'+'.join(e)}" for w, t, d, e in LEARN_CASES])  # fmt: skip
def test_learn_is_the_host_statements(request, shape_facts, which, dtype, damping, entities):
    """``basic.learn`` against ``BiasModel.learn``, mean and biases bit for bit.  A user without ratings has bias 0.

    On the cancelling ratings a reversed chain changes the f32 biases of most items and of many users, with f64
    and with f32 centring, and that is asserted for the configurations that learn both with damping 0, the
    outputs ``bo.reversed_chain_changes`` counts.  So an entity pass that adds out of COO order fails there.  On the
    bench's ratings and the noisy copy every order gives the same biases: those cases check agreement only."""
    it = {"bench": "ml25m", "noisy": "noisy", "cancelling": "cancelling"}[which]
    it = request.getfixturevalue(it)
    pair = basic.damping_pair(damping)
    dev = basic.learn(Dataset(it), damping, entities=set(entities), centered_dtype=dtype)
    host = BiasModel.learn(it, pair, dtype, entities)
    check_same(dev, host)
    if dev.user_biases is not None:
        assert (dev.user_biases[shape_facts["empty_users"]] == 0).all()
    if which == "cancelling" and damping == 0.0 and len(entities) == 2:
        items_changed, users_changed = bo.reversed_chain_changes(it, dtype)
        print(f"\n[bias-scale] reversed chains change {items_changed} item and {users_changed} user biases")
        assert items_changed > it.n_items // 2 and users_changed > it.n_users // 5


# ---------------------------------------------------------------------------------------------------------------
# the query call shared by the ranking tests
# ---------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def query_call(ml25m, shape_facts):
    """32,768 queries (a user id with that user's history, as tools/basic_bench.py makes them) with a sample of
    queries at evenly spread positions, the first and the last among them: the 8 longest histories, 2 users
    without ratings, the heaviest user's items with f32 and with f64 ratings (a fold-in offset), an unknown user
    with and without a history, a query without a user whose items are all but the 3,000 least rated, and random
    users.  Returns ``(queries, positions, labels)``."""
    it = ml25m
    lens = shape_facts["user_counts"]
    vocab = Dataset(it).items
    rng = np.random.default_rng(1)
    ptr = np.concatenate([[0], np.cumsum(lens)])

    def history(u, rating=None):
        lo, hi = ptr[u], ptr[u + 1]
        fields = {} if rating is None else {"rating": it.ratings[lo:hi].astype(rating)}
        return ItemList(item_nums=it.items[lo:hi], vocabulary=vocab, **fields)

    longest = np.argsort(-lens, kind="stable")[:8]
    empty = shape_facts["empty_users"][:2]
    rand = rng.choice(np.flatnonzero(lens > 0), 24, replace=False)
    sample = [(f"longest/{u}", RecQuery(int(u), history(u))) for u in longest]
    sample += [(f"empty/{u}", RecQuery(int(u), history(u))) for u in empty]
    sample += [("rated_f32", RecQuery(int(longest[0]), history(longest[0], np.float32)))]
    sample += [("rated_f64", RecQuery(int(longest[1]), history(longest[1], np.float64)))]
    sample += [("unknown", RecQuery(it.n_users + 5, None)), ("unknown_with_items", RecQuery(-3, history(rand[0])))]
    # every item but the 3,000 least rated excluded: the candidates' counts are small and mostly tied
    popular = np.argsort(-shape_facts["item_counts"], kind="stable")[: it.n_items - 3_000]
    sample += [("least_rated_tail", RecQuery(None, ItemList(item_nums=np.sort(popular).astype(np.int32), vocabulary=vocab)))]
    sample += [(f"random/{u}", RecQuery(int(u), history(u))) for u in rand]

    users = np.sort(rng.choice(it.n_users, QUERIES, replace=False))
    queries = [RecQuery(int(u), history(u)) for u in users]
    pos = np.linspace(0, QUERIES - 1, len(sample)).round().astype(np.int64)
    assert pos[0] == 0 and pos[-1] == QUERIES - 1 and len(np.unique(pos)) == len(sample)
    for p, (_label, q) in zip(pos, sample):
        queries[p] = q
    return queries, pos, [label for label, _q in sample]


# ---------------------------------------------------------------------------------------------------------------
# BiasScorer and PopScorer ranking
# ---------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def offset_scorers(cuda_lib, ml25m, shape_facts):
    """The trained scorers.  The popularity scores are the reference's pandas statements over the host's
    ``np.bincount``, so the rankings' host reference does not rest on the device's counts."""
    ds = Dataset(ml25m)
    out = {"bias": BiasScorer(damping=5.0)}
    out.update({f"pop-{mode}": PopScorer(score=mode) for mode in ("quantile", "rank", "count")})
    counts = pd.Series(shape_facts["item_counts"], index=pd.Index(ds.items.ids(), name="item_id"), name="count")
    for name, m in out.items():
        m.train(ds)
        if name != "bias":
            want = np.require(m._train_internal(counts).values, np.float32)
            assert np.array_equal(m.item_scores.view(np.int32), want.view(np.int32)), name
    return out


@pytest.mark.parametrize("exclude", ["query", None])
@pytest.mark.parametrize("n", [100, 1024])
@pytest.mark.parametrize("scorer", ["bias", "pop-quantile", "pop-rank", "pop-count"])
def test_offset_recommend_is_the_host_composition(offset_scorers, query_call, scorer, n, exclude):
    """One ``recommend_batch`` call of 32,768 queries; the sampled ones against the host composition.  For count
    scores at n = 1024 the tie group at the cut reaches past n, so that the heap alone decides which tied items
    survive.  With nothing excluded every query ranks the same list, and there the 1,024th count's tie group ends
    inside the top 1,024; with the query's items excluded it reaches past n for some sampled users (5 of 39 when
    this was written) and always for the query that leaves only the 3,000 least rated items, whose counts are
    mostly tied."""
    m = offset_scorers[scorer]
    queries, pos, labels = query_call
    recs = m.recommend_batch(queries, n, exclude=exclude)
    assert len(recs) == QUERIES
    sample = [queries[p] for p in pos]
    if scorer == "bias":
        all_items = ItemList(item_nums=np.arange(len(m.items), dtype=np.int32), vocabulary=m.items)
        host = [bo.bias_scores(m.model, m.users, m.items, q, all_items) for q in sample]
        off = m.query_offsets(sample)[labels.index("rated_f64")]
        assert off != np.float64(np.float32(off))  # an offset the kernel adds in f64, not an f32 value
    else:
        host = [m.item_scores] * len(sample)
    for p, label, q, s in zip(pos, labels, sample, host):
        try:
            check_ranking([recs[p]], [s], [q], m.items, n, exclude=exclude == "query")
        except AssertionError as e:
            raise AssertionError(f"{label} at position {p}, n={n}") from e
    if scorer == "pop-count" and n == 1024 and exclude == "query":
        past = []
        for label, q, s in zip(labels, sample, host):
            s = np.array(s, dtype=np.float32)
            if q.query_items is not None:
                nums = q.query_items.numbers(vocabulary=m.items, missing="negative")
                s[nums[nums >= 0]] = np.nan
            cut = np.sort(s[~np.isnan(s)])[::-1][n - 1]
            if (s >= cut).sum() > n:
                past.append(label)
        print(f"\n[bias-scale] count ties past n = {n} (exclude={exclude}): {len(past)} of {len(sample)}: {past}")
        assert "least_rated_tail" in past and len(past) > 1


# ---------------------------------------------------------------------------------------------------------------
# BiasedSVD
# ---------------------------------------------------------------------------------------------------------------


def _sub_csr(X: sps.csr_array, rows: np.ndarray):
    """The rows ``rows`` of ``X`` as ``(indptr, indices, values)``, entries in stored order."""
    lens = np.diff(X.indptr)[rows]
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    take = np.concatenate([np.arange(X.indptr[r], X.indptr[r + 1]) for r in rows]).astype(np.int64)
    return ptr, X.indices[take], X.data[take]


@pytest.fixture(scope="module")
def svd_model(cuda_lib, noisy):
    """``BiasedSVDScorer(embedding_size=64)`` trained on the noisy ratings under a fixed NumPy seed, the residual
    operand rebuilt on the device from its bias model, the host residuals in both orientations, and the sampled
    rows of each orientation: the 16 longest, the empty user rows and 200 random rows."""
    np.random.seed(SVD_SEED)
    m = BiasedSVDScorer(embedding_size=SVD_K)
    m.train(Dataset(noisy))
    b = m.bias
    X = so.residuals(noisy.users, noisy.items, noisy.ratings, noisy.n_users, noisy.n_items, b.global_bias,
                     b.item_biases, b.user_biases)  # fmt: skip
    X.sort_indices()
    XT = sps.csr_array(X.T)
    XT.sort_indices()
    rng = np.random.default_rng(74)
    rows = {}
    for name, M in (("users", X), ("items", XT)):
        lens = np.diff(M.indptr)
        longest = np.argsort(-lens, kind="stable")[:16]
        empty = np.flatnonzero(lens == 0)
        rand = rng.choice(np.setdiff1d(np.arange(M.shape[0]), np.concatenate([longest, empty])), 200, replace=False)
        rows[name] = np.concatenate([longest, empty, rand])
    assert np.diff(XT.indptr)[rows["items"][0]] == HEAVIEST_ITEM
    assert np.diff(X.indptr)[rows["users"][0]] == LONGEST_USER
    assert (np.diff(X.indptr)[rows["users"]] == 0).any()
    x = svd.residual_operand(b, noisy, _lib.require_device())
    return {"m": m, "X": X, "XT": XT, "x": x, "rows": rows}


def test_svd_residual_operand(svd_model):
    """``svd.residual_operand`` is ``so.residuals`` in both orientations: offsets, indices and value bits."""
    x, X, XT = svd_model["x"], svd_model["X"], svd_model["XT"]
    for dm, want in ((x.rows, X), (x.cols, XT)):
        assert np.array_equal(dm.h_indptr, want.indptr)
        assert np.array_equal(dm.indices.cpu().numpy(), want.indices)
        assert np.array_equal(_bits(dm.values.cpu().numpy()), _bits(want.data))


@pytest.mark.parametrize("orient", ["users", "items"])
def test_svd_spmm_on_sampled_rows(svd_model, orient):
    """``engine.spmm`` over the whole operand at W = 26, 64 and 74 against ``so.spmm`` of the sampled rows' sub-CSR
    (one host call: the columns of a product are independent)."""
    x = svd_model["x"]
    dm, order, M = (x.rows, x.rows_order, svd_model["X"]) if orient == "users" else (x.cols, x.cols_order,
                                                                                   svd_model["XT"])  # fmt: skip
    rows = svd_model["rows"][orient]
    rng = np.random.default_rng(len(rows))
    dense = [rng.standard_normal((M.shape[1], W)).astype(np.float32) for W in SPMM_WIDTHS]
    want = so.spmm(*_sub_csr(M, rows), np.concatenate(dense, axis=1))
    c = 0
    for W, d in zip(SPMM_WIDTHS, dense):
        got = engine.spmm(dm, order, torch.from_numpy(d).to(dm.indptr.device))
        got = got[torch.from_numpy(rows).to(got.device)].cpu().numpy()
        assert np.array_equal(_bits(got), _bits(want[:, c : c + W])), f"{orient}, W={W}"
        c += W


def test_svd_user_components_and_singular_values(svd_model):
    """``user_components`` is ``so.spmm(X, components_.T)`` on the sampled user rows, bit for bit; the singular
    values are within SV_TOL of ``so.truncated_svd`` from the same start matrix (cuSOLVER's LU, QR and SVD agree
    with LAPACK's to rounding only)."""
    m, X = svd_model["m"], svd_model["X"]
    rows = svd_model["rows"]["users"]
    want = so.spmm(*_sub_csr(X, rows), np.ascontiguousarray(m.components_.T))
    assert np.array_equal(_bits(m.user_components[rows]), _bits(want))
    q0 = so.start_matrix(X.shape, SVD_K, np.random.RandomState(SVD_SEED))
    _vt, s, _xt = so.truncated_svd(X, SVD_K, m.config.n_iter, q0)
    assert np.abs(m.singular_values_ / s - 1).max() < SV_TOL


@pytest.mark.parametrize("n", [100, 1024])
def test_svd_recommend_is_score_matrix_topn(svd_model, query_call, n):
    """``recommend_batch(exclude="query")`` over the 32,768-query call; the sampled queries against ``argtopn`` of
    their ``score_matrix`` columns with the history set to NaN.  An unknown user gets an empty list."""
    m = svd_model["m"]
    queries, pos, labels = query_call
    recs = m.recommend_batch(queries, n, exclude="query")
    assert len(recs) == QUERIES
    sample = [queries[p] for p in pos]
    S = m.score_matrix(sample).cpu().numpy()
    for b, (p, label, q) in enumerate(zip(pos, labels, sample)):
        col = S[:, b].copy()
        if q.query_items is not None:
            nums = q.query_items.numbers(vocabulary=m.items, missing="negative")
            col[nums[nums >= 0]] = np.nan
        want = oracle.argtopn(col, n)
        assert np.array_equal(recs[p].numbers(), want), f"{label} at position {p}"
        assert np.array_equal(_bits(recs[p].scores()), _bits(col[want])), f"{label} at position {p}"
    assert len(recs[pos[labels.index("unknown")]]) == 0
