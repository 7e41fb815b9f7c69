"""
BiasScorer and PopScorer on the device: ``lk_bias_learn`` bit for bit against the host statements
(``basic.BiasModel.learn``), ``lk_offset_score_batch`` rankings against the host composition (``__call__``, exclusion,
``argtopn``), and the trained scorers against the recordings of the reference's own classes.
"""

import math
import pickle

import numpy as np
import pytest

import basic_oracle as bo
import basic_ref_sandbox as brs
from lkpy_b200 import basic, engine
from lkpy_b200.basic import BiasModel
from lkpy_b200.basic import BiasScorer, PopScorer
from lkpy_b200.components import Dataset, ItemList, RecQuery, TrainingOptions
from lkpy_b200.data import Interactions
from test_basic import our_queries, reference_golden

pytestmark = pytest.mark.gpu

DAMPINGS = [0.0, 5, 0.1, (3.0, 0.5), {"user": 2.5}, {"item": 0.1}]
ENTITIES = [("user", "item"), ("user",), ("item",)]


@pytest.fixture(scope="module")
def skewed():
    """120 k users and 3,000 items (plus 4 items and 3 users without ratings); item 17 has 100 k ratings, the other
    ratings follow a skewed item draw.  Ratings are halves with a noise term, so that sums round."""
    rng = np.random.default_rng(7)
    n_users, n_items = 120_003, 3_004
    heavy = np.sort(rng.choice(120_000, 100_000, replace=False))
    u = rng.integers(0, 120_000, 400_000)
    i = np.minimum(rng.zipf(1.3, 400_000), 2_999)
    keys = np.unique(np.concatenate([u * n_items + i, heavy * n_items + 17]))
    users, items = (keys // n_items).astype(np.int32), (keys % n_items).astype(np.int32)
    r = (rng.integers(1, 11, len(keys)) * 0.5 + rng.standard_normal(len(keys)) * 1e-3).astype(np.float32)
    assert (items == 17).sum() >= 100_000
    return Interactions(users, items, r, n_users, n_items)


@pytest.fixture(scope="module")
def cancelling(skewed):
    """``skewed``'s users and items with ``bo.cancelling_ratings``: the learner input on which the order of the
    entity chains shows in the f32 biases, with f64 and with f32 centring."""
    it = Interactions(skewed.users, skewed.items, bo.cancelling_ratings(skewed, np.random.default_rng(8)),
                      skewed.n_users, skewed.n_items)  # fmt: skip
    for dtype in (np.float64, np.float32):
        items_changed, users_changed = bo.reversed_chain_changes(it, dtype)
        assert items_changed > 1000 and users_changed > 1000, (dtype, items_changed, users_changed)
    return it


def check_same(dev: BiasModel, host: BiasModel) -> None:
    assert dev.global_bias == host.global_bias and dev.damping == host.damping
    for a, b in ((dev.item_biases, host.item_biases), (dev.user_biases, host.user_biases)):
        assert (a is None) == (b is None)
        if a is not None:
            assert a.dtype == np.float32 and np.array_equal(a.view(np.int32), b.view(np.int32))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("damping", DAMPINGS, ids=str)
@pytest.mark.parametrize("entities", ENTITIES, ids="+".join)
@pytest.mark.parametrize("which", ["ml_small", "skewed", "cancelling"])
def test_learn_is_the_host_statements(request, which, entities, damping, dtype):
    it = request.getfixturevalue(which)
    dev = basic.learn(Dataset(it), damping, entities=set(entities), centered_dtype=dtype)
    pair = basic.damping_pair(damping)
    check_same(dev, BiasModel.learn(it, pair, dtype, entities))


@pytest.mark.parametrize("n", [1, 8, 9, 128, 129, 2**20 + 3, 2**23, 2**23 + 8, 25_000_095, 2**27 + 3])
def test_learn_mean_on_awkward_lengths(n):
    """Up to 2^20 + 3 every depth-16 subtree is a leaf reached at depth 13 or above.  At 2^23 each of the 2^16
    subtrees holds exactly 128 values; at 2^23 + 8 some walkers recurse one level; 25,000,095 is the benchmark's
    count; at 2^27 + 3 every walker recurses four levels or more, and every combine level has inner nodes.

    The ratings are halves with a noise term and a random sign.  With positive ratings only, the total is so much
    larger than the rounding of the partial sums that every order gives the same bits; with signs the total is a
    small difference of large partial sums, and the exact sum rounded once differs from NumPy's."""
    rng = np.random.default_rng(n)
    users = np.sort(rng.integers(0, max(n // 50, 1), n)).astype(np.int32)
    items = rng.integers(0, 1000, n).astype(np.int32)
    r = (rng.integers(1, 11, n) * 0.5 + rng.standard_normal(n) * 0.01).astype(np.float32)
    r = np.where(rng.random(n) < 0.5, -r, r)
    it = Interactions(users, items, r, int(users.max()) + 1, 1000)  # COO order by user is all the mean needs
    m = basic.learn(Dataset(it), 0.0, entities=set())
    want = np.mean(r)
    assert np.float32(m.global_bias).view(np.int32) == want.view(np.int32)
    if n >= 2**20:
        # the input tells summation orders apart: the exact sum rounded once gives other bits
        exact = np.float32(np.float64(np.float32(math.fsum(r.astype(np.float64)))) / n)
        assert exact.view(np.int32) != want.view(np.int32)
    if n >= 2**23:
        sizes = np.array([bo.mean_node(n, bo.MEAN_DEPTH, p)[1] for p in range(1 << bo.MEAN_DEPTH)])
        assert sizes.sum() == n
        if n == 2**23:
            assert (sizes == 128).all()
        else:
            assert sizes.max() > 128  # the walkers' pairwise sums recurse
        if n >= 2**27:
            assert sizes.min() >= 2048  # four levels or more below the cut


def trained_bias(ml_small, **cfg) -> BiasScorer:
    m = BiasScorer(**cfg)
    m.train(Dataset(ml_small))
    return m


def query_set(ml_small):
    """Known users, unknown users, and queries carrying ratings (one of them all NaN)."""
    qs = [RecQuery(ml_small.user_ids[u], None) for u in range(0, ml_small.n_users, 37)]
    qs += [RecQuery(-5, None), RecQuery(None, None)]
    rows = np.flatnonzero(ml_small.users == 3)
    ids = np.append(ml_small.item_ids[ml_small.items[rows]], -77)
    qs.append(RecQuery(ml_small.user_ids[3], ItemList(item_ids=ids, rating=np.append(ml_small.ratings[rows], 4.0))))
    qs.append(RecQuery(-5, ItemList(item_ids=ids[:5], rating=np.full(5, np.nan, np.float32))))
    qs.append(RecQuery(None, ItemList(item_ids=ids[:7])))  # a history without ratings: excluded, no fold-in
    return qs


def history_nums(q, items) -> np.ndarray:
    return np.zeros(0, np.int32) if q.query_items is None else q.query_items.numbers(vocabulary=items, missing="negative")


def check_ranking(recs, host_scores, queries, items, n: int, exclude: bool = True) -> None:
    for r, s, q in zip(recs, host_scores, queries):
        idx, val = bo.ranked(s, history_nums(q, items) if exclude else [], n)
        assert np.array_equal(r.numbers(), idx)
        assert np.array_equal(r.scores().view(np.int32), val.view(np.int32))


@pytest.mark.parametrize("cfg", [{}, {"damping": 5.0}, {"damping": {"user": 2.0}}, {"entities": {"item"}},
                                 {"entities": {"user"}, "damping": 0.3}], ids=str)  # fmt: skip
@pytest.mark.parametrize("n", [1, 10, 100, 1024])
def test_bias_recommend_is_the_host_composition(ml_small, cfg, n):
    m = trained_bias(ml_small, **cfg)
    qs = query_set(ml_small)
    all_items = ItemList(item_nums=np.arange(ml_small.n_items), vocabulary=m.items)
    host = [bo.bias_scores(m.model, m.users, m.items, q, all_items) for q in qs]
    check_ranking(m.recommend_batch(qs, n), host, qs, m.items, n)
    check_ranking(m.recommend_batch(qs, n, exclude=None), host, qs, m.items, n, exclude=False)


def test_bias_scores_unknown_items_and_users(ml_small):
    m = trained_bias(ml_small, damping=5.0)
    qs = query_set(ml_small)
    targets = [ItemList(item_ids=np.append(ml_small.item_ids[::13], [-1, -2])) for _ in qs]
    got = m.score_batch(qs, targets)
    for q, t, r in zip(qs, targets, got):
        want = bo.bias_scores(m.model, m.users, m.items, q, t)
        assert not np.isnan(want).any() and np.array_equal(r.scores().view(np.int32), want.view(np.int32))
    one = m(qs[-3], targets[0])
    assert np.array_equal(one.scores(), got[-3].scores())


@pytest.mark.parametrize("mode", brs.POP_SCORES)
@pytest.mark.parametrize("n", [1, 50, 1024])
def test_pop_recommend_is_the_host_composition(ml_small, mode, n):
    """Count scores are mostly ties: the heap decides which tied items are kept, and in what order."""
    m = PopScorer(score=mode)
    m.train(Dataset(ml_small))
    counts = np.bincount(ml_small.items, minlength=ml_small.n_items)
    if mode == "count":
        assert np.array_equal(m.item_scores, counts.astype(np.float32))
    qs = query_set(ml_small)
    check_ranking(m.recommend_batch(qs, n), [m.item_scores] * len(qs), qs, m.items, n)
    t = ItemList(item_ids=np.append(ml_small.item_ids[:40], -3))
    s = m.score_batch([qs[0]], [t])[0].scores()
    assert np.array_equal(s, m(t).scores(), equal_nan=True) and np.isnan(s[-1])


def test_n_beyond_the_candidates(ml_small):
    """``n`` larger than the catalogue: every candidate is listed, exclusions left out."""
    small = Interactions(ml_small.users[:300], ml_small.items[:300] % 50, ml_small.ratings[:300],
                         int(ml_small.users[299]) + 1, 50)  # fmt: skip
    for m in (BiasScorer(damping=1.0), PopScorer(score="count")):
        m.train(Dataset(small))
        qs = [RecQuery(1, ItemList(item_nums=np.array([3, 4, 4, 9], np.int32), vocabulary=m.items)), RecQuery(2, None)]
        recs = m.recommend_batch(qs, 80)
        assert [len(r) for r in recs] == [47, 50]
        all_items = ItemList(item_nums=np.arange(50), vocabulary=m.items)
        host = [bo.bias_scores(m.model, m.users, m.items, q, all_items) if isinstance(m, BiasScorer) else m.item_scores
                for q in qs]  # fmt: skip
        check_ranking(recs, host, qs, m.items, 80)


def test_pickle_and_retrain(ml_small):
    for m in (trained_bias(ml_small, damping=5.0), PopScorer(score="quantile")):
        if not m.is_trained():
            m.train(Dataset(ml_small))
        qs = query_set(ml_small)
        before = m.recommend_batch(qs, 20)
        m2 = pickle.loads(pickle.dumps(m))
        assert "_d_base" not in m2.__dict__
        for a, b in zip(before, m2.recommend_batch(qs, 20)):
            assert np.array_equal(a.numbers(), b.numbers()) and np.array_equal(a.scores(), b.scores())
        m2.train(Dataset(Interactions(ml_small.users[:10], ml_small.items[:10], ml_small.ratings[:10], 1, 9066)),
                 TrainingOptions(retrain=False))  # fmt: skip
        assert np.array_equal(m2.recommend_batch(qs[:1], 5)[0].numbers(), before[0].numbers()[:5])


@pytest.mark.parametrize("name", list(brs.BIAS_CONFIGS))
def test_bias_scorer_is_the_reference(ml_small, name):
    g = reference_golden(f"basic_bias_{name}", ml_small)
    m = trained_bias(ml_small, **brs.BIAS_CONFIGS[name])
    assert m.model.global_bias == float(g["global_bias"])
    if m.model.item_biases is not None:
        assert np.array_equal(m.model.item_biases.view(np.int32), g["item_biases"].view(np.int32))
    if m.model.user_biases is not None:
        assert np.array_equal(m.model.user_biases.view(np.int32), g["user_biases"].view(np.int32))
    targets = ItemList(item_ids=brs.score_item_ids(ml_small))
    qs = our_queries(ml_small, m.items)
    for r, want in zip(m.score_batch(qs, [targets] * len(qs)), g["scores"]):
        assert np.array_equal(r.scores().view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("mode", ["rank", "count"])
def test_pop_scorer_is_the_reference(ml_small, mode):
    g = reference_golden(f"basic_pop_{mode}", ml_small)
    m = PopScorer(score=mode)
    m.train(Dataset(ml_small))
    assert np.array_equal(m.item_scores.view(np.int32), g["item_scores"].view(np.int32))
    got = m(ItemList(item_ids=brs.score_item_ids(ml_small))).scores()
    assert np.array_equal(got, g["scores"], equal_nan=True)


def test_offset_scores_match_numpy_in_f64(ml_small):
    """``f32 += f64`` under NEP 50: computed in f64, rounded once — including offsets an f32 add would round."""
    import torch

    rng = np.random.default_rng(3)
    base = (rng.standard_normal(5000) * 3).astype(np.float32)
    off = rng.standard_normal(70) * 1e-3 + rng.standard_normal(70)
    S = engine.offset_scores(torch.from_numpy(base).cuda(), 70, torch.from_numpy(off)).cpu().numpy()
    for q in range(70):
        want = base.copy()
        want += off[q]
        assert np.array_equal(S[q].view(np.int32), want.view(np.int32))
