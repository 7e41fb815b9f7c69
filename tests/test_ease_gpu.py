"""
EASE on the GPU: training bit for bit against the reference's statements run with torch on the same device, and
scoring and top-n bit for bit against ``tests/ease_oracle.py``.
"""

import pickle

import numpy as np
import pytest
import torch

import ease_oracle as eo
import oracle
from lkpy_b200 import data
from lkpy_b200.components import Dataset, ItemList, Vocabulary
from lkpy_b200.ease import EASEScorer

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def trained(ml_small):
    m = EASEScorer(regularization=2.5)
    m.train(Dataset(ml_small))
    return m


def _synth_scorer(W: np.ndarray) -> EASEScorer:
    """A scorer around a given weight matrix, as after unpickling."""
    m = EASEScorer()
    m.items = Vocabulary(np.arange(W.shape[0]) + 1000, "item")
    m._weights_host = W
    return m


def test_train_matches_reference_statements(cuda_lib, ml_small, trained):
    it = ml_small
    cooc = eo.gram(it.n_users, it.n_items, it.users, it.items, 2.5)
    want = eo.normalise(eo.invert_torch(cooc.copy(), "cuda"))
    got = trained.weights
    assert got.dtype == np.float32 and got.shape == (it.n_items, it.n_items)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    # and close to the f64 inverse: the f32 Cholesky's norm-wise error is of order kappa * eps_f32
    ref = np.linalg.inv(cooc.astype(np.float64))
    ref = ref / -np.diag(ref).reshape(1, -1)
    np.fill_diagonal(ref, 0)
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    print(f"ml-latest-small: weights vs f64 inverse, relative Frobenius error {err:.3g}")
    assert err < 1e-2
    assert trained.is_trained() and len(trained.items) == it.n_items


def test_train_scipy_solver(cuda_lib, ml_small, trained, monkeypatch):
    monkeypatch.setenv("LK_EASE_SOLVER", "scipy")
    m = EASEScorer(regularization=2.5)
    m.train(Dataset(ml_small))
    it = ml_small
    want = eo.normalise(eo.invert_scipy(eo.gram(it.n_users, it.n_items, it.users, it.items, 2.5)))
    assert np.array_equal(m.weights.view(np.int32), want.view(np.int32))


def _queries(ds, rng, n=30):
    it = ds.interactions
    qs = []
    for u in rng.choice(it.n_users, n, replace=False):
        nums = ds.user_history(int(u)).numbers()
        if len(nums) and u % 3 == 0:  # repeated history items count once
            nums = np.concatenate([nums, nums[: max(1, len(nums) // 3)]])
        qs.append(nums)
    qs.append(np.zeros(0, np.int32))  # empty history
    qs.append(np.array([0, 0, 0], np.int32))
    return qs


def test_score_batch(cuda_lib, ml_small, trained):
    ds = Dataset(ml_small)
    W = trained.weights
    rng = np.random.default_rng(1)
    qs = _queries(ds, rng)
    ids = ds.items.ids()
    unknown = ids.max() + 1
    hist = [ItemList(item_ids=np.concatenate([ids[q], [unknown]]) if len(q) else ids[q]) for q in qs]
    hist.append(ItemList(item_ids=np.array([unknown, unknown + 1])))  # no known history item
    tgt_nums = rng.integers(0, len(ids), 300)
    tgt = ItemList(item_ids=np.concatenate([ids[tgt_nums], [unknown]]))
    got = trained.score_batch(hist, [tgt] * len(hist))
    for q, g in zip(qs + [np.zeros(0, np.int32)], got):
        full = eo.score(W, q)
        want = np.concatenate([full[tgt_nums], [np.nan]]).astype(np.float32)
        s = g.scores()
        assert np.array_equal(np.isnan(s), np.isnan(want))
        ok = ~np.isnan(want)
        assert np.array_equal(s[ok].view(np.int32), want[ok].view(np.int32))
        if len(eo.history(q)):  # tolerance parity with the reference's BLAS GEMV
            blas = eo.score_blas(W, q)[tgt_nums]
            np.testing.assert_allclose(s[:-1], blas, rtol=0, atol=1e-5 * max(1.0, float(np.abs(blas).max())))
    one = trained(hist[0], tgt)
    assert np.array_equal(one.scores(), got[0].scores(), equal_nan=True)


def _check_recommend(m, W, qs, ns, exclude):
    hist = [ItemList(item_nums=q, vocabulary=m.items) for q in qs]
    n_items = W.shape[0]
    for n in ns:
        got = m.recommend_batch(hist, n, exclude=exclude)
        assert len(got) == len(qs)
        for q, g in zip(qs, got):
            s = eo.score(W, q).copy()
            if not len(eo.history(q)):
                assert len(g) == 0
                continue
            if exclude == "query":
                s[eo.history(q)] = np.nan
            want = oracle.argtopn(s, min(n, n_items))
            assert np.array_equal(g.numbers(), want), (n, exclude)
            assert np.array_equal(g.scores().view(np.int32), s[want].view(np.int32))


@pytest.mark.parametrize("exclude", ["query", None])
def test_recommend_batch(cuda_lib, ml_small, trained, exclude):
    ds = Dataset(ml_small)
    qs = _queries(ds, np.random.default_rng(2))
    _check_recommend(trained, trained.weights, qs, (1, 10, 100, 1024), exclude)


@pytest.mark.parametrize("exclude", ["query", None])
def test_recommend_batch_ties(cuda_lib, exclude):
    """Weights on a coarse grid, so that many scores tie and lists end inside runs of equal scores."""
    rng = np.random.default_rng(7)
    n_items = 2500
    W = (rng.integers(-2, 3, (n_items, n_items)) * 0.25).astype(np.float32)
    W[rng.random((n_items, n_items)) < 0.9] = 0.0
    m = _synth_scorer(W)
    qs = [rng.choice(n_items, k, replace=False) for k in (1, 2, 5, 40)] + [np.zeros(0, np.int64)]
    _check_recommend(m, W, qs, (1, 10, 100, 1024), exclude)
    # the cut falls inside a run of equal scores: the 100th and the 101st best tie
    cut_ties = [np.sort(eo.score(W, q))[::-1][99:101] for q in qs if len(q) > 1]
    assert any(t[0] == t[1] for t in cut_ties)


@pytest.mark.parametrize("n_items", [20_000, 20_003])  # float4 rows, and the scalar path of an unaligned width
def test_mid_size_shape(cuda_lib, n_items):
    """Twenty column tiles; histories of one item and of several thousand."""
    rng = np.random.default_rng(n_items)
    W = rng.standard_normal((n_items, n_items), dtype=np.float32)
    m = _synth_scorer(W)
    qs = [np.array([n_items - 1]), rng.choice(n_items, 4000, replace=False), rng.choice(n_items, 37),
          np.zeros(0, np.int64)]  # fmt: skip
    hist = [ItemList(item_nums=q, vocabulary=m.items) for q in qs]
    tgt = ItemList(item_nums=np.arange(n_items), vocabulary=m.items)
    for q, g in zip(qs, m.score_batch(hist, [tgt] * len(qs))):
        want = eo.score(W, q)
        assert np.array_equal(g.scores().view(np.int32), want.view(np.int32))
    _check_recommend(m, W, qs, (100, 1024), "query")


def test_pickle_round_trip(cuda_lib, ml_small, trained):
    ds = Dataset(ml_small)
    hist = [ds.user_history(3), ds.user_history(11)]
    a = trained.recommend_batch(hist, 20)
    m2 = pickle.loads(pickle.dumps(trained))
    assert "_state" not in pickle.loads(pickle.dumps(trained)).__dict__
    assert np.array_equal(m2.weights, trained.weights)
    b = m2.recommend_batch(hist, 20)
    for x, y in zip(a, b):
        assert np.array_equal(x.numbers(), y.numbers()) and np.array_equal(x.scores(), y.scores())


def test_train_on_synthetic_interactions(cuda_lib):
    """A width that is a multiple of 4 (the float4 scoring path on trained weights) and a retrain."""
    it = data.synth_interactions(1500, 1200, 40_000, seed=9)
    m = EASEScorer()
    m.train(Dataset(it))
    want = eo.train(it.n_users, it.n_items, it.users, it.items, 1.0, "cuda")
    assert np.array_equal(m.weights.view(np.int32), want.view(np.int32))
    q = np.unique(it.items[:50])
    got = m.score_batch([ItemList(item_nums=q, vocabulary=m.items)], [ItemList(item_nums=np.arange(1200),
                                                                              vocabulary=m.items)])[0]  # fmt: skip
    assert np.array_equal(got.scores().view(np.int32), eo.score(want, q).view(np.int32))
    torch.cuda.synchronize()
