"""
BiasedSVD on the device: ``lk_spmm`` and the residual matrix bit for bit against tests/svd_oracle.py, ``train`` against
the reference's recordings (tests/golden/reference_classes/biased_svd_k*.npz) and against the restatement on a tall
matrix, the reference test's 3 x 3 case, and the batched scoring interface.
"""

import pickle

import numpy as np
import pytest
import scipy.sparse as sps
import torch

import basic_oracle as bo
import oracle
import svd_oracle as so
import svd_ref_sandbox as srs
import test_svd as host
from lkpy_b200 import engine, svd
from lkpy_b200.basic import BiasModel
from lkpy_b200.components import Dataset, ItemList, RecQuery
from lkpy_b200.data import InteractionCSR, Interactions
from lkpy_b200.svd import BiasedSVDScorer

pytestmark = pytest.mark.gpu
# cuSOLVER's LU, QR and SVD stand in for SciPy's LAPACK (f32 both): the factors agree to rounding only
SV_TOL, SCORE_TOL, VT_TOL = 1e-4, 1e-4, 1e-3


def _device_csr(m) -> engine.DeviceCSR:
    m = sps.csr_array(m)
    m.sort_indices()
    return engine.DeviceCSR.from_host(InteractionCSR.from_scipy(m))


def _bits(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _test_matrix() -> sps.csr_array:
    """300 x 3000 with empty rows, short rows and one row of every column (a long row, walked by several warps
    when W > 32)."""
    rng = np.random.default_rng(5)
    lens = rng.integers(0, 40, 300)
    lens[::17] = 0
    lens[123] = 3000
    rows = np.repeat(np.arange(300), lens)
    cols = np.concatenate([np.sort(rng.choice(3000, n, replace=False)) for n in lens])
    vals = rng.standard_normal(len(rows)).astype(np.float32)
    return sps.csr_array((vals, (rows, cols)), shape=(300, 3000))


@pytest.mark.parametrize("W", [1, 17, 64, 74, 138])
def test_spmm_is_the_restatement(ml_small, W):
    _bias, X = host.ml_residuals(ml_small)
    rng = np.random.default_rng(W)
    for m in (X, sps.csr_array(X.T), _test_matrix(), sps.csr_array(_test_matrix().T)):
        dm = _device_csr(m)
        d = rng.standard_normal((m.shape[1], W)).astype(np.float32)
        got = engine.spmm(dm, engine.spmm_order(dm), torch.from_numpy(d).cuda()).cpu().numpy()
        want = so.spmm(dm.h_indptr, dm.indices.cpu().numpy(), dm.values.cpu().numpy(), d)
        assert np.array_equal(_bits(got), _bits(want))


def test_residual_matrix_is_step_two(ml_small):
    bias, X = host.ml_residuals(ml_small)
    x = svd.residual_operand(bias, ml_small, torch.device("cuda"))
    XT = sps.csr_array(X.T)
    XT.sort_indices()
    for dm, want in ((x.rows, X), (x.cols, XT)):
        assert np.array_equal(dm.h_indptr, want.indptr) and np.array_equal(dm.indices.cpu().numpy(), want.indices)
        assert np.array_equal(_bits(dm.values.cpu().numpy()), _bits(want.data))


def _rel(a, b) -> float:
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _golden_queries(ml_small):
    out = []
    for uid, hist, ratings in srs.queries(ml_small):
        out.append(RecQuery(uid, None if hist is None else ItemList(item_ids=hist, rating=ratings)))
    return out


@pytest.mark.parametrize("k", host.GOLDEN_K)
def test_train_follows_the_reference(ml_small, k):
    g = host.reference_golden(ml_small, k)
    np.random.seed(srs.SEED)
    m = BiasedSVDScorer(embedding_size=k)
    m.train(Dataset(ml_small))
    state = np.random.get_state()
    assert np.array_equal(state[1], g["state_keys"]) and state[2] == g["state_pos"]
    assert np.array_equal([state[3], state[4]], g["state_gauss"])
    assert m.components_.shape == (k, ml_small.n_items) and m.user_components.shape == (ml_small.n_users, k)
    assert m.components_.dtype == m.user_components.dtype == m.singular_values_.dtype == np.float32
    assert np.array_equal(m.bias.user_biases, g["user_biases"]) and np.array_equal(m.bias.item_biases, g["item_biases"])
    assert np.abs(m.singular_values_ / g["singular_values"] - 1).max() < SV_TOL
    assert np.abs(m.components_[:, srs.ROWS_I] - g["components"]).max() < VT_TOL
    assert _rel(m.user_components[srs.ROWS_U], g["user_components"]) < VT_TOL
    items = ItemList(item_ids=srs.score_item_ids(ml_small))
    got = np.stack([m(q, items).scores() for q in _golden_queries(ml_small)])
    want = g["scores"]
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.isnan(got[-2]).all() and np.isnan(got[:, -1]).all()  # unknown user, unknown item
    ok = ~np.isnan(want)
    assert np.abs(got[ok] / want[ok] - 1).max() < SCORE_TOL


def _swapped(ml_small) -> Interactions:
    """ml-latest-small with the roles swapped: 9,066 users and 671 items, a tall matrix (not transposed)."""
    order = np.lexsort((ml_small.users, ml_small.items))
    return Interactions(ml_small.items[order], ml_small.users[order], ml_small.ratings[order], ml_small.n_items,
                        ml_small.n_users, ml_small.item_ids, ml_small.user_ids)  # fmt: skip


@pytest.mark.parametrize("n_iter", [2, 5])
def test_tall_matrix_follows_the_restatement(ml_small, n_iter):
    it = _swapped(ml_small)
    k = 16
    np.random.seed(7)
    m = BiasedSVDScorer(embedding_size=k, n_iter=n_iter, damping={"user": 2.0, "item": 4.0})
    m.train(Dataset(it))
    bias = BiasModel.learn(it, (2.0, 4.0), np.float32)
    X = so.residuals(it.users, it.items, it.ratings, it.n_users, it.n_items, bias.global_bias, bias.item_biases,
                     bias.user_biases)  # fmt: skip
    vt, s, xt = so.truncated_svd(X, k, n_iter, so.start_matrix(X.shape, k, np.random.RandomState(7)))
    assert np.abs(m.singular_values_ / s - 1).max() < SV_TOL
    assert np.abs(m.components_ - vt).max() < VT_TOL
    assert _rel(m.user_components, xt) < VT_TOL


def test_reference_three_by_three_case():
    """The reference's own test data: 3 users x 3 items with ``features=2``, where k + 10 exceeds both sides and
    the LU shrinks the basis."""
    # (item, user, rating) = (1, 10, 4), (1, 12, 3), (2, 10, 5), (3, 13, 2), numbered and sorted by (user, item)
    it = Interactions(np.array([0, 0, 1, 2], np.int32), np.array([0, 1, 0, 2], np.int32),
                      np.array([4.0, 5.0, 3.0, 2.0], np.float32), 3, 3, np.array([10, 12, 13]), np.array([1, 2, 3]))  # fmt: skip
    ds = Dataset(it)
    m = BiasedSVDScorer(features=2, damping=0)
    m.train(ds)
    assert m.user_components.shape == (3, 2) and m.components_.shape == (2, 3)
    s = m(10, ItemList(item_ids=[3])).scores()
    assert len(s) == 1 and 0 <= s[0] <= 5
    assert np.isnan(m(10, ItemList(item_ids=[4])).scores()).all()
    assert np.isnan(m(50, ItemList(item_ids=[3])).scores()).all()


def test_scorer_batched_interface_against_host_bias(ml_small):
    ds = Dataset(ml_small)
    np.random.seed(3)
    m = BiasedSVDScorer(embedding_size=16)
    m.train(ds)
    users = (0, 5, 77, 300)
    uids = [ds.users.id(u) for u in users]
    queries = [RecQuery(uids[0], None), RecQuery(uids[1], ds.user_history(5))]
    queries += [RecQuery(uid, ds.user_history(u)) for uid, u in zip(uids[2:], users[2:])] + [RecQuery(-999, None)]
    S = m.score_matrix(queries).cpu().numpy()
    assert np.isnan(S[:, -1]).all() and not np.isnan(S[:, :-1]).any()
    for exclude in (None, "query"):
        recs = m.recommend_batch(queries, 25, exclude=exclude)
        assert len(recs[-1]) == 0
        for b, rec in enumerate(recs[:-1]):
            col = S[:, b].copy()
            if exclude == "query" and queries[b].query_items is not None:
                col[queries[b].query_items.numbers(vocabulary=m.items)] = np.nan
            want = oracle.argtopn(col, 25)
            assert np.array_equal(rec.numbers(), want)
            assert np.array_equal(_bits(rec.scores()), _bits(col[want]))
    targets = [ItemList(item_ids=np.concatenate([ds.items.ids()[b::7], [-5]])) for b in range(len(queries))]
    scored = m.score_batch(queries, targets)
    for b, (tgt, out) in enumerate(zip(targets, scored)):
        s = out.scores()
        assert np.isnan(s[-1])  # unknown item
        nums = tgt.numbers(vocabulary=m.items, missing="negative")[:-1]
        assert np.array_equal(_bits(s[:-1]), _bits(S[nums, b]))
        assert np.array_equal(_bits(m(queries[b], tgt).scores()), _bits(s))
    assert np.isnan(scored[-1].scores()).all()  # unknown user
    # the score chain: user components . item components (f32 FMA chain), + (f32(g) + ib), + user bias
    ib = (m.bias.item_biases + m.bias.global_bias).astype(np.float32)
    for b, u in ((0, 0), (2, 77)):
        ub = m.bias.user_biases[u] if b == 0 else bo.rated_user_bias(m.bias, m.items, queries[b].query_items)
        want = (m.components_.T.astype(np.float64) @ m.user_components[u] + ib) + np.float32(ub)
        assert np.allclose(S[:, b], want, rtol=1e-5, atol=1e-5)
    m2 = pickle.loads(pickle.dumps(m))
    assert np.array_equal(m2.user_components, m.user_components) and m2.bias.global_bias == m.bias.global_bias
    assert np.array_equal(_bits(m2.score_matrix(queries[:2]).cpu().numpy()), _bits(S[:, :2]))


def test_spmm_rejects_a_mismatched_operand():
    dm = _device_csr(_test_matrix())
    with pytest.raises(ValueError):
        engine.spmm(dm, engine.spmm_order(dm), torch.zeros((10, 4), device="cuda"))
