"""
NMF on the device: ``lk_nmf_cd_sweep`` and ``lk_f32_seq_sum`` bit for bit against scikit-learn's sweep and NumPy's
sequential sum, one device iteration against the host restatement, training against ``non_negative_factorization``
under the same seed (both SVD orientations, and the random initialisation), and the batched scoring interface.
"""

import pickle
import warnings

import numpy as np
import pytest
import scipy.sparse as sps
import torch

import nmf_oracle as no
import oracle
import test_nmf as host
from lkpy_b200 import engine, nmf
from lkpy_b200.components import Dataset, ItemList, RecQuery
from lkpy_b200.nmf import NMFConfig, NMFScorer

pytestmark = pytest.mark.gpu

#: ML-25M's user and item counts
ML25M_ROWS = (162_541, 59_047)


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def device_sweep(W, HHt, XHt):
    w = dev(W)
    pg = torch.empty((W.shape[1], W.shape[0]), dtype=torch.float32, device="cuda")
    engine.nmf_cd_sweep(w, dev(HHt), dev(XHt), pg)
    v = engine.f32_seq_sum([pg.view(-1)]).cpu().numpy()[0]
    return w.cpu().numpy(), pg.cpu().numpy(), v


@pytest.mark.parametrize("k", host.SWEEP_K)
def test_sweep_is_sklearn(k):
    cdnmf = pytest.importorskip("sklearn.decomposition._cdnmf_fast")
    W, HHt, XHt = host.sweep_case(k)
    theirs = W.copy()
    v = cdnmf._update_cdnmf_fast(theirs, HHt, XHt, np.arange(k, dtype=np.intp))
    w, pg, dv = device_sweep(W, HHt, XHt)
    assert np.array_equal(_bits(w), _bits(theirs))
    assert host.same_bits(dv, v)
    ref = W.copy()
    assert np.array_equal(_bits(pg), _bits(no.cd_sweep(ref, HHt, XHt)))


@pytest.mark.parametrize("n", ML25M_ROWS)
def test_sweep_at_ml25m_rows(n):
    cdnmf = pytest.importorskip("sklearn.decomposition._cdnmf_fast")
    W, HHt, XHt = host.sweep_case(64, n=n, seed=n)
    theirs = W.copy()
    v = cdnmf._update_cdnmf_fast(theirs, HHt, XHt, np.arange(64, dtype=np.intp))
    w, _pg, dv = device_sweep(W, HHt, XHt)
    assert np.array_equal(_bits(w), _bits(theirs))
    assert host.same_bits(dv, v)


def test_seq_sum_adversarial():
    cases = host.adversarial_sums()
    xs = [dev(x) if len(x) else torch.empty(0, device="cuda") for x in cases.values()]
    got = []
    for i in range(0, len(xs), 8):  # at most 8 sums per call, run concurrently
        got += list(engine.f32_seq_sum(xs[i : i + 8]).cpu().numpy())
    with np.errstate(over="ignore", invalid="ignore"):
        for (name, x), g in zip(cases.items(), got):
            assert host.same_bits(g, host.cumsum_f32(x)), name


def test_seq_sum_ten_million():
    x = host.violation_like()
    y = host.violation_like(3_800_000, seed=12)
    got = engine.f32_seq_sum([dev(x), dev(y)]).cpu().numpy()
    assert host.same_bits(got[0], host.cumsum_f32(x)) and host.same_bits(got[1], host.cumsum_f32(y))


def indicator(users, items, n_rows, n_cols):
    return sps.csr_matrix((np.ones(len(users), np.float32), (users, items)), shape=(n_rows, n_cols))


def test_iteration_is_the_restatement(ml_small):
    """One device iteration from the same W and H: the Grams (f64, rounded once) and everything after them match the
    host restatement bit for bit."""
    X = indicator(ml_small.users, ml_small.items, ml_small.n_users, ml_small.n_items)
    x = nmf.indicator_operand(ml_small.users, ml_small.items, ml_small.n_users, ml_small.n_items, "cuda")
    rng = np.random.default_rng(4)
    W = np.abs(rng.standard_normal((X.shape[0], 32))).astype(np.float32) * np.float32(0.1)
    H = np.abs(rng.standard_normal((32, X.shape[1]))).astype(np.float32) * np.float32(0.1)
    d = engine.NmfDescent(x, dev(W), dev(H.T), 0.5, 0.25, 2.0, 1.0)
    v_W, v_H = d.iteration()
    Wh, Hth = W.copy(), np.ascontiguousarray(H.T)
    XT = sps.csr_matrix(X.T)
    assert np.array_equal(_bits(engine.nmf_gram(dev(Hth)).cpu().numpy()), _bits(no.gram(Hth)))
    want_W = no.cd_half(X, Wh, Hth, 0.5, 2.0)
    want_H = no.cd_half(XT, Hth, Wh, 0.25, 1.0)
    assert np.array_equal(_bits(d.W.cpu().numpy()), _bits(Wh))
    assert np.array_equal(_bits(d.Ht.cpu().numpy()), _bits(Hth))
    assert host.same_bits(v_W, want_W) and host.same_bits(v_H, want_H)


def rel(a, b) -> float:
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def against_sklearn(users, items, n_rows, n_cols, k, seed=5):
    """The device factorisation and scikit-learn's under the same seed, with the global states after each."""
    skd = pytest.importorskip("sklearn.decomposition")
    X = indicator(users, items, n_rows, n_cols)
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        W, H, n_iter = skd.non_negative_factorization(X, n_components=k)
    their_state = np.random.get_state()
    order = np.lexsort((items, users))
    x = nmf.indicator_operand(users[order], items[order], n_rows, n_cols, "cuda")
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dW, dH, d_iter = nmf.factorize(x, NMFConfig(embedding_size=k))
    our_state = np.random.get_state()
    assert np.array_equal(our_state[1], their_state[1]) and our_state[2] == their_state[2]
    return (W, H, n_iter), (dW.cpu().numpy(), dH.cpu().numpy(), d_iter)


# Measured on an H100 against scikit-learn 1.9.0 on ml-latest-small under seed 5 (relative Frobenius; the iteration
# counts were equal in every case):
#   wide, k = 16: W 3.0e-5, H 3.1e-5, W H 2.2e-6      tall, k = 16: W 2.7e-5, H 3.6e-5, W H 2.3e-5
#   wide, k = 64: W 2.8e-3, H 3.7e-3, W H 2.1e-3      tall, k = 64: W 1.9e-4, H 1.7e-4, W H 1.2e-4
# The differences start in the initialisation (cuSOLVER's SVD for LAPACK's) and the Grams (f64, rounded once), and
# grow over the iterations; the bounds leave a factor of about three over the largest.
FACTOR_TOL = 1e-2
PRODUCT_TOL = 6e-3


@pytest.mark.parametrize("k", [16, 64])
@pytest.mark.parametrize("tall", [False, True])
def test_factorize_is_non_negative_factorization(ml_small, k, tall):
    """Wide ml-latest-small (users as rows: the transposed SVD) and tall (items as rows: the ML-25M case)."""
    u, i, nu, ni = ml_small.users, ml_small.items, ml_small.n_users, ml_small.n_items
    if tall:
        u, i, nu, ni = i, u, ni, nu
    (W, H, n_iter), (dW, dH, d_iter) = against_sklearn(u, i, nu, ni, k)
    errs = rel(dW, W), rel(dH, H), rel(dW.astype(np.float64) @ dH, W.astype(np.float64) @ H)
    print(f"k={k} tall={tall}: n_iter {d_iter} vs {n_iter}; W {errs[0]:.2e} H {errs[1]:.2e} WH {errs[2]:.2e}")
    assert d_iter == n_iter
    assert errs[0] < FACTOR_TOL and errs[1] < FACTOR_TOL and errs[2] < PRODUCT_TOL


def test_random_initialisation():
    """k above min(n_rows, n_cols): scikit-learn's ``"random"`` initialisation, drawn from the global state."""
    rng = np.random.default_rng(9)
    users = np.repeat(np.arange(12), 5)
    items = np.concatenate([rng.choice(40, 5, replace=False) for _ in range(12)])
    (W, H, n_iter), (dW, dH, d_iter) = against_sklearn(users, items, 12, 40, 16)
    assert d_iter == n_iter
    assert rel(dW.astype(np.float64) @ dH, W.astype(np.float64) @ H) < 1e-4


def test_max_iter_warns(ml_small):
    with pytest.warns(UserWarning, match="Maximum number of iterations 3"):
        NMFScorer(embedding_size=8, max_iter=3).train(Dataset(ml_small))


def test_scorer_batched_interface(ml_small):
    ds = Dataset(ml_small)
    np.random.seed(3)
    m = NMFScorer(embedding_size=16)
    m.train(ds)
    assert m.user_components.shape == (ml_small.n_users, 16) and m.item_components.shape == (ml_small.n_items, 16)
    assert m.user_components.dtype == np.float32 and (m.user_components >= 0).all() and m.n_iter_ > 1
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
    assert np.isnan(scored[-1].scores()).all()  # unknown user, with or without a history
    assert np.isnan(m(RecQuery(-999, ds.user_history(5)), targets[0]).scores()).all()
    for b, u in ((0, 0), (2, 77)):  # W[u] . H[:, i], one f32 FMA chain against the f64 product
        want = m.item_components.astype(np.float64) @ m.user_components[u]
        assert np.allclose(S[:, b], want, rtol=1e-5, atol=1e-6)
    m2 = pickle.loads(pickle.dumps(m))
    assert np.array_equal(m2.user_components, m.user_components) and m2.n_iter_ == m.n_iter_
    assert np.array_equal(_bits(m2.score_matrix(queries[:2]).cpu().numpy()), _bits(S[:, :2]))
