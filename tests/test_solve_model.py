"""
NumPy model of the tf32 three-term split that als_tc.cu uses for fp32-accurate Grams on the tensor cores
(CPU only): operands split into tf32 `hi` (low 13 mantissa bits cleared) and `lo = x - hi` (truncated to
tf32 again by the MMA), products hi·hi + hi·lo + lo·hi accumulated in f32.  The model applies the split in
a harsher setting than the kernel's Gram: the rank-16 trailing updates of a blocked Cholesky (and a block
Gauss-Jordan variant), where its error compounds over every update.  No kernel factors that way; the
kernel's own accuracy is checked by the GPU tests.  What the model shows about the arithmetic: the
three-term split is as accurate as f32, a two-term split is not.
"""

import numpy as np
import pytest

f32 = np.float32
NB = 16


def _tf32(x: np.ndarray) -> np.ndarray:
    return (np.ascontiguousarray(x, dtype=f32).view(np.uint32) & np.uint32(0xFFFFE000)).view(f32)


def _xxt(X: np.ndarray, Y: np.ndarray, terms: int) -> np.ndarray:
    """X @ Y.T as the split MMAs deliver it (f32 accumulation)."""
    xh, yh = _tf32(X), _tf32(Y)
    xl, yl = _tf32(X - xh), _tf32(Y - yh)
    acc = (xh @ yh.T).astype(f32)
    if terms >= 2:
        acc = (acc + (xh @ yl.T).astype(f32)).astype(f32)
    if terms >= 3:
        acc = (acc + (xl @ yh.T).astype(f32)).astype(f32)
    return acc


def _chol_f32(A):
    return np.linalg.cholesky(A.astype(np.float64)).astype(f32)  # a 16x16 block: rounding once is the model


def _tri(L, B):  # X with X L^T = B
    return np.linalg.solve(L.astype(np.float64), B.T.astype(np.float64)).T.astype(f32)


def solve_blocked(A, y, terms=3, gauss_jordan=False):
    A = A.astype(f32).copy()
    y = y.astype(f32).copy()
    n = len(A)
    Ls, z = {}, np.zeros(n, f32)
    for j in range(0, n, NB):
        J = slice(j, j + NB)
        L = _chol_f32(A[J, J])
        Ls[j] = L
        zj = np.linalg.solve(L.astype(np.float64), y[J].astype(np.float64)).astype(f32)
        z[J] = zj
        rows = [w for w in range(0, n, NB) if (w != j if gauss_jordan else w > j)]
        X = np.zeros((n, NB), f32)
        for w in rows:
            X[w : w + NB] = _tri(L, A[w : w + NB, J])
            y[w : w + NB] = (y[w : w + NB] - X[w : w + NB] @ zj).astype(f32)
        c0 = j + NB
        if c0 < n:
            A[:, c0:] = (A[:, c0:] - _xxt(X, X[c0:], terms)).astype(f32)
        if not gauss_jordan:
            A[c0:, J] = X[c0:]  # L panel, read by the back substitution
    x = np.zeros(n, f32)
    if gauss_jordan:  # block-diagonal system left: L_jj L_jj^T x_j = y_j
        for j, L in Ls.items():
            t = np.linalg.solve(L.astype(np.float64), y[j : j + NB].astype(np.float64)).astype(f32)
            x[j : j + NB] = np.linalg.solve(L.T.astype(np.float64), t.astype(np.float64)).astype(f32)
        return x
    for j in range(n - NB, -1, -NB):  # block back substitution on z
        rhs = z[j : j + NB].astype(np.float64)
        for w in range(j + NB, n, NB):
            rhs -= A[w : w + NB, j : j + NB].T.astype(np.float64) @ x[w : w + NB]
        x[j : j + NB] = np.linalg.solve(Ls[j].T.astype(np.float64), rhs.astype(f32).astype(np.float64)).astype(f32)
    return x


def _system(rng, cond):
    Q, _ = np.linalg.qr(rng.standard_normal((64, 64)))
    lam = np.logspace(0, np.log10(cond), 64) * 0.1
    A = ((Q * lam) @ Q.T).astype(f32)
    A = ((A + A.T) / 2).astype(f32)
    return A, rng.standard_normal(64).astype(f32)


def _err(x, A, y):
    ref = np.linalg.solve(A.astype(np.float64), y.astype(np.float64))
    return float(np.linalg.norm(x - ref) / np.linalg.norm(ref))


def _lapack_f32(A, y):
    import scipy.linalg as sl

    return sl.cho_solve(sl.cho_factor(A.astype(f32), lower=True), y.astype(f32)).astype(f32)


@pytest.mark.parametrize("cond", [1e1, 1e3, 1e5])
def test_three_term_split_matches_f32_cholesky(cond):
    rng = np.random.default_rng(int(cond))
    e_model, e_gj, e_lapack, e_two = [], [], [], []
    for _ in range(12):
        A, y = _system(rng, cond)
        e_lapack.append(_err(_lapack_f32(A, y), A, y))
        e_model.append(_err(solve_blocked(A, y, 3), A, y))
        e_gj.append(_err(solve_blocked(A, y, 3, gauss_jordan=True), A, y))
        e_two.append(_err(solve_blocked(A, y, 2), A, y))
    m_l, m_m, m_g, m_2 = map(np.mean, (e_lapack, e_model, e_gj, e_two))
    # (the model truncates `lo` to tf32 as well, the harshest reading of the hardware)
    assert m_m < 5.0 * m_l + 1e-6, (m_m, m_l)  # f32-level accuracy
    assert m_g < 6.0 * m_l + 1e-6, (m_g, m_l)  # Gauss-Jordan: a small factor at most
    assert m_2 > 10.0 * m_m, (m_2, m_m)  # dropping lo.hi is a 2^-12 relative error per product: visible


def test_model_agrees_with_plain_solution_on_als_like_system():
    rng = np.random.default_rng(1)
    Q = (rng.standard_normal((3000, 64)) * 0.1).astype(f32)
    M = Q[rng.choice(3000, 150, replace=False)]
    A = ((Q.T @ Q + 0.1 * np.eye(64)) / 40.0 + M.T @ M).astype(f32)  # an implicit-ALS system scaled by 1 / v
    y = (41.0 / 40.0 * M.sum(0)).astype(f32)
    for gj in (False, True):
        assert _err(solve_blocked(A, y, 3, gauss_jordan=gj), A, y) < 5e-6
