"""
Restatements behind the BiasedSVD tests (host, NumPy and SciPy):

* ``spmm``: the sparse x dense product as ``lk_spmm`` defines it, one sequential f32 sum per output element over the
  row's stored entries, product and sum each rounded; SciPy's ``A @ D``, ``A.T @ D`` and ``D.T @ A`` equal it bit for
  bit (tests/test_svd.py);
* ``residuals``: step 2 of ``BiasedSVDScorer.train``, the f32 bias residuals as a SciPy CSR matrix;
* ``truncated_svd``: ``TruncatedSVD(k, algorithm="randomized", n_iter=n_iter).fit_transform`` from a given start matrix,
  statement for statement with scikit-learn's ``_randomized_range_finder`` / ``_randomized_svd`` / ``svd_flip``.
"""

from __future__ import annotations

import numpy as np
import scipy.linalg as la
import scipy.sparse as sps

N_OVERSAMPLES = 10


def spmm(indptr, indices, values, dense: np.ndarray) -> np.ndarray:
    """``A @ dense`` for the CSR ``(indptr, indices, values)``: row r's sum walks its entries in stored order from
    +0.0f, ``acc = acc + v * dense[j]`` in f32.  All rows advance together, one stored position at a time."""
    dense = np.asarray(dense, dtype=np.float32)
    indptr = np.asarray(indptr, dtype=np.int64)
    n_rows = len(indptr) - 1
    lens = np.diff(indptr)
    acc = np.zeros((n_rows, dense.shape[1]), dtype=np.float32)
    for t in range(int(lens.max()) if n_rows else 0):
        rows = np.flatnonzero(lens > t)
        p = indptr[rows] + t
        acc[rows] = acc[rows] + np.asarray(values, np.float32)[p, None] * dense[np.asarray(indices)[p]]
    return acc


def residuals(users, items, ratings, n_users: int, n_items: int, global_bias: float, item_biases, user_biases):
    """``r - g``, ``-= ib[col]``, ``-= ub[row]`` on the f32 ratings (g a Python float, so rounded to f32 first),
    then the CSR matrix (sorted indices), as ``BiasedSVDScorer.train`` builds it."""
    data = np.asarray(ratings, dtype=np.float32) - global_bias
    data -= item_biases[items]
    data -= user_biases[users]
    return sps.coo_array((data, (users, items)), shape=(n_users, n_items)).tocsr()


def start_matrix(x_shape, k: int, random_state: np.random.RandomState) -> np.ndarray:
    """scikit-learn's draw: ``normal(size=(M.shape[1], k + 10))`` in f64, then f32; M is Xᵀ for a wide X."""
    return random_state.normal(size=(min(x_shape), k + N_OVERSAMPLES)).astype(np.float32)


def truncated_svd(X, k: int, n_iter: int, q0: np.ndarray):
    """``(components_ [k, n_cols], singular_values_ [k], X @ components_.T)`` of ``TruncatedSVD.fit_transform`` on the
    f32 CSR ``X`` with start matrix ``q0``."""
    transpose = X.shape[0] < X.shape[1]
    M = X.T if transpose else X
    Q = q0
    if n_iter <= 2:
        normalizer = lambda a: (a, None)  # noqa: E731
    else:
        normalizer = lambda a: la.lu(a, permute_l=True, check_finite=False)  # noqa: E731
    for _ in range(n_iter):
        Q, _ = normalizer(M @ Q)
        Q, _ = normalizer(M.T @ Q)
    Q, _ = la.qr(M @ Q, mode="economic", check_finite=False)
    B = Q.T @ M
    Uhat, s, Vt = la.svd(B, full_matrices=False, lapack_driver="gesdd")
    U = Q @ Uhat
    if transpose:
        U, s, Vt = Vt[:k, :].T, s[:k], U[:, :k].T
    else:
        U, s, Vt = U[:, :k], s[:k], Vt[:k, :]
    # svd_flip(U, Vt, u_based_decision=False)
    signs = np.sign(Vt[np.arange(Vt.shape[0]), np.argmax(np.abs(Vt), axis=1)])
    Vt = Vt * signs[:, None]
    return Vt, s, X @ Vt.T
