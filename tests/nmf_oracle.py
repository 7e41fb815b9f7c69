"""
Restatements behind the NMF tests (host, NumPy and SciPy):

* ``cd_sweep``: scikit-learn's ``_update_cdnmf_fast(W, HHt, XHt, arange(k))``, vectorised over the rows, each product
  and sum rounded to f32 separately (no FMA); returns the |pg| of every (t, i) in t-major order, as
  ``lk_nmf_cd_sweep`` writes them;
* ``seq_sum``: the left-to-right f32 sum ``np.cumsum(x, dtype=float32)[-1]`` by the binade-segmented integer scan
  ``lk_f32_seq_sum`` runs;
* ``gram`` and ``fit``: the coordinate-descent loop of ``_fit_coordinate_descent`` with the Gram computed in f64 and
  rounded once to f32, as the device computes it.
"""

from __future__ import annotations

import numpy as np

LIMIT = 1 << 24  # ulps in a binade
BIG = 1 << 26  # an increment that certainly leaves the binade
CHUNK = 1 << 16  # elements examined per step of seq_sum


def cd_sweep(W: np.ndarray, HHt: np.ndarray, XHt: np.ndarray) -> np.ndarray:
    """One ``_update_cdnmf_fast`` call on f32 ``W`` [n, k] (updated in place); returns |pg| [k, n]."""
    n, k = W.shape
    pg_abs = np.empty((k, n), dtype=np.float32)
    for t in range(k):
        grad = -XHt[:, t]
        for r in range(k):
            grad = grad + HHt[t, r] * W[:, r]
        wt = W[:, t]
        pg = np.where(wt == 0, np.where(grad < 0, grad, np.float32(0)), grad)
        pg_abs[t] = np.abs(pg)
        hess = HHt[t, t]
        if hess != 0:
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                v = wt - grad / hess
            W[:, t] = np.where(np.float32(0) > v, np.float32(0), v)
    return pg_abs


def _segment(s: np.float32) -> tuple[int, int]:
    """(log2 of the ulp, s / ulp) of the binade holding s; [0, 2^-125) is one binade with ulp 2^-149."""
    b = int(np.float32(s).view(np.uint32))
    ex = b >> 23
    if ex <= 1:
        return -149, b
    return ex - 150, (b & 0x7FFFFF) | 0x800000


def _value(ue: int, cnt: int) -> np.float32:
    if ue == -149:
        return np.uint32(cnt).view(np.float32)
    return np.uint32(((ue + 150) << 23) | (cnt & 0x7FFFFF)).view(np.float32)


def _increments(x: np.ndarray, ue: int):
    """Per element: the increment in ulps of 2^ue when not a tie, the tie flag, and the floor for ties."""
    b = x.view(np.uint32).astype(np.int64) & 0x7FFFFFFF
    ex = b >> 23
    mant = b & 0x7FFFFF
    m = np.where(ex == 0, mant, mant | 0x800000)
    sh = ue - np.where(ex == 0, -149, ex - 150)
    left = np.clip(-sh, 0, 26)
    q_left = np.where(-sh >= 26, BIG, np.minimum(m << left, BIG))
    s = np.clip(sh, 1, 26)
    f = m >> s
    rem = m & ((np.int64(1) << s) - 1)
    half = np.int64(1) << (s - 1)
    tie = (sh > 0) & (rem == half)
    inc = np.where(sh <= 0, q_left, f + (rem > half))
    inc = np.where(ex == 0xFF, BIG, inc)
    tie &= ex != 0xFF
    return inc, tie, f


def seq_sum(x: np.ndarray) -> np.float32:
    """``np.cumsum(x, dtype=float32)[-1]`` (0 for an empty x) of non-negative f32 values, by binade segments: inside
    one, a step adds ``rne(x / ulp)`` ulps, which depends on the running sum only through its parity on exact ties
    (a tie leaves the parity even).  The first element that would leave the binade is added in f32, and the scan
    restarts after it."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    n = len(x)
    s = np.float32(0)
    j = 0
    while j < n:
        if np.isnan(s):
            return s
        if np.isinf(s):
            return np.float32(np.nan) if np.isnan(x[j:]).any() else s
        ue, cnt = _segment(s)
        par = cnt & 1
        xs = x[j : j + CHUNK]
        inc, tie, f = _increments(xs, ue)
        # parity before each element: the start's parity, or 0 after the last tie, flipped by every odd increment
        odd = np.where(tie, 0, inc & 1)
        flips = np.cumsum(odd) - odd  # odd increments before each element
        idx = np.arange(len(xs))
        last_tie = np.maximum.accumulate(np.where(tie, idx, -1))
        prev_tie = np.concatenate(([-1], last_tie[:-1]))  # the last tie strictly before each element
        flips_at_tie = np.where(prev_tie >= 0, flips[np.maximum(prev_tie, 0)], 0)
        parity = np.where(prev_tie >= 0, 0, par) ^ ((flips - flips_at_tie) & 1)
        inc = np.where(tie, f + ((parity + f) & 1), inc)
        after = cnt + np.cumsum(inc)
        out = np.flatnonzero(after >= LIMIT)
        if len(out) == 0:
            s = _value(ue, int(after[-1]))
            j += len(xs)
            continue
        c = int(out[0])
        before = cnt if c == 0 else int(after[c - 1])
        with np.errstate(over="ignore", invalid="ignore"):
            s = np.float32(_value(ue, before) + xs[c])
        j += c + 1
    return s


def gram(Q: np.ndarray) -> np.ndarray:
    """``Q.T @ Q`` in f64, rounded once to f32."""
    Q = Q.astype(np.float64)
    return (Q.T @ Q).astype(np.float32)


def cd_half(X, W, Ht, l1_reg: float, l2_reg: float) -> np.float32:
    """``_update_coordinate_descent(X, W, Ht, ...)`` with the f64 Gram: W updated in place, the f32 violation."""
    k = Ht.shape[1]
    HHt = gram(Ht)
    XHt = np.asarray(X @ Ht, dtype=np.float32)
    if l2_reg != 0.0:
        HHt.flat[:: k + 1] += l2_reg
    if l1_reg != 0.0:
        XHt -= l1_reg
    return seq_sum(cd_sweep(W, HHt, XHt).ravel())


def fit(X, W, H, max_iter: int = 200, tol: float = 1e-4, l1_reg_W=0.0, l1_reg_H=0.0, l2_reg_W=0.0, l2_reg_H=0.0):
    """``_fit_coordinate_descent`` from the initial W [n_rows, k] and H [k, n_cols]: ``(W, H, n_iter)``."""
    import scipy.sparse as sps

    X = sps.csr_array(X)
    XT = sps.csr_array(X.T)
    W = np.ascontiguousarray(W, dtype=np.float32).copy()
    Ht = np.ascontiguousarray(H.T, dtype=np.float32).copy()
    violation_init = None
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        violation = 0.0
        violation += float(cd_half(X, W, Ht, l1_reg_W, l2_reg_W))
        violation += float(cd_half(XT, Ht, W, l1_reg_H, l2_reg_H))
        if n_iter == 1:
            violation_init = violation
        if violation_init == 0:
            break
        if violation / violation_init <= tol:
            break
    return W, Ht.T, n_iter
