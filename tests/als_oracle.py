"""
Host restatement of the ALS scores ``lk_als_recommend_batch`` computes (``lkpy_b200/csrc/als_recommend.cu``):
for item i and query b,

    s = +0.0f;  for d = 0 .. k-1:  s = fmaf(Q[i,d], X[b,d], s)      one fp32 FMA chain, ascending d
    s = s + item_offset[i];  s = s + query_offset[b]                f32 adds, each when given

NumPy has no fused multiply-add, so each step is an exactly rounded fmaf built from f64 parts:
  * the product of two f32 values has at most 48 significant bits, so ``p = q * x`` in f64 is exact;
  * TwoSum gives ``p + s = t + e`` exactly, with ``t = fl64(p + s)`` and |e| at most half an f64 ulp of t;
  * rounding t to f32 is the correct rounding of t + e, except when t lies exactly halfway between two f32
    values and e != 0: then e decides the direction, away from the nearest-even choice when it points that way.
    (e is 2^29 times smaller than an f32 ulp, so it can change nothing else.)
Signed zeros, subnormal results and the f32 range behave as in ``fmaf``.  Used by the tests and ``smoke()``;
``tests/test_als_recommend.py`` checks it against the C library's ``fmaf``.
"""

from __future__ import annotations

import numpy as np


def _fmaf64(p: np.ndarray, c: np.ndarray) -> np.ndarray:
    """Correctly rounded f32 ``p + c`` for an exact f64 product p of two f32 values and f32 values c (as f64)."""
    t = p + c
    bp = t - c  # TwoSum (Knuth): e = (p - bp) + (c - (t - bp)), exact
    e = (p - bp) + (c - (t - bp))
    r = t.astype(np.float32)
    d = t - r  # exact (Sterbenz): from r towards t
    # only where t is off the f32 grid and the TwoSum error is nonzero can t be a midpoint that e moves
    idx = np.flatnonzero((d != 0) & (e != 0))
    if idx.size:
        ri, di, ei = r.flat[idx], d.flat[idx], e.flat[idx]
        nb = np.nextafter(ri, np.where(di > 0, np.float32(np.inf), np.float32(-np.inf)))
        mid = di == (nb.astype(np.float64) - ri) / 2  # t halfway to the f32 neighbour on its side
        # at a tie, t + e lies beyond the midpoint (round to nb) when e points the same way as d
        up = mid & ((ei > 0) == (di > 0))
        r.flat[idx[up]] = nb[up]
    return r


def fmaf(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    """Element-wise correctly rounded f32 ``a * b + c`` for finite f32 arrays (broadcasting)."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)  # exact
    c64 = np.broadcast_to(np.asarray(c, np.float32), p.shape).astype(np.float64)
    return _fmaf64(p, c64)


def als_scores(Q: np.ndarray, X: np.ndarray, item_offset=None, query_offset=None) -> np.ndarray:
    """The scores ``[n_items, n_queries]`` (f32, item-major) of every item in ``Q [n_items, k]`` for every query
    in ``X [n_queries, k]``, as the module docstring states them."""
    Q = np.ascontiguousarray(Q, dtype=np.float32)
    X = np.ascontiguousarray(X, dtype=np.float32)
    if Q.ndim != 2 or X.ndim != 2 or Q.shape[1] != X.shape[1]:
        raise ValueError("Q and X must be 2-D with the same number of columns")
    n_items, k = Q.shape
    XT = X.T.astype(np.float64)  # [k, n_queries]
    out = np.empty((n_items, X.shape[0]), dtype=np.float32)
    rows = max(1, 65536 // max(X.shape[0], 1))  # blocks that stay in cache
    for i0 in range(0, n_items, rows):
        Qb = Q[i0 : i0 + rows].astype(np.float64)
        s = np.zeros((Qb.shape[0], X.shape[0]), dtype=np.float64)
        for d in range(k):
            s = _fmaf64(Qb[:, d, None] * XT[None, d, :], s).astype(np.float64)
        out[i0 : i0 + rows] = s
    if item_offset is not None:
        out = out + np.asarray(item_offset, dtype=np.float32)[:, None]
    if query_offset is not None:
        out = out + np.asarray(query_offset, dtype=np.float32)[None, :]
    return out.astype(np.float32, copy=False)
