"""
Host restatements behind the stochastic ranker's tests: NumPy's PCG64 on Python ints with the jump constants derived
independently of ``engine.pcg64_jump``, the reference's key statements (``stochastic/_ranker.py:119-156``) in
NumPy, and argtopn's heap replay (``src/accel/indirect/heap.rs``, ``src/accel/data/sorting.rs:131-170``) over f64
keys.
"""

from __future__ import annotations

import numpy as np

MULT = 0x2360ED051FC65DA44385DF649FCCF645
M64, M128 = (1 << 64) - 1, (1 << 128) - 1


def step(state: int, inc: int) -> int:
    return (state * MULT + inc) & M128


def xsl_rr(state: int) -> int:
    hi, lo = state >> 64, state & M64
    x, rot = hi ^ lo, hi >> 58
    return ((x >> rot) | (x << ((64 - rot) & 63))) & M64


def raw(state: int, inc: int, k: int) -> tuple[list[int], int]:
    """``k`` raw outputs from ``(state, inc)`` (step, then output the new state), and the state they leave."""
    out = []
    for _ in range(k):
        state = step(state, inc)
        out.append(xsl_rr(state))
    return out, state


def jump(j: int) -> tuple[int, int]:
    """``(M^j, G_j)`` with ``G_j = (M^j - 1) / (M - 1)``: M - 1 is even, so the quotient is taken exactly modulo
    ``(M - 1) 2^128`` before dividing."""
    mod = (MULT - 1) << 128
    return pow(MULT, j, 1 << 128), ((pow(MULT, j, mod) - 1) % mod) // (MULT - 1)


def jump_table_words() -> np.ndarray:
    rows = [jump(j) for j in range(33)] + [jump(1 << t) for t in range(64)]
    return np.array([[m >> 64, m & M64, g >> 64, g & M64] for m, g in rows], dtype=np.uint64).reshape(-1)


def weights(s: np.ndarray, transform: str | None) -> np.ndarray:
    """The selection weights of the scaled f32 scores ``s`` (all finite): NumPy 2 promotion keeps them f32."""
    if transform == "softmax":
        e = np.exp(s - np.max(s))
        return e / np.sum(e)
    if transform == "linear":
        lb, ub = np.min(s).item(), np.max(s).item()
        r = ub - lb
        if r > 0:
            t = (s - lb) / np.float32(r)
            tot = np.sum(t)
            if tot > 0:
                return t / tot
        return np.ones_like(s) / len(s)
    return s


def keys(scores: np.ndarray, transform: str | None, scale: float, gen: np.random.Generator) -> np.ndarray:
    """The f64 keys of the finite f32 ``scores``, drawing ``len(scores)`` uniforms from ``gen``."""
    s = np.asarray(scores, dtype=np.float32) * scale
    w = weights(s, transform)
    u = gen.uniform(0, 1, len(s))
    return np.log(u) / np.maximum(w, np.finfo(np.float32).smallest_normal)


def _down(hv: list, hk: list, pos: int, lim: int) -> None:
    v, k = hv[pos], hk[pos]
    while True:
        mn, mv = pos, v
        left, right = 2 * pos + 1, 2 * pos + 2
        if left < lim and hv[left] < mv:
            mn, mv = left, hv[left]
        if right < lim and hv[right] < mv:
            mn = right
        if mn == pos:
            break
        hv[pos], hk[pos] = hv[mn], hk[mn]
        pos = mn
    hv[pos], hk[pos] = v, k


def argtopn(vals: np.ndarray, n: int) -> np.ndarray:
    """argtopn: the ``n`` largest non-NaN values, offered in order to the indirect min-heap, then heap-sorted."""
    n = int(min(max(n, 0), len(vals)))
    hv: list[float] = []
    hk: list[int] = []
    if n == 0:
        return np.zeros(0, np.int32)
    for i, v in enumerate(np.asarray(vals, dtype=np.float64).tolist()):
        if v != v:
            continue
        if len(hv) < n:
            hv.append(v)
            hk.append(i)
            pos = len(hv) - 1
            while pos > 0:
                parent = (pos - 1) // 2
                if not hv[parent] > v:
                    break
                hv[pos], hk[pos] = hv[parent], hk[parent]
                pos = parent
            hv[pos], hk[pos] = v, i
        elif v > hv[0]:
            hv[0], hk[0] = v, i
            _down(hv, hk, 0, n)
    for m in range(len(hv) - 1, 0, -1):
        hv[0], hv[m], hk[0], hk[m] = hv[m], hv[0], hk[m], hk[0]
        _down(hv, hk, 0, m)
    return np.array(hk, dtype=np.int32)


def rank(scores: np.ndarray, n: int | None, transform: str | None, scale: float, gen: np.random.Generator):
    """One ``__call__`` on a list with these scores: ``(positions in the list, their keys)``; ``n=None`` ranks every
    valid item (a stable descending sort, one order the reference's unstable sort may give)."""
    scores = np.asarray(scores, dtype=np.float32)
    valid = np.flatnonzero(np.isfinite(scores))
    if len(valid) == 0:
        return np.zeros(0, np.int64), np.zeros(0)
    k = keys(scores[valid], transform, scale, gen)
    pick = np.argsort(-k, kind="stable") if n is None else argtopn(k, n)
    return valid[pick], k[pick]
