"""
Host restatement of LensKit's co-occurrence counting and association scoring, the reference the GPU results
are compared with bit for bit.

* ``count_cooc`` / ``dense_cooc``: the loop of ``count_cooc_parallel`` (src/accel/data/cooc.rs:197-212) — every
  position pair p <= q of a group, equal items to the diagonal, others to (min, max) — vectorised per group,
  with the result layout of ``SymmetricPairCounter::finish`` / ``DensePairCounter::finish``.
* ``assoc_values``: the NumPy statements of ``AssociationScorer.train`` (association.py:117-124).
* ``score``: ``AssociationScorer.__call__``'s dense rows and ``np.mean`` / ``np.max`` (association.py:150-155);
  ``score_sequential`` is the order the GPU kernel uses, pinned against ``np.mean`` by the tests.
"""

from __future__ import annotations

import numpy as np
import scipy.sparse as sps


def _pairs(n_groups: int, n_items: int, groups: np.ndarray, items: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """(row, col) of every position pair p <= q of every group, in the group's input order."""
    groups = np.asarray(groups, dtype=np.int64)
    items = np.asarray(items, dtype=np.int64)
    ptr = np.concatenate([[0], np.cumsum(np.bincount(groups, minlength=n_groups))]).astype(np.int64)
    rows, cols = [], []
    for g in range(n_groups):
        its = items[ptr[g] : ptr[g + 1]]
        p, q = np.triu_indices(len(its))  # p <= q: `for ci in &items[i..n]`
        rows.append(its[p])
        cols.append(its[q])
    if not rows:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(rows), np.concatenate(cols)


def _tally(n_items: int, r: np.ndarray, c: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Diagonal counts and the strict upper triangle (row-major, columns ascending) of the pairs."""
    diag_m = r == c
    diag = np.bincount(r[diag_m], minlength=n_items).astype(np.int64)
    lo, hi = np.minimum(r[~diag_m], c[~diag_m]), np.maximum(r[~diag_m], c[~diag_m])
    keys, cnt = np.unique(lo * n_items + hi, return_counts=True)
    return diag, (keys // n_items).astype(np.int32), (keys % n_items).astype(np.int32), cnt.astype(np.int64)


def count_cooc(n_groups: int, n_items: int, groups, items, diagonal: bool = True) -> list[tuple]:
    """``[(row, col, count) ...]``: the diagonal (all items) if ``diagonal``, the upper triangle, its transpose."""
    diag, row, col, cnt = _tally(n_items, *_pairs(n_groups, n_items, groups, items))
    out = [(np.arange(n_items, dtype=np.int32), np.arange(n_items, dtype=np.int32), diag.astype(np.int32))] if diagonal else []
    return out + [(row, col, cnt.astype(np.int32)), (col, row, cnt.astype(np.int32))]


def dense_cooc(n_groups: int, n_items: int, groups, items, diagonal: bool = True) -> np.ndarray:
    diag, row, col, cnt = _tally(n_items, *_pairs(n_groups, n_items, groups, items))
    m = np.zeros((n_items, n_items), dtype=np.float32)
    m[row, col] = cnt.astype(np.float32)
    m[col, row] = cnt.astype(np.float32)
    if diagonal:
        m[np.arange(n_items), np.arange(n_items)] = diag.astype(np.float32)
    return m


def count_matrix(n_groups: int, n_items: int, groups, items) -> sps.csr_array:
    """X[g, i] = occurrences of i in g: off the diagonal, C = XᵀX (sum_g #i #j)."""
    g = np.asarray(groups, dtype=np.int64)
    return sps.csr_array((np.ones(len(g), np.int64), (g, np.asarray(items, np.int64))), shape=(n_groups, n_items))


def assoc_values(row, col, count, item_counts, n_groups: int, method: str, damping: float) -> np.ndarray:
    """association.py:117-124, statement for statement."""
    cooc_vals = np.asarray(count).astype(np.float32)
    cooc_vals /= item_counts[row] + damping
    if method == "lift":
        cooc_vals *= n_groups
        cooc_vals /= item_counts[col] + damping
    return cooc_vals


def assoc_matrix(n_groups: int, n_items: int, groups, items, method: str, damping: float) -> sps.csr_array:
    """What ``AssociationScorer.train`` stores: no diagonal, both triangles, rows sorted by column."""
    _diag, row, col, cnt = _tally(n_items, *_pairs(n_groups, n_items, groups, items))
    r = np.concatenate([row, col])
    c = np.concatenate([col, row])
    v = np.concatenate([cnt, cnt])
    item_counts = np.bincount(np.asarray(items, np.int64), minlength=n_items).astype(np.int32)
    vals = assoc_values(r, c, v, item_counts, n_groups, method, damping)
    m = sps.csr_array((vals, (r, c)), shape=(n_items, n_items))
    m.sort_indices()
    return m


def score(assoc: sps.csr_array, refs: np.ndarray, max_nbrs: int | None) -> np.ndarray:
    """Scores of every item (association.py:145-155); all NaN without reference items."""
    refs = np.asarray(refs, dtype=np.int64)
    if len(refs) == 0:
        return np.full(assoc.shape[1], np.nan, dtype=np.float32)
    assoc_mat = assoc[refs, :].todense()
    if max_nbrs == 1:
        return np.asarray(np.max(assoc_mat, axis=0), dtype=np.float32)
    return np.asarray(np.mean(assoc_mat, axis=0), dtype=np.float32)


def score_sequential(dense_rows: np.ndarray) -> np.ndarray:
    """The mean as the kernel computes it: f32 adds in row order from +0, then f32(f64(sum) / f64(R))."""
    s = np.zeros(dense_rows.shape[1], dtype=np.float32)
    for row in dense_rows:
        s = s + row.astype(np.float32)
    return (s.astype(np.float64) / np.float64(len(dense_rows))).astype(np.float32)
