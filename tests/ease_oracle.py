"""
Host restatement of LensKit's EASE scorer (``src/lenskit/knn/ease.py``), what the GPU results are compared with.

* ``train``: the statements of ``EASEScorer.train`` — the dense Gram with its diagonal (``cooc_oracle.dense_cooc``,
  what ``co_occurrences(include_self=True, dense=True)`` returns), ``cooc[di] += regularization``, the inverse, and
  ``mat /= -np.diag(mat)``, ``mat[di] = 0`` — with the inverse of ``_chol_invert_torch`` on a given torch device
  (the same calls, so on the same device and torch build the weights are the reference's bit for bit) or of
  ``_chol_invert_scipy``.
* ``score``: the order ``lk_ease_score_batch`` fixes — history deduplicated and ascending, f32 adds from +0.0.
* ``score_blas``: ``EASEScorer.__call__``'s own ``q_vec @ weights`` (BLAS, order unspecified).
"""

from __future__ import annotations

import numpy as np
import torch

import cooc_oracle as co


def gram(n_users: int, n_items: int, users, items, regularization: float) -> np.ndarray:
    cooc = co.dense_cooc(n_users, n_items, users, items, diagonal=True)
    di = np.diag_indices(n_items)
    cooc[di] += regularization  # NumPy 2: the Python float is weakly typed, one f32 add per entry
    return cooc


def invert_torch(cooc: np.ndarray, device) -> np.ndarray:
    """``_chol_invert_torch`` (ease.py) on ``device``."""
    with torch.inference_mode():
        cooc_t = torch.from_numpy(cooc).to(device)
        decomp, info = torch.linalg.cholesky_ex(cooc_t)
        if info.item():
            raise RuntimeError(f"matrix minor {info.item()} is not positive-definite.")
        inv = torch.cholesky_inverse(decomp, out=cooc_t)
        return inv.cpu().numpy()


def invert_scipy(cooc: np.ndarray) -> np.ndarray:
    import scipy.linalg as spla

    return spla.inv(cooc, assume_a="pos", overwrite_a=True)


def normalise(mat: np.ndarray) -> np.ndarray:
    mat /= -np.diag(mat).reshape(1, -1)
    mat[np.diag_indices(mat.shape[0])] = 0
    return mat


def train(n_users: int, n_items: int, users, items, regularization: float = 1.0, device="cpu") -> np.ndarray:
    """The weight matrix of ``EASEScorer.train`` with the torch inverse on ``device`` (``"scipy"``: LAPACK)."""
    cooc = gram(n_users, n_items, users, items, regularization)
    mat = invert_scipy(cooc) if device == "scipy" else invert_torch(cooc, device)
    return normalise(mat)


def history(hist) -> np.ndarray:
    """The rows that count: known items, deduplicated, ascending (``q_vec[q_good] = 1.0``)."""
    h = np.asarray(hist, dtype=np.int64)
    return np.unique(h[h >= 0])


def score(weights: np.ndarray, hist) -> np.ndarray:
    """Scores of every item: ``s = +0.0f; for h in H ascending: s = s + W[h]`` in f32; all NaN without history."""
    h = history(hist)
    if len(h) == 0:
        return np.full(weights.shape[1], np.nan, dtype=np.float32)
    s = np.zeros(weights.shape[1], dtype=np.float32)
    for r in h:
        s = s + weights[r]
    return s


def score_blas(weights: np.ndarray, hist) -> np.ndarray:
    """``EASEScorer.__call__``: ``q_vec @ self.weights`` with a dense 0/1 f32 query vector."""
    h = history(hist)
    if len(h) == 0:
        return np.full(weights.shape[1], np.nan, dtype=np.float32)
    q_vec = np.zeros(weights.shape[0], dtype=np.float32)
    q_vec[h] = 1.0
    return q_vec @ weights
