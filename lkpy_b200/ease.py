"""
EASE scorer on the H100 engine — the component surface of ``lenskit.knn.ease.EASEScorer``
(``src/lenskit/knn/ease.py``).

Same config (``regularization``), the same ``LK_EASE_SOLVER`` training variable, the same trained attributes
(``items``, ``weights``) and the same per-query ``__call__``; plus ``score_batch`` and ``recommend_batch``, the
batched form of candidate selector → scorer → ``TopNRanker`` with scoring and top-n selection in one kernel.

Training follows ``EASEScorer.train`` statement for statement, on the device: the item Gram with its diagonal
(``lk_cooc_count`` + ``lk_cooc_diagonal`` + ``lk_cooc_dense``, what ``co_occurrences(include_self=True,
dense=True)`` returns), the regularisation added to the diagonal, the reference's own torch calls for the inverse
(``torch.linalg.cholesky_ex`` and ``torch.cholesky_inverse``, cuSOLVER) and the column normalisation.  The weight
matrix (n_items² f32: 13.9 GB at the ML-25M shape) stays on the device as the scorer's state; the NumPy ``weights``
is built on first access and when pickling.  Scoring (``lk_ease_score_batch``) reads only the history rows.
"""

from __future__ import annotations

import os
import threading
import warnings
from typing import Callable, Literal

import numpy as np
import torch
from pydantic import BaseModel, PositiveFloat

from . import _lib, engine
from .components import Component, ItemList, Trainable, TrainingOptions, _as_dataset
from .batch import check_exclude, empty_list, history_csr, rank_size, ranked_lists, target_scores

MIN_SCIPY_VERSION = "1.17"
#: one device Cholesky at a time (ease.py's ``_chol_lock``)
_chol_lock = threading.Lock()


class EASEConfig(BaseModel, extra="forbid"):
    regularization: PositiveFloat = 1


def _chol_invert_torch(gram: torch.Tensor) -> torch.Tensor:
    """``_chol_invert_torch`` of ease.py on the matrix's own device: the inverse overwrites ``gram``."""
    with torch.inference_mode():
        with _chol_lock:
            decomp, info = torch.linalg.cholesky_ex(gram)
        if info.item():
            raise RuntimeError(f"matrix minor {info.item()} is not positive-definite.")
        return torch.cholesky_inverse(decomp, out=gram)


def _chol_invert_scipy(gram: np.ndarray) -> np.ndarray:
    """``_chol_invert_scipy`` of ease.py: LAPACK on the host, in place."""
    import scipy
    import scipy.linalg as spla
    from packaging.version import Version

    if Version(scipy.__version__) < Version(MIN_SCIPY_VERSION):
        raise RuntimeError("SciPy solver requires SciPy 1.17 or later")
    return spla.inv(gram, assume_a="pos", overwrite_a=True)


def _check_solver(solver: str | None) -> None:
    if solver and solver not in ("torch", "scipy"):
        raise ValueError(f"unsupported option: LK_EASE_SOLVER={solver}")


def _invert(gram: Callable[[], torch.Tensor], solver: str | None) -> torch.Tensor:
    """
    The inverse of the regularised Gram that ``gram()`` builds, on the Gram's device.  As in ``EASEScorer.train``:
    torch unless ``solver == "scipy"``; with ``solver`` unset a ``torch.OutOfMemoryError`` falls back to SciPy,
    with it set the error is raised.  The fallback builds the Gram again, since a failed in-place inverse may have
    left it partly overwritten.
    """
    if solver != "scipy":
        try:
            return _chol_invert_torch(gram())
        except torch.OutOfMemoryError as e:
            if solver:
                raise e
            warnings.warn(f"failed to allocate PyTorch memory to solve, falling back to SciPy: {e}", RuntimeWarning)
    g = gram()
    dev = g.device
    host = g.cpu().numpy()
    del g
    return torch.from_numpy(np.ascontiguousarray(_chol_invert_scipy(host), dtype=np.float32)).to(dev)


def _normalise(mat: torch.Tensor) -> torch.Tensor:
    """``mat /= -np.diag(mat).reshape(1, -1); mat[di] = 0``: every column divided by its negated diagonal entry
    (f32 division, correctly rounded on both sides), then a zero diagonal."""
    mat /= torch.diagonal(mat).neg().reshape(1, -1)
    mat.fill_diagonal_(0.0)
    return mat


class EASEScorer(Component, Trainable):
    CONFIG_CLASS = EASEConfig
    config: EASEConfig

    items = None

    def is_trained(self) -> bool:
        return "_state" in self.__dict__ or "_weights_host" in self.__dict__

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        solver = os.environ.get("LK_EASE_SOLVER")
        _check_solver(solver)
        ds = _as_dataset(data)
        dev = _lib.require_device()
        it = ds.interactions
        reg = float(self.config.regularization)

        def gram() -> torch.Tensor:
            # co_occurrences("item", include_self=True, dense=True), then cooc[di] += regularization: the Python
            # float is weakly typed under NumPy 2, so each diagonal entry is one f32 add, as torch's add_ does
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
            plan = engine.CoocPlan.create(it.n_users, it.n_items, up(it.users), up(it.items))
            indptr, cols, counts = plan.count(full_rows=False)
            g = plan.dense(indptr, cols, counts, plan.diagonal())
            g.diagonal().add_(reg)
            return g  # the count CSR and the plan are released here, before the inverse

        self._state = engine.EaseState(_normalise(_invert(gram, solver)))
        self.__dict__.pop("_weights_host", None)
        self.items = ds.items

    @property
    def weights(self) -> np.ndarray:
        """Item interpolation weights (f32 ``[n_items, n_items]``, history items on rows, targets on columns)."""
        w = self.__dict__.get("_weights_host")
        if w is None:
            st = self.__dict__.get("_state")
            if st is None:
                raise AttributeError("weights")  # untrained: hasattr(scorer, "weights") is False
            w = st.weights.cpu().numpy()
            self._weights_host = w
        return w

    def _device_state(self) -> engine.EaseState:
        st = self.__dict__.get("_state")
        if st is None:  # e.g. after unpickling
            st = engine.EaseState.create(self.weights, _lib.require_device())
            self._state = st
        return st

    def __getstate__(self):
        self.weights  # noqa: B018 — the host matrix is what gets pickled
        d = dict(self.__dict__)
        d.pop("_state", None)
        return d

    def score_batch(self, queries, targets: list[ItemList]) -> list[ItemList]:
        """Score ``targets[i]`` for query ``queries[i]`` (a history ``ItemList`` or a ``RecQuery``), in one launch.
        Unknown targets, and every target of a query without known history items, score NaN."""
        st = self._device_state()
        dev = st.weights.device
        # q_vec[q_good] = 1.0 counts a repeated item once: each history ascending without repeats
        _has, h_ptr, h_items = history_csr(queries, self.items, dev, unique=True)
        return target_scores(st.score(h_ptr, h_items), targets, self.items)

    def __call__(self, query, items: ItemList) -> ItemList:
        return self.score_batch([query], [items])[0]

    def recommend_batch(self, queries, n: int, *, exclude: Literal["query"] | None = "query") -> list[ItemList]:
        """
        Top-``n`` items for every query, scored and selected on the device in one launch: for each query the result
        of ``TrainingItemsCandidateSelector`` (every item, minus the query's items when ``exclude="query"``),
        ``__call__`` and ``TopNRanker``, bit for bit with the scores of ``score_batch``.  A query without known
        history items gets an empty list.
        """
        check_exclude(exclude)
        st = self._device_state()
        dev = st.weights.device
        n_eff = rank_size(n, st.n_items)
        if n_eff == 0:
            return [empty_list(self.items) for _ in queries]
        _has, h_ptr, h_items = history_csr(queries, self.items, dev, unique=True)
        excl = (h_ptr, h_items) if exclude == "query" else (None, None)
        idx, val, cnt = st.recommend(h_ptr, h_items, n_eff, *excl)
        return ranked_lists(self.items, len(queries), range(len(queries)), idx, val, cnt)
