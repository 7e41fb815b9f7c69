"""
SLIM scorer on the H100 engine — the component surface of ``lenskit.knn.slim.SLIMScorer``
(``src/lenskit/knn/slim.py``).

Same config (``l1_reg``, ``l2_reg``, ``max_iters``, ``max_nbrs``), the same trained attributes (``items``, ``weights``:
the *transposed* weight matrix, history items on rows) and the same per-query ``__call__``; plus ``score_batch`` and
``recommend_batch``, the batched form of candidate selector → scorer → ``TopNRanker`` with scoring and top-n
selection in one kernel.

Training runs ``lk_slim_train`` (``engine.SlimPlan``) over the interaction structure, the same computation as the
reference's ``_accel.slim.train_slim``.  The transposed weights stay on the device as the scorer's state; the SciPy
``weights`` is built on first access and when pickling.  Scoring is ``x @ weights`` with x the 0/1 row of the known
history items in query order, repeats kept: the association scoring kernel's plain sum (``lk_assoc_score_batch``,
``agg`` 2), which adds the history rows' entries in that order, as SciPy's sparse product does.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch
from pydantic import BaseModel, PositiveFloat, PositiveInt

from . import _lib, engine
from .components import Component, ItemList, Trainable, TrainingOptions, _as_dataset
from .batch import check_exclude, empty_list, history_csr, rank_size, ranked_lists, target_scores

_AGG_SUM = 2


class SLIMConfig(BaseModel, extra="forbid"):
    l1_reg: PositiveFloat = 1.0
    l2_reg: PositiveFloat = 1.0
    max_iters: PositiveInt = 100
    max_nbrs: PositiveInt | None = None


def _transpose(n: int, indptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor):
    """The transpose of a square device CSR, columns ascending in every row (what SciPy's ``.T.tocsr()`` gives)."""
    dev = indptr.device
    rows = torch.repeat_interleave(torch.arange(n, device=dev), indptr[1:] - indptr[:-1])
    order = torch.argsort(cols.long() * n + rows)
    t_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(torch.bincount(cols.long(), minlength=n), 0, out=t_ptr[1:])
    return t_ptr, rows[order].to(torch.int32), vals[order]


class SLIMScorer(Component, Trainable):
    CONFIG_CLASS = SLIMConfig
    config: SLIMConfig

    items = None

    def is_trained(self) -> bool:
        return getattr(self, "_state", None) is not None or "_weights_host" in self.__dict__

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        dev = _lib.require_device()
        it = ds.interactions
        n = it.n_items
        u, i = torch.from_numpy(it.users).to(dev).long(), torch.from_numpy(it.items).to(dev).long()

        def structure(rows, cols, n_rows, n_cols):  # rows by number, columns ascending within a row
            ip = torch.zeros(n_rows + 1, dtype=torch.int64, device=dev)
            torch.cumsum(torch.bincount(rows, minlength=n_rows), 0, out=ip[1:])
            return ip, (torch.sort(rows * max(n_cols, 1) + cols).values % max(n_cols, 1)).to(torch.int32)

        ui_p, ui_c = structure(u, i, it.n_users, n)
        iu_p, iu_c = structure(i, u, n, it.n_users)
        c = self.config
        plan = engine.SlimPlan.create(it.n_users, n, ui_p, ui_c, iu_p, iu_c, c.l1_reg, c.l2_reg, c.max_iters,
                                      c.max_nbrs)  # fmt: skip
        indptr, cols, vals = plan.train()
        del plan
        self._state = engine.AssocState.create(n, *_transpose(n, indptr, cols, vals), device=dev)
        self.__dict__.pop("_weights_host", None)
        self.items = ds.items

    @property
    def weights(self):
        """The transposed SLIM weights, history items on rows and targets on columns (SciPy ``csr_array``)."""
        m = self.__dict__.get("_weights_host")
        if m is None:
            m = self._weights_host = self._state.host_csr()
        return m

    def _device_state(self) -> engine.AssocState:
        st = getattr(self, "_state", None)
        if st is None:  # e.g. after unpickling
            m = self.weights
            st = engine.AssocState.create(m.shape[0], m.indptr, m.indices, m.data, _lib.require_device())
            self._state = st
        return st

    def __getstate__(self):
        self.weights  # noqa: B018 — the host matrix is what gets pickled
        d = dict(self.__dict__)
        d.pop("_state", None)
        return d

    def score_batch(self, queries, targets: list[ItemList]) -> list[ItemList]:
        """Score ``targets[i]`` for query ``queries[i]`` (a history ``ItemList`` or a ``RecQuery``), in one launch.
        A query without history scores NaN everywhere; one whose items are all unknown scores 0."""
        st = self._device_state()
        dev = st.indptr.device
        has, r_ptr, r_items = history_csr(queries, self.items, dev)
        return target_scores(st.score(r_ptr, r_items, _AGG_SUM), targets, self.items, has)

    def __call__(self, query, items: ItemList) -> ItemList:
        return self.score_batch([query], [items])[0]

    def recommend_batch(self, queries, n: int, *, exclude: Literal["query"] | None = "query") -> list[ItemList]:
        """
        Top-``n`` items for every query, scored and selected on the device in one launch: for each query the result
        of ``TrainingItemsCandidateSelector`` (every item, minus the query's items when ``exclude="query"``),
        ``__call__`` and ``TopNRanker``, bit for bit.  A query without history gets an empty list; one whose items
        are all unknown ranks the all-zero scores in ``argtopn``'s tie order.
        """
        check_exclude(exclude)
        st = self._device_state()
        dev = st.indptr.device
        n_eff = rank_size(n, st.n_items)
        if n_eff == 0:
            return [empty_list(self.items) for _ in queries]
        has, r_ptr, r_items = history_csr(queries, self.items, dev)
        excl = (r_ptr, r_items) if exclude == "query" else (None, None)
        idx, val, cnt = st.recommend(r_ptr, r_items, _AGG_SUM, n_eff, *excl)
        at = np.flatnonzero(has)  # the kernel ranks the all-zero sums of a query without history: dropped
        sel = torch.from_numpy(at).to(dev)
        return ranked_lists(self.items, len(queries), at, idx[sel], val[sel], cnt[sel])
