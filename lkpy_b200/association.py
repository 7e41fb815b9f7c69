"""
Association-rule scorer on the H100 engine — the component surface of
``lenskit.knn.association.AssociationScorer`` (``src/lenskit/knn/association.py``).

Same config (``method``, ``damping``, ``max_nbrs``), same trained attributes (``items``, ``item_freqs``,
``assoc_scores``) and the same per-query ``__call__``; plus ``score_batch`` and ``recommend_batch``, the batched
form of candidate selector → scorer → ``TopNRanker`` with scoring and top-n selection in one kernel.

Training counts the co-occurrences on the device (``lk_cooc_count``, full rows) and turns each count into its
association value in the same pass.  At the ML-25M shape the matrix has about 1.6e9 entries, so it stays on the
device as the scorer's state: the SciPy ``assoc_scores`` is built on first access and when pickling.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch
from pydantic import BaseModel, NonNegativeFloat, PositiveInt

from . import _lib, engine
from .components import Component, ItemList, Trainable, TrainingOptions, _as_dataset
from .batch import check_exclude, empty_list, history_csr, rank_size, ranked_lists, target_scores


class AssociationConfig(BaseModel, extra="forbid"):
    method: Literal["probability", "lift"] = "probability"
    damping: NonNegativeFloat = 0.0
    max_nbrs: PositiveInt | None = None


class AssociationScorer(Component, Trainable):
    CONFIG_CLASS = AssociationConfig
    config: AssociationConfig

    items = None
    item_freqs: np.ndarray

    def is_trained(self) -> bool:
        return hasattr(self, "item_freqs")

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        dev = _lib.require_device()
        it = ds.interactions
        # Dataset.item_stats()["count"]: the interaction count per item, int64 like the reference's Arrow aggregate
        counts = np.bincount(it.items, minlength=it.n_items).astype(np.int64)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        plan = engine.CoocPlan.create(it.n_users, it.n_items, up(it.users), up(it.items))
        method = _lib.LK_ASSOC_LIFT if self.config.method == "lift" else _lib.LK_ASSOC_PROBABILITY
        indptr, cols, vals = plan.count(full_rows=True, method=method, item_count=up(counts.astype(np.int32)),
                                        damping=float(self.config.damping))  # fmt: skip
        del plan
        self._state = engine.AssocState.create(it.n_items, indptr, cols, vals, dev)
        self.__dict__.pop("_assoc_host", None)
        self.items = ds.items
        self.item_freqs = counts

    @property
    def assoc_scores(self):
        """Association values, reference items on rows and targets on columns (SciPy ``csr_array``, rows sorted)."""
        m = self.__dict__.get("_assoc_host")
        if m is None:
            m = self._assoc_host = self._state.host_csr()
        return m

    def _device_state(self) -> engine.AssocState:
        st = getattr(self, "_state", None)
        if st is None:  # e.g. after unpickling
            m = self.assoc_scores
            st = engine.AssocState.create(m.shape[0], m.indptr, m.indices, m.data, _lib.require_device())
            self._state = st
        return st

    def __getstate__(self):
        self.assoc_scores  # noqa: B018 — the host matrix is what gets pickled
        d = dict(self.__dict__)
        d.pop("_state", None)
        return d

    def _agg(self) -> int:
        if self.config.max_nbrs is None:
            return 0
        if self.config.max_nbrs == 1:
            return 1
        raise NotImplementedError("limited reference items not yet implemented")  # association.py:155

    def score_batch(self, queries, targets: list[ItemList]) -> list[ItemList]:
        """Score ``targets[i]`` for query ``queries[i]`` (a history ``ItemList`` or a ``RecQuery``), in one launch."""
        agg = self._agg()
        st = self._device_state()
        dev = st.indptr.device
        _has, r_ptr, r_items = history_csr(queries, self.items, dev)
        return target_scores(st.score(r_ptr, r_items, agg), targets, self.items)

    def __call__(self, query, items: ItemList) -> ItemList:
        return self.score_batch([query], [items])[0]

    def recommend_batch(self, queries, n: int, *, exclude: Literal["query"] | None = "query") -> list[ItemList]:
        """
        Top-``n`` items for every query, scored and selected on the device in one launch: for each query the result
        of ``TrainingItemsCandidateSelector`` (every item, minus the query's items when ``exclude="query"``),
        ``__call__`` and ``TopNRanker``, bit for bit.  Zero scores are ranked like any other; a query without known
        reference items gets an empty list.
        """
        check_exclude(exclude)
        agg = self._agg()
        st = self._device_state()
        dev = st.indptr.device
        n_eff = rank_size(n, st.n_items)
        if n_eff == 0:
            return [empty_list(self.items) for _ in queries]
        _has, r_ptr, r_items = history_csr(queries, self.items, dev)
        excl = (r_ptr, r_items) if exclude == "query" else (None, None)
        idx, val, cnt = st.recommend(r_ptr, r_items, agg, n_eff, *excl)
        return ranked_lists(self.items, len(queries), range(len(queries)), idx, val, cnt)
