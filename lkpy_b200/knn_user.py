"""
User-kNN scorer on the H100 engine (SURVEY.md §8f N3) — the component surface of
``lenskit.knn.user.UserKNNScorer`` (``src/lenskit/knn/user.py:41-300``).

Training memorises the centred ratings and the unit-normalised user vectors exactly as the reference
does (``user.py:112-155``, SciPy on the host: it is the model, not a hot path).  Scoring a query is two
device steps:

(i) the neighbour search ``user_vectors @ ratings`` with the self-exclusion and the ``min_sim`` mask
(``user.py:189-214``): ``lk_uknn_search`` (``knn_user.cu``) gathers, for each of the query's items, the
item's column of the f64 user vectors and accumulates the similarities in f64 in ascending item order,
an unfused multiply and add per step — SciPy's own order and rounding, so the neighbour set and the f32
weights are the reference's bit for bit.  Known users' queries are their rows of the user vectors on the
device; provided histories are built on the host with the reference's rules (unknown items dropped, a
repeated item keeps its last value, explicit ratings centred by their f32 mean, implicit 1.0).

(ii) the neighbourhood aggregation of ``_accel.knn.user_score_items_{explicit,implicit}``
(``src/accel/knn/user_score.rs:21-98``): the accumulator kernel of ``knn_score.cu`` in user mode —
weights from the neighbour list, values from the rating matrix — bit-exact against the oracle's
ScoreAccumulator emulation (``tests/test_user_knn_gpu.py``).

``score_batch`` runs each step once for many queries, and the neighbour lists pass from (i) to (ii)
without leaving the device.  ``recommend_batch`` does the same over all items and selects each query's top n
in the aggregation kernel (its ranking mode, ``lk_knn_recommend_batch``), the batched form of scorer →
``TopNRanker``.  Both device states are built on first use and are not pickled.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import scipy.sparse.linalg as spla
import torch
from pydantic import AliasChoices, BaseModel, Field, PositiveFloat, PositiveInt, field_validator
from scipy.sparse import csr_array

from . import _lib, engine
from .components import Component, ItemList, RecQuery, Trainable, TrainingOptions, _as_dataset
from .data import InteractionCSR
from .batch import check_exclude, empty_list, history_csr, rank_size, ranked_lists


class UserKNNConfig(BaseModel, extra="forbid"):
    max_nbrs: PositiveInt = Field(20, validation_alias=AliasChoices("max_nbrs", "nnbrs", "k"))
    min_nbrs: PositiveInt = 1
    min_sim: PositiveFloat = 1.0e-6
    feedback: Literal["explicit", "implicit"] = "explicit"

    @field_validator("min_sim", mode="after")
    @staticmethod
    def clamp_min_sim(sim) -> float:
        return max(sim, float(np.finfo(np.float64).smallest_normal))

    @field_validator("max_nbrs", mode="after")
    @staticmethod
    def check_max_nbrs(n) -> int:
        if n > engine.KNN_SCORE_MAX_NBRS:
            raise ValueError(f"max_nbrs={n} exceeds the engine limit of {engine.KNN_SCORE_MAX_NBRS}")
        return n

    @property
    def explicit(self) -> bool:
        return self.feedback == "explicit"


class UserKNNScorer(Component, Trainable):
    CONFIG_CLASS = UserKNNConfig
    config: UserKNNConfig

    users = None
    items = None
    user_means: np.ndarray | None = None
    user_vectors: csr_array
    user_ratings: InteractionCSR

    def is_trained(self) -> bool:
        return hasattr(self, "user_ratings")

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        it = ds.interactions
        vals = it.ratings if self.config.explicit else np.ones(it.nnz, dtype=np.float32)
        rmat = csr_array(it.coo(vals.astype(np.float32))).astype(np.float32)
        rmat.sort_indices()
        means = None
        if self.config.explicit:  # user.py:131-145
            counts = np.diff(rmat.indptr)
            sums = rmat.sum(axis=1)
            means = np.zeros(sums.shape, dtype=np.float32)
            np.divide(sums, counts, out=means, where=counts > 0)
            rmat.data = rmat.data - np.repeat(means, counts)
        norms = spla.norm(rmat, 2, axis=1)  # user.py:147-155
        cmat = rmat / np.maximum(norms, np.finfo("f4").smallest_normal).reshape(-1, 1)
        self.user_vectors = cmat.tocsr()
        self.user_ratings = InteractionCSR.from_scipy(rmat)
        self.users = ds.users
        self.user_means = means
        self.items = ds.items

    # -- inference -----------------------------------------------------------
    def _device_state(self) -> engine.KnnScorerState:
        st = self.__dict__.get("_state")
        if st is None:
            r = self.user_ratings
            st = engine.KnnScorerState.create(
                r.shape[1], r.indptr, r.indices, r.values if self.config.explicit else None,
                _lib.require_device(), user_mode=True,
            )  # fmt: skip
            self.__dict__["_state"] = st
        return st

    def _neighbour_state(self) -> engine.UserNeighbourState:
        ns = self.__dict__.get("_nbr_state")
        if ns is None:
            ns = engine.UserNeighbourState.create(self.user_vectors, _lib.require_device())
            self.__dict__["_nbr_state"] = ns
        return ns

    def __getstate__(self):
        d = dict(self.__dict__)
        d.pop("_state", None)
        d.pop("_nbr_state", None)
        return d

    def _query(self, query: RecQuery):
        """``_get_user_data`` (user.py:257-300) as a neighbour-search query: (query, user mean) or None, where the
        query is the user's number (its row of the user vectors) or ``(items, values, self)`` for a history."""
        index = self.users.number(query.user_id, missing=None) if query.user_id is not None else None
        if query.query_items is None:
            if index is None:
                return None
            umean = float(self.user_means[index]) if self.config.explicit else 0.0
            return int(index), umean
        if len(query.query_items) == 0:
            return None
        ui_nos = query.query_items.numbers(vocabulary=self.items, missing="negative")
        urv = None
        if self.config.explicit:
            urv = query.query_items.field("rating")
            if urv is None:
                return None
        items, vals, umean = engine.history_query(ui_nos, urv)
        return (items, vals, None if index is None else int(index)), umean

    def score_batch(self, queries: list, targets: list[ItemList]) -> list[ItemList]:
        """``__call__`` for many queries: one neighbour search and one neighbourhood aggregation on the device for
        all of them; the neighbour lists go from the search to the aggregation without leaving the device."""
        st = self._device_state()
        dev = st.sim_cols.device
        specs, at, means = [], [], []
        for i, (q, items) in enumerate(zip(queries, targets)):
            qd = self._query(RecQuery.create(q)) if len(items) > 0 else None
            if qd is not None:
                specs.append(qd[0])
                at.append(i)
                means.append(qd[1])
        metas = [None] * len(targets)
        t_ptr, tgts = [0], []
        nb_indptr = None
        if specs:
            ns = self._neighbour_state()
            nb_indptr, nb_rows, nb_sims = ns.neighbours(ns.queries(specs), self.config.min_sim)
            n_nbrs = np.diff(nb_indptr.cpu().numpy())
            for j, i in enumerate(at):
                if n_nbrs[j] == 0:  # no neighbour: every score is null
                    t_ptr.append(t_ptr[-1])
                    continue
                iidx = targets[i].numbers(vocabulary=self.items, missing="negative").astype(np.int32)
                ki = iidx >= 0
                tgts.append(iidx[ki])  # only known items are passed down (user.py:218-221)
                metas[i] = (ki, means[j], j)
                t_ptr.append(t_ptr[-1] + int(ki.sum()))
        sc = np.zeros(0, np.float32)
        if t_ptr[-1] > 0:
            scores, _counts = st.score(
                nb_indptr, nb_rows, nb_sims, torch.tensor(t_ptr, dtype=torch.int64, device=dev),
                torch.from_numpy(np.concatenate(tgts).astype(np.int32)).to(dev),
                self.config.max_nbrs, self.config.min_nbrs,
            )  # fmt: skip
            sc = scores.cpu().numpy()
        out = []
        for i, items in enumerate(targets):
            if metas[i] is None:
                out.append(ItemList(items, scores=np.nan))
                continue
            ki, umean, j = metas[i]
            full = np.full(len(items), np.nan, dtype=np.float32)
            full[ki] = sc[t_ptr[j] : t_ptr[j + 1]] + np.float32(umean)  # scores += umean (user.py:243-244)
            out.append(ItemList(items, scores=full))
        return out

    def __call__(self, query, items: ItemList) -> ItemList:
        return self.score_batch([query], [items])[0]

    def recommend_batch(self, queries, n: int, *, exclude: Literal["query"] | None = "query") -> list[ItemList]:
        """
        Top-``n`` items for every query: one neighbour search, then scoring and selection over all items in one
        launch (``KnnScorerState.recommend`` in user mode).  For each query the result of
        ``TrainingItemsCandidateSelector`` (every item, minus the known items of ``query.query_items`` when
        ``exclude="query"``; a query given only a user id excludes nothing), ``__call__`` and ``TopNRanker``, bit
        for bit.  A query without neighbours or usable data gets an empty list.
        """
        check_exclude(exclude)
        st = self._device_state()
        dev = st.sim_cols.device
        n_eff = rank_size(n, st.n_items)
        rqs = [RecQuery.create(q) for q in queries]
        if n_eff == 0:
            return [empty_list(self.items) for _ in rqs]
        specs, at, means = [], [], []
        for i, rq in enumerate(rqs):
            qd = self._query(rq)
            if qd is not None:
                specs.append(qd[0])
                at.append(i)
                means.append(qd[1])
        if not specs:
            return [empty_list(self.items) for _ in rqs]
        ns = self._neighbour_state()
        nb_indptr, nb_rows, nb_sims = ns.neighbours(ns.queries(specs), self.config.min_sim)
        excl = (None, None)
        if exclude == "query":  # the known items of query_items; a query given only a user id excludes nothing
            excl = history_csr([rqs[i] for i in at], self.items, dev)[1:]
        idx, val, _nbrs, cnt = st.recommend(
            nb_indptr, nb_rows, nb_sims, self.config.max_nbrs, self.config.min_nbrs, n_eff,
            query_offset=torch.tensor(means, dtype=torch.float32, device=dev),  # scores += umean (user.py:243-244)
            excl_indptr=excl[0], excl_items=excl[1],
        )  # fmt: skip
        # cnt is 0 for a query without neighbours: every score is null
        return ranked_lists(self.items, len(rqs), at, idx, val, cnt)
