"""
User-kNN scorer on the H100 engine (SURVEY.md §8f N3) — the component surface of
``lenskit.knn.user.UserKNNScorer`` (``src/lenskit/knn/user.py:41-300``).

Training memorises the centred ratings and the unit-normalised user vectors exactly as the reference
does (``user.py:112-155``, SciPy on the host: it is the model, not a hot path).  Scoring a query is
(i) the neighbour similarities ``user_vectors @ ratings`` with the ``min_sim`` mask (``user.py:189-214``,
kept on the host as in the reference) and (ii) the neighbourhood aggregation of
``_accel.knn.user_score_items_{explicit,implicit}`` (``src/accel/knn/user_score.rs:21-98``), which
runs on the device: the accumulator kernel of ``knn_score.cu`` in user mode — weights from the
neighbour list, values from the rating matrix — bit-exact against the oracle's ScoreAccumulator
emulation (``tests/test_user_knn_gpu.py``).  ``score_batch`` aggregates many queries in one launch.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import scipy.sparse.linalg as spla
import torch
from pydantic import AliasChoices, BaseModel, Field, PositiveFloat, PositiveInt, field_validator
from scipy.sparse import csr_array

from . import _lib, engine
from .als import _as_dataset
from .components import Component, ItemList, RecQuery, Trainable, TrainingOptions
from .data import InteractionCSR


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

    def __getstate__(self):
        d = dict(self.__dict__)
        d.pop("_state", None)
        return d

    def _user_data(self, query: RecQuery):
        """``_get_user_data`` (user.py:257-300): (user index or None, dense rating vector, user mean) or None."""
        index = self.users.number(query.user_id, missing=None) if query.user_id is not None else None
        if query.query_items is None:
            if index is None:
                return None
            row = self.user_vectors[[int(index)], :].toarray()[0, :]
            umean = float(self.user_means[index]) if self.config.explicit else 0.0
            return int(index), row, umean
        if len(query.query_items) == 0:
            return None
        ratings = np.zeros(len(self.items), dtype=np.float32)
        ui_nos = query.query_items.numbers(vocabulary=self.items, missing="negative")
        ui_mask = ui_nos >= 0
        if self.config.explicit:
            urv = query.query_items.field("rating")
            if urv is None:
                return None
            urv = np.require(urv, dtype=np.float32)
            umean = float(urv.mean())
            ratings[ui_nos[ui_mask]] = urv[ui_mask] - umean
        else:
            umean = 0.0
            ratings[ui_nos[ui_mask]] = 1.0
        return index, ratings, umean

    def _neighbours(self, query: RecQuery):
        """The neighbour list of a query (user.py:189-214): (neighbour rows int32, similarities f32, mean) or None."""
        ud = self._user_data(query)
        if ud is None:
            return None
        uidx, ratings, umean = ud
        nbr_sims = self.user_vectors @ ratings
        if uidx is not None:
            nbr_sims[uidx] = 0  # zero out the self-similarity
        mask = nbr_sims >= self.config.min_sim
        if not mask.any():
            return None
        return np.flatnonzero(mask).astype(np.int32), nbr_sims[mask].astype(np.float32), umean

    def score_batch(self, queries: list, targets: list[ItemList]) -> list[ItemList]:
        """``__call__`` for many queries: the neighbourhood aggregation of all of them in one device launch."""
        st = self._device_state()
        dev = st.sim_cols.device
        r_ptr, t_ptr = [0], [0]
        nbrs, sims, tgts, metas = [], [], [], []
        for q, items in zip(queries, targets):
            q = RecQuery.create(q)
            nb = self._neighbours(q) if len(items) > 0 else None
            iidx = items.numbers(vocabulary=self.items, missing="negative").astype(np.int32)
            if nb is None:
                metas.append(None)
                r_ptr.append(r_ptr[-1])
                t_ptr.append(t_ptr[-1])
                continue
            ki = iidx >= 0
            nbrs.append(nb[0])
            sims.append(nb[1])
            tgts.append(iidx[ki])  # only known items are passed down (user.py:218-221)
            metas.append((ki, nb[2]))
            r_ptr.append(r_ptr[-1] + len(nb[0]))
            t_ptr.append(t_ptr[-1] + int(ki.sum()))
        cat = lambda xs, dt: torch.from_numpy(np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)).to(dev)  # noqa: E731
        sc = np.zeros(0, np.float32)
        if t_ptr[-1] > 0:
            scores, _counts = st.score(
                torch.tensor(r_ptr, dtype=torch.int64, device=dev), cat(nbrs, np.int32), cat(sims, np.float32),
                torch.tensor(t_ptr, dtype=torch.int64, device=dev), cat(tgts, np.int32),
                self.config.max_nbrs, self.config.min_nbrs,
            )  # fmt: skip
            sc = scores.cpu().numpy()
        out = []
        for i, items in enumerate(targets):
            if metas[i] is None:
                out.append(ItemList(items, scores=np.nan))
                continue
            ki, umean = metas[i]
            full = np.full(len(items), np.nan, dtype=np.float32)
            full[ki] = sc[t_ptr[i] : t_ptr[i + 1]] + np.float32(umean)  # scores += umean (user.py:243-244)
            out.append(ItemList(items, scores=full))
        return out

    def __call__(self, query, items: ItemList) -> ItemList:
        return self.score_batch([query], [items])[0]
