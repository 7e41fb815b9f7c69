"""
Item-kNN scorer on the H100 engine — the component surface of
``lenskit.knn.item.ItemKNNScorer`` (``src/lenskit/knn/item.py:41-295``).

Same config fields / aliases (``max_nbrs``/``nnbrs``/``k``, ``min_nbrs``,
``min_sim`` with its float64 clamp, ``save_nbrs``, ``feedback``, the unused
``block_size``), same trained attributes (``items``, ``item_means``,
``item_counts``, ``sim_matrix``), same per-query ``__call__``; plus
``score_batch`` which scores many queries in one launch (the reference scores
one query per call on one thread), and ``recommend_batch``, the batched form of
candidate selector → scorer → ``TopNRanker``, whose scoring and top-n selection
run together in one kernel (``lk_knn_recommend_batch``).
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch
from pydantic import AliasChoices, BaseModel, Field, PositiveFloat, PositiveInt, field_validator

from . import _lib, engine
from .batch import check_exclude, empty_list, rank_size, ranked_lists
from .components import Component, ItemList, RecQuery, Trainable, TrainingOptions, _as_dataset
from .data import InteractionCSR, knn_item_matrices


class ItemKNNConfig(BaseModel, extra="forbid"):
    max_nbrs: PositiveInt = Field(20, validation_alias=AliasChoices("max_nbrs", "nnbrs", "k"))
    min_nbrs: PositiveInt = 1
    min_sim: PositiveFloat = 1.0e-6
    save_nbrs: PositiveInt | None = None
    feedback: Literal["explicit", "implicit"] = "explicit"
    block_size: int = 250  # accepted and ignored, as in the reference (SURVEY.md App. A)
    prep: Literal["device", "host"] = "device"
    "Engine option: where centring / normalisation / transposition run (bit-identical either way)."

    @field_validator("min_sim", mode="after")
    @staticmethod
    def clamp_min_sim(sim) -> float:
        return max(sim, float(np.finfo(np.float64).smallest_normal))

    @field_validator("max_nbrs", mode="after")
    @staticmethod
    def check_max_nbrs(n) -> int:
        # engine limit (the reference has none): a target's accumulator heap lives in thread-local
        # memory of the scoring kernel — reported here, not at the first scoring call
        if n > engine.KNN_SCORE_MAX_NBRS:
            raise ValueError(f"max_nbrs={n} exceeds the engine limit of {engine.KNN_SCORE_MAX_NBRS}")
        return n

    @property
    def explicit(self) -> bool:
        return self.feedback == "explicit"


class ItemKNNScorer(Component, Trainable):
    CONFIG_CLASS = ItemKNNConfig
    config: ItemKNNConfig

    items = None
    item_means: np.ndarray | None = None
    item_counts: np.ndarray
    sim_matrix: InteractionCSR

    def is_trained(self) -> bool:
        return hasattr(self, "sim_matrix")

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        dev = _lib.require_device()
        it = ds.interactions
        if self.config.prep == "device":
            # knn/item.py:141-157,202-228 on the device (prep.cu): the COO triplets go up once, the f32
            # inputs of the build are the same bits the SciPy path produces (tests/test_prep_gpu.py)
            from . import prep

            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
            d_ui, d_iu, d_means = prep.knn_item_matrices_device(
                up(it.users), up(it.items), up(it.ratings) if self.config.explicit else None,
                it.n_users, it.n_items, self.config.explicit,
            )  # fmt: skip
            means = None if d_means is None else d_means.cpu().numpy()
            if means is not None and bool(torch.all(d_ui.values == 0)):
                import warnings

                warnings.warn("Ratings seem to have the same value, centering is not recommended.", UserWarning)
        else:
            # host prep with the reference's own SciPy calls
            ui, iu, means = knn_item_matrices(it, self.config.explicit)
            d_ui, d_iu = engine.DeviceCSR.from_host(ui, dev), engine.DeviceCSR.from_host(iu, dev)
        self.prep_where = "device (prep.cu)" if self.config.prep == "device" else "host (SciPy)"
        plan = engine.KnnBuildPlan.create(d_ui, d_iu)
        if self.config.save_nbrs:
            cols, vals, cnt = plan.build_topk(self.config.min_sim, int(self.config.save_nbrs))
            indptr, c, v = engine.topk_rows_to_csr(cols, vals, cnt)
        else:
            indptr, c, v = plan.build_unbounded(self.config.min_sim)
        n = ds.item_count
        self._state = engine.KnnScorerState.create(n, indptr, c, v, dev)
        self.items = ds.items
        self.item_means = means
        self.sim_matrix = InteractionCSR(indptr.cpu().numpy(), c.cpu().numpy(), v.cpu().numpy(), (n, n))
        self.item_counts = np.diff(self.sim_matrix.indptr)

    # -- inference -----------------------------------------------------------
    def _device_state(self) -> engine.KnnScorerState:
        st = getattr(self, "_state", None)
        if st is None:  # e.g. after unpickling
            s = self.sim_matrix
            st = engine.KnnScorerState.create(s.shape[0], s.indptr, s.indices, s.values, _lib.require_device())
            self._state = st
        return st

    def __getstate__(self):
        d = dict(self.__dict__)
        d.pop("_state", None)
        return d

    def score_batch(self, queries: list[ItemList], targets: list[ItemList]) -> list[ItemList]:
        """Score ``targets[i]`` for history ``queries[i]``, all in one device launch."""
        st = self._device_state()
        dev = st.sim_cols.device
        r_ptr, t_ptr = [0], [0]
        r_items, r_vals, t_items = [], [], []
        for hist, tgt in zip(queries, targets):
            rn = hist.numbers(vocabulary=self.items, missing="negative").astype(np.int32)
            tn = tgt.numbers(vocabulary=self.items, missing="negative").astype(np.int32)
            if self.config.explicit:
                rv = hist.field("rating")
                if rv is None:
                    raise RuntimeError("explicit-feedback scorer must have ratings")
                rv = rv.astype(np.float32, copy=True)
                ok = rn >= 0
                rv[ok] -= self.item_means[rn[ok]]  # knn/item.py:262-271
                r_vals.append(rv)
            r_items.append(rn)
            t_items.append(tn)
            r_ptr.append(r_ptr[-1] + len(rn))
            t_ptr.append(t_ptr[-1] + len(tn))
        cat = lambda xs, dt: torch.from_numpy(np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)).to(dev)  # noqa: E731
        scores, counts = st.score(
            torch.tensor(r_ptr, dtype=torch.int64, device=dev),
            cat(r_items, np.int32),
            cat(r_vals, np.float32) if self.config.explicit else None,
            torch.tensor(t_ptr, dtype=torch.int64, device=dev),
            cat(t_items, np.int32),
            self.config.max_nbrs,
            self.config.min_nbrs,
        )
        sc = scores.cpu().numpy()
        ct = counts.cpu().numpy()
        out = []
        for i, tgt in enumerate(targets):
            s = sc[t_ptr[i] : t_ptr[i + 1]].copy()
            tn = t_items[i]
            if self.config.explicit:
                ok = tn >= 0
                s[ok] += self.item_means[tn[ok]]  # knn/item.py:281-282
            out.append(ItemList(tgt, scores=s, nbr_counts=ct[t_ptr[i] : t_ptr[i + 1]]))
        return out

    def __call__(self, query, items: ItemList) -> ItemList:
        query = RecQuery.create(query)
        ratings = query.query_items
        if ratings is None or len(ratings) == 0:
            return ItemList(items, scores=np.nan)  # knn/item.py:238-245
        return self.score_batch([ratings], [items])[0]

    def recommend_batch(self, queries, n: int, *, exclude: Literal["query"] | None = "query") -> list[ItemList]:
        """
        Top-``n`` items for every query, scored and selected on the device in one launch: for each query the
        result of ``TrainingItemsCandidateSelector`` (every item, minus the query's items when
        ``exclude="query"``), ``__call__`` and ``TopNRanker``, bit for bit, with ``nbr_counts``.  A query without
        history gets an empty list.
        """
        check_exclude(exclude)
        st = self._device_state()
        dev = st.sim_cols.device
        n_eff = rank_size(n, st.n_items)
        hists = [RecQuery.create(q).query_items for q in queries]
        if n_eff == 0:
            return [empty_list(self.items) for _ in hists]
        at, r_ptr, r_items, r_vals = [], [0], [], []
        for i, hist in enumerate(hists):
            if hist is None or len(hist) == 0:  # knn/item.py:238-245: every score is null
                continue
            rn = hist.numbers(vocabulary=self.items, missing="negative").astype(np.int32)
            if self.config.explicit:
                rv = hist.field("rating")
                if rv is None:
                    raise RuntimeError("explicit-feedback scorer must have ratings")
                rv = rv.astype(np.float32, copy=True)
                ok = rn >= 0
                rv[ok] -= self.item_means[rn[ok]]  # knn/item.py:262-271
                r_vals.append(rv)
            at.append(i)
            r_items.append(rn)
            r_ptr.append(r_ptr[-1] + len(rn))
        if not at:
            return [empty_list(self.items) for _ in hists]
        ref_ptr = torch.tensor(r_ptr, dtype=torch.int64, device=dev)
        ref_items = torch.from_numpy(np.concatenate(r_items)).to(dev)
        idx, val, nbrs, cnt = st.recommend(
            ref_ptr, ref_items,
            torch.from_numpy(np.concatenate(r_vals)).to(dev) if self.config.explicit else None,
            self.config.max_nbrs, self.config.min_nbrs, n_eff,
            item_offset=torch.from_numpy(self.item_means).to(dev) if self.config.explicit else None,
            # the candidates leave out the query's own items: its history, already on the device
            excl_indptr=ref_ptr if exclude == "query" else None,
            excl_items=ref_items if exclude == "query" else None,
        )  # fmt: skip
        return ranked_lists(self.items, len(hists), at, idx, val, cnt, nbr_counts=nbrs)
