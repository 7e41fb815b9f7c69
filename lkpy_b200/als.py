"""
ALS scorers on the H100 engine — the component surface of ``lenskit.als``.

Mirrors (same names, config fields and aliases, training/epoch contract):

* ``ALSConfig`` / ``ImplicitMFConfig`` / ``BiasedMFConfig``
  (``src/lenskit/als/_common.py:36-78``, ``_implicit.py:24-32``, ``_explicit.py:25-29``)
* ``ImplicitMFScorer`` / ``BiasedMFScorer`` and their trainers
  (``_implicit.py:35-175``, ``_explicit.py:32-118``, ``_common.py:113-356``)

What differs: factor tables and the two CSR orientations live in HBM for the
whole training run; a half-epoch is ``lk_als_otor`` + ``lk_als_half_epoch`` on
the device; ``user_embeddings`` / ``item_embeddings`` are materialised on the
host after every epoch (the model must be usable after each ``train_epoch()``,
``training.py:364-370``).  The engine-only option ``gather_dtype="bfloat16"``
gathers a bf16 copy of the opposite factor table (BASELINE.json config 2).
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch
from pydantic import AliasChoices, BaseModel, Field, PositiveFloat, PositiveInt, field_validator

from . import _lib, engine
from .components import Component, Dataset, ItemList, ModelTrainer, RecQuery, TrainingOptions, UsesTrainer
from .data import InteractionCSR, Interactions


class ALSConfig(BaseModel):
    embedding_size: PositiveInt = Field(default=64, validation_alias=AliasChoices("embedding_size", "features"))
    epochs: PositiveInt = 10
    regularization: PositiveFloat | tuple[PositiveFloat, PositiveFloat] = 0.1
    user_embeddings: bool | Literal["prefer"] = True
    gather_dtype: Literal["float32", "bfloat16"] = "float32"
    "Engine option: storage type of the gathered (opposite) factor rows."

    @field_validator("embedding_size", mode="after")
    @staticmethod
    def check_embedding_size(k) -> int:
        # engine limit (the reference has none), reported at configuration time
        if k > engine.ALS_MAX_FEATURES:
            raise ValueError(f"embedding_size={k} exceeds the engine limit of {engine.ALS_MAX_FEATURES}")
        return k

    @property
    def user_reg(self) -> float:
        r = self.regularization
        return float(r[0]) if isinstance(r, tuple) else float(r)

    @property
    def item_reg(self) -> float:
        r = self.regularization
        return float(r[1]) if isinstance(r, tuple) else float(r)


class ImplicitMFConfig(ALSConfig):
    weight: float = 40
    use_ratings: bool = False


class BiasedMFConfig(ALSConfig):
    damping: float | tuple[float, float] = 5.0


def _as_dataset(data) -> Dataset:
    if isinstance(data, Dataset):
        return data
    if isinstance(data, Interactions):
        return Dataset(data)
    raise TypeError("expected a Dataset or Interactions")


class ALSBase(UsesTrainer, Component):
    """``ALSBase`` (als/_common.py:113-192)."""

    users = None
    items = None
    user_embeddings: np.ndarray | None = None
    item_embeddings: np.ndarray | None = None

    def is_trained(self) -> bool:
        return self.item_embeddings is not None

    def new_user_embedding(self, user_num, items: ItemList):  # pragma: no cover
        raise NotImplementedError

    def finalize_scores(self, user_num, items: ItemList, user_bias) -> ItemList:
        return items

    def __call__(self, query, items: ItemList) -> ItemList:
        query = RecQuery.create(query)
        user_num = None
        if query.user_id is not None and self.users is not None:
            user_num = self.users.number(query.user_id, missing=None)
        u_offset = None
        u_feat = None
        if (
            query.query_items is not None
            and len(query.query_items) > 0
            and self.config.user_embeddings != "prefer"
        ):
            u_feat, u_offset = self.new_user_embedding(user_num, query.query_items)
        if u_feat is None:
            if user_num is None or self.user_embeddings is None:
                return ItemList(items, scores=np.nan)
            u_feat = self.user_embeddings[user_num, :]
        item_nums = items.numbers(vocabulary=self.items, missing="negative")
        mask = item_nums >= 0
        scores = np.full((len(items),), np.nan, dtype=np.float32)
        scores[mask] = self.item_embeddings[item_nums[mask], :] @ u_feat
        return self.finalize_scores(user_num, ItemList(items, scores=scores), u_offset)

    # ------------------------------------------------------------------------------------------
    # Batched inference on the device (SURVEY.md §8f N1 + N2): what the reference does one query at
    # a time — ALSBase.__call__ (als/_common.py:133-175), fold-in (_implicit.py:77-130), TopNRanker
    # → ItemList.top_n → argtopn (basic/topn.py:32-69, data/_items.py:942-998,
    # src/accel/data/sorting.rs:131-170) — for a whole batch of queries with the factors resident
    # in HBM: fold-in rows by the training kernel, scores by one library GEMM (Q · Xᵀ, item-major so
    # the selection kernel's scan is coalesced), top-N by lk_topn_columns.
    # ------------------------------------------------------------------------------------------

    def _device_items(self) -> torch.Tensor:
        dev = _lib.require_device()
        cached = self.__dict__.get("_d_items_cache")
        if cached is None or cached[0] is not self.item_embeddings:
            t = torch.from_numpy(np.ascontiguousarray(self.item_embeddings, dtype=np.float32)).to(dev)
            self.__dict__["_d_items_cache"] = cached = (self.item_embeddings, t)
        return cached[1]

    def fold_in_batch(self, histories: list[ItemList]) -> torch.Tensor:  # pragma: no cover
        raise NotImplementedError

    def batch_offsets(self, user_nums: np.ndarray, fold_bias: np.ndarray | None):
        """(per-item offset [n_items] or None, per-query offset [B] or None) added to Q · Xᵀ."""
        return None, None

    def embed_batch(self, queries) -> tuple[torch.Tensor, np.ndarray, np.ndarray, np.ndarray | None]:
        """
        Query embeddings on the device: ``(X [B, k], scorable [B] bool, user_nums [B] (-1 unknown),
        fold-in user offsets or None)`` with the precedence rules of ``__call__``.
        """
        dev = _lib.require_device()
        queries = [RecQuery.create(q) for q in queries]
        k = self.item_embeddings.shape[1]
        B = len(queries)
        user_nums = np.full(B, -1, dtype=np.int64)
        for b, q in enumerate(queries):
            if q.user_id is not None and self.users is not None:
                num = self.users.number(q.user_id, missing=None)
                if num is not None:
                    user_nums[b] = num
        fold = np.array(
            [q.query_items is not None and len(q.query_items) > 0 and self.config.user_embeddings != "prefer"
             for q in queries], dtype=bool,
        )  # fmt: skip
        X = torch.zeros((B, k), dtype=torch.float32, device=dev)
        scorable = fold.copy()
        fold_bias = None
        if fold.any():
            rows = np.flatnonzero(fold)
            emb, fold_bias_rows = self.fold_in_batch([queries[b].query_items for b in rows])
            X[torch.from_numpy(rows).to(dev)] = emb
            if fold_bias_rows is not None:
                fold_bias = np.full(B, np.nan, dtype=np.float32)
                fold_bias[rows] = fold_bias_rows
        known = ~fold & (user_nums >= 0) & (self.user_embeddings is not None)
        if known.any():
            rows = np.flatnonzero(known)
            emb = torch.from_numpy(np.ascontiguousarray(self.user_embeddings[user_nums[rows]], dtype=np.float32))
            X[torch.from_numpy(rows).to(dev)] = emb.to(dev)
            scorable |= known
        return X, scorable, user_nums, fold_bias

    def score_matrix(self, queries) -> torch.Tensor:
        """Scores of every item for every query, item-major: [n_items, B] f32, NaN columns for unscorable queries."""
        X, scorable, user_nums, fold_bias = self.embed_batch(queries)
        S = self._device_items() @ X.T  # [n_items, B]; fp32 GEMM (allow_tf32 is off by default)
        item_off, query_off = self.batch_offsets(user_nums, fold_bias)
        if item_off is not None:
            S += torch.from_numpy(item_off.astype(np.float32)).to(S.device)[:, None]
        if query_off is not None:
            S += torch.from_numpy(query_off.astype(np.float32)).to(S.device)[None, :]
        if not scorable.all():
            S[:, torch.from_numpy(np.flatnonzero(~scorable)).to(S.device)] = float("nan")
        return S

    def recommend_batch(self, queries, n: int) -> list[ItemList]:
        """Top-``n`` items for every query: the batched form of scorer → ``TopNRanker``."""
        S = self.score_matrix(queries)
        n_eff = min(int(n), S.shape[0])
        if n_eff <= 0:
            return [ItemList([], scores=np.empty(0, dtype=np.float32)) for _ in range(S.shape[1])]
        idx, val, cnt = engine.topn_columns(S, n_eff)
        idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy()
        out = []
        for b in range(S.shape[1]):
            c = int(cnt[b])
            out.append(
                ItemList(item_ids=self.items.ids(idx[b, :c]), item_nums=idx[b, :c].copy(), vocabulary=self.items,
                         scores=val[b, :c].copy())
            )  # fmt: skip
        return out


def _solve_cholesky(A: np.ndarray, y: np.ndarray) -> np.ndarray:
    """``lenskit.math.solve.solve_cholesky`` (math/solve.py:17-41); host fold-in only."""
    from scipy.linalg import cho_factor, cho_solve

    return np.require(cho_solve(cho_factor(A), y), dtype=A.dtype)


class ALSTrainerBase(ModelTrainer):
    """``ALSTrainerBase`` (als/_common.py:195-356) with device-resident state."""

    MODE = _lib.LK_ALS_IMPLICIT
    kernel_events: list | None = None  # bench.py: (start, end) CUDA events around each row-solve launch

    def __init__(self, scorer: ALSBase, data, options: TrainingOptions):
        from .prep import DeviceInteractions, coo_to_csr_pair

        self.scorer = scorer
        self.device = _lib.require_device()
        self.rng = options.random_generator()
        k = self.config.embedding_size
        if isinstance(data, DeviceInteractions):
            # interactions already in HBM (scale-out configurations): R and Rᵀ are built on the device
            # (prep.coo_to_csr_pair, the role of als/_common.py:216-219); there is no host copy
            from .components import Vocabulary

            scorer.users = Vocabulary(np.arange(data.n_users), "user")
            scorer.items = Vocabulary(np.arange(data.n_items), "item")
            self.ui_host = self.iu_host = None
            self.ui, self.iu, _ = coo_to_csr_pair(
                data.users, data.items, self.prepare_values_device(data), data.n_users, data.n_items
            )
            n_users, n_items = data.n_users, data.n_items
        else:
            ds = _as_dataset(data)
            scorer.users = ds.users
            scorer.items = ds.items
            coo = self.prepare_matrix(ds)
            self.ui_host = InteractionCSR.from_scipy(coo)
            self.iu_host = InteractionCSR.from_scipy(coo.T)
            self.ui = engine.DeviceCSR.from_host(self.ui_host, self.device)
            self.iu = engine.DeviceCSR.from_host(self.iu_host, self.device)
            n_users, n_items = ds.user_count, ds.item_count
        self._make_plans(k)
        self.otor_ws = engine.OtorWorkspace.create(k, self.device)

        # items first, then users, from one generator (als/_common.py:287-301)
        q0 = self.initial_params(n_items, k)
        p0 = self.initial_params(n_users, k)
        self.d_items = torch.from_numpy(q0).to(self.device)
        self.d_users = torch.from_numpy(p0).to(self.device)
        self.bf16 = self.config.gather_dtype == "bfloat16"
        self.d_items_bf16 = torch.empty_like(self.d_items, dtype=torch.bfloat16) if self.bf16 else None
        self.d_users_bf16 = torch.empty_like(self.d_users, dtype=torch.bfloat16) if self.bf16 else None
        self.epochs_trained = 0
        self._sync_host()

    @property
    def config(self):
        return self.scorer.config

    def _chunk_nnz(self, k: int) -> int:
        weighted = self.MODE == _lib.LK_ALS_IMPLICIT and getattr(self.config, "use_ratings", False)
        bf16_uniform = self.config.gather_dtype == "bfloat16" and not weighted
        # shorter parts for the tensor-core Gram at k = 128 and on the tf32 paths (engine.TF32_CHUNK_NNZ*: part
        # lengths carried over from an earlier tensor-core design, not re-measured on the H100)
        if k == 128:
            return engine.TF32_CHUNK_NNZ if bf16_uniform else engine.TF32_CHUNK_NNZ_K128
        if k == 64 and not bf16_uniform:
            return engine.TF32_CHUNK_NNZ
        return engine.DEFAULT_CHUNK_NNZ

    def _make_plans(self, k: int) -> None:
        c = self._chunk_nnz(k)
        self.u_plan = engine.ALSHalfPlan.create(self.ui, k, c)
        self.i_plan = engine.ALSHalfPlan.create(self.iu, k, c)

    # -- hooks -------------------------------------------------------------
    def prepare_matrix(self, data: Dataset):  # pragma: no cover
        raise NotImplementedError

    def prepare_values_device(self, data) -> torch.Tensor:  # pragma: no cover
        raise NotImplementedError("this trainer has no device-resident input path")

    def initial_params(self, nrows: int, ncols: int) -> np.ndarray:  # pragma: no cover
        raise NotImplementedError

    # -- epoch ---------------------------------------------------------------
    def _half(self, plan, this, other, other_bf16, reg: float, replicas=None, replica_row0: int = 0,
              before_solve=None) -> torch.Tensor:  # fmt: skip
        plan.sqdelta.zero_()
        otor = None
        gather = other
        if self.MODE == _lib.LK_ALS_IMPLICIT:
            otor = engine.als_otor(other, reg, self.otor_ws, other_bf16)
            if other_bf16 is not None:
                gather = other_bf16
        elif other_bf16 is not None:
            other_bf16.copy_(other)
            gather = other_bf16
        if before_solve is not None:
            before_solve()  # e.g. wait for the upload of `this` that ran beside the OtOr pass
        if self.kernel_events is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        engine.als_half_epoch(
            plan, self.MODE, this, gather, otor=otor, reg=reg, replicas=replicas, replica_row0=replica_row0
        )
        if self.kernel_events is not None:
            e1.record()
            self.kernel_events.append((e0, e1))
        return plan.sqdelta

    def train_epoch_device(self) -> tuple[torch.Tensor, torch.Tensor]:
        """One epoch entirely on the device; returns the two Σ‖Δ‖² scalars (device)."""
        self.u_plan.status.zero_()
        self.i_plan.status.zero_()
        du = self._half(self.u_plan, self.d_users, self.d_items, self.d_items_bf16, self.config.user_reg)
        di = self._half(self.i_plan, self.d_items, self.d_users, self.d_users_bf16, self.config.item_reg)
        self.epochs_trained += 1
        return du, di

    def solve_kernel_name(self) -> str:
        """Which row-solve kernel the configuration runs (bench.py's roofline label)."""
        k = self.config.embedding_size
        on = _lib.get_option("LK_ALS_TC") != 0
        tf32 = _lib.get_option("LK_ALS_TF32") != 0

        def one(plan, other) -> str:
            # the conditions under which launch_als_tc (als_tc.cu) takes the launch
            weighted = self.MODE == _lib.LK_ALS_IMPLICIT and not plan.vals_uniform
            if not on or k not in (64, 128) or other.data_ptr() % 16 != 0:
                return "als_half_kernel"
            if weighted and not plan.uniform_val >= 0.0:  # sqrt(v) needs non-negative confidences
                return "als_half_kernel"
            if (not self.bf16 or weighted) and not tf32:
                return "als_half_kernel"
            return "als_tc_kernel"

        users = one(self.u_plan, self.d_items_bf16 if self.bf16 else self.d_items)
        items = one(self.i_plan, self.d_users_bf16 if self.bf16 else self.d_users)
        return users if users == items else f"{users} (user half) / {items} (item half)"

    def launches_per_epoch(self) -> int:
        """Kernels of this library launched by one epoch (two halves: OtOr partial + reduce + row solve)."""
        return 6 if self.MODE == _lib.LK_ALS_IMPLICIT else 2

    def _raise_on_status(self) -> None:
        for plan in (self.u_plan, self.i_plan):
            st = int(plan.status.item())
            if st:
                raise RuntimeError(f"ALS solve error: array minor of row {st - 1} is not positive")

    def train_epoch(self) -> dict[str, float]:
        du, di = self.train_epoch_device()
        self._sync_host()
        self._raise_on_status()
        return {"deltaP": float(np.sqrt(du.item())), "deltaQ": float(np.sqrt(di.item()))}

    def _copy_stream(self) -> torch.cuda.Stream:
        s = self.__dict__.get("_copy_stream_obj")
        if s is None:
            s = self.__dict__["_copy_stream_obj"] = torch.cuda.Stream(device=self.device)
        return s

    def train_epoch_e2e(self, host_users: torch.Tensor, host_items: torch.Tensor) -> dict[str, float]:
        """
        One epoch with the factor tables taken from, and returned to, pinned host
        tensors (the host-array contract of ``train_*_matrix``); the CSR stays in HBM.
        The copies that do not sit on the dependency chain are hidden: Q goes up first (the user
        half's OtOr pass starts on it while P is still in flight on the copy stream), and P — final
        after the user half — comes down on the copy stream underneath the item half.
        """
        main = torch.cuda.current_stream()
        side = self._copy_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            self.d_users.copy_(host_users, non_blocking=True)  # old P: only the Δ-norm needs it
        self.d_items.copy_(host_items, non_blocking=True)
        self.u_plan.status.zero_()
        self.i_plan.status.zero_()
        du = self._half(self.u_plan, self.d_users, self.d_items, self.d_items_bf16, self.config.user_reg,
                        before_solve=lambda: main.wait_stream(side))  # fmt: skip
        side.wait_stream(main)
        with torch.cuda.stream(side):
            host_users.copy_(self.d_users, non_blocking=True)  # under the item half
        di = self._half(self.i_plan, self.d_items, self.d_users, self.d_users_bf16, self.config.item_reg)
        self.epochs_trained += 1
        host_items.copy_(self.d_items, non_blocking=True)
        main.wait_stream(side)
        deltas = torch.cat([du, di]).cpu()  # device->host read of the step's result; synchronises
        return {"deltaP": float(np.sqrt(deltas[0])), "deltaQ": float(np.sqrt(deltas[1]))}

    def _sync_host(self) -> None:
        self.scorer.user_embeddings = self.d_users.cpu().numpy()
        self.scorer.item_embeddings = self.d_items.cpu().numpy()

    def finalize(self) -> None:
        self._sync_host()
        if not self.config.user_embeddings:
            self.scorer.user_embeddings = None
            self.scorer.users = None

    def get_parameters(self) -> dict[str, object]:
        return {"user_embeddings": self.scorer.user_embeddings, "item_embeddings": self.scorer.item_embeddings}

    def load_parameters(self, state) -> None:
        self.d_users.copy_(torch.from_numpy(np.ascontiguousarray(state["user_embeddings"], dtype=np.float32)))
        self.d_items.copy_(torch.from_numpy(np.ascontiguousarray(state["item_embeddings"], dtype=np.float32)))
        self._sync_host()


# ---------------------------------------------------------------------------
# implicit feedback
# ---------------------------------------------------------------------------


class ImplicitMFScorer(ALSBase):
    """``ImplicitMFScorer`` (als/_implicit.py:35-130)."""

    CONFIG_CLASS = ImplicitMFConfig
    config: ImplicitMFConfig
    _OtOr: np.ndarray

    def create_trainer(self, data, options):
        return ImplicitMFTrainer(self, data, options)

    def new_user_embedding(self, user_num, user_items: ItemList):
        ri = user_items.numbers(vocabulary=self.items, missing="negative")
        good = ri >= 0
        if self.config.use_ratings:
            ratings = user_items.field("rating")
            if ratings is None:
                raise ValueError("no ratings in user items")
            val = ratings[good] * self.config.weight
        else:
            val = np.full((int(good.sum()),), self.config.weight)
        val = val.astype(self.item_embeddings.dtype)
        M = self.item_embeddings[ri[good], :]
        A = self._OtOr + (M.T * val) @ M
        y = M.T @ (val + 1.0)
        return _solve_cholesky(A, y.astype(A.dtype)), None

    def fold_in_batch(self, histories: list[ItemList]):
        """
        ``new_user_embedding`` for a batch of histories on the device: the histories become the rows
        of a CSR matrix and one ``lk_als_half_epoch`` (the training kernel, fp32 item table) solves
        them all — same math as ``_train_new_row`` (``_implicit.py:109-130``).
        """
        dev = _lib.require_device()
        k = self.item_embeddings.shape[1]
        cols, vals, indptr = [], [], [0]
        for h in histories:
            ri = h.numbers(vocabulary=self.items, missing="negative")
            good = ri >= 0
            if self.config.use_ratings:
                ratings = h.field("rating")
                if ratings is None:
                    raise ValueError("no ratings in user items")
                v = np.asarray(ratings)[good] * self.config.weight
            else:
                v = np.full(int(good.sum()), self.config.weight)
            c = ri[good].astype(np.int32)
            order = np.argsort(c, kind="stable")  # the CSR container wants ascending columns
            cols.append(c[order])
            vals.append(np.asarray(v, dtype=np.float32)[order])
            indptr.append(indptr[-1] + len(c))
        csr = InteractionCSR(
            np.asarray(indptr, dtype=np.int32),
            np.concatenate(cols) if cols else np.empty(0, np.int32),
            np.concatenate(vals) if vals else np.empty(0, np.float32),
            (len(histories), self.item_embeddings.shape[0]),
        )
        dm = engine.DeviceCSR.from_host(csr, dev)
        plan = engine.ALSHalfPlan.create(dm, k)
        d_items = self._device_items()
        ws = engine.OtorWorkspace.create(k, dev)
        otor = engine.als_otor(d_items, float(self.config.user_reg), ws, None)
        x = torch.zeros((len(histories), k), dtype=torch.float32, device=dev)
        plan.sqdelta.zero_()
        plan.status.zero_()
        engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, x, d_items, otor=otor)
        if int(plan.status.item()):
            raise RuntimeError("ALS solve error: a fold-in system is not positive definite")
        return x, None


class ImplicitMFTrainer(ALSTrainerBase):
    MODE = _lib.LK_ALS_IMPLICIT

    def prepare_matrix(self, data: Dataset):
        it = data.interactions
        base = it.ratings if self.config.use_ratings else np.ones(it.nnz, dtype=np.float32)
        vals = (np.require(base, dtype=np.float32) * self.config.weight).astype(np.float32)
        return it.coo(vals)

    def prepare_values_device(self, data) -> torch.Tensor:
        base = data.ratings if self.config.use_ratings else torch.ones_like(data.ratings)
        return (base.to(torch.float32) * float(self.config.weight)).to(torch.float32)

    def initial_params(self, nrows: int, ncols: int) -> np.ndarray:
        mat = self.rng.standard_normal((nrows, ncols), dtype=np.float32) * 0.01
        mat *= mat
        return mat

    def _save_user_otor(self) -> None:
        q = self.scorer.item_embeddings
        self.scorer._OtOr = q.T @ q + np.eye(q.shape[1], dtype=q.dtype) * self.config.user_reg

    def train_epoch(self):
        res = super().train_epoch()
        self._save_user_otor()
        return res

    def finalize(self):
        self._sync_host()
        self._save_user_otor()
        super().finalize()


# ---------------------------------------------------------------------------
# explicit feedback
# ---------------------------------------------------------------------------


class BiasModel:
    """The part of ``lenskit.basic.BiasModel`` (basic/bias.py:84-150) BiasedMF needs."""

    def __init__(self, global_bias, item_biases, user_biases, damping):
        self.global_bias = global_bias
        self.item_biases = item_biases
        self.user_biases = user_biases
        self.damping = damping

    @classmethod
    def learn(cls, it: Interactions, damping) -> "BiasModel":
        d_user, d_item = damping if isinstance(damping, tuple) else (damping, damping)
        g = float(np.mean(it.ratings))
        centered = it.ratings.astype(np.float64) - g
        counts = np.full(it.n_items, float(d_item))
        sums = np.zeros(it.n_items)
        np.add.at(counts, it.items, 1)
        np.add.at(sums, it.items, centered)
        ib = np.zeros(it.n_items, dtype=np.float32)
        np.divide(sums, counts, out=ib, where=counts > 0, casting="unsafe")
        centered = centered - ib[it.items]
        counts = np.full(it.n_users, float(d_user))
        sums = np.zeros(it.n_users)
        np.add.at(counts, it.users, 1)
        np.add.at(sums, it.users, centered)
        ub = np.zeros(it.n_users, dtype=np.float32)
        np.divide(sums, counts, out=ub, where=counts > 0, casting="unsafe")
        return cls(g, ib, ub, (d_user, d_item))

    def transform(self, it: Interactions) -> np.ndarray:
        return (it.ratings - self.global_bias - self.item_biases[it.items] - self.user_biases[it.users]).astype(
            np.float32
        )


class BiasedMFScorer(ALSBase):
    """``BiasedMFScorer`` (als/_explicit.py:32-91)."""

    CONFIG_CLASS = BiasedMFConfig
    config: BiasedMFConfig
    bias: BiasModel

    def create_trainer(self, data, options):
        return BiasedMFTrainer(self, data, options)

    def new_user_embedding(self, user_num, items: ItemList):
        inums = items.numbers(vocabulary=self.items, missing="negative")
        ratings = items.field("rating")
        assert ratings is not None
        mask = (inums >= 0) & np.isfinite(ratings)
        uoff = ratings - self.bias.global_bias
        uoff[inums >= 0] -= self.bias.item_biases[inums[inums >= 0]]
        u_bias = float(np.sum(uoff) / (np.sum(np.isfinite(uoff)) + self.bias.damping[0]))
        if not np.isfinite(u_bias):  # BiasModel.compute_for_items zeroes a NaN user bias (basic/bias.py)
            u_bias = 0.0
        biases = np.full(len(items), self.bias.global_bias, dtype=np.float32)
        biases[inums >= 0] += self.bias.item_biases[inums[inums >= 0]]
        rv = (ratings - biases - u_bias)[mask].astype(np.float32)
        nf = self.item_embeddings.shape[1]
        if mask.sum() == 0:
            return np.zeros(nf, dtype=np.float32), u_bias
        M = self.item_embeddings[inums[mask], :]
        A = M.T @ M + np.eye(nf, dtype=np.float32) * self.config.user_reg * int(mask.sum())
        return np.require(_solve_cholesky(A, (M.T @ rv).astype(A.dtype)), dtype=np.float32), u_bias

    def finalize_scores(self, user_num, items: ItemList, user_bias) -> ItemList:
        scores = items.scores()
        if user_bias is None:
            user_bias = float(self.bias.user_biases[user_num]) if user_num is not None else 0.0
        inums = items.numbers(vocabulary=self.items, missing="negative")
        biases = np.full(len(items), self.bias.global_bias + user_bias, dtype=np.float32)
        biases[inums >= 0] += self.bias.item_biases[inums[inums >= 0]]
        return ItemList(items, scores=scores + biases)

    def fold_in_batch(self, histories: list[ItemList]):
        """
        ``new_user_embedding`` for a batch of histories on the device: the bias-removed ratings of every
        history become one row of a CSR matrix and ONE explicit half-epoch (``lk_als_half_epoch`` mode 1,
        ``A = MᵀM + reg·n·I``, ``b = Mᵀr`` — the math of ``_train_bias_row_cholesky``,
        ``_explicit.py:121-147``) solves them all.  The user offsets follow ``BiasModel.compute_for_items``
        (a non-finite offset counts as 0); ratings that are not finite are left out of the row.
        """
        dev = _lib.require_device()
        k = self.item_embeddings.shape[1]
        cols, vals, indptr, offs = [], [], [0], []
        for h in histories:
            inums = h.numbers(vocabulary=self.items, missing="negative")
            ratings = h.field("rating")
            assert ratings is not None
            ratings = np.asarray(ratings, dtype=np.float32)
            known = inums >= 0
            uoff = ratings - self.bias.global_bias
            uoff[known] -= self.bias.item_biases[inums[known]]
            u_bias = float(np.sum(uoff) / (np.sum(np.isfinite(uoff)) + self.bias.damping[0]))
            if not np.isfinite(u_bias):
                u_bias = 0.0
            offs.append(u_bias)
            mask = known & np.isfinite(ratings)
            biases = self.bias.global_bias + self.bias.item_biases[inums[mask]]
            rv = (ratings[mask] - biases - u_bias).astype(np.float32)
            c = inums[mask].astype(np.int32)
            order = np.argsort(c, kind="stable")  # the CSR container wants ascending columns
            cols.append(c[order])
            vals.append(rv[order])
            indptr.append(indptr[-1] + len(c))
        csr = InteractionCSR(
            np.asarray(indptr, dtype=np.int32),
            np.concatenate(cols) if cols else np.empty(0, np.int32),
            np.concatenate(vals) if vals else np.empty(0, np.float32),
            (len(histories), self.item_embeddings.shape[0]),
        )
        plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), k)
        x = torch.zeros((len(histories), k), dtype=torch.float32, device=dev)  # empty histories stay 0 (:134-135)
        plan.sqdelta.zero_()
        plan.status.zero_()
        engine.als_half_epoch(plan, _lib.LK_ALS_EXPLICIT, x, self._device_items(), reg=float(self.config.user_reg))
        if int(plan.status.item()):
            raise RuntimeError("ALS solve error: a fold-in system is not positive definite")
        return x, np.asarray(offs, dtype=np.float32)

    def batch_offsets(self, user_nums: np.ndarray, fold_bias: np.ndarray | None):
        """``finalize_scores`` for a batch: global + item bias per item, user bias per query."""
        ub = np.where(user_nums >= 0, self.bias.user_biases[np.maximum(user_nums, 0)], 0.0).astype(np.float32)
        if fold_bias is not None:
            ub = np.where(np.isnan(fold_bias), ub, fold_bias).astype(np.float32)
        return (self.bias.item_biases + self.bias.global_bias).astype(np.float32), ub


class BiasedMFTrainer(ALSTrainerBase):
    MODE = _lib.LK_ALS_EXPLICIT

    def prepare_matrix(self, data: Dataset):
        it = data.interactions
        self.scorer.bias = BiasModel.learn(it, self.config.damping)
        return it.coo(self.scorer.bias.transform(it))

    def initial_params(self, nrows: int, ncols: int) -> np.ndarray:
        mat = self.rng.standard_normal((nrows, ncols), dtype=np.float32)
        mat /= np.linalg.norm(mat, axis=1).reshape((nrows, 1))
        return mat
