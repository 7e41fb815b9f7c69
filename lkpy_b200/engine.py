"""
Device-side engine: torch tensors in, C-ABI calls out.

PyTorch is used for device memory, streams and (in ``lkpy_b200.parallel``)
``torch.distributed`` only.  Every compute step is a call into
``liblkpy_b200.so``; nothing here falls back to torch math.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import threading
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from ._lib import (
    LkAlsArgs, LkAlsRecArgs, LkAssocScoreArgs, LkBiasLearnArgs, LkCoocArgs, LkEaseScoreArgs, LkFlexmfSampleArgs,
    LkFlexmfStepArgs, LkF32SeqSumArgs, LkKnnBuildArgs, LkKnnGeom, LkKnnRankArgs, LkKnnScoreArgs, LkNmfCdSweepArgs,
    LkFairArgs, LkItemExposureArgs, LkOffsetScoreArgs, LkRankMetricsArgs, LkSlimArgs, LkSpmmArgs, LkStochasticArgs,
    LkUknnSearchArgs, check, lib, ptr, stream_ptr,
)  # fmt: skip
from .data import InteractionCSR

DEFAULT_CHUNK_NNZ = 4096
#: rows of the fp32 / weighted tensor-core path (als_tc.cu, tf32 x3) are cut shorter, and the parts are summed with
#: round-to-nearest by the CUDA cores.  These lengths were chosen for an earlier tensor-core design whose
#: accumulators truncated; they are carried over unmeasured for the mma.sync accumulator of the H100 kernel
TF32_CHUNK_NNZ = 1024
#: fp32 rows / per-nonzero weights at k = 128: a quarter of that length (carried over the same way; it kept the
#: 100 M-interaction item rows inside the 1e-4 tolerance on that design)
TF32_CHUNK_NNZ_K128 = 256
#: engine limits the reference does not have (DESIGN.md §6): validated up front by the configs
ALS_MAX_FEATURES = 128
KNN_SCORE_MAX_NBRS = 128
KNN_MERGE_SMEM_LIMIT = 200 * 1024  # n_halves * save_nbrs * 16 B must fit (lk_knn_merge_topk)


@dataclass
class DeviceCSR:
    """A CSR matrix resident in HBM (int32 offsets/indices, f32 values)."""

    indptr: torch.Tensor
    indices: torch.Tensor
    values: torch.Tensor
    shape: tuple[int, int]
    h_indptr: np.ndarray  # host copy of the offsets, for planning

    @classmethod
    def from_host(cls, m: InteractionCSR, device=None, pin: bool = False) -> "DeviceCSR":
        device = device or _lib.require_device()
        if m.indptr.dtype != np.int32:
            raise _lib.EngineError("matrices with nnz >= 2**31 need row sharding first")

        def up(a):
            t = torch.from_numpy(np.ascontiguousarray(a))
            if pin:
                t = t.pin_memory()
            return t.to(device, non_blocking=pin)

        return cls(up(m.indptr), up(m.indices), up(m.values), m.shape, np.ascontiguousarray(m.indptr))

    @property
    def nnz(self) -> int:
        return int(self.h_indptr[-1])


# ---------------------------------------------------------------------------
# ALS
# ---------------------------------------------------------------------------


@dataclass
class ALSHalfPlan:
    """Row-chunk schedule and workspaces for one side (user or item) of ALS."""

    matrix: DeviceCSR
    k: int
    chunk_nnz: int
    chunks: torch.Tensor
    n_chunks: int
    n_split_rows: int
    n_slots: int
    partials: torch.Tensor | None
    split_counters: torch.Tensor | None
    work_counter: torch.Tensor
    sqdelta: torch.Tensor
    status: torch.Tensor
    vals_uniform: bool = False
    uniform_val: float = 0.0

    @classmethod
    def create(cls, matrix: DeviceCSR, k: int, chunk_nnz: int = DEFAULT_CHUNK_NNZ) -> "ALSHalfPlan":
        L = lib()
        dev = matrix.indptr.device
        n_rows = matrix.shape[0]
        hp = matrix.h_indptr
        nc, ns, nslot = C.c_int64(), C.c_int64(), C.c_int64()
        check(
            L.lk_als_plan_size(hp.ctypes.data, n_rows, chunk_nnz, C.byref(nc), C.byref(ns), C.byref(nslot)),
            "lk_als_plan_size",
        )
        h_chunks = np.empty((max(nc.value, 1), 8), dtype=np.int32)
        check(L.lk_als_plan_fill(hp.ctypes.data, n_rows, chunk_nnz, h_chunks.ctypes.data), "lk_als_plan_fill")
        slot_f = L.lk_als_slot_floats(k)
        if slot_f < 0:
            raise _lib.EngineError(f"embedding size {k} not supported (max {L.lk_als_max_features()})")
        partials = counters = None
        if ns.value > 0:
            partials = torch.empty(nslot.value * slot_f, dtype=torch.float32, device=dev)
            counters = torch.zeros(ns.value, dtype=torch.int32, device=dev)
        uniform, uval = False, 0.0
        if matrix.nnz > 0:
            lo, hi = torch.aminmax(matrix.values)
            uniform, uval = bool(lo == hi), float(lo)
        return cls(
            vals_uniform=uniform,
            uniform_val=uval,
            matrix=matrix,
            k=k,
            chunk_nnz=chunk_nnz,
            chunks=torch.from_numpy(h_chunks).to(dev),
            n_chunks=nc.value,
            n_split_rows=ns.value,
            n_slots=nslot.value,
            partials=partials,
            split_counters=counters,
            work_counter=torch.zeros(1, dtype=torch.int32, device=dev),
            sqdelta=torch.zeros(1, dtype=torch.float64, device=dev),
            status=torch.zeros(1, dtype=torch.int32, device=dev),
        )


@dataclass
class OtorWorkspace:
    scratch: torch.Tensor
    otor: torch.Tensor

    @classmethod
    def create(cls, k: int, device) -> "OtorWorkspace":
        n = lib().lk_als_otor_scratch_floats(k)
        if n < 0:
            raise _lib.EngineError(f"embedding size {k} not supported")
        return cls(
            torch.empty(n, dtype=torch.float32, device=device),
            torch.empty((k, k), dtype=torch.float32, device=device),
        )


def als_otor(
    other: torch.Tensor, reg: float, ws: OtorWorkspace, other_bf16: torch.Tensor | None = None
) -> torch.Tensor:
    """OtOr = OᵀO + reg·I on device; optionally fills the bf16 copy of ``other``."""
    assert other.dtype == torch.float32 and other.is_contiguous()
    n, k = other.shape
    if other_bf16 is not None:
        assert other_bf16.dtype == torch.bfloat16 and other_bf16.shape == other.shape
    check(
        lib().lk_als_otor(ptr(other), n, k, float(reg), ptr(ws.otor), ptr(other_bf16), ptr(ws.scratch), stream_ptr()),
        "lk_als_otor",
    )
    return ws.otor


def als_half_epoch(
    plan: ALSHalfPlan,
    mode: int,
    this: torch.Tensor,
    other: torch.Tensor,
    *,
    otor: torch.Tensor | None = None,
    reg: float = 0.0,
    replicas: list[torch.Tensor] | None = None,
    replica_row0: int = 0,
    cancel: torch.Tensor | None = None,
) -> None:
    """
    Enqueue one half-epoch.  ``this`` [n_rows,k] f32 is updated in place;
    ``other`` is f32 or bf16.  ``plan.sqdelta`` accumulates Σ‖Δ‖² and
    ``plan.status`` reports a non-PD row; the caller zeroes / reads them.
    """
    m = plan.matrix
    assert this.dtype == torch.float32 and this.is_contiguous()
    assert other.is_contiguous() and other.shape[1] == this.shape[1] == plan.k
    assert this.shape[0] == m.shape[0] and other.shape[0] == m.shape[1]
    a = LkAlsArgs()
    a.mode = mode
    a.k = plan.k
    a.n_rows = m.shape[0]
    a.n_other = other.shape[0]
    a.d_indptr, a.d_cols, a.d_vals = ptr(m.indptr), ptr(m.indices), ptr(m.values)
    a.d_this = ptr(this)
    a.d_other = ptr(other)
    if other.dtype == torch.float32:
        a.other_dtype = _lib.LK_DTYPE_F32
    elif other.dtype == torch.bfloat16:
        a.other_dtype = _lib.LK_DTYPE_BF16
    else:
        raise TypeError(f"unsupported factor dtype {other.dtype}")
    reps = replicas or []
    a.n_replicas = len(reps)
    for i, r in enumerate(reps):
        a.d_replicas[i] = r if isinstance(r, int) else ptr(r)
    a.replica_row0 = replica_row0
    a.d_otor = ptr(otor)
    a.reg = float(reg)
    a.d_chunks = ptr(plan.chunks)
    a.n_chunks = plan.n_chunks
    a.d_partials = ptr(plan.partials)
    a.d_split_counters = ptr(plan.split_counters)
    a.n_split_rows = plan.n_split_rows
    a.d_work_counter = ptr(plan.work_counter)
    a.d_sqdelta = ptr(plan.sqdelta)
    a.d_status = ptr(plan.status)
    a.vals_uniform = 1 if plan.vals_uniform else 0
    a.uniform_val = plan.uniform_val
    # optional device flag: non-zero stops the hand-out of rows (cooperative cancel); rows already handed out
    # finish, which for the k = 64 tensor-core kernel includes the one chunk each CTA claims ahead
    a.d_cancel = ptr(cancel)
    check(lib().lk_als_half_epoch(C.byref(a), stream_ptr()), "lk_als_half_epoch")


# ---------------------------------------------------------------------------
# item-kNN build
# ---------------------------------------------------------------------------


@dataclass
class KnnBuildPlan:
    """Tiling, tile pointers and cost-ordered work units for one (UI, IU) pair."""

    ui: DeviceCSR
    iu: DeviceCSR
    geom: LkKnnGeom
    tile_ptr: torch.Tensor
    cost: torch.Tensor  # int64 [n_items]
    order: torch.Tensor  # int32 [n_items], most expensive first
    tie_scratch: torch.Tensor
    work_counter: torch.Tensor
    status: torch.Tensor
    extra: dict = field(default_factory=dict)
    world: int = 1  # GPUs sharing the build: sets how finely hot items are cut into column pieces
    MAX_PIECES = 8
    #: a piece repeats the unit's loads and does 1/P of its shared-memory updates: modelled cost share of the loads
    LOAD_SHARE = 0.45

    @classmethod
    def create(cls, ui: DeviceCSR, iu: DeviceCSR, world: int = 1) -> "KnnBuildPlan":
        L = lib()
        dev = ui.indptr.device
        n_users, n_items = ui.shape
        assert iu.shape == (n_items, n_users)
        g = LkKnnGeom()
        check(L.lk_knn_geometry(n_users, n_items, C.byref(g)), "lk_knn_geometry")
        tile_ptr = torch.empty(max(1, n_users * (g.n_subtiles + 1)), dtype=torch.int32, device=dev)
        cost = torch.empty(n_items, dtype=torch.int64, device=dev)
        tie = torch.empty(max(1, L.lk_knn_tie_scratch_ints(C.byref(g))), dtype=torch.int32, device=dev)
        plan = cls(
            ui, iu, g, tile_ptr, cost, torch.empty(0, dtype=torch.int32, device=dev), tie,
            torch.zeros(1, dtype=torch.int32, device=dev),
            torch.zeros(1, dtype=torch.int32, device=dev),
            world=max(1, int(world)),
        )  # fmt: skip
        plan.prepare()
        return plan

    def prepare(self) -> None:
        """(Re)compute tile pointers, row costs, the cost-ordered item list and the work units."""
        L = lib()
        g = self.geom
        check(
            L.lk_knn_tile_pointers(
                C.byref(g), ptr(self.ui.indptr), ptr(self.ui.indices), ptr(self.tile_ptr), stream_ptr()
            ),
            "lk_knn_tile_pointers",
        )
        check(
            L.lk_knn_row_cost(
                C.byref(g), ptr(self.ui.indptr), ptr(self.iu.indptr), ptr(self.iu.indices), ptr(self.cost), stream_ptr()
            ),
            "lk_knn_row_cost",
        )
        self.order = torch.argsort(self.cost, descending=True, stable=True).to(torch.int32)
        self.extra.pop("units", None)

    def units(self, split_hot: bool):
        """
        Work units {item, half, piece, n_pieces}, item-major, with their schedule (most expensive first).
        ``split_hot`` (truncated build only): an (item, half) unit whose product count exceeds half a
        CTA's fair share of the whole build on ``world`` GPUs is cut into 2 / 4 / 8 column pieces
        (``knn_build.cu``) — without it the five hottest ML-25M-shaped items pin one CTA each for longer
        than an 8-GPU build should take.  No host sync: everything is computed on the device.
        """
        key = ("units", bool(split_hot))
        cached = self.extra.get("units")
        if cached is not None and cached[0] == key:
            return cached[1]
        dev = self.cost.device
        H, n_items = self.geom.n_halves, self.geom.n_items
        cost = self.cost.to(torch.float64)
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        n_cta = sms * self.geom.ctas_per_sm * self.world
        pieces = torch.ones(n_items, dtype=torch.int64, device=dev)
        if split_hot:
            fair = cost.sum() / n_cta  # products per CTA if the build were perfectly balanced
            want = (cost / H) / (0.5 * fair).clamp_min(1.0)
            pieces = torch.where(want > 4, 8, torch.where(want > 2, 4, torch.where(want > 1, 2, 1))).to(torch.int64)
            pieces = pieces.clamp_max(self.MAX_PIECES)
        per_item = pieces * H
        unit_ptr = torch.zeros(n_items + 1, dtype=torch.int64, device=dev)
        torch.cumsum(per_item, 0, out=unit_ptr[1:])
        item_of = torch.repeat_interleave(torch.arange(n_items, device=dev), per_item)
        local = torch.arange(item_of.numel(), device=dev) - unit_ptr[item_of]
        p_of = pieces[item_of]
        units = torch.stack([item_of, local // p_of, local % p_of, p_of], dim=1).to(torch.int32).contiguous()
        ucost = (cost[item_of] / H) * (self.LOAD_SHARE + (1.0 - self.LOAD_SHARE) / p_of.to(torch.float64))
        sched = torch.argsort(ucost, descending=True, stable=True).to(torch.int32)
        out = {
            "units": units, "unit_ptr": unit_ptr.to(torch.int32), "sched": sched, "item_of": item_of,
            "max_units": int(H * (self.MAX_PIECES if split_hot else 1)), "n_units": int(units.shape[0]),
        }  # fmt: skip
        self.extra["units"] = (key, out)
        return out

    #: optional device int32 flag checked by the build kernel whenever a CTA fetches a work unit
    cancel: torch.Tensor | None = None

    def _args(self, u: dict, sched: torch.Tensor, min_sim: float, save_nbrs: int) -> LkKnnBuildArgs:
        a = LkKnnBuildArgs()
        a.d_cancel = ptr(self.cancel)
        a.geom = self.geom
        a.d_ui_indptr, a.d_ui_cols, a.d_ui_vals = ptr(self.ui.indptr), ptr(self.ui.indices), ptr(self.ui.values)
        a.d_iu_indptr, a.d_iu_cols, a.d_iu_vals = ptr(self.iu.indptr), ptr(self.iu.indices), ptr(self.iu.values)
        a.d_tile_ptr = ptr(self.tile_ptr)
        a.d_units, a.d_unit_ptr, a.max_units_per_item = ptr(u["units"]), ptr(u["unit_ptr"]), u["max_units"]
        a.d_sched = ptr(sched)
        a.n_work = sched.numel()
        a.min_sim = float(np.float32(min_sim))
        a.save_nbrs = int(save_nbrs)
        a.d_tie_scratch = ptr(self.tie_scratch)
        a.d_work_counter = ptr(self.work_counter)
        a.d_status = ptr(self.status)
        return a

    def _sched_for(self, u: dict, order: torch.Tensor | None) -> torch.Tensor:
        """The schedule restricted to the units of the items in ``order`` (item-sharded build)."""
        if order is None:
            return u["sched"]
        mine = torch.zeros(self.geom.n_items, dtype=torch.bool, device=order.device)
        mine[order.long()] = True
        sched = u["sched"]
        return sched[mine[u["item_of"][sched.long()]]].contiguous()

    def build_topk(
        self, min_sim: float, save_nbrs: int, order: torch.Tensor | None = None
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """
        Truncated build: returns fixed-width rows (cols [n_items,K] sorted by
        column, vals, counts).  Rows not in ``order`` have count 0.
        """
        L = lib()
        dev = self.ui.indptr.device
        n_items, K = self.geom.n_items, int(save_nbrs)
        u = self.units(split_hot=True)
        if u["max_units"] * K * 16 > KNN_MERGE_SMEM_LIMIT:  # checked before the build runs, not after it
            raise _lib.EngineError(
                f"save_nbrs={K} with {u['max_units']} work units per item exceeds the merge limit "
                f"(units * save_nbrs <= {KNN_MERGE_SMEM_LIMIT // 16}); use save_nbrs=None"
            )
        sched = self._sched_for(u, order)
        ws = self.extra.get(("topk", K, u["n_units"]))
        if ws is None:  # workspaces are allocated once per plan and K, reused by every build
            ws = (
                torch.empty(u["n_units"] * K, dtype=torch.int32, device=dev),
                torch.empty(u["n_units"] * K, dtype=torch.float32, device=dev),
                torch.empty(u["n_units"], dtype=torch.int32, device=dev),
            )
            self.extra[("topk", K, u["n_units"])] = ws
        part_cols, part_vals, part_cnt = ws
        part_cnt.zero_()
        self.status.zero_()
        a = self._args(u, sched, min_sim, K)
        a.d_part_cols, a.d_part_vals, a.d_part_cnt = ptr(part_cols), ptr(part_vals), ptr(part_cnt)
        check(L.lk_knn_build(C.byref(a), stream_ptr()), "lk_knn_build")
        out_cols = torch.empty((n_items, K), dtype=torch.int32, device=dev)
        out_vals = torch.empty((n_items, K), dtype=torch.float32, device=dev)
        out_cnt = torch.empty(n_items, dtype=torch.int32, device=dev)
        check(
            L.lk_knn_merge_topk(C.byref(a), ptr(out_cols), ptr(out_vals), ptr(out_cnt), stream_ptr()),
            "lk_knn_merge_topk",
        )
        return out_cols, out_vals, out_cnt

    def build_unbounded(
        self, min_sim: float, order: torch.Tensor | None = None, capacity: int | None = None
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Unbounded build (``save_nbrs=None``): CSR (int64 indptr, cols, vals) on device."""
        L = lib()
        dev = self.ui.indptr.device
        n_items, H = self.geom.n_items, self.geom.n_halves
        u = self.units(split_hot=False)  # one unit per (item, half): pool segments stay in column order
        sched = self._sched_for(u, order)
        rows = self.order if order is None else order.to(torch.int32).contiguous()
        if capacity is None:
            # every kept pair shares a user: at most sum of the processed rows' product counts
            capacity = int(min(int(self.cost[rows.long()].sum().item()), rows.numel() * max(n_items - 1, 1)))
        cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        self.status.zero_()
        a = self._args(u, sched, min_sim, 0)

        def launch(pool_cols, pool_vals, pool_off, part_cnt):
            a.d_part_cnt = ptr(part_cnt)
            a.d_pool_cols, a.d_pool_vals, a.pool_capacity = ptr(pool_cols), ptr(pool_vals), pool_cols.numel()
            a.d_pool_off, a.d_pool_cursor = ptr(pool_off), ptr(cursor)
            check(L.lk_knn_build(C.byref(a), stream_ptr()), "lk_knn_build")
            return int(self.status.item())

        def gather(indptr, cols, vals):
            rc = L.lk_knn_pool_to_csr(C.byref(a), ptr(indptr), ptr(cols), ptr(vals), stream_ptr())
            check(rc, "lk_knn_pool_to_csr")

        return pool_to_csr(
            dev, n_items, H, capacity, torch.float32, launch, gather, "similarity pool overflow; pass a larger capacity"
        )


def pool_to_csr(dev, n_rows: int, units_per_row: int, capacity: int, vals_dtype, launch, gather, overflow: str):
    """
    The host side of a tiled kernel's bump pool (``tiles.cuh``): allocates a pool of ``capacity`` (at least 1)
    entries and the per-unit segment offsets and counts of ``n_rows * units_per_row`` units, row-major;
    ``launch(pool_cols, pool_vals, pool_off, part_cnt)`` runs the kernel and returns the status word, 1 raising
    :class:`EngineError` with ``overflow``; ``gather(indptr, cols, vals)`` copies the segments, in unit order, into
    the CSR.  Returns the device CSR (int64 indptr [n_rows + 1], int32 columns, values of ``vals_dtype``).
    """
    capacity = max(int(capacity), 1)
    pool_cols = torch.empty(capacity, dtype=torch.int32, device=dev)
    pool_vals = torch.empty(capacity, dtype=vals_dtype, device=dev)
    pool_off = torch.zeros(n_rows * units_per_row, dtype=torch.int64, device=dev)
    part_cnt = torch.zeros(n_rows * units_per_row, dtype=torch.int32, device=dev)
    if launch(pool_cols, pool_vals, pool_off, part_cnt) == 1:
        raise _lib.EngineError(overflow)
    indptr = torch.zeros(n_rows + 1, dtype=torch.int64, device=dev)
    torch.cumsum(part_cnt.view(n_rows, units_per_row).sum(dim=1, dtype=torch.int64), 0, out=indptr[1:])
    nnz = int(indptr[-1].item())
    cols = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
    vals = torch.empty(max(nnz, 1), dtype=vals_dtype, device=dev)
    gather(indptr, cols, vals)
    return indptr, cols[:nnz], vals[:nnz]


def topk_rows_to_csr(
    cols: torch.Tensor, vals: torch.Tensor, cnt: torch.Tensor
) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Compact fixed-width top-K rows into CSR (int64 offsets, the LargeList layout)."""
    n, K = cols.shape
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=cols.device)
    torch.cumsum(cnt.to(torch.int64), 0, out=indptr[1:])
    mask = torch.arange(K, device=cols.device)[None, :] < cnt[:, None]
    return indptr, cols[mask], vals[mask]


# ---------------------------------------------------------------------------
# item-kNN scoring
# ---------------------------------------------------------------------------


@dataclass
class KnnScorerState:
    """Similarity matrix in HBM; per-warp slot maps and scratch are sized to the batches actually scored."""

    n_items: int
    sim_indptr: torch.Tensor  # int64
    sim_cols: torch.Tensor
    sim_vals: torch.Tensor | None  # None: user mode with implicit feedback (structure only)
    max_warps: int
    work_counter: torch.Tensor
    status: torch.Tensor
    slotmap: torch.Tensor | None = None  # [warps, n_items] int32, all -1 between calls; grown on demand
    scratch: dict = field(default_factory=dict)  # contribution pool and cursor, the dense kernel's per-CTA rows
    lock: object = field(default_factory=threading.Lock)  # the mutable device state above is per-state
    #: user-kNN scoring (user_score.rs:21-98): the matrix is users x items ratings, a query's "history" is its
    #: neighbour list and carries the weights (lk_knn_score_args.user_mode)
    user_mode: bool = False
    n_rows: int = 0

    def _slotmap(self, n_queries: int) -> tuple[torch.Tensor, int]:
        """One slot-map row per working warp: min(n_queries, full grid) rows (a single query takes
        n_items * 4 B, not grid * n_items * 4 B)."""
        warps = max(1, min(int(n_queries), self.max_warps))
        if self.slotmap is None or self.slotmap.shape[0] < warps:
            self.slotmap = None
            self.slotmap = torch.full((warps, self.n_items), -1, dtype=torch.int32, device=self.sim_cols.device)
        return self.slotmap, int(self.slotmap.shape[0])

    @classmethod
    def create(cls, n_items: int, indptr, cols, vals, device=None, user_mode: bool = False) -> "KnnScorerState":
        """``n_items`` = number of columns (targets).  Item mode: the square similarity matrix; user mode: the
        users x items (centred) rating matrix, ``vals`` None for implicit feedback."""
        device = device or _lib.require_device()
        warps = int(lib().lk_knn_score_warps())

        def dev(t, dt):
            t = torch.as_tensor(t)
            return t.to(device=device, dtype=dt).contiguous()

        ip = dev(indptr, torch.int64)
        return cls(
            n_items,
            ip,
            dev(cols, torch.int32),
            None if vals is None else dev(vals, torch.float32),
            warps,
            torch.zeros(1, dtype=torch.int32, device=device),
            torch.zeros(1, dtype=torch.int32, device=device),
            user_mode=bool(user_mode),
            n_rows=int(ip.numel() - 1),
        )

    def score(
        self,
        ref_indptr: torch.Tensor,
        ref_items: torch.Tensor,
        ref_vals: torch.Tensor | None,
        tgt_indptr: torch.Tensor,
        tgt_items: torch.Tensor,
        max_nbrs: int,
        min_nbrs: int,
    ) -> tuple[torch.Tensor, torch.Tensor]:
        """Score a batch of queries; returns (scores with NaN nulls, counts with -1 nulls)."""
        nt = tgt_items.numel()
        lists = torch.empty((3, nt), dtype=torch.int32, device=self.sim_cols.device)  # offset, cursor, count

        def target_lists(a: LkKnnScoreArgs) -> None:
            slotmap, a.slotmap_warps = self._slotmap(ref_indptr.numel() - 1)
            a.d_tgt_indptr, a.d_tgt_items, a.d_slotmap = ptr(tgt_indptr), ptr(tgt_items), ptr(slotmap)
            a.d_list_off, a.d_list_cur, a.d_list_cnt = ptr(lists[0]), ptr(lists[1]), ptr(lists[2])

        return self._launch((nt,), ref_indptr, ref_items, ref_vals, max_nbrs, min_nbrs, target_lists)

    def _pool_for(self, ref_items: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """Contribution pool: one 16-byte entry per (history entry, matrix-row entry) pair of the batch."""
        dev = self.sim_cols.device
        n_rows = self.n_rows if self.user_mode else self.n_items
        r = ref_items.long()
        ok = (r >= 0) & (r < n_rows)
        rr = r.clamp(0, n_rows - 1)
        total = int(((self.sim_indptr[rr + 1] - self.sim_indptr[rr]) * ok).sum().item())
        pool = self.scratch.get("pool")
        if pool is None or pool.numel() < 4 * max(total, 1):
            # the old pool goes first: user-mode pools of a few hundred queries take tens of GB
            pool = self.scratch["pool"] = None
            pool = torch.empty(4 * max(total, 1), dtype=torch.int32, device=dev)
            self.scratch["pool"] = pool
            self.scratch["pool_cursor"] = torch.zeros(1, dtype=torch.int64, device=dev)
        return pool, self.scratch["pool_cursor"]

    def score_all_items(
        self, ref_indptr: torch.Tensor, ref_items: torch.Tensor, ref_vals: torch.Tensor | None, max_nbrs: int, min_nbrs: int
    ) -> tuple[torch.Tensor, torch.Tensor]:
        """
        Score every query against ALL items (the batch runner's case): returns (scores [n_queries, n_items]
        with NaN nulls, counts [n_queries, n_items]).  Runs ``knn_score_dense_kernel`` — a CTA per query,
        cost proportional to the contributions plus one streaming fill of the output.
        """
        shape = (ref_indptr.numel() - 1, self.n_items)
        return self._launch(shape, ref_indptr, ref_items, ref_vals, max_nbrs, min_nbrs, self._per_cta_rows)

    def _per_cta_rows(self, a: LkKnnScoreArgs) -> None:
        """The dense kernel's per-CTA state: a slot map (item -> touched-target number; zero between queries and
        between launches) and two compact rows indexed by touched-target number."""
        ctas = int(lib().lk_knn_score_dense_ctas())
        rows = self.scratch.get("dense")
        if rows is None:
            dev, n = self.sim_cols.device, ctas * self.n_items
            rows = self.scratch["dense"] = (
                torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
                torch.zeros(n, dtype=torch.int32, device=dev),
            )  # fmt: skip
        off, cur, slotmap = rows
        a.d_list_off, a.d_list_cur = ptr(off), ptr(cur)
        a.d_slotmap, a.slotmap_warps = ptr(slotmap), ctas

    def recommend(
        self,
        ref_indptr: torch.Tensor,
        ref_items: torch.Tensor,
        ref_vals: torch.Tensor | None,
        max_nbrs: int,
        min_nbrs: int,
        n: int,
        item_offset: torch.Tensor | None = None,
        query_offset: torch.Tensor | None = None,
        excl_indptr: torch.Tensor | None = None,
        excl_items: torch.Tensor | None = None,
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """
        Top-``n`` of every query over ALL items, scored and selected in one launch (``lk_knn_recommend_batch``,
        the dense kernel's ranking mode): the final score of item i for query q is
        ``(score + item_offset[i]) + query_offset[q]`` (f32), the items ``excl_items[excl_indptr[q]:excl_indptr[q+1]]``
        are never recommended to q, and the selection is ``argtopn``'s, ties included.  Returns
        ``(idx [B, n] int32 item numbers, -1 padding; val [B, n] f32, NaN padding; nbrs [B, n] int32 accumulator
        lengths, 0 padding; cnt [B] int32)``.
        """
        _check_max_nbrs(max_nbrs)
        n = _check_topn(n)
        dev = self.sim_cols.device
        B = ref_indptr.numel() - 1
        idx, val, cnt = _topn_outputs(B, n, dev)
        nbrs = torch.empty((B, n), dtype=torch.int32, device=dev)
        if excl_items is not None and excl_items.numel() == 0:  # NULL address; never read (bounded by the indptr)
            excl_items = torch.full((1,), -1, dtype=torch.int32, device=dev)

        def launch(a: LkKnnScoreArgs) -> None:
            self._per_cta_rows(a)
            spill = self.scratch.get("spill")
            if spill is None:  # the touched-target tail of a query past the CTA's shared-memory list
                spill = torch.empty(int(lib().lk_knn_score_dense_ctas()) * self.n_items, dtype=torch.int32, device=dev)
                self.scratch["spill"] = spill
            r = LkKnnRankArgs()
            r.n = n
            r.d_item_offset, r.d_query_offset = ptr(item_offset), ptr(query_offset)
            r.d_excl_indptr, r.d_excl_items = ptr(excl_indptr), ptr(excl_items)
            r.d_spill = ptr(spill)
            r.d_out_idx, r.d_out_val, r.d_out_nbrs, r.d_out_cnt = ptr(idx), ptr(val), ptr(nbrs), ptr(cnt)
            check(lib().lk_knn_recommend_batch(C.byref(a), C.byref(r), stream_ptr()), "lk_knn_recommend_batch")

        if B > 0:
            self._run(ref_indptr, ref_items, ref_vals, max_nbrs, min_nbrs, launch, "lk_knn_recommend_batch")
        return idx, val, nbrs, cnt[:B]

    def _launch(self, out_shape, ref_indptr, ref_items, ref_vals, max_nbrs, min_nbrs, fill_mode):
        """``score`` and ``score_all_items``: the outputs and ``lk_knn_score_batch`` around :meth:`_run`.
        ``fill_mode(args)`` sets the mode's own fields (with the lock held; the scratch they point to must outlive
        this call)."""
        _check_max_nbrs(max_nbrs)
        dev = self.sim_cols.device
        scores = torch.empty(out_shape, dtype=torch.float32, device=dev)
        counts = torch.empty(out_shape, dtype=torch.int32, device=dev)
        if scores.numel() == 0:  # no targets (or no queries): nothing to score
            return scores, counts

        def launch(a: LkKnnScoreArgs) -> None:
            fill_mode(a)
            a.d_scores, a.d_counts = ptr(scores), ptr(counts)
            check(lib().lk_knn_score_batch(C.byref(a), stream_ptr()), "lk_knn_score_batch")

        self._run(ref_indptr, ref_items, ref_vals, max_nbrs, min_nbrs, launch, "lk_knn_score_batch")
        return scores, counts

    def _run(self, ref_indptr, ref_items, ref_vals, max_nbrs, min_nbrs, launch, what: str) -> None:
        """What every launch shares: the empty-history placeholder, the common ``lk_knn_score_args`` fields, the
        lock, the wait and the status word.  ``launch(args)`` completes the arguments and calls the entry point
        ``what`` (with the lock held)."""
        dev = self.sim_cols.device
        if ref_items.numel() == 0:
            # every history is empty: the address of an empty tensor is NULL, which the library rejects; the
            # kernels never read these placeholders because the indptr bounds every read
            ref_items = torch.full((1,), -1, dtype=torch.int32, device=dev)
            ref_vals = None if ref_vals is None else torch.zeros(1, dtype=torch.float32, device=dev)
        with self.lock:  # status word, work counter, pool and slot maps are shared by the callers of one state
            a = LkKnnScoreArgs()
            pool, cursor = self._pool_for(ref_items)
            a.n_items = self.n_items
            a.d_sim_indptr, a.d_sim_cols, a.d_sim_vals = ptr(self.sim_indptr), ptr(self.sim_cols), ptr(self.sim_vals)
            a.n_queries = ref_indptr.numel() - 1
            a.d_ref_indptr, a.d_ref_items, a.d_ref_vals = ptr(ref_indptr), ptr(ref_items), ptr(ref_vals)
            a.max_nbrs, a.min_nbrs = int(max_nbrs), int(min_nbrs)
            a.d_work_counter, a.d_status = ptr(self.work_counter), ptr(self.status)
            a.user_mode, a.n_matrix_rows = (1 if self.user_mode else 0), self.n_rows
            a.d_pool, a.pool_entries, a.d_pool_cursor = ptr(pool), pool.numel() // 4, ptr(cursor)
            self.status.zero_()
            launch(a)
            torch.cuda.current_stream().synchronize()
            st = int(self.status.item())
        if st == 2:
            raise ValueError("similarity is null")
        if st == 3:
            raise _lib.EngineError(f"{what}: contribution pool too small")


def _check_max_nbrs(max_nbrs: int) -> None:
    if not 1 <= int(max_nbrs) <= KNN_SCORE_MAX_NBRS:
        raise ValueError(f"max_nbrs must be in 1..{KNN_SCORE_MAX_NBRS}")


# ---------------------------------------------------------------------------
# user-kNN neighbour search
# ---------------------------------------------------------------------------


def history_query(item_nums: np.ndarray, ratings: np.ndarray | None) -> tuple[np.ndarray, np.ndarray, float]:
    """
    The sparse query vector of a provided history, as ``UserKNNScorer._get_user_data`` builds it densely
    (``user.py:274-298``): ``item_nums`` are the history's item numbers (negative = unknown item, dropped),
    ``ratings`` its ratings (explicit feedback: centred by their f32 mean over the whole history, unknown
    items included) or None (implicit feedback: 1.0).  A repeated item keeps its LAST value, as the
    reference's ``ratings[idx] = ...`` does.  Returns (items int32 strictly ascending, values f64, mean).
    """
    nums = np.asarray(item_nums, dtype=np.int64)
    if ratings is None:
        umean = 0.0
        vals = np.ones(len(nums), dtype=np.float32)
    else:
        urv = np.require(ratings, dtype=np.float32)
        umean = float(urv.mean())
        vals = urv - umean  # f32 arithmetic, as the reference's f32 rating vector
    known = nums >= 0
    nums, vals = nums[known], vals[known]
    # last occurrence wins: the first occurrence in the reversed history
    items, first = np.unique(nums[::-1], return_index=True)
    vals = vals[::-1][first]
    return items.astype(np.int32), vals.astype(np.float64), umean


@dataclass
class UserQueries:
    """A batch of neighbour-search queries on the device: query q is entries ``[begin[q], end[q])`` of
    ``items`` / ``vals`` (rows of ``V`` for known users, or uploaded histories); ``self_`` the user
    excluded from its neighbours, or -1."""

    begin: torch.Tensor  # int64 [B]
    end: torch.Tensor  # int64 [B]
    items: torch.Tensor  # int32
    vals: torch.Tensor  # float64
    self_: torch.Tensor  # int32 [B]

    @property
    def n(self) -> int:
        return int(self.begin.numel())


@dataclass
class UserNeighbourState:
    """
    The unit-normalised f64 user vectors in HBM in both orientations — ``V`` (users x items, the rows of
    known-user queries) and ``VT`` (items x users, what the search gathers) — with the accumulator
    geometry and tile pointers of ``lk_uknn_search``.  At the ML-25M shape (25 M ratings) V and VT take
    12 B per rating each, 600 MB together, and the tile pointers 46 MB.
    """

    n_users: int
    n_items: int
    v_indptr: torch.Tensor  # int32 [n_users + 1]
    v_items: torch.Tensor  # int32
    v_vals: torch.Tensor  # float64
    h_v_indptr: np.ndarray
    vt_indptr: torch.Tensor  # int32 [n_items + 1]
    vt_users: torch.Tensor
    vt_vals: torch.Tensor
    geom: LkKnnGeom
    tile_ptr: torch.Tensor
    work_counter: torch.Tensor
    status: torch.Tensor
    cursor: torch.Tensor
    lock: object = field(default_factory=threading.Lock)

    @classmethod
    def create(cls, user_vectors, device=None, ctas_per_sm: int = 0) -> "UserNeighbourState":
        """``user_vectors``: the SciPy CSR (f64) of ``UserKNNScorer.train``."""
        import scipy.sparse as sps

        device = device or _lib.require_device()
        v = sps.csr_array(user_vectors, dtype=np.float64)
        v.sort_indices()
        vt = sps.csr_array(v.T)
        vt.sort_indices()
        if v.nnz >= 2**31:
            raise _lib.EngineError("user vectors with nnz >= 2**31 are not supported")
        n_users, n_items = v.shape
        L = lib()
        g = LkKnnGeom()
        check(L.lk_uknn_geometry(n_users, n_items, int(ctas_per_sm), C.byref(g)), "lk_uknn_geometry")

        def up(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(device)

        vt_indptr, vt_users = up(vt.indptr, np.int32), up(vt.indices, np.int32)
        tile_ptr = torch.empty(max(1, n_items * (g.n_subtiles + 1)), dtype=torch.int32, device=device)
        if n_items > 0:
            check(
                L.lk_knn_tile_pointers(C.byref(g), ptr(vt_indptr), ptr(vt_users), ptr(tile_ptr), stream_ptr()),
                "lk_knn_tile_pointers",
            )
        z = lambda dt: torch.zeros(1, dtype=dt, device=device)  # noqa: E731
        return cls(
            n_users, n_items, up(v.indptr, np.int32), up(v.indices, np.int32), up(v.data, np.float64),
            np.ascontiguousarray(v.indptr, dtype=np.int64), vt_indptr, vt_users, up(vt.data, np.float64),
            g, tile_ptr, z(torch.int32), z(torch.int32), z(torch.int64),
        )  # fmt: skip

    @property
    def device(self):
        return self.v_indptr.device

    def known_queries(self, users) -> UserQueries:
        """Queries that are rows of ``V``: only the user numbers are uploaded; each user is its own self."""
        u = torch.as_tensor(np.asarray(users, dtype=np.int64)).to(self.device)
        if u.numel() and (int(u.min()) < 0 or int(u.max()) >= self.n_users):
            raise IndexError("user number out of range")
        ip = self.v_indptr.to(torch.int64)
        return UserQueries(ip[u].contiguous(), ip[u + 1].contiguous(), self.v_items, self.v_vals, u.to(torch.int32))

    def queries(self, specs) -> UserQueries:
        """
        A mixed batch.  Each spec is a known user number (its row of ``V``) or a tuple ``(items, vals, self)``
        from :func:`history_query` (``self`` a user number or None).  Known rows are gathered on the device.
        """
        if all(not isinstance(s, tuple) for s in specs):
            return self.known_queries([int(s) for s in specs])
        dev = self.device
        hv = self.h_v_indptr
        k_at = [i for i, s in enumerate(specs) if not isinstance(s, tuple)]
        k_users = np.array([int(specs[i]) for i in k_at], dtype=np.int64)
        k_len = (hv[k_users + 1] - hv[k_users]) if len(k_at) else np.zeros(0, np.int64)
        k_start = np.concatenate([[0], np.cumsum(k_len)]).astype(np.int64)
        k_tot = int(k_start[-1])
        hist = [specs[i] for i in range(len(specs)) if isinstance(specs[i], tuple)]
        h_len = np.array([len(h[0]) for h in hist], dtype=np.int64)
        h_start = k_tot + np.concatenate([[0], np.cumsum(h_len)]).astype(np.int64)
        begin = np.empty(len(specs), np.int64)
        end = np.empty(len(specs), np.int64)
        self_ = np.empty(len(specs), np.int32)
        begin[k_at], end[k_at], self_[k_at] = k_start[:-1], k_start[1:], k_users
        h_at = [i for i, s in enumerate(specs) if isinstance(s, tuple)]
        begin[h_at], end[h_at] = h_start[:-1], h_start[1:]
        self_[h_at] = [-1 if h[2] is None else int(h[2]) for h in hist]
        items = torch.empty(max(1, int(h_start[-1])), dtype=torch.int32, device=dev)
        vals = torch.zeros(max(1, int(h_start[-1])), dtype=torch.float64, device=dev)
        if k_tot:  # V rows, gathered on the device: position p of known query j comes from hv[u_j] + p - k_start[j]
            shift = torch.from_numpy(hv[k_users] - k_start[:-1]).to(dev)
            src = torch.repeat_interleave(shift, torch.from_numpy(k_len).to(dev), output_size=k_tot)
            src += torch.arange(k_tot, device=dev)
            items[:k_tot] = self.v_items[src]
            vals[:k_tot] = self.v_vals[src]
        if len(hist) and h_start[-1] > k_tot:
            items[k_tot : h_start[-1]] = torch.from_numpy(np.concatenate([h[0] for h in hist]).astype(np.int32)).to(dev)
            vals[k_tot : h_start[-1]] = torch.from_numpy(np.concatenate([h[1] for h in hist]).astype(np.float64)).to(dev)
        t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
        return UserQueries(t(begin), t(end), items, vals, t(self_))

    def _args(self, qs: UserQueries, min_sim: float) -> LkUknnSearchArgs:
        a = LkUknnSearchArgs()
        a.geom = self.geom
        a.d_vt_indptr, a.d_vt_users, a.d_vt_vals = ptr(self.vt_indptr), ptr(self.vt_users), ptr(self.vt_vals)
        a.d_tile_ptr = ptr(self.tile_ptr)
        a.n_queries = qs.n
        a.d_q_begin, a.d_q_end, a.d_q_items, a.d_q_vals = ptr(qs.begin), ptr(qs.end), ptr(qs.items), ptr(qs.vals)
        a.d_q_self = ptr(qs.self_)
        a.min_sim = float(min_sim)
        a.d_work_counter, a.d_status, a.d_pool_cursor = ptr(self.work_counter), ptr(self.status), ptr(self.cursor)
        return a

    def query_cost(self, qs: UserQueries) -> torch.Tensor:
        """Products of each query's search: the summed ``VT`` row lengths of its items (int64 [B])."""
        cost = torch.zeros(max(qs.n, 1), dtype=torch.int64, device=self.device)
        check(lib().lk_uknn_query_cost(C.byref(self._args(qs, 1.0)), ptr(cost), stream_ptr()), "lk_uknn_query_cost")
        return cost[: qs.n]

    def neighbours(
        self, qs: UserQueries, min_sim: float, capacity: int | None = None
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """
        Every query's neighbours ``{v : sim >= min_sim, v != self}`` in ascending ``v``: device CSR (int64
        indptr [B+1], int32 users, f32 similarities) — the user-mode neighbour lists of
        ``KnnScorerState.score``.  ``capacity``: survivor pool entries (default: the bound
        Σ_q min(products_q, n_users)); a pool too small raises :class:`EngineError`.
        """
        if not min_sim > 0:
            raise ValueError("min_sim must be positive")
        dev, B, H = self.device, qs.n, self.geom.n_halves
        if B == 0:
            indptr = torch.zeros(1, dtype=torch.int64, device=dev)
            return indptr, torch.empty(0, dtype=torch.int32, device=dev), torch.empty(0, dtype=torch.float32, device=dev)
        if B * H >= 2**31:
            raise _lib.EngineError(f"{B} queries x {H} user tiles exceed the work-unit numbering; split the batch")
        L = lib()
        cost = self.query_cost(qs)
        order = torch.argsort(cost, descending=True, stable=True)
        order = order[cost[order] > 0]  # a query without products has no neighbours and needs no unit
        sched = (order[:, None] * H + torch.arange(H, device=dev)[None, :]).reshape(-1).to(torch.int32)
        if capacity is None:
            capacity = int(cost.clamp_max(self.n_users).sum().item())
        a = self._args(qs, min_sim)
        a.d_sched, a.n_work = ptr(sched), sched.numel()

        def launch(pool_rows, pool_sims, pool_off, part_cnt):
            with self.lock:  # work counter, cursor and status word are per state
                a.d_pool_rows, a.d_pool_sims, a.pool_capacity = ptr(pool_rows), ptr(pool_sims), pool_rows.numel()
                a.d_pool_off, a.d_part_cnt = ptr(pool_off), ptr(part_cnt)
                check(L.lk_uknn_search(C.byref(a), stream_ptr()), "lk_uknn_search")
                return int(self.status.item())

        def gather(indptr, rows, sims):
            rc = L.lk_uknn_pool_to_csr(C.byref(a), ptr(indptr), ptr(rows), ptr(sims), stream_ptr())
            check(rc, "lk_uknn_pool_to_csr")

        return pool_to_csr(
            dev, B, H, capacity, torch.float32, launch, gather,
            "lk_uknn_search: neighbour pool overflow; pass a larger capacity",
        )  # fmt: skip


# ---------------------------------------------------------------------------
# batched top-N (SURVEY.md §8f N2)
# ---------------------------------------------------------------------------


def topn_columns(scores: torch.Tensor, n: int, with_values: bool = True):
    """
    Top-``n`` of every column of ``scores`` [n_items, n_vectors] (f32, unit column stride) with
    the reference's ``argtopn`` semantics (``lk_topn_columns``): returns
    ``(idx [n_vectors, n] int32 with -1 padding, val [n_vectors, n] f32 or None, cnt [n_vectors] int32)``.
    """
    _lib.require_device()
    if scores.dtype != torch.float32 or scores.dim() != 2 or (scores.shape[1] > 1 and scores.stride(1) != 1):
        raise TypeError("scores must be a 2-D float32 tensor with contiguous columns")
    n_rows, n_cols = scores.shape
    n = _check_topn(n)
    idx, val, cnt = _topn_outputs(n_cols, n, scores.device)
    val = val if with_values else None
    check(
        lib().lk_topn_columns(
            ptr(scores), n_rows, n_cols, scores.stride(0) if n_rows > 1 else max(n_cols, 1), n,
            ptr(idx), ptr(val), ptr(cnt), stream_ptr(),
        ),
        "lk_topn_columns",
    )  # fmt: skip
    return idx, val, cnt[:n_cols]


def als_recommend(
    items: torch.Tensor,
    queries: torch.Tensor,
    n: int | None = None,
    item_offset: torch.Tensor | None = None,
    query_offset: torch.Tensor | None = None,
    excl_indptr: torch.Tensor | None = None,
    excl_items: torch.Tensor | None = None,
):
    """
    ALS scores of every item for every query (``lk_als_recommend_batch``): one fp32 FMA chain per score over
    ascending d, ``s = fmaf(items[i, d], queries[b, d], s)`` from +0, then ``+ item_offset[i]`` and
    ``+ query_offset[b]`` (f32).  ``items`` is [n_items, k], ``queries`` [B, k], both f32 with k in 1..128.

    ``n=None`` (score mode) returns the item-major matrix ``S [n_items, B]`` f32.  An integer ``n`` (rank mode,
    1..``lk_topn_max()``) returns ``(idx [B, n] int32 item numbers, -1 padding; val [B, n] f32, NaN padding;
    cnt [B] int32)``: for every query, ``argtopn`` over all items minus
    ``excl_items[excl_indptr[b]:excl_indptr[b+1]]`` (any order; repeats, negative and unknown numbers are
    ignored), ties included, without storing the score matrix.  The grid has one CTA per 64 queries, each
    sweeping every item, so small batches leave the GPU idle: batch widely.
    """
    _lib.require_device()
    if items.dtype != torch.float32 or queries.dtype != torch.float32 or items.dim() != 2 or queries.dim() != 2:
        raise TypeError("items and queries must be 2-D float32 tensors")
    n_items, k = items.shape
    B = queries.shape[0]
    if queries.shape[1] != k:
        raise ValueError(f"queries have {queries.shape[1]} columns, items {k}")
    dev = queries.device
    items, queries = items.contiguous(), queries.contiguous()
    a = LkAlsRecArgs()
    a.n_items, a.k, a.n_queries = n_items, k, B
    a.d_items, a.d_queries = ptr(items), ptr(queries)
    if item_offset is not None:
        item_offset = item_offset.to(device=dev, dtype=torch.float32).contiguous()
    if query_offset is not None:
        query_offset = query_offset.to(device=dev, dtype=torch.float32).contiguous()
    a.d_item_offset, a.d_query_offset = ptr(item_offset), ptr(query_offset)
    if n is None:
        S = torch.empty((n_items, B), dtype=torch.float32, device=dev)
        a.n, a.d_scores = 0, ptr(S)
        check(lib().lk_als_recommend_batch(C.byref(a), stream_ptr()), "lk_als_recommend_batch")
        return S
    ws_bytes = int(lib().lk_als_recommend_workspace_bytes(B, _check_topn(n)))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes > 0 else None
    a.d_workspace = ptr(ws)
    return _rank_launch(a, lib().lk_als_recommend_batch, "lk_als_recommend_batch", n, n_items, B, dev, excl_indptr,
                        excl_items)  # fmt: skip


def _check_topn(n) -> int:
    """``n`` as an int, or ``ValueError`` unless it is in 1..``lk_topn_max()``."""
    n_max = int(lib().lk_topn_max())
    if not 1 <= int(n) <= n_max:
        raise ValueError(f"n must be in 1..{n_max}")
    return int(n)


def _topn_outputs(B: int, n: int, dev):
    """The outputs of a top-n launch over B queries: ``idx [B, n]`` int32, ``val [B, n]`` f32 and ``cnt`` int32
    (at least one entry, so that its address is never NULL)."""
    idx = torch.empty((B, n), dtype=torch.int32, device=dev)
    val = torch.empty((B, n), dtype=torch.float32, device=dev)
    return idx, val, torch.empty(max(B, 1), dtype=torch.int32, device=dev)


def _rank_launch(args, entry, name: str, n: int, n_items: int, B: int, dev, excl_indptr, excl_items):
    """
    The rank mode of a fused scoring entry point: sorts the exclusions (:func:`_sorted_exclusions`), sets ``n``, the
    exclusions and the outputs in ``args``, calls ``entry(args, stream)`` and returns ``(idx [B, n], val [B, n],
    cnt [B])``.  ``args`` carries the mode's own fields already.
    """
    n = _check_topn(n)
    idx, val, cnt = _topn_outputs(B, n, dev)
    if B == 0:
        return idx, val, cnt[:0]
    if excl_indptr is not None:
        excl_indptr, excl_items = _sorted_exclusions(excl_indptr, excl_items, n_items, B, dev)
    args.n = n
    args.d_excl_indptr, args.d_excl_items = ptr(excl_indptr), ptr(excl_items)
    args.d_out_idx, args.d_out_val, args.d_out_cnt = ptr(idx), ptr(val), ptr(cnt)
    check(entry(C.byref(args), stream_ptr()), name)
    return idx, val, cnt[:B]


def _sorted_exclusions(indptr: torch.Tensor, items: torch.Tensor, n_items: int, B: int, dev):
    """The exclusion lists as the kernel takes them: item numbers in 0..n_items-1, ascending within each query."""
    indptr = indptr.to(device=dev, dtype=torch.int64)
    items = items.to(device=dev, dtype=torch.int64)
    if indptr.numel() != B + 1:
        raise ValueError(f"excl_indptr must have {B + 1} entries")
    seg = torch.repeat_interleave(torch.arange(B, device=dev), indptr[1:] - indptr[:-1])
    ok = (items >= 0) & (items < n_items)
    seg, items = seg[ok], items[ok]
    keys = torch.sort(seg * n_items + items).values
    out_ptr = torch.zeros(B + 1, dtype=torch.int64, device=dev)
    out_ptr[1:] = torch.cumsum(torch.bincount(seg, minlength=B), 0)
    out_items = (keys - (keys // max(n_items, 1)) * n_items).to(torch.int32)
    if out_items.numel() == 0:  # a non-NULL address the kernel never reads (bounded by the indptr)
        out_items = torch.full((1,), -1, dtype=torch.int32, device=dev)
    return out_ptr, out_items


# ---------------------------------------------------------------------------
# co-occurrence counting and association scoring
# ---------------------------------------------------------------------------


@dataclass
class CoocPlan:
    """
    The inputs of ``lk_cooc_count`` for one (groups, items) interaction list: the groups x items CSR (GI, a
    group's items ascending, repeats kept), its transpose IG (one entry per occurrence), the column tiling and
    GI's tile pointers.  At the ML-25M shape (25 M interactions) GI and IG take 100 MB each and the tile
    pointers 32 MB.
    """

    n_groups: int
    n_items: int
    gi_indptr: torch.Tensor  # int32 [n_groups + 1]
    gi_items: torch.Tensor
    ig_indptr: torch.Tensor  # int32 [n_items + 1]
    ig_groups: torch.Tensor
    geom: LkKnnGeom
    tile_ptr: torch.Tensor
    work_counter: torch.Tensor
    status: torch.Tensor
    cursor: torch.Tensor
    #: optional device int32 flag checked by the count kernel whenever a CTA fetches a work unit
    cancel: torch.Tensor | None = None

    @classmethod
    def create(cls, n_groups: int, n_items: int, groups: torch.Tensor, items: torch.Tensor) -> "CoocPlan":
        """``groups`` / ``items``: int32 device tensors of equal length, ``groups`` ascending, every number in range
        (the caller validates)."""
        if n_items < 1:
            raise ValueError("n_items must be positive")
        if groups.numel() >= 2**31:
            raise _lib.EngineError("co-occurrence input with 2**31 or more entries is not supported")
        dev = groups.device
        g, i = groups.to(torch.int64), items.to(torch.int64)

        def offsets(keys: torch.Tensor, n: int) -> torch.Tensor:
            ip = torch.zeros(n + 1, dtype=torch.int64, device=dev)
            torch.cumsum(torch.bincount(keys, minlength=n), 0, out=ip[1:])
            return ip.to(torch.int32)

        gi_items = (torch.sort(g * n_items + i).values % n_items).to(torch.int32)
        ig_groups = (torch.sort(i * max(n_groups, 1) + g).values % max(n_groups, 1)).to(torch.int32)
        gi_indptr, ig_indptr = offsets(g, n_groups), offsets(i, n_items)
        L = lib()
        geom = LkKnnGeom()
        check(L.lk_cooc_geometry(n_groups, n_items, C.byref(geom)), "lk_cooc_geometry")
        tile_ptr = torch.empty(max(1, n_groups * (geom.n_subtiles + 1)), dtype=torch.int32, device=dev)
        if gi_items.numel() == 0:
            gi_items = torch.zeros(1, dtype=torch.int32, device=dev)  # a non-NULL address, never read
            ig_groups = torch.zeros(1, dtype=torch.int32, device=dev)
        check(
            L.lk_knn_tile_pointers(C.byref(geom), ptr(gi_indptr), ptr(gi_items), ptr(tile_ptr), stream_ptr()),
            "lk_knn_tile_pointers",
        )
        z = lambda dt: torch.zeros(1, dtype=dt, device=dev)  # noqa: E731
        return cls(
            n_groups, n_items, gi_indptr, gi_items, ig_indptr, ig_groups, geom, tile_ptr,
            z(torch.int32), z(torch.int32), z(torch.int64),
        )  # fmt: skip

    def _args(self, full_rows: bool) -> LkCoocArgs:
        a = LkCoocArgs()
        a.geom = self.geom
        a.d_gi_indptr, a.d_gi_items = ptr(self.gi_indptr), ptr(self.gi_items)
        a.d_ig_indptr, a.d_ig_groups = ptr(self.ig_indptr), ptr(self.ig_groups)
        a.d_tile_ptr = ptr(self.tile_ptr)
        a.full_rows = 1 if full_rows else 0
        a.d_work_counter, a.d_status, a.d_pool_cursor = ptr(self.work_counter), ptr(self.status), ptr(self.cursor)
        a.d_cancel = ptr(self.cancel)
        return a

    def row_cost(self, full_rows: bool) -> torch.Tensor:
        """Pair updates of every row (int64 [n_items]): its columns > item, or all of them with ``full_rows``."""
        cost = torch.empty(self.n_items, dtype=torch.int64, device=self.gi_indptr.device)
        check(lib().lk_cooc_row_cost(C.byref(self._args(full_rows)), ptr(cost), stream_ptr()), "lk_cooc_row_cost")
        return cost

    def count(
        self,
        full_rows: bool = False,
        method: int = _lib.LK_COOC_COUNT,
        item_count: torch.Tensor | None = None,
        damping: float = 0.0,
        attach=None,
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """
        The co-occurrence rows as a device CSR (int64 indptr [n_items+1], int32 columns ascending, values): the
        strict upper triangle, or every off-diagonal entry with ``full_rows``.  Values are the int32 counts, or with
        ``method`` ``LK_ASSOC_PROBABILITY`` / ``LK_ASSOC_LIFT`` (full rows only) the f32 association values of
        ``AssociationScorer.train`` from ``item_count`` (int32 [n_items]) and ``damping``.  ``attach(counter,
        units)``, if given, is called before the launch and returns the device cancel flag.
        """
        dev = self.gi_indptr.device
        n, H, CW = self.n_items, self.geom.n_halves, self.geom.warps * self.geom.tile_cols
        cost = self.row_cost(full_rows)
        order = torch.argsort(cost, descending=True, stable=True)
        order = order[cost[order] > 0]  # a row without pair updates has no entries and needs no unit
        h = torch.arange(H, device=dev)
        units = order[:, None] * H + h[None, :]
        if not full_rows:  # tiles left of the diagonal hold no column > item
            units = units[(h[None, :] + 1) * CW > order[:, None] + 1]
        sched = units.reshape(-1).to(torch.int32).contiguous()
        width = (n - 1 - torch.arange(n, device=dev)) if not full_rows else torch.full((n,), n - 1, device=dev)
        capacity = int(torch.minimum(cost, width).sum().item())  # a row has at most min(cost, width) entries
        max_cost = int(cost.max().item()) if n else 0
        a = self._args(full_rows)
        if attach is not None:
            self.cancel = attach(self.work_counter, sched.numel())
            a.d_cancel = ptr(self.cancel)
        a.method, a.d_item_count, a.damping = int(method), ptr(item_count), float(damping)
        a.max_row_cost = max_cost
        a.d_sched, a.n_work = ptr(sched), sched.numel()

        def launch(pool_cols, pool_vals, pool_off, part_cnt):
            a.d_pool_cols, a.d_pool_vals, a.pool_capacity = ptr(pool_cols), ptr(pool_vals), pool_cols.numel()
            a.d_pool_off, a.d_part_cnt = ptr(pool_off), ptr(part_cnt)
            check(lib().lk_cooc_count(C.byref(a), stream_ptr()), "lk_cooc_count")
            return int(self.status.item())

        def gather(indptr, cols, vals):
            rc = lib().lk_cooc_pool_to_csr(C.byref(a), ptr(indptr), ptr(cols), ptr(vals), stream_ptr())
            check(rc, "lk_cooc_pool_to_csr")

        indptr, cols, vals = pool_to_csr(
            dev, n, H, capacity, torch.int32, launch, gather, "lk_cooc_count: pool overflow"
        )
        if method != _lib.LK_COOC_COUNT:
            vals = vals.view(torch.float32)
        return indptr, cols, vals

    def diagonal(self) -> torch.Tensor:
        """``sum_g #i (#i + 1) / 2`` for every item (int32 [n_items]); a count of 2**31 or more raises."""
        d = torch.zeros(self.n_items, dtype=torch.int64, device=self.gi_indptr.device)
        check(lib().lk_cooc_diagonal(C.byref(self._args(False)), ptr(d), stream_ptr()), "lk_cooc_diagonal")
        if self.n_items and int(d.max().item()) >= 2**31:
            raise _lib.EngineError("a diagonal co-occurrence count exceeds int32")
        return d.to(torch.int32)

    def dense(self, indptr: torch.Tensor, cols: torch.Tensor, counts: torch.Tensor, diag: torch.Tensor | None):
        """``dense_cooc``'s matrix from the upper-triangle CSR of :meth:`count` and, optionally, :meth:`diagonal`."""
        n = self.n_items
        out = torch.zeros((n, n), dtype=torch.float32, device=indptr.device)
        d64 = None if diag is None else diag.to(torch.int64)
        check(
            lib().lk_cooc_dense(n, ptr(indptr), ptr(_nonempty(cols)), ptr(_nonempty(counts)), ptr(d64), ptr(out),
                                stream_ptr()),
            "lk_cooc_dense",
        )  # fmt: skip
        return out


def _nonempty(t: torch.Tensor) -> torch.Tensor:
    """A tensor with a non-NULL address: the library rejects NULL, and bounded reads never touch the placeholder."""
    return t if t.numel() else torch.zeros(1, dtype=t.dtype, device=t.device)


@dataclass
class AssocState:
    """The association matrix in HBM (int64 offsets, rows sorted by column) with the tiling and row-relative tile
    pointers of ``lk_assoc_score_batch``.  Read-only once built: every call allocates its own outputs, so concurrent
    callers need no lock."""

    n_items: int
    indptr: torch.Tensor  # int64 [n_items + 1]
    cols: torch.Tensor  # int32
    vals: torch.Tensor  # float32
    geom: LkKnnGeom
    tile_ptr: torch.Tensor

    @classmethod
    def create(cls, n_items: int, indptr, cols, vals, device=None) -> "AssocState":
        device = device or _lib.require_device()
        dev = lambda t, dt: _nonempty(torch.as_tensor(t).to(device=device, dtype=dt).contiguous())  # noqa: E731
        ip, c, v = dev(indptr, torch.int64), dev(cols, torch.int32), dev(vals, torch.float32)
        g = LkKnnGeom()
        check(lib().lk_cooc_geometry(n_items, n_items, C.byref(g)), "lk_cooc_geometry")
        tp = torch.empty(max(1, n_items * (g.n_subtiles + 1)), dtype=torch.int32, device=device)
        check(lib().lk_assoc_tile_pointers(C.byref(g), ptr(ip), ptr(c), ptr(tp), stream_ptr()), "lk_assoc_tile_pointers")
        return cls(n_items, ip, c, v, g, tp)

    def _args(self, ref_indptr: torch.Tensor, ref_items: torch.Tensor, agg: int) -> LkAssocScoreArgs:
        a = LkAssocScoreArgs()
        a.geom = self.geom
        a.d_indptr, a.d_cols, a.d_vals, a.d_tile_ptr = ptr(self.indptr), ptr(self.cols), ptr(self.vals), ptr(self.tile_ptr)
        a.n_queries = ref_indptr.numel() - 1
        a.agg = int(agg)
        a.d_ref_indptr, a.d_ref_items = ptr(ref_indptr), ptr(_nonempty(ref_items))
        return a

    def score(self, ref_indptr: torch.Tensor, ref_items: torch.Tensor, agg: int) -> torch.Tensor:
        """
        Scores of every item for every query (f32 [B, n_items]): query q's reference rows are
        ``ref_items[ref_indptr[q]:ref_indptr[q+1]]`` in query order (all in range); ``agg`` 0 is the mean over them
        (``max_nbrs=None``), 1 the maximum (``max_nbrs=1``); a query without rows scores NaN everywhere.
        """
        B = ref_indptr.numel() - 1
        out = torch.empty((B, self.n_items), dtype=torch.float32, device=self.indptr.device)
        if B == 0:
            return out
        a = self._args(ref_indptr, ref_items, agg)
        a.n, a.d_scores = 0, ptr(out)
        check(lib().lk_assoc_score_batch(C.byref(a), stream_ptr()), "lk_assoc_score_batch")
        return out

    def recommend(
        self, ref_indptr: torch.Tensor, ref_items: torch.Tensor, agg: int, n: int,
        excl_indptr: torch.Tensor | None = None, excl_items: torch.Tensor | None = None,
    ):  # fmt: skip
        """
        Top-``n`` of every query over all items minus ``excl_items[excl_indptr[q]:excl_indptr[q+1]]`` (any order),
        with ``argtopn``'s order and ties: ``(idx [B, n] int32, -1 padding; val [B, n] f32, NaN padding; cnt [B])``.
        """
        return _rank_launch(self._args(ref_indptr, ref_items, agg), lib().lk_assoc_score_batch, "lk_assoc_score_batch",
                            n, self.n_items, ref_indptr.numel() - 1, self.indptr.device, excl_indptr, excl_items)

    def host_csr(self):
        """The matrix on the host as a SciPy ``csr_array`` (rows sorted)."""
        import scipy.sparse as sps

        nnz = int(self.indptr[-1].item())
        return sps.csr_array((self.vals[:nnz].cpu().numpy(), self.cols[:nnz].cpu().numpy(), self.indptr.cpu().numpy()),
                             shape=(self.n_items, self.n_items))  # fmt: skip


# ---------------------------------------------------------------------------
# EASE scoring
# ---------------------------------------------------------------------------


@dataclass
class EaseState:
    """The EASE weight matrix in HBM (f32 [n_items, n_items], row-major).  Read-only once built: every call
    allocates its own outputs, so concurrent callers need no lock."""

    weights: torch.Tensor

    @property
    def n_items(self) -> int:
        return int(self.weights.shape[0])

    @classmethod
    def create(cls, weights, device=None) -> "EaseState":
        device = device or _lib.require_device()
        w = torch.as_tensor(weights).to(device=device, dtype=torch.float32).contiguous()
        if w.dim() != 2 or w.shape[0] != w.shape[1] or w.shape[0] < 1:
            raise ValueError("EASE weights must be a non-empty square matrix")
        if w.shape[0] >= 2**31:
            raise _lib.EngineError("EASE with 2**31 or more items is not supported")
        return cls(w)

    def _args(self, hist_indptr: torch.Tensor, hist_items: torch.Tensor) -> LkEaseScoreArgs:
        a = LkEaseScoreArgs()
        a.n_items, a.d_w = self.n_items, ptr(self.weights)
        a.n_queries = hist_indptr.numel() - 1
        a.d_hist_indptr, a.d_hist_items = ptr(hist_indptr), ptr(_nonempty(hist_items))
        return a

    def score(self, hist_indptr: torch.Tensor, hist_items: torch.Tensor) -> torch.Tensor:
        """
        Scores of every item for every query (f32 [B, n_items]): query q's history is ``hist_items[hist_indptr[q]:
        hist_indptr[q+1]]``, ascending without repeats (``batch.history_csr(..., unique=True)``); each score is the f32 sum of the
        history rows' entries in that order; a query without history scores NaN everywhere.
        """
        B = hist_indptr.numel() - 1
        out = torch.empty((B, self.n_items), dtype=torch.float32, device=self.weights.device)
        if B == 0:
            return out
        a = self._args(hist_indptr, hist_items)
        a.n, a.d_scores = 0, ptr(out)
        check(lib().lk_ease_score_batch(C.byref(a), stream_ptr()), "lk_ease_score_batch")
        return out

    def recommend(
        self, hist_indptr: torch.Tensor, hist_items: torch.Tensor, n: int,
        excl_indptr: torch.Tensor | None = None, excl_items: torch.Tensor | None = None,
    ):  # fmt: skip
        """
        Top-``n`` of every query over all items minus ``excl_items[excl_indptr[q]:excl_indptr[q+1]]`` (any order),
        with ``argtopn``'s order and ties: ``(idx [B, n] int32, -1 padding; val [B, n] f32, NaN padding; cnt [B])``.
        A query without history gets an empty list.
        """
        return _rank_launch(self._args(hist_indptr, hist_items), lib().lk_ease_score_batch, "lk_ease_score_batch", n,
                            self.n_items, hist_indptr.numel() - 1, self.weights.device, excl_indptr, excl_items)


# ---------------------------------------------------------------------------
# Sparse x dense products and the randomized SVD (BiasedSVD)
# ---------------------------------------------------------------------------


def spmm_order(m: DeviceCSR) -> torch.Tensor:
    """The rows of ``m`` longest first (int32, ties ascending): the order ``lk_spmm`` hands rows to warps."""
    return torch.argsort(m.indptr[1:] - m.indptr[:-1], descending=True, stable=True).to(torch.int32)


def spmm(m: DeviceCSR, order: torch.Tensor, dense: torch.Tensor) -> torch.Tensor:
    """
    ``m @ dense`` (``lk_spmm``), f32 [n_rows, W]: every element one sequential sum over the row's stored entries,
    product and sum each rounded, which is SciPy's f32 product bit for bit.  ``order`` is :func:`spmm_order` of ``m``.
    """
    if dense.dtype != torch.float32 or dense.dim() != 2 or dense.shape[0] != m.shape[1] or dense.shape[1] < 1:
        raise ValueError(f"dense operand must be f32 [{m.shape[1]}, W >= 1], not {dense.dtype} {tuple(dense.shape)}")
    dense = dense.contiguous()
    out = torch.empty((m.shape[0], dense.shape[1]), dtype=torch.float32, device=dense.device)
    a = LkSpmmArgs()
    a.n_rows, a.n_src, a.width, a.nnz = m.shape[0], m.shape[1], dense.shape[1], m.nnz
    a.d_indptr, a.d_indices, a.d_values = ptr(m.indptr), ptr(_nonempty(m.indices)), ptr(_nonempty(m.values))
    a.d_order, a.d_dense, a.d_out = ptr(order), ptr(dense), ptr(out)
    check(lib().lk_spmm(C.byref(a), stream_ptr()), "lk_spmm")
    return out


def lu_permuted_l(a: torch.Tensor) -> torch.Tensor:
    """
    ``scipy.linalg.lu(a, permute_l=True)[0]``, the product P L of ``a = P L U``, from ``torch.linalg.lu_factor_ex``
    (getrf).  P is never formed: the pivots (min(m, n) row swaps, read on the host) become a row permutation that is
    applied to L as a gather.  Shape [m, min(m, n)].
    """
    m, n = a.shape
    r = min(m, n)
    lu, piv, _info = torch.linalg.lu_factor_ex(a)  # a singular U is no error, as in SciPy
    L = lu[:, :r].tril(-1)
    L.diagonal().fill_(1.0)
    perm = np.arange(m)
    for i, t in enumerate(piv.cpu().numpy().astype(np.int64) - 1):  # LAPACK's 1-based swaps, applied in order
        perm[i], perm[t] = perm[t], perm[i]
    inv = np.empty(m, dtype=np.int64)
    inv[perm] = np.arange(m)  # row perm[i] of P L is row i of L
    return L[torch.from_numpy(inv).to(a.device)]


@dataclass
class SvdOperand:
    """
    A sparse matrix M for the randomized SVD, with Mᵀ beside it: both orientations in HBM and each one's row order
    for ``lk_spmm``.  ``M @ D`` is ``spmm(rows)``, ``Mᵀ @ D`` is ``spmm(cols)``.
    """

    rows: DeviceCSR
    cols: DeviceCSR
    rows_order: torch.Tensor
    cols_order: torch.Tensor

    @classmethod
    def create(cls, rows: DeviceCSR, cols: DeviceCSR) -> "SvdOperand":
        return cls(rows, cols, spmm_order(rows), spmm_order(cols))

    @property
    def shape(self) -> tuple[int, int]:
        return self.rows.shape

    def mul(self, d: torch.Tensor) -> torch.Tensor:
        return spmm(self.rows, self.rows_order, d)

    def tmul(self, d: torch.Tensor) -> torch.Tensor:
        return spmm(self.cols, self.cols_order, d)

    @property
    def T(self) -> "SvdOperand":
        return SvdOperand(self.cols, self.rows, self.cols_order, self.rows_order)


def randomized_svd(x: SvdOperand, q0: torch.Tensor, k: int, n_iter: int, stage=None):
    """
    ``TruncatedSVD(k, algorithm="randomized", n_iter=n_iter).fit`` of the f32 matrix X (scikit-learn's
    ``_randomized_svd`` with ``flip_sign=False``, then ``svd_flip(u_based_decision=False)``) on the device: returns
    ``(components_ [k, n_cols], singular_values_ [k])``.  M is Xᵀ when X has fewer rows than columns, else X; ``q0``
    is the start matrix [M.shape[1], k + oversamples].  The sparse products run on ``lk_spmm`` (SciPy's bit for
    bit); the LU (with ``n_iter > 2``), QR and SVD are torch's (cuSOLVER) in f32.  ``stage(name)``, when given, is
    a context manager entered around each step (benchmark timing).
    """
    stage = stage or (lambda _name: contextlib.nullcontext())
    with _prefer_cusolver():
        return _randomized_svd(x, q0, k, n_iter, stage)


@contextlib.contextmanager
def _prefer_cusolver():
    """torch's dense factorisations on cuSOLVER for the duration (its default may pick MAGMA's batched LU, which is
    meant for many small matrices and says so on stdout); the caller's preference is restored after."""
    before = torch.backends.cuda.preferred_linalg_library()
    torch.backends.cuda.preferred_linalg_library("cusolver")
    try:
        yield
    finally:
        torch.backends.cuda.preferred_linalg_library(before)


def randomized_svd_usv(x: SvdOperand, q0: torch.Tensor, k: int, n_iter: int, stage=None):
    """
    scikit-learn's ``_randomized_svd(X, k, n_iter=n_iter)`` with ``flip_sign=True`` on the device, as NMF's
    ``nndsvda`` initialisation calls it: returns ``(U [n_rows, k], s [k], Vt [k, n_cols])`` of the f32 matrix X.
    Each component's sign makes the entry of largest magnitude (the first such) of X's left singular vector
    positive: ``svd_flip(U, Vt)`` without transposition, ``svd_flip(..., u_based_decision=False)`` on Xᵀ's factors
    with it.  ``q0`` and the products, LU, QR and SVD are as in :func:`randomized_svd`.
    """
    stage = stage or (lambda _name: contextlib.nullcontext())
    with _prefer_cusolver():
        transpose, Q, Uh, s, Vt = _randomized_basis(x, q0, n_iter, stage)
        with stage("svd"):
            left = (Q @ Uh[:, :k], Vt[:k].T)  # M's left singular vectors, and its right ones
            u, vt = (left[1], left[0].T) if transpose else (left[0], left[1].T)
        with stage("flip"):
            pick = u.abs().argmax(dim=0, keepdim=True)
            sign = torch.sign(torch.gather(u, 0, pick))
            u, vt = u * sign, vt * sign.T
    return u.contiguous(), s[:k].contiguous(), vt.contiguous()


def _randomized_basis(x: SvdOperand, q0: torch.Tensor, n_iter: int, stage):
    """The range finder and the small SVD of ``_randomized_svd``: ``(transpose, Q, Uh, s, Vt)`` with M = Xᵀ when
    ``transpose``, else X, and ``Q.T @ M = Uh diag(s) Vt``."""
    transpose = x.shape[0] < x.shape[1]
    M = x.T if transpose else x
    Q = q0
    normalise = n_iter > 2  # power_iteration_normalizer="auto": LU, or nothing with n_iter <= 2
    for _ in range(n_iter):
        for product in (M.mul, M.tmul):
            with stage("spmm_power"):
                Q = product(Q)
            if normalise:
                with stage("lu"):
                    Q = lu_permuted_l(Q)
    with stage("spmm_power"):
        Y = M.mul(Q)
    with stage("qr"):
        Q = torch.linalg.qr(Y, mode="reduced")[0]
    with stage("spmm_project"):
        B = M.tmul(Q).T  # Q.T @ M, which SciPy computes as (Mᵀ @ Q).T
    with stage("svd"):
        Uh, s, Vt = torch.linalg.svd(B, full_matrices=False)
    return transpose, Q, Uh, s, Vt


def _randomized_svd(x: SvdOperand, q0: torch.Tensor, k: int, n_iter: int, stage):
    transpose, Q, Uh, s, Vt = _randomized_basis(x, q0, n_iter, stage)
    with stage("svd"):
        vt = (Q @ Uh[:, :k]).T if transpose else Vt[:k]  # the right singular vectors of X
    with stage("flip"):
        # svd_flip(u_based_decision=False): each row's sign is that of its first entry of largest magnitude
        pick = vt.abs().argmax(dim=1, keepdim=True)
        vt = vt * torch.sign(torch.gather(vt, 1, pick))
    return vt.contiguous(), s[:k].contiguous()


# ---------------------------------------------------------------------------
# NMF coordinate descent (NMFScorer)
# ---------------------------------------------------------------------------


def nmf_gram(q: torch.Tensor) -> torch.Tensor:
    """``Q.T @ Q`` [k, k]: in f64, rounded once to f32 (scikit-learn's is an f32 sgemm; see DESIGN.md §4.17)."""
    q = q.double()
    return (q.T @ q).float().contiguous()


def nmf_cd_sweep(w: torch.Tensor, hht: torch.Tensor, xht: torch.Tensor, pg: torch.Tensor) -> None:
    """One ``_update_cdnmf_fast(W, HHt, XHt, arange(k))`` (``lk_nmf_cd_sweep``): W [n, k] updated in place, every
    |projected gradient| written to ``pg`` [k, n]."""
    n, k = w.shape
    for t, shape in ((w, (n, k)), (hht, (k, k)), (xht, (n, k)), (pg, (k, n))):
        if t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"NMF sweep operands must be contiguous f32 of shapes W [n, k], HHt [k, k], XHt [n, k], "
                             f"pg [k, n]; got {tuple(t.shape)} for {shape}")  # fmt: skip
    a = LkNmfCdSweepArgs()
    a.n, a.k = n, k
    a.d_w, a.d_hht, a.d_xht, a.d_pg = ptr(w), ptr(hht), ptr(xht), ptr(pg)
    check(lib().lk_nmf_cd_sweep(C.byref(a), stream_ptr()), "lk_nmf_cd_sweep")


def f32_seq_sum(xs: list[torch.Tensor]) -> torch.Tensor:
    """The left-to-right f32 sums ``np.cumsum(x, dtype=float32)[-1]`` of the non-negative f32 tensors ``xs`` (at
    most 8), computed concurrently by ``lk_f32_seq_sum``: a device tensor [len(xs)]."""
    out = torch.empty(len(xs), dtype=torch.float32, device=xs[0].device)
    sums = (LkF32SeqSumArgs * len(xs))()
    for i, x in enumerate(xs):
        if x.dtype != torch.float32 or not x.is_contiguous():
            raise ValueError("f32_seq_sum needs contiguous f32 tensors")
        sums[i].n, sums[i].d_x, sums[i].d_out = x.numel(), ptr(x), out.data_ptr() + 4 * i
    check(lib().lk_f32_seq_sum(sums, len(xs), stream_ptr()), "lk_f32_seq_sum")
    return out


@dataclass
class NmfDescent:
    """
    ``_fit_coordinate_descent`` on the device for the indicator matrix X (both orientations in ``x``): W [n_rows, k]
    and Ht [n_cols, k] in HBM, updated in place by :meth:`iteration`, and the two |pg| buffers of the sweeps.
    """

    x: SvdOperand
    W: torch.Tensor
    Ht: torch.Tensor
    l1_W: float = 0.0
    l1_H: float = 0.0
    l2_W: float = 0.0
    l2_H: float = 0.0
    pg_W: torch.Tensor = field(init=False)
    pg_H: torch.Tensor = field(init=False)

    def __post_init__(self):
        k = self.W.shape[1]
        self.pg_W = torch.empty((k, self.W.shape[0]), dtype=torch.float32, device=self.W.device)
        self.pg_H = torch.empty((k, self.Ht.shape[0]), dtype=torch.float32, device=self.W.device)

    def half(self, product, w, ht, l1: float, l2: float, pg, stage) -> None:
        """``_update_coordinate_descent(X, W, Ht, l1, l2)`` without its violation sum: Gram, product, sweep."""
        with stage("gram"):
            hht = nmf_gram(ht)
            if l2 != 0.0:
                hht.diagonal().add_(l2)  # in f32, as NumPy adds a Python float to an f32 array
        with stage("spmm"):
            xht = product(ht)
            if l1 != 0.0:
                xht.sub_(l1)
        with stage("sweep"):
            nmf_cd_sweep(w, hht, xht, pg)

    def iteration(self, stage=None) -> tuple[float, float]:
        """One iteration: the W sweep, the H sweep, then both violations (f32, returned as Python floats)."""
        stage = stage or (lambda _name: contextlib.nullcontext())
        self.half(self.x.mul, self.W, self.Ht, self.l1_W, self.l2_W, self.pg_W, stage)
        self.half(self.x.tmul, self.Ht, self.W, self.l1_H, self.l2_H, self.pg_H, stage)
        with stage("sum"):
            v = f32_seq_sum([self.pg_W.view(-1), self.pg_H.view(-1)]).cpu().numpy()
        return float(v[0]), float(v[1])


def nndsvd(u: torch.Tensor, s: torch.Tensor, vt: torch.Tensor, fill: float) -> tuple[torch.Tensor, torch.Tensor]:
    """
    The NNDSVD step of scikit-learn's ``_initialize_nmf`` (``init="nndsvda"``) on the device: W [n_rows, k] and
    H [k, n_cols] from X's SVD, entries below 1e-6 set to 0 and then every 0 to ``fill`` (``X.mean()``).  The norms
    are square roots of f32 sums of squares taken in f64, and the products of norms are f64, as there; f32 sums in
    another order than BLAS's, so W and H agree with scikit-learn's to rounding.
    """
    W = torch.zeros_like(u)
    H = torch.zeros_like(vt)
    W[:, 0] = torch.sqrt(s[0]) * u[:, 0].abs()
    H[0, :] = torch.sqrt(s[0]) * vt[0, :].abs()
    if u.shape[1] > 1:
        x, y = u[:, 1:], vt[1:, :].T  # one column per component
        xp, yp = x.clamp(min=0), y.clamp(min=0)
        xn, yn = x.clamp(max=0).abs(), y.clamp(max=0).abs()
        nrm = lambda a: (a * a).sum(dim=0).double().sqrt()  # noqa: E731
        xpn, ypn, xnn, ynn = nrm(xp), nrm(yp), nrm(xn), nrm(yn)
        mp, mn = xpn * ypn, xnn * ynn
        pos = mp > mn
        uu = torch.where(pos, xp / xpn.float(), xn / xnn.float())
        vv = torch.where(pos, yp / ypn.float(), yn / ynn.float())
        lbd = torch.sqrt(s[1:] * torch.where(pos, mp, mn).float())
        W[:, 1:] = lbd * uu
        H[1:, :] = (lbd * vv).T
    W[W < 1e-6] = 0
    H[H < 1e-6] = 0
    W[W == 0] = fill
    H[H == 0] = fill
    return W.contiguous(), H.contiguous()


# ---------------------------------------------------------------------------
# SLIM training
# ---------------------------------------------------------------------------


@dataclass
class SlimPlan:
    """
    The inputs of ``lk_slim_train`` for one training run: the UI and IU structures (int32 offsets and indices, rows
    in the caller's stored order), the f32 regularisation, the iteration and neighbour limits, and the target items
    most expensive first.  ``columns`` restricts training to some target items (their rows are computed exactly as
    in a full run; the others stay empty), so that a sample of the items can be checked or timed.
    """

    n_users: int
    n_items: int
    ui_indptr: torch.Tensor
    ui_cols: torch.Tensor
    iu_indptr: torch.Tensor
    iu_cols: torch.Tensor
    l1_reg: float
    l2_reg: float
    max_iters: int
    max_nbrs: int  # -1: SLIM
    sched: torch.Tensor  # int32 target items, most expensive first
    capacity_bound: int  # entries the result can have at most
    work_counter: torch.Tensor
    status: torch.Tensor
    cursor: torch.Tensor
    #: optional device int32 flag checked whenever a warp fetches a target item
    cancel: torch.Tensor | None = None

    @classmethod
    def create(
        cls, n_users: int, n_items: int, ui_indptr, ui_cols, iu_indptr, iu_cols, l1_reg: float, l2_reg: float,
        max_iters: int, max_nbrs: int | None, columns=None,
    ) -> "SlimPlan":  # fmt: skip
        """Device tensors in (any integer dtype; nnz < 2**31).  Raises ``ValueError`` for an index out of range or an
        IU row that repeats a user (coordinate descent updates each of a row's residuals once per entry)."""
        if n_items < 1 or n_users < 0:
            raise ValueError("SLIM needs at least one item")
        dev = ui_indptr.device
        i32 = lambda t: _nonempty(torch.as_tensor(t).to(device=dev, dtype=torch.int32).contiguous())  # noqa: E731
        for name, ip, c, rows, ncols in (("ui_matrix", ui_indptr, ui_cols, n_users, n_items),
                                         ("iu_matrix", iu_indptr, iu_cols, n_items, n_users)):  # fmt: skip
            if ip.numel() != rows + 1 or int(ip[-1].item()) != c.numel():
                raise ValueError(f"{name}: offsets do not match the shape")
            if c.numel() >= 2**31:
                raise _lib.EngineError("SLIM input with 2**31 or more entries is not supported")
            if c.numel() and (int(c.min().item()) < 0 or int(c.max().item()) >= ncols):
                raise ValueError(f"{name}: index out of range")
        nnz = iu_cols.numel()
        if nnz:
            row = torch.repeat_interleave(torch.arange(n_items, device=dev), (iu_indptr[1:] - iu_indptr[:-1]).long())
            key = torch.sort(row * max(n_users, 1) + iu_cols.long()).values
            if bool((key[1:] == key[:-1]).any()):
                raise ValueError("iu_matrix: a row repeats a user")
        ui_p, ui_c, iu_p, iu_c = i32(ui_indptr), i32(ui_cols), i32(iu_indptr), i32(iu_cols)
        # cost of target i: sum over its users of their UI row lengths, the entries the active-set walk reads
        geom = LkKnnGeom()
        check(lib().lk_cooc_geometry(max(n_users, 0), n_items, C.byref(geom)), "lk_cooc_geometry")
        ca = LkCoocArgs()
        ca.geom, ca.full_rows = geom, 1
        ca.d_gi_indptr, ca.d_gi_items, ca.d_ig_indptr, ca.d_ig_groups = ptr(ui_p), ptr(ui_c), ptr(iu_p), ptr(iu_c)
        cost = torch.empty(n_items, dtype=torch.int64, device=dev)
        check(lib().lk_cooc_row_cost(C.byref(ca), ptr(cost), stream_ptr()), "lk_cooc_row_cost")
        if columns is None:
            cols = torch.arange(n_items, device=dev)
        else:
            cols = torch.unique(torch.as_tensor(columns, device=dev).long())
            if cols.numel() and (int(cols[0].item()) < 0 or int(cols[-1].item()) >= n_items):
                raise ValueError("columns: item out of range")
        sched = cols[torch.argsort(cost[cols], descending=True, stable=True)].to(torch.int32).contiguous()
        k = -1 if max_nbrs is None or int(max_nbrs) >= n_items else int(max_nbrs)
        width = min(n_items - 1, k) if k >= 0 else n_items - 1
        bound = int(torch.clamp(cost[cols], max=max(width, 0)).sum().item())
        z = lambda dt: torch.zeros(1, dtype=dt, device=dev)  # noqa: E731
        return cls(
            n_users, n_items, ui_p, ui_c, iu_p, iu_c, float(np.float32(l1_reg)), float(np.float32(l2_reg)),
            int(max_iters), k, sched, bound, z(torch.int32), z(torch.int32), z(torch.int64),
        )  # fmt: skip

    def train(self, attach=None, capacity: int | None = None):
        """
        The weight rows as a device CSR (int64 indptr [n_items+1], int32 columns ascending, f32 values).
        ``attach(counter, units)``, if given, is called before the launch and returns the device cancel flag.  The
        result pool starts at ``capacity`` entries (a guess by default) and a run that overflows it is repeated
        with a larger pool, up to the bound that cannot overflow.
        """
        dev = self.ui_indptr.device
        n = self.n_items
        a = LkSlimArgs()
        a.n_users, a.n_items = self.n_users, n
        a.d_ui_indptr, a.d_ui_cols = ptr(self.ui_indptr), ptr(self.ui_cols)
        a.d_iu_indptr, a.d_iu_cols = ptr(self.iu_indptr), ptr(self.iu_cols)
        a.l1_reg, a.l2_reg, a.max_iters, a.max_nbrs = self.l1_reg, self.l2_reg, self.max_iters, self.max_nbrs
        a.d_sched, a.n_work = ptr(self.sched), self.sched.numel()
        a.d_work_counter, a.d_status, a.d_pool_cursor = ptr(self.work_counter), ptr(self.status), ptr(self.cursor)
        if attach is not None:
            self.cancel = attach(self.work_counter, self.sched.numel())
        a.d_cancel = ptr(self.cancel)
        ws_bytes = C.c_int64()
        check(lib().lk_slim_workspace_bytes(self.n_users, n, self.sched.numel(), C.byref(ws_bytes)),
              "lk_slim_workspace_bytes")  # fmt: skip
        ws = torch.zeros(max(int(ws_bytes.value), 1), dtype=torch.uint8, device=dev)
        a.d_workspace, a.workspace_bytes = ptr(ws), ws.numel()
        if capacity is None:
            capacity = max(4 * self.iu_cols.numel(), 1 << 22)
        capacity = max(1, min(int(capacity), self.capacity_bound))
        overflowed = False

        def launch(pool_cols, pool_vals, pool_off, part_cnt):
            nonlocal overflowed
            a.d_pool_cols, a.d_pool_vals, a.pool_capacity = ptr(pool_cols), ptr(pool_vals), pool_cols.numel()
            a.d_pool_off, a.d_part_cnt = ptr(pool_off), ptr(part_cnt)
            check(lib().lk_slim_train(C.byref(a), stream_ptr()), "lk_slim_train")
            st = int(self.status.item())
            overflowed = st == 1
            return st

        def gather(indptr, cols, vals):
            check(lib().lk_slim_pool_to_csr(C.byref(a), ptr(indptr), ptr(cols), ptr(vals), stream_ptr()),
                  "lk_slim_pool_to_csr")  # fmt: skip

        while True:
            try:
                return pool_to_csr(dev, n, 1, capacity, torch.float32, launch, gather, "lk_slim_train: pool overflow")
            except _lib.EngineError:
                if not overflowed or capacity >= self.capacity_bound:
                    raise
                capacity = min(4 * capacity, self.capacity_bound)


# ---------------------------------------------------------------------------
# FlexMF implicit and explicit
# ---------------------------------------------------------------------------

FLEXMF_LOSSES = {"logistic": _lib.LK_FLEXMF_LOGISTIC, "pairwise": _lib.LK_FLEXMF_PAIRWISE, "mse": _lib.LK_FLEXMF_MSE}
FLEXMF_REG_METHODS = {None: _lib.LK_FLEXMF_REG_NONE, "L2": _lib.LK_FLEXMF_REG_L2, "AdamW": _lib.LK_FLEXMF_REG_ADAMW}
FLEXMF_MAX_ATTEMPTS = 10  # rejected draws per negative, as the reference's sampler
FLEXMF_UNIT = 64  # occurrences of a row per gradient unit (flexmf.cu)
_ADAM_BETA1, _ADAM_BETA2, _ADAM_EPS = 0.9, 0.999, 1e-8  # torch.optim defaults


def flexmf_workspace_bytes(batch: int, n_neg: int, k: int) -> int:
    out = C.c_int64()
    check(lib().lk_flexmf_workspace_bytes(batch, n_neg, k, C.byref(out)), "lk_flexmf_workspace_bytes")
    return int(out.value)


def flexmf_adam_scalars(reg_method: str | None, lr: float, regularization: float, step: int) -> dict[str, float]:
    """The step-dependent scalars of ``lk_flexmf_step``, computed in double as torch's optimisers do."""
    bc1, bc2 = 1 - _ADAM_BETA1**step, 1 - _ADAM_BETA2**step
    if reg_method == "AdamW":
        return {"decay": 1 - lr * regularization, "step_size": lr / bc1, "bias2_sqrt": bc2**0.5}
    return {"decay": 1.0, "step_size": lr * bc2**0.5 / bc1, "bias2_sqrt": 1.0}


@dataclass
class _FlexmfGroups:
    """One side's occurrences in a run of batches, grouped for ``lk_flexmf_step`` (``lk_flexmf_groups``)."""

    occ: torch.Tensor
    unit_start: torch.Tensor
    unit_uniq: torch.Tensor
    uniq_row: torch.Tensor
    uniq_unit: torch.Tensor
    step_uniq: np.ndarray  # host: first uniq of every step, and the total
    step_unit: np.ndarray  # host: first unit of every step, and the total

    @classmethod
    def build(cls, keys: torch.Tensor, entries: torch.Tensor, n_rows: int, n_steps: int) -> "_FlexmfGroups":
        """``keys`` = step * n_rows + row of every occurrence, ``entries`` ascending within a step.  Index plumbing
        only (a stable sort, flags and prefix sums); the additions these groups order are the kernel's."""
        dev = keys.device
        E = keys.numel()
        if E >= 2**31:  # uniq and unit numbers are int32 in lk_flexmf_groups
            raise _lib.EngineError(f"{E} row occurrences in one run of batches; the grouping holds fewer than 2**31")
        skey, order = torch.sort(keys, stable=True)  # stable: entries stay ascending within a (step, row)
        new_row = torch.ones(E, dtype=torch.bool, device=dev)
        new_row[1:] = skey[1:] != skey[:-1]
        uniq_at = torch.nonzero(new_row).flatten()
        uniq_of = torch.cumsum(new_row, 0) - 1
        # every run of one (step, row) is cut from its own start, so a batch's units do not depend on its neighbours
        new_unit = (torch.arange(E, device=dev) - uniq_at[uniq_of]) % FLEXMF_UNIT == 0
        unit_at = torch.nonzero(new_unit).flatten()
        unit_uniq = uniq_of[unit_at].to(torch.int32)
        uniq_unit = torch.searchsorted(unit_at, uniq_at)
        ukey = skey[uniq_at]
        step_uniq = torch.searchsorted(ukey, torch.arange(n_steps + 1, device=dev) * n_rows)
        uniq_unit = torch.cat([uniq_unit, torch.tensor([unit_at.numel()], device=dev)])
        step_unit = uniq_unit[step_uniq]
        return cls(
            entries[order].contiguous(), torch.cat([unit_at, torch.tensor([E], device=dev)]), unit_uniq,
            (ukey % n_rows).to(torch.int32), uniq_unit.to(torch.int32), step_uniq.cpu().numpy(), step_unit.cpu().numpy(),
        )  # fmt: skip

    def fill(self, g, step: int, mark: torch.Tensor | None) -> int:
        g.d_occ, g.d_unit_start, g.d_unit_uniq = ptr(self.occ), ptr(self.unit_start), ptr(self.unit_uniq)
        g.d_uniq_row, g.d_uniq_unit, g.d_mark = ptr(self.uniq_row), ptr(self.uniq_unit), ptr(mark)
        g.unit0, g.uniq0 = int(self.step_unit[step]), int(self.step_uniq[step])
        g.n_uniq = int(self.step_uniq[step + 1] - self.step_uniq[step])
        return int(self.step_unit[step + 1] - self.step_unit[step])


@dataclass
class _FlexmfBatches:
    users: torch.Tensor
    pos: torch.Tensor
    neg: torch.Tensor  # [S, n]; [S, 0] for MSE
    ratings: torch.Tensor | None  # [S] MSE targets
    u_groups: _FlexmfGroups
    i_groups: _FlexmfGroups
    n_steps: int


class FlexMFState:
    """
    Device state of one FlexMF training run: the four parameter tables with their Adam moments, the users x items
    CSR the sampler tests membership in, the step workspace, the optimiser step count and the sampler seed.  The
    only caller of ``lk_flexmf_sample_negatives`` and ``lk_flexmf_step``.

    ``params`` maps the reference's state-dict names (``u_bias.weight`` / ``i_bias.weight`` [n, 1], optional;
    ``u_embed.weight`` / ``i_embed.weight`` [n, k]) to f32 arrays or tensors; ``users`` / ``items`` are the training
    interactions sorted by (user, item).  ``loss="mse"`` (the explicit model) takes ``negative_count=0`` and
    ``ratings``, the f32 target of every interaction (the centred rating), which is permuted with the samples.
    """

    def __init__(self, params: dict, users, items, *, loss: str, reg_method: str | None, negative_count: int = 1,
                 popular: bool = False, batch_size: int = 8192, learning_rate: float = 0.01,
                 regularization: float = 0.01, positive_weight: float = 1.0, seed: int = 0, ratings=None,
                 device=None):  # fmt: skip
        dev = device or _lib.require_device()
        if loss not in FLEXMF_LOSSES:
            raise ValueError(f"loss={loss!r} is not one of {sorted(FLEXMF_LOSSES)}")
        if reg_method not in FLEXMF_REG_METHODS:
            raise ValueError(f"reg_method={reg_method!r} is not one of 'AdamW', 'L2', None")
        if (loss == "mse") != (int(negative_count) == 0):
            raise ValueError(f"loss={loss!r} with negative_count={negative_count}: MSE takes 0 negatives, the others 1 or more")
        if (loss == "mse") != (ratings is not None):
            raise ValueError("ratings are the MSE targets: given with loss='mse' and only then")
        self.loss, self.reg_method, self.n_neg, self.popular = loss, reg_method, int(negative_count), bool(popular)
        self.batch_size, self.lr, self.reg = int(batch_size), float(learning_rate), float(regularization)
        self.positive_weight, self.seed = float(positive_weight), int(seed) & (2**64 - 1)
        self.params: dict[str, torch.Tensor] = {}
        for name in ("u_bias.weight", "i_bias.weight", "u_embed.weight", "i_embed.weight"):
            if params.get(name) is not None:
                self.params[name] = torch.as_tensor(params[name]).to(dev, torch.float32).contiguous().clone()
        self.n_users, self.k = self.params["u_embed.weight"].shape
        self.n_items = self.params["i_embed.weight"].shape[0]
        if self.params["i_embed.weight"].shape[1] != self.k or not 1 <= self.k <= ALS_MAX_FEATURES:
            raise ValueError(f"embedding sizes must agree and be in 1..{ALS_MAX_FEATURES}")
        self.moments = {n: (torch.zeros_like(t), torch.zeros_like(t)) for n, t in self.params.items()}
        self.users = torch.as_tensor(users).to(dev, torch.int32).contiguous()
        self.items = torch.as_tensor(items).to(dev, torch.int32).contiguous()
        self.ratings = None if ratings is None else torch.as_tensor(ratings).to(dev, torch.float32).contiguous()
        if self.ratings is not None and self.ratings.shape != self.items.shape:
            raise ValueError("one rating per interaction")
        self.ui_indptr = torch.zeros(self.n_users + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.bincount(self.users.long(), minlength=self.n_users), 0, out=self.ui_indptr[1:])
        if self.items.numel() >= 2**31:
            raise _lib.EngineError("more than 2**31 - 1 interactions need sharding first")
        self.ui_indptr = self.ui_indptr.to(torch.int32)
        dense = reg_method == "AdamW"
        self.u_mark = torch.zeros(self.n_users, dtype=torch.int64, device=dev) if dense else None
        self.i_mark = torch.zeros(self.n_items, dtype=torch.int64, device=dev) if dense else None
        self.workspace = torch.empty(flexmf_workspace_bytes(self.batch_size, self.n_neg, self.k), dtype=torch.uint8,
                                     device=dev)  # fmt: skip
        self.steps_done = 0
        self.device = dev

    def sample(self, rows: torch.Tensor, step0: int | None = None, *, n: int | None = None,
               popular: bool | None = None, max_attempts: int = FLEXMF_MAX_ATTEMPTS) -> torch.Tensor:  # fmt: skip
        """Negatives [len(rows), n] for the users ``rows``, cut into batches of ``batch_size`` whose step numbers
        start at ``step0`` (default: the steps done so far)."""
        rows = rows.to(self.device, torch.int32).contiguous()
        a = LkFlexmfSampleArgs()
        a.n_users, a.n_items, a.d_ui_indptr, a.d_ui_cols = self.n_users, self.n_items, ptr(self.ui_indptr), ptr(self.items)
        a.d_coo_items, a.nnz, a.d_rows, a.n_samples = ptr(self.items), self.items.numel(), ptr(rows), rows.numel()
        a.batch_size, a.n, a.max_attempts = self.batch_size, self.n_neg if n is None else int(n), int(max_attempts)
        a.popular = int(self.popular if popular is None else popular)
        a.seed, a.step0 = self.seed, self.steps_done if step0 is None else int(step0)
        out = torch.empty((rows.numel(), a.n), dtype=torch.int32, device=self.device)
        a.d_out = ptr(out)
        check(lib().lk_flexmf_sample_negatives(C.byref(a), stream_ptr()), "lk_flexmf_sample_negatives")
        return out

    def _step_args(self) -> LkFlexmfStepArgs:
        a = LkFlexmfStepArgs()
        a.n_users, a.n_items, a.k, a.n_neg = self.n_users, self.n_items, self.k, self.n_neg
        a.loss, a.reg_method = FLEXMF_LOSSES[self.loss], FLEXMF_REG_METHODS[self.reg_method]
        a.positive_weight, a.regularization = self.positive_weight, self.reg
        a.one_minus_beta1, a.beta2, a.one_minus_beta2, a.eps = 1 - _ADAM_BETA1, _ADAM_BETA2, 1 - _ADAM_BETA2, _ADAM_EPS
        for field_, name in (("u_emb", "u_embed.weight"), ("i_emb", "i_embed.weight"), ("u_bias", "u_bias.weight"),
                             ("i_bias", "i_bias.weight")):  # fmt: skip
            if name in self.params:
                m, v = self.moments[name]
                setattr(a, f"d_{field_}", ptr(self.params[name]))
                setattr(a, f"d_{field_}_m", ptr(m))
                setattr(a, f"d_{field_}_v", ptr(v))
        a.d_workspace, a.workspace_bytes = ptr(self.workspace), self.workspace.numel()
        return a

    def plan_batches(self, users: torch.Tensor, pos: torch.Tensor, neg: torch.Tensor | None = None, *,
                     ratings: torch.Tensor | None = None) -> "_FlexmfBatches":  # fmt: skip
        """
        Everything about a run of consecutive batches (``batch_size`` samples each, the last may be short) that does
        not depend on the model: the negatives (``neg`` [S, n], default this state's sampler at the current step
        count; none for MSE, which takes the targets ``ratings`` [S] instead) and the grouping of every batch's
        rows.  Made once for all the steps, so an epoch pays one sampler launch and two sorts instead of one of each
        per step.
        """
        dev, B, n = self.device, self.batch_size, self.n_neg
        users = users.to(dev, torch.int32).contiguous()
        pos = pos.to(dev, torch.int32).contiguous()
        S = users.numel()
        if self.loss == "mse":
            if neg is not None or ratings is None or ratings.numel() != S:
                raise ValueError(f"MSE batches take no negatives and {S} ratings")
            ratings = ratings.to(dev, torch.float32).contiguous()
            neg = torch.empty((S, 0), dtype=torch.int32, device=dev)
        else:
            if ratings is not None:
                raise ValueError(f"loss={self.loss!r} takes no ratings")
            neg = self.sample(users) if neg is None else neg.to(dev, torch.int32).contiguous()
        if S == 0 or pos.numel() != S or tuple(neg.shape) != (S, n):
            raise ValueError(f"expected {S} > 0 users, as many positives and negatives of shape ({S}, {n})")
        n_steps = -(-S // B)
        at = torch.arange(S, device=dev)
        step_of, local = at // B, (at % B).to(torch.int32)
        ug = _FlexmfGroups.build(step_of * self.n_users + users.long(), local, self.n_users, n_steps)
        slots = torch.cat([pos[:, None], neg], dim=1).long()
        entries = local[:, None] * (n + 1) + torch.arange(n + 1, device=dev, dtype=torch.int32)[None, :]
        ig = _FlexmfGroups.build((step_of[:, None] * self.n_items + slots).flatten(), entries.flatten(),
                                 self.n_items, n_steps)  # fmt: skip
        return _FlexmfBatches(users, pos, neg, ratings, ug, ig, n_steps)

    def run_batches(self, plan: "_FlexmfBatches") -> torch.Tensor:
        """The steps of ``plan``, four launches each; the batch losses as a device vector, not synchronised on."""
        B, n, S = self.batch_size, self.n_neg, plan.users.numel()
        if self.steps_done + plan.n_steps >= 2**31:
            raise _lib.EngineError("the optimiser step count must stay below 2**31")
        losses = torch.empty(plan.n_steps, dtype=torch.float32, device=self.device)
        a = self._step_args()
        stream = stream_ptr()
        for s in range(plan.n_steps):
            lo, hi = s * B, min(S, (s + 1) * B)
            a.batch, a.step = hi - lo, self.steps_done + 1
            for name, value in flexmf_adam_scalars(self.reg_method, self.lr, self.reg, a.step).items():
                setattr(a, name, value)
            a.d_users, a.d_pos = plan.users.data_ptr() + 4 * lo, plan.pos.data_ptr() + 4 * lo
            a.d_neg = plan.neg.data_ptr() + 4 * lo * n if n > 0 else None
            a.d_ratings = plan.ratings.data_ptr() + 4 * lo if plan.ratings is not None else None
            a.n_u_units = plan.u_groups.fill(a.u_groups, s, self.u_mark)
            a.n_i_units = plan.i_groups.fill(a.i_groups, s, self.i_mark)
            a.d_loss = losses.data_ptr() + 4 * s
            check(lib().lk_flexmf_step(C.byref(a), stream), "lk_flexmf_step")
            self.steps_done += 1
        return losses

    def train_batches(self, users: torch.Tensor, pos: torch.Tensor, neg: torch.Tensor | None = None, *,
                      ratings: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
        """``run_batches(plan_batches(...))``."""
        return self.run_batches(self.plan_batches(users, pos, neg, ratings=ratings))

    def step(self, users: torch.Tensor, pos: torch.Tensor, neg: torch.Tensor | None = None, *,
             ratings: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
        """One minibatch (at most ``batch_size`` samples); the loss as a device scalar."""
        if users.numel() > self.batch_size:
            raise ValueError(f"a step takes at most batch_size={self.batch_size} samples")
        return self.train_batches(users, pos, neg, ratings=ratings)[0]

    def epoch(self, perm: torch.Tensor) -> torch.Tensor:
        """One pass over the training interactions in the order ``perm``; the batch losses (device)."""
        perm = perm.to(self.device, torch.int64)
        ratings = None if self.ratings is None else self.ratings[perm]
        return self.train_batches(self.users[perm], self.items[perm], ratings=ratings)


# ---------------------------------------------------------------------------
# Bias model and offset scoring (BiasScorer, PopScorer)
# ---------------------------------------------------------------------------


def longest_first(indptr: torch.Tensor) -> torch.Tensor:
    """The rows of a CSR offset array longest first (int32, ties ascending)."""
    return torch.argsort(indptr[1:] - indptr[:-1], descending=True, stable=True).to(torch.int32)


def bias_learn(
    ratings: torch.Tensor, items: torch.Tensor, user_indptr: torch.Tensor, item_indptr: torch.Tensor,
    item_ratings: torch.Tensor, damping: tuple[float, float], *, item_pass: bool = True, user_pass: bool = True,
    centered_f64: bool = False,
):  # fmt: skip
    """
    ``BiasModel.learn`` on the device (``lk_bias_learn``), bit for bit with the host statements: returns the global
    mean (f32 [1]) and the item and user biases (f32 [n_items] and [n_users], or None for a pass left out).
    ``ratings`` and ``items`` are the COO arrays sorted by (user, item), ``user_indptr`` their user offsets, and
    ``item_ratings`` the ratings item-major (ascending user within an item) with offsets ``item_indptr`` (int32).
    ``damping`` is ``(user, item)``; ``centered_f64`` centres in f64 (an f64 rating matrix) instead of f32.
    """
    dev = ratings.device
    n_users, n_items = user_indptr.numel() - 1, item_indptr.numel() - 1
    a = LkBiasLearnArgs()
    a.nnz, a.n_users, a.n_items = ratings.numel(), n_users, n_items
    a.d_ratings, a.d_items = ptr(ratings), ptr(items)
    a.d_user_indptr, a.d_item_indptr, a.d_item_ratings = ptr(user_indptr), ptr(item_indptr), ptr(item_ratings)
    user_order, item_order = longest_first(user_indptr), longest_first(item_indptr)
    a.d_user_order, a.d_item_order = ptr(user_order), ptr(item_order)
    a.centered_f64 = int(centered_f64)
    a.damping_user, a.damping_item = float(damping[0]), float(damping[1])
    ws = torch.empty(int(lib().lk_bias_learn_workspace_bytes()), dtype=torch.uint8, device=dev)
    mean = torch.empty(1, dtype=torch.float32, device=dev)
    ib = torch.empty(n_items, dtype=torch.float32, device=dev) if item_pass else None
    ub = torch.empty(n_users, dtype=torch.float32, device=dev) if user_pass else None
    a.d_workspace, a.d_mean = ptr(ws), ptr(mean)
    a.d_item_bias, a.d_user_bias = ptr(_nonempty_or_none(ib)), ptr(_nonempty_or_none(ub))
    check(lib().lk_bias_learn(C.byref(a), stream_ptr()), "lk_bias_learn")
    return mean, ib, ub


def _nonempty_or_none(t: torch.Tensor | None) -> torch.Tensor | None:
    return None if t is None else _nonempty(t)


def offset_scores(
    base: torch.Tensor, n_queries: int, offset: torch.Tensor | None = None, n: int | None = None,
    excl_indptr: torch.Tensor | None = None, excl_items: torch.Tensor | None = None,
):  # fmt: skip
    """
    Scores ``s(q, i) = f32(f64(base[i]) + offset[q])`` (``lk_offset_score_batch``) for ``n_queries`` queries:
    ``base`` f32 [n_items], ``offset`` f64 [n_queries] or None for 0.  ``n=None`` (score mode) returns
    ``S [B, n_items]``.  An integer ``n`` (rank mode) returns ``(idx [B, n] int32, -1 padding; val [B, n] f32, NaN
    padding; cnt [B] int32)``: ``argtopn`` over every item minus ``excl_items[excl_indptr[q]:excl_indptr[q+1]]``
    (any order; repeats, negative and unknown numbers are ignored), ties included.
    """
    _lib.require_device()
    dev = base.device
    base = base.to(torch.float32).contiguous()
    n_items = base.numel()
    if n_items >= 2**31:
        raise _lib.EngineError("offset scoring with 2**31 or more items is not supported")
    if offset is not None:
        offset = offset.to(device=dev, dtype=torch.float64).contiguous()
        if offset.numel() != n_queries:
            raise ValueError(f"offset has {offset.numel()} entries for {n_queries} queries")
    a = LkOffsetScoreArgs()
    a.n_items, a.n_queries = n_items, n_queries
    a.d_base, a.d_offset = ptr(base), ptr(offset)
    if n is None:
        S = torch.empty((n_queries, n_items), dtype=torch.float32, device=dev)
        a.n, a.d_scores = 0, ptr(S)
        check(lib().lk_offset_score_batch(C.byref(a), stream_ptr()), "lk_offset_score_batch")
        return S
    return _rank_launch(a, lib().lk_offset_score_batch, "lk_offset_score_batch", n, n_items, n_queries, dev,
                        excl_indptr, excl_items)  # fmt: skip


# ---------------------------------------------------------------------------
# stochastic top-n (StochasticTopNRanker)
# ---------------------------------------------------------------------------

#: NumPy's PCG64 multiplier (PCG_DEFAULT_MULTIPLIER_128)
PCG64_MULT = 0x2360ED051FC65DA44385DF649FCCF645
_M64, _M128 = (1 << 64) - 1, (1 << 128) - 1
#: the bytes one split of a stochastic batch may take for its workspace, and in key mode for its key matrix
STOCHASTIC_SPLIT_BYTES = 1 << 30
_STOCH_TRANSFORMS = {None: _lib.LK_STOCH_NONE, "softmax": _lib.LK_STOCH_SOFTMAX, "linear": _lib.LK_STOCH_LINEAR}


def pcg64_jump(j: int) -> tuple[int, int]:
    """``(M^j, G_j) mod 2^128`` with ``G_j = sum(M^k for k < j)``: ``j`` PCG64 steps take a state ``s`` to
    ``M^j s + G_j inc``.  Square-and-multiply on Python ints."""
    mul, add, m, g = 1, 0, PCG64_MULT, 1
    while j:
        if j & 1:
            mul, add = (m * mul) & _M128, (m * add + g) & _M128
        m, g = (m * m) & _M128, (m * g + g) & _M128
        j >>= 1
    return mul, add


def pcg64_words(state: int, inc: int) -> list[int]:
    """A PCG64 ``(state, inc)`` as the four u64 words ``lk_stochastic_topn`` takes."""
    return [state >> 64, state & _M64, inc >> 64, inc & _M64]


def stochastic_jump_table() -> np.ndarray:
    """``lk_stochastic_topn``'s ``d_jump``: ``(M^j, G_j)`` for j = 0..32, then for j = 2^t, t = 0..63."""
    rows = [pcg64_jump(j) for j in range(33)] + [pcg64_jump(1 << t) for t in range(64)]
    return np.array([pcg64_words(m, g) for m, g in rows], dtype=np.uint64).reshape(-1)


_jump_tables: dict = {}


def _device_jump_table(dev) -> torch.Tensor:
    t = _jump_tables.get(dev)
    if t is None:
        t = _jump_tables[dev] = torch.from_numpy(stochastic_jump_table().view(np.int64)).to(dev)
    return t


def stochastic_topn(
    scores: torch.Tensor, n: int | None, *, transform: str | None, scale: float, states: np.ndarray, shared: bool,
    excl_indptr: torch.Tensor | None = None, excl_items: torch.Tensor | None = None, with_keys: bool = False,
):  # fmt: skip
    """
    Plackett–Luce top-``n`` of every row of ``scores`` [B, L] (f32, any strides: a contiguous matrix or the
    transpose of an item-major one) by exponential keys (``lk_stochastic_topn``, include/lkpy_b200.h has the
    arithmetic).  Position i of row b is valid when its score is finite and it is not among
    ``excl_items[excl_indptr[b]:excl_indptr[b+1]]`` (any order; repeats and out-of-range numbers are ignored).
    ``states`` holds PCG64 states as u64 words ``[B, 4]`` (each row its own stream) or, with ``shared``, ``[1, 4]``
    (one stream through the rows in order).

    Returns ``(idx [B, w] int32 positions, -1 padding; val [B, w] f32 scores, NaN padding; key [B, w] f64 or None;
    cnt [B] int32 list lengths; drawn)``, where ``w`` is ``n``, or ``L`` for ``n=None`` (every valid position) and
    ``drawn`` a device int64 [1] holding the draws of a shared stream.  ``n`` in 1..``lk_topn_max()`` is the rank
    mode; ``None`` and larger ``n`` take every key (key mode) and sort each row's keys on the device, truncated to
    ``n``.  Equal keys may then come out in any order, as the reference's unstable sort allows.  Batches are split
    so that each launch's workspace and keys stay within ``STOCHASTIC_SPLIT_BYTES``.
    """
    _lib.require_device()
    if scores.dtype != torch.float32 or scores.dim() != 2:
        raise TypeError("scores must be a 2-D float32 tensor")
    if transform not in _STOCH_TRANSFORMS:
        raise ValueError(f"unknown transform {transform!r}")
    tcode = _STOCH_TRANSFORMS[transform]
    dev = scores.device
    B, L = scores.shape
    if L > 2**31 - 65:
        raise _lib.EngineError("stochastic ranking of 2**31 - 64 or more positions is not supported")
    if n is not None and n < 1:
        raise ValueError("n must be positive or None")
    rank = n is not None and n <= int(lib().lk_topn_max())
    width = n if rank else (L if n is None else min(n, L))
    states = np.ascontiguousarray(states, dtype=np.uint64).reshape(-1, 4)
    if states.shape[0] != (1 if shared else B):
        raise ValueError(f"states must have {1 if shared else B} rows")
    d_states = torch.from_numpy(states.view(np.int64)).to(dev)
    drawn = torch.zeros(1, dtype=torch.int64, device=dev)
    idx = torch.full((B, width), -1, dtype=torch.int32, device=dev)
    val = torch.full((B, width), float("nan"), dtype=torch.float32, device=dev)
    key = torch.full((B, width), float("nan"), dtype=torch.float64, device=dev) if with_keys or not rank else None
    cnt = torch.zeros(max(B, 1), dtype=torch.int32, device=dev)
    if B == 0 or L == 0:
        return idx, val, key if with_keys else None, cnt[:B], drawn
    if excl_indptr is not None:
        excl_indptr, excl_items = _sorted_exclusions(excl_indptr, excl_items, L, B, dev)
    per_row = int(lib().lk_stochastic_workspace_bytes(1, L, tcode)) + (0 if rank else 8 * L)
    chunk = max(1, min(B, STOCHASTIC_SPLIT_BYTES // per_row))
    ws_bytes = int(lib().lk_stochastic_workspace_bytes(chunk, L, tcode))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    keys = None if rank else torch.empty((chunk, L), dtype=torch.float64, device=dev)
    jump = _device_jump_table(dev)
    for c0 in range(0, B, chunk):
        c1 = min(B, c0 + chunk)
        a = LkStochasticArgs()
        a.n_queries, a.n_items = c1 - c0, L
        a.d_scores, a.row_stride, a.item_stride = ptr(scores[c0:c1]), scores.stride(0), scores.stride(1)
        if excl_indptr is not None:
            a.d_excl_indptr, a.d_excl_items = ptr(excl_indptr[c0:]), ptr(excl_items)
        a.transform, a.scale, a.shared_stream = tcode, float(scale), int(shared)
        a.d_state, a.d_jump, a.d_position = ptr(d_states if shared else d_states[c0:c1]), ptr(jump), ptr(drawn)
        a.d_workspace, a.workspace_bytes = ptr(ws), ws_bytes
        a.d_out_cnt = ptr(cnt[c0:c1])
        if rank:
            a.n = n
            a.d_out_idx, a.d_out_val = ptr(idx[c0:c1]), ptr(val[c0:c1])
            a.d_out_key = ptr(key[c0:c1]) if with_keys else None
        else:
            a.n, a.d_keys = 0, ptr(keys)
        check(lib().lk_stochastic_topn(C.byref(a), stream_ptr()), "lk_stochastic_topn")
        if not rank:
            # a sort of each row's keys, invalid positions (NaN) last; the valid count cuts the row
            k = torch.nan_to_num(keys[: c1 - c0], nan=float("-inf"))
            sk, order = torch.sort(k, dim=1, descending=True)
            c = cnt[c0:c1].clamp(max=width)
            keep = torch.arange(width, device=dev)[None, :] < c[:, None]
            take = order[:, :width]
            idx[c0:c1] = torch.where(keep, take, -1).to(torch.int32)
            val[c0:c1] = torch.where(keep, scores[c0:c1].gather(1, take), float("nan"))
            key[c0:c1] = torch.where(keep, sk[:, :width], float("nan"))
            cnt[c0:c1] = c
    return idx, val, key if with_keys else None, cnt[:B], drawn


# ---------------------------------------------------------------------------
# FA*IR re-ranking (FAIRReranker)
# ---------------------------------------------------------------------------


def fair_rerank(
    m: np.ndarray, n: int, protected, *, indptr=None, lengths=None, scores: torch.Tensor | None = None,
    candidates: int | None = None, excl_indptr: torch.Tensor | None = None, excl_items: torch.Tensor | None = None,
):  # fmt: skip
    """
    The FA*IR merge (``lk_fair_rerank``; include/lkpy_b200.h states it) of a batch, to at most ``n`` entries
    (1..``lk_topn_max()``) under the minimum protected counts ``m`` (the trained ``m_list``, at least ``n`` entries).

    * Lists: ``indptr`` [B + 1] offsets into ``protected`` (one bool per position of the concatenated lists) and
      ``lengths`` [B], each list's output length (at most ``n`` and its list length).  Returns ``(idx [B, n] int32
      positions within each list, -1 padding; None; cnt [B] int32)``.
    * Scores: ``scores`` [B, n_items] f32 on the device (any strides), ``protected`` one bool per item, and
      ``candidates`` N (1..``lk_topn_max()``): each row's list is argtopn's top N, the items
      ``excl_items[excl_indptr[b]:excl_indptr[b+1]]`` (any order; repeats and out-of-range numbers are ignored)
      offered as NaN, and is merged to ``min(n, its length)``.  Returns ``(idx [B, n] int32 item numbers, -1
      padding; val [B, n] f32 scores, NaN padding; cnt [B] int32)``.
    """
    dev = _lib.require_device()
    n = _check_topn(n)
    m = np.asarray(m, dtype=np.int64)
    if m.ndim != 1 or len(m) < n:
        raise ValueError(f"m must hold at least n={n} entries")
    a = LkFairArgs()
    if scores is not None:
        if scores.dtype != torch.float32 or scores.dim() != 2:
            raise TypeError("scores must be a 2-D float32 tensor")
        if candidates is None or not 1 <= int(candidates) <= int(lib().lk_topn_max()):
            raise ValueError(f"candidates must be in 1..{int(lib().lk_topn_max())}")
        dev = scores.device
        B, L = scores.shape
        if L > 2**31 - 33:
            raise _lib.EngineError("re-ranking from 2**31 - 32 or more items is not supported")
        prot = torch.as_tensor(np.asarray(protected, dtype=bool).view(np.uint8)).to(dev)
        if prot.numel() != L:
            raise ValueError(f"protected must have one flag per item ({L})")
        a.mode, a.n_candidates, a.n_items = _lib.LK_FAIR_SCORES, int(candidates), L
        a.d_scores, a.row_stride, a.item_stride = ptr(scores), scores.stride(0), scores.stride(1)
        a.d_item_protected = ptr(prot)
        val = torch.full((B, n), float("nan"), dtype=torch.float32, device=dev)
        a.d_out_val = ptr(val)
        if excl_indptr is not None and B > 0:
            excl_indptr, excl_items = _sorted_exclusions(excl_indptr, excl_items, L, B, dev)
            a.d_excl_indptr, a.d_excl_items = ptr(excl_indptr), ptr(excl_items)
    else:
        indptr = np.asarray(indptr, dtype=np.int64)
        lengths = np.asarray(lengths, dtype=np.int32)
        flags = np.asarray(protected, dtype=bool)
        B = len(indptr) - 1
        if B < 0 or len(lengths) != B or indptr[0] != 0 or np.any(np.diff(indptr) < 0) or indptr[-1] != len(flags):
            raise ValueError("indptr must be B + 1 ascending offsets from 0 to the flag count, with B lengths")
        if np.any(np.diff(indptr) >= 2**31 - 32):
            raise _lib.EngineError("lists of 2**31 - 32 or more positions are not supported")
        if np.any(lengths < 0) or np.any(lengths > np.minimum(np.diff(indptr), n)):
            raise ValueError("each length must be in 0..min(n, its list length)")
        d_indptr = torch.from_numpy(indptr).to(dev)
        d_flags = torch.from_numpy(np.concatenate([flags.view(np.uint8), np.zeros(1, np.uint8)])).to(dev)
        d_len = torch.from_numpy(lengths).to(dev)
        a.mode, a.d_list_indptr, a.d_list_protected, a.d_list_len = _lib.LK_FAIR_LISTS, ptr(d_indptr), ptr(d_flags), ptr(d_len)
        val = None
    idx = torch.full((B, n), -1, dtype=torch.int32, device=dev)
    cnt = torch.zeros(max(B, 1), dtype=torch.int32, device=dev)
    if B == 0 or (scores is not None and scores.shape[1] == 0):
        return idx, val, cnt[:B]
    d_m = torch.from_numpy(m[:n].astype(np.int32)).to(dev)
    a.n_queries, a.n, a.d_m = B, n, ptr(d_m)
    a.d_out_idx, a.d_out_cnt = ptr(idx), ptr(cnt)
    check(lib().lk_fair_rerank(C.byref(a), stream_ptr()), "lk_fair_rerank")
    return idx, val, cnt[:B]


# ---------------------------------------------------------------------------
# ranking metrics (lkpy_b200.metrics)
# ---------------------------------------------------------------------------


def rank_metrics(specs: list[dict], rec_indptr: torch.Tensor, rec_items: torch.Tensor, test_indptr: torch.Tensor,
                 test_items: torch.Tensor, nrel: torch.Tensor, weights: np.ndarray, norms: np.ndarray) -> torch.Tensor:  # fmt: skip
    """
    ``lk_rank_metrics`` (include/lkpy_b200.h states each metric) over B lists: ``rec_indptr`` [B + 1] int64 and
    ``rec_items`` int32 (-1 for unknown items) on the device, the test sets as a device CSR of ascending unique item
    numbers, ``nrel`` [B] int64 the test lengths, and one record per metric (the keys of ``lk_metric_spec``) with
    offsets into the host f64 tables ``weights`` and ``norms``.  Returns ``out [M, B]`` f64 on the device.
    """
    dev = rec_indptr.device
    B, M = rec_indptr.numel() - 1, len(specs)
    out = torch.empty((M, max(B, 0)), dtype=torch.float64, device=dev)
    if B <= 0 or M == 0:
        return out
    d_w = torch.from_numpy(np.concatenate([np.asarray(weights, np.float64), np.zeros(1)])).to(dev)
    d_n = torch.from_numpy(np.concatenate([np.asarray(norms, np.float64), np.zeros(1)])).to(dev)
    for m0 in range(0, M, _lib.LK_RANK_METRICS_MAX):
        group = specs[m0 : m0 + _lib.LK_RANK_METRICS_MAX]
        a = LkRankMetricsArgs()
        a.n_lists, a.n_metrics = B, len(group)
        a.d_rec_indptr, a.d_rec_items = ptr(rec_indptr), ptr(rec_items)
        a.d_test_indptr, a.d_test_items, a.d_nrel = ptr(test_indptr), ptr(test_items), ptr(nrel)
        a.d_weights, a.d_norms, a.d_out = ptr(d_w), ptr(d_n), ptr(out[m0:])
        for j, sp in enumerate(group):
            for k, v in sp.items():
                setattr(a.metrics[j], k, v)
        check(lib().lk_rank_metrics(C.byref(a), stream_ptr()), "lk_rank_metrics")
    return out


def item_exposure(n_items: int, items: torch.Tensor, lists: torch.Tensor, ranks: torch.Tensor,
                  weights: np.ndarray | None) -> torch.Tensor:  # fmt: skip
    """
    ``lk_item_exposure``: the per-item totals [n_items] f64 of the entries ``items`` / ``lists`` / ``ranks`` (int32 on
    the device, in list order): 1.0 per entry when ``weights`` is None, else ``weights[rank]`` added one by one in
    entry order; of an item's entries in one list only the last counts.  The entries are sorted stably by item here.
    """
    dev = items.device
    totals = torch.zeros(n_items, dtype=torch.float64, device=dev)
    if n_items == 0:
        return totals
    sorted_items, order = torch.sort(items, stable=True)
    d_w = None if weights is None else torch.from_numpy(np.asarray(weights, np.float64)).to(dev)
    a = LkItemExposureArgs()
    a.n_items, a.n_entries = n_items, items.numel()
    a.d_sorted_items, a.d_order = ptr(sorted_items), ptr(order)
    a.d_entry_list, a.d_entry_rank = ptr(lists), ptr(ranks)
    a.d_weights, a.d_totals = ptr(d_w), ptr(totals)
    check(lib().lk_item_exposure(C.byref(a), stream_ptr()), "lk_item_exposure")
    return totals
