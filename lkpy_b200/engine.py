"""
Device-side engine: torch tensors in, C-ABI calls out.

PyTorch is used for device memory, streams and (in ``lkpy_b200.parallel``)
``torch.distributed`` only.  Every compute step is a call into
``liblkpy_b200.so``; nothing here falls back to torch math.
"""

from __future__ import annotations

import ctypes as C
import threading
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from ._lib import LkAlsArgs, LkKnnBuildArgs, LkKnnGeom, LkKnnScoreArgs, check, lib, ptr, stream_ptr
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
#: optional int64[8] device tensor receiving per-phase cycle counters of the ALS kernels (diagnostics)
PROF_BUFFER = None


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
    a.d_prof = ptr(PROF_BUFFER)
    a.d_cancel = ptr(cancel)  # optional device flag: non-zero stops the hand-out of rows (cooperative cancel)
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
        capacity = max(capacity, 1)
        pool_cols = torch.empty(capacity, dtype=torch.int32, device=dev)
        pool_vals = torch.empty(capacity, dtype=torch.float32, device=dev)
        pool_off = torch.zeros(n_items * H, dtype=torch.int64, device=dev)
        part_cnt = torch.zeros(n_items * H, dtype=torch.int32, device=dev)
        cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        self.status.zero_()
        a = self._args(u, sched, min_sim, 0)
        a.d_part_cnt = ptr(part_cnt)
        a.d_pool_cols, a.d_pool_vals, a.pool_capacity = ptr(pool_cols), ptr(pool_vals), capacity
        a.d_pool_off, a.d_pool_cursor = ptr(pool_off), ptr(cursor)
        check(L.lk_knn_build(C.byref(a), stream_ptr()), "lk_knn_build")
        if int(self.status.item()) == 1:
            raise _lib.EngineError("similarity pool overflow; pass a larger capacity")
        counts = part_cnt.view(n_items, H).sum(dim=1, dtype=torch.int64)
        indptr = torch.zeros(n_items + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=indptr[1:])
        nnz = int(indptr[-1].item())
        out_cols = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
        out_vals = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
        check(
            L.lk_knn_pool_to_csr(C.byref(a), ptr(indptr), ptr(out_cols), ptr(out_vals), stream_ptr()),
            "lk_knn_pool_to_csr",
        )
        torch.cuda.current_stream().synchronize()
        return indptr, out_cols[:nnz], out_vals[:nnz]


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
    heap_scratch: dict = field(default_factory=dict)  # (max_nbrs, warps) -> per-warp heap states
    lock: object = field(default_factory=threading.Lock)  # the mutable device state above is per-state
    #: user-kNN scoring (user_score.rs:21-98): the matrix is users x items ratings, a query's "history" is its
    #: neighbour list and carries the weights (lk_knn_score_args.user_mode)
    user_mode: bool = False
    n_rows: int = 0
    HEAP_TARGETS_PER_WARP = 2048
    USE_LISTS = True  # list-based kernel (parallel over the history); False: the sequential kernel
    #: dense kernel: batches of at least this many queries are handed out longest history first.  Off by default:
    #: measured 3.0 vs 2.7 ms per 4,096 ML-25M-shaped users (the heaviest queries, started together, contend for
    #: L2), and a random position costs a wide batch less than that (tools/score_prof.py toggles it)
    DENSE_LPT_MIN_QUERIES = 1 << 30

    def kernel_name(self) -> str:
        lists = self.USE_LISTS and _lib.get_option("LK_KNN_SCORE_SEQ") != 1
        return "knn_score_lists_kernel" if lists else "knn_score_kernel"

    def _slotmap(self, n_queries: int) -> tuple[torch.Tensor, int]:
        """One slot-map row per working warp: min(n_queries, full grid) rows (a single query takes
        n_items * 4 B, not grid * n_items * 4 B)."""
        warps = max(1, min(int(n_queries), self.max_warps))
        if self.slotmap is None or self.slotmap.shape[0] < warps:
            self.slotmap = None
            self.slotmap = torch.full((warps, self.n_items), -1, dtype=torch.int32, device=self.sim_cols.device)
        return self.slotmap, int(self.slotmap.shape[0])

    def _heap(self, max_nbrs: int, warps: int) -> tuple[torch.Tensor, int]:
        """Heap states of the sequential kernel (only allocated when that kernel will run)."""
        per_warp = self.HEAP_TARGETS_PER_WARP * (2 + 2 * (int(max_nbrs) + 1))
        key = int(max_nbrs)
        t = self.heap_scratch.get(key)
        if t is None or t.numel() < warps * per_warp:
            t = torch.empty(warps * per_warp, dtype=torch.float32, device=self.sim_cols.device)
            self.heap_scratch[key] = t
        return t, per_warp

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
        if not 1 <= int(max_nbrs) <= KNN_SCORE_MAX_NBRS:
            raise ValueError(f"max_nbrs must be in 1..{KNN_SCORE_MAX_NBRS}")
        with self.lock:  # status word, work counter, pool and slot maps are shared by the callers of one state
            return self._score_locked(ref_indptr, ref_items, ref_vals, tgt_indptr, tgt_items, max_nbrs, min_nbrs)

    def _pool_for(self, ref_items: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """Contribution pool: one 16-byte entry per (history entry, matrix-row entry) pair of the batch."""
        dev = self.sim_cols.device
        n_rows = self.n_rows if self.user_mode else self.n_items
        r = ref_items.long()
        ok = (r >= 0) & (r < n_rows)
        rr = r.clamp(0, n_rows - 1)
        total = int(((self.sim_indptr[rr + 1] - self.sim_indptr[rr]) * ok).sum().item())
        pool = self.heap_scratch.get("pool")
        if pool is None or pool.numel() < 4 * max(total, 1):
            pool = torch.empty(4 * max(total, 1), dtype=torch.int32, device=dev)
            self.heap_scratch["pool"] = pool
            self.heap_scratch["pool_cursor"] = torch.zeros(1, dtype=torch.int64, device=dev)
        return pool, self.heap_scratch["pool_cursor"]

    def score_all_items(
        self, ref_indptr: torch.Tensor, ref_items: torch.Tensor, ref_vals: torch.Tensor | None, max_nbrs: int, min_nbrs: int
    ) -> tuple[torch.Tensor, torch.Tensor]:
        """
        Score every query against ALL items (the batch runner's case): returns (scores [n_queries, n_items]
        with NaN nulls, counts [n_queries, n_items]).  Runs ``knn_score_dense_kernel`` — a CTA per query,
        cost proportional to the contributions plus one streaming fill of the output.
        """
        if not 1 <= int(max_nbrs) <= KNN_SCORE_MAX_NBRS:
            raise ValueError(f"max_nbrs must be in 1..{KNN_SCORE_MAX_NBRS}")
        with self.lock:
            dev = self.sim_cols.device
            nq, ni = ref_indptr.numel() - 1, self.n_items
            scores = torch.empty((nq, ni), dtype=torch.float32, device=dev)
            counts = torch.empty((nq, ni), dtype=torch.int32, device=dev)
            ctas = int(lib().lk_knn_score_dense_ctas())
            # per-CTA state of the dense kernel: a slot map (item -> touched-target number; zero between queries
            # and between launches) and two compact rows indexed by touched-target number
            ws = self.heap_scratch.get("dense_ws")
            if ws is None:
                ws = self.heap_scratch["dense_ws"] = (
                    torch.empty(ctas * ni, dtype=torch.int32, device=dev), torch.empty(ctas * ni, dtype=torch.int32, device=dev),
                    torch.zeros(ctas * ni, dtype=torch.int32, device=dev),
                )  # fmt: skip
            off, cur, spill = ws
            self.status.zero_()
            pool, cursor = self._pool_for(ref_items)
            a = LkKnnScoreArgs()
            a.n_items = ni
            a.d_sim_indptr, a.d_sim_cols, a.d_sim_vals = ptr(self.sim_indptr), ptr(self.sim_cols), ptr(self.sim_vals)
            a.n_queries = nq
            a.d_ref_indptr, a.d_ref_items, a.d_ref_vals = ptr(ref_indptr), ptr(ref_items), ptr(ref_vals)
            a.max_nbrs, a.min_nbrs = int(max_nbrs), int(min_nbrs)
            a.d_acc_ws, a.d_acc_tw = ptr(off), ptr(cur)
            a.d_scores, a.d_counts = ptr(scores), ptr(counts)
            a.d_work_counter, a.d_status = ptr(self.work_counter), ptr(self.status)
            a.user_mode, a.n_matrix_rows = (1 if self.user_mode else 0), self.n_rows
            a.d_pool, a.pool_entries, a.d_pool_cursor = ptr(pool), pool.numel() // 4, ptr(cursor)
            a.d_slotmap, a.slotmap_warps = ptr(spill), ctas  # per-CTA slot maps (all zero between launches)
            order = None
            if nq >= self.DENSE_LPT_MIN_QUERIES:
                # longest histories first: a query costs what its history contributes, and the launch ends with
                # its last query
                order = torch.argsort(ref_indptr[1:] - ref_indptr[:-1], descending=True).to(torch.int32)
                a.d_deferred = ptr(order)
            check(lib().lk_knn_score_batch(C.byref(a), stream_ptr()), "lk_knn_score_batch")
            torch.cuda.current_stream().synchronize()
            st = int(self.status.item())
            if st == 2:
                raise ValueError("similarity is null")
            if st == 3:
                raise _lib.EngineError("lk_knn_score_batch: contribution pool too small")
        return scores, counts

    def _score_locked(self, ref_indptr, ref_items, ref_vals, tgt_indptr, tgt_items, max_nbrs, min_nbrs):
        dev = self.sim_cols.device
        nq = ref_indptr.numel() - 1
        nt = tgt_items.numel()
        scores = torch.empty(max(nt, 1), dtype=torch.float32, device=dev)
        counts = torch.empty(max(nt, 1), dtype=torch.int32, device=dev)
        acc_ws = torch.empty(max(nt, 1), dtype=torch.float32, device=dev)
        acc_tw = torch.empty(max(nt, 1), dtype=torch.float32, device=dev)
        acc_cnt = torch.empty(max(nt, 1), dtype=torch.int32, device=dev)
        self.status.zero_()
        slotmap, warps = self._slotmap(nq)
        a = LkKnnScoreArgs()
        a.n_items = self.n_items
        a.d_sim_indptr, a.d_sim_cols, a.d_sim_vals = ptr(self.sim_indptr), ptr(self.sim_cols), ptr(self.sim_vals)
        a.n_queries = nq
        a.d_ref_indptr, a.d_ref_items, a.d_ref_vals = ptr(ref_indptr), ptr(ref_items), ptr(ref_vals)
        a.d_tgt_indptr, a.d_tgt_items = ptr(tgt_indptr), ptr(tgt_items)
        a.max_nbrs, a.min_nbrs = int(max_nbrs), int(min_nbrs)
        a.d_slotmap, a.slotmap_warps = ptr(slotmap), warps
        a.d_acc_ws, a.d_acc_tw, a.d_acc_cnt = ptr(acc_ws), ptr(acc_tw), ptr(acc_cnt)
        a.d_scores, a.d_counts = ptr(scores), ptr(counts)
        a.d_work_counter, a.d_status = ptr(self.work_counter), ptr(self.status)
        a.user_mode, a.n_matrix_rows = (1 if self.user_mode else 0), self.n_rows
        use_lists = self.USE_LISTS and ref_items.numel() > 0 and _lib.get_option("LK_KNN_SCORE_SEQ") != 1
        if use_lists:
            # contribution pool for the list-based kernel: one 16-byte entry per (reference item,
            # similarity-row entry) pair of the batch
            pool, cursor = self._pool_for(ref_items)
            a.d_pool, a.pool_entries = ptr(pool), pool.numel() // 4
            a.d_pool_cursor = ptr(cursor)
        else:
            # the sequential kernel is the one that reads the per-warp heap states
            heap, per_warp = self._heap(max_nbrs, warps)
            a.d_heap_scratch, a.heap_floats_per_warp = ptr(heap), per_warp
        check(lib().lk_knn_score_batch(C.byref(a), stream_ptr()), "lk_knn_score_batch")
        # keep scratch alive until the stream has consumed it
        torch.cuda.current_stream().synchronize()
        st = int(self.status.item())
        if st == 2:
            raise ValueError("similarity is null")
        if st == 3:
            raise _lib.EngineError("lk_knn_score_batch: contribution pool too small")
        return scores[:nt], counts[:nt]


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
    n = int(n)
    if not 1 <= n <= int(lib().lk_topn_max()):
        raise ValueError(f"n must be in 1..{int(lib().lk_topn_max())}")
    dev = scores.device
    idx = torch.empty((n_cols, n), dtype=torch.int32, device=dev)
    val = torch.empty((n_cols, n), dtype=torch.float32, device=dev) if with_values else None
    cnt = torch.empty((max(n_cols, 1),), dtype=torch.int32, device=dev)
    check(
        lib().lk_topn_columns(
            ptr(scores), n_rows, n_cols, scores.stride(0) if n_rows > 1 else max(n_cols, 1), n,
            ptr(idx), ptr(val), ptr(cnt), stream_ptr(),
        ),
        "lk_topn_columns",
    )  # fmt: skip
    return idx, val, cnt[:n_cols]
