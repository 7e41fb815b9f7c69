"""
Drop-in surface of the reference's native accelerator module for the two hot
paths — the same function names, argument meaning and error behaviour as
``lenskit._accel.als`` / ``lenskit._accel.knn`` (stubs
``src/lenskit/_accel/als.pyi``, ``knn.pyi``) and the ``AccelTask`` protocol of
``src/lenskit/parallel/_task.py:60-100`` — executed on the H100 through the C
ABI.  A maintainer rebinding ``from lenskit._accel import als`` /
``from lenskit import _accel`` to this module gets the GPU engine under the
unchanged Python components (see INTEGRATION.md).

Host arrays in, host arrays out: ``this`` is mutated in place like the NumPy
borrow at ``implicit.rs:57-58``; device copies of the CSR operands are cached
per matrix object so that the ten half-epochs of a training run upload it once.
"""

from __future__ import annotations

import threading
from types import SimpleNamespace
from typing import Any, Callable, Generic, TypeVar

import numpy as np
import torch

from . import _lib, engine
from .data import InteractionCSR

R = TypeVar("R")
UPDATE_INTERVAL = 0.2  # parallel/_task.py:22
RESULT_CHUNK_ROWS = 1 << 16  # rows per LargeList chunk returned by compute_similarities


class AccelTask(Generic[R]):
    """
    Mirror of the Rust ``AccelTask`` pyclass (``src/accel/tasks/mod.rs:33-106``):
    ``invoke`` once, ``cancel`` and ``current_progress`` from another thread while it runs.

    Both are live: the kernels hand out work from a device counter and re-read a device cancel flag
    every time a CTA fetches work (``fetch_work``, common.cuh).  ``cancel()`` raises the flag from a
    side stream — rows / similarity rows already started finish, nothing new starts, ``invoke`` raises
    — and ``current_progress()`` copies the counter out on that side stream without disturbing the
    compute stream (the role of ``CancelAdapter``, ``implicit.rs:72-73``).
    """

    def __init__(self, fn: Callable[["AccelTask"], R], total: int | None = None):
        self._fn = fn
        self._invoked = False
        self._cancelled = threading.Event()
        self._done = False
        self._total = total
        self._flag: torch.Tensor | None = None  # device cancel flag (created when the task starts)
        self._counter: torch.Tensor | None = None  # device work counter of the running kernel
        self._units = 1  # counter ticks for the whole job
        self._side: torch.cuda.Stream | None = None

    # -- called by the task body -------------------------------------------------
    def _attach(self, counter: torch.Tensor, units: int) -> torch.Tensor:
        """Register the running kernel's work counter; returns the device cancel flag to hand to it."""
        dev = counter.device
        self._side = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(self._side):
            self._flag = torch.zeros(1, dtype=torch.int32, device=dev)
            if self._cancelled.is_set():
                self._flag.fill_(1)
        self._side.synchronize()
        self._counter, self._units = counter, max(1, int(units))
        return self._flag

    def _check_cancelled(self) -> None:
        if self._cancelled.is_set():
            raise RuntimeError("task cancelled")

    # -- the protocol --------------------------------------------------------------
    def invoke(self, *, pool: Any = None) -> R:
        if self._invoked:
            raise RuntimeError("task already invoked")  # tasks/mod.rs:64-70
        self._invoked = True
        self._check_cancelled()
        res = self._fn(self)
        self._done = True
        return res

    def cancel(self) -> None:
        self._cancelled.set()
        if self._flag is not None and self._side is not None:
            with torch.cuda.stream(self._side):
                self._flag.fill_(1)

    def current_progress(self) -> int | tuple[int, int] | None:
        if self._total is None:
            return None
        if self._done:
            return (self._total, self._total)
        if self._counter is None or self._side is None:
            return (0, self._total)
        with torch.cuda.stream(self._side):
            ticks = int(self._counter.to("cpu", non_blocking=False).item())
        return (min(self._total, self._total * min(ticks, self._units) // self._units), self._total)


def run_accel_task(task: AccelTask[R], *, progress: Any = None) -> R:
    """``lenskit.parallel.run_accel_task`` (parallel/_task.py:25-57)."""
    box: dict[str, Any] = {}
    done = threading.Event()

    def body():
        try:
            box["v"] = task.invoke(pool=None)
        except BaseException as e:  # noqa: BLE001
            box["e"] = e
        done.set()

    th = threading.Thread(target=body, name="AccelTask", daemon=False)
    th.start()
    try:
        while not done.wait(UPDATE_INTERVAL if progress is not None else None):
            cp = task.current_progress()
            if progress is not None and isinstance(cp, tuple):
                progress.update(completed=cp[0], total=cp[1])
    except KeyboardInterrupt:
        task.cancel()
        raise
    th.join()
    if "e" in box:
        raise RuntimeError("accelerator task failed with exception") from box["e"]
    return box["v"]


# ---------------------------------------------------------------------------
# operand conversion / caching
# ---------------------------------------------------------------------------


def _arrow_list_parts(arr):
    """(offsets, struct-or-index child, n_columns or None) of an Arrow List / LargeList array, following
    ``CSRMatrix::from_arrow`` (src/accel/sparse/csr.rs:160-209); extension arrays (the reference's
    ``SparseRowArray``, data/matrix.py:318-540) are unwrapped to their storage."""
    import pyarrow as pa

    ncol = None
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    if isinstance(arr, pa.ExtensionArray):
        ncol = getattr(arr.type, "dimension", None)
        arr = arr.storage
    if not (pa.types.is_list(arr.type) or pa.types.is_large_list(arr.type)):
        raise TypeError(f"expected a List or LargeList array, got {arr.type}")  # csr.rs:160-195
    if arr.null_count:
        raise TypeError("sparse rows must not be null")
    return arr, ncol


def as_host_csr(m: Any, n_cols: int | None = None) -> InteractionCSR:
    """
    Accept what the reference's entry points accept — an Arrow ``List`` / ``LargeList`` of
    ``Struct{index: int32, value: float32}`` (or of plain int32 indices: structure only), possibly
    wrapped in the ``SparseRowArray`` extension type or chunked (csr.rs:160-209) — plus this package's
    ``InteractionCSR`` and SciPy CSR matrices.  Arrow buffers are viewed, not copied, where their types
    already match (offsets, int32 indices, float32 values).
    """
    if isinstance(m, InteractionCSR):
        return m
    try:
        import pyarrow as pa
    except ImportError:  # pragma: no cover
        pa = None
    if pa is not None and isinstance(m, (pa.Array, pa.ChunkedArray)):
        arr, dim = _arrow_list_parts(m)
        off = arr.offsets.to_numpy(zero_copy_only=False)
        child = arr.values  # the flattened child, not sliced by the offsets
        if isinstance(child, pa.ExtensionArray):
            child = child.storage
        if pa.types.is_struct(child.type):
            names = [child.type.field(i).name for i in range(child.type.num_fields)]
            if "index" not in names or "value" not in names:
                raise TypeError("sparse row elements must be Struct{index, value}")
            idx, val = child.field("index"), child.field("value")
            if isinstance(idx, pa.ExtensionArray):
                dim = dim or getattr(idx.type, "dimension", None)
                idx = idx.storage
            if not pa.types.is_int32(idx.type):
                raise TypeError(f"sparse row indices must be int32, got {idx.type}")
            if not pa.types.is_float32(val.type):
                raise TypeError(f"sparse row values must be float32, got {val.type}")
            vals = val.to_numpy(zero_copy_only=False)
        elif pa.types.is_int32(child.type):
            idx, vals = child, None
        else:
            raise TypeError(f"sparse row elements must be Struct{{index,value}} or int32, got {child.type}")
        cols = idx.to_numpy(zero_copy_only=False)
        base, end = (int(off[0]), int(off[-1])) if len(off) else (0, 0)
        if base or end != len(cols):  # a slice of a longer array: its children are not sliced
            off = off - base
            cols, vals = cols[base:end], (None if vals is None else vals[base:end])
        ncol = n_cols or dim or (int(cols.max()) + 1 if len(cols) else 0)
        if vals is None:
            vals = np.ones(len(cols), dtype=np.float32)
        return InteractionCSR(np.ascontiguousarray(off), np.ascontiguousarray(cols),
                              np.ascontiguousarray(vals), (len(off) - 1, int(ncol)))  # fmt: skip
    if hasattr(m, "offsets") and hasattr(m, "indices") and hasattr(m, "values"):  # SparseRowArray-like duck type
        off = m.offsets.to_numpy(zero_copy_only=False)
        idx = m.indices.to_numpy(zero_copy_only=False)
        val = m.values.to_numpy(zero_copy_only=False)
        ncol = n_cols or getattr(m, "dimension", int(idx.max()) + 1 if len(idx) else 0)
        return InteractionCSR(
            np.ascontiguousarray(off), np.ascontiguousarray(idx, dtype=np.int32),
            np.ascontiguousarray(val, dtype=np.float32), (len(off) - 1, int(ncol)),
        )  # fmt: skip
    if hasattr(m, "indptr") and hasattr(m, "data"):
        return InteractionCSR.from_scipy(m)
    raise TypeError(f"cannot interpret {type(m).__name__} as a CSR matrix")  # csr.rs:160-195


SPARSE_IDX_EXT_NAME = "lenskit.sparse_index"  # data/matrix.py:35
_own_index_type: Any = None


def sparse_index_type(dimension: int):
    """
    The Arrow type of the ``index`` field of a sparse row: int32 storage under the reference's
    ``lenskit.sparse_index`` extension type, whose metadata carries the row dimension
    (``SparseIndexType``, data/matrix.py:104-146; the Rust consumer attaches it at
    sparse/consumer.rs:109).  ``SparseRowArray.from_array`` (knn/item.py:177) refuses a result whose index
    field is a plain int32.  Inside a process that has imported lenskit the reference's own class is used
    (it is the one its ``isinstance`` checks look for); otherwise a class with the same extension name and
    serialisation — left unregistered, so that a later ``import lenskit`` can still register its own.
    """
    import sys

    import pyarrow as pa

    ref = getattr(sys.modules.get("lenskit.data.matrix"), "SparseIndexType", None)
    if ref is not None:
        return ref(int(dimension))
    global _own_index_type
    if _own_index_type is None:
        import json

        class SparseIndexType(pa.ExtensionType):
            def __init__(self, dimension: int):
                self.dimension = int(dimension)
                super().__init__(pa.int32(), SPARSE_IDX_EXT_NAME)

            def __arrow_ext_serialize__(self) -> bytes:
                return json.dumps({"dimension": self.dimension}).encode()

            @classmethod
            def __arrow_ext_deserialize__(cls, storage_type, serialized):
                return cls(json.loads(serialized.decode())["dimension"])

        _own_index_type = SparseIndexType
    return _own_index_type(int(dimension))


def csr_to_arrow_chunks(csr: InteractionCSR, rows_per_chunk: int | None = None) -> list:
    """
    The result layout of ``compute_similarities`` (``ArrowCSRConsumer``, src/accel/sparse/consumer.rs:96-142):
    a list of ``LargeListArray<Struct{index: sparse_index(n_cols) over int32, value: float32}>`` chunks in row
    order, which the caller concatenates and wraps (``pa.chunked_array(...).combine_chunks()`` then
    ``SparseRowArray.from_array``, knn/item.py:173-177).  The struct children view the CSR's own buffers; a
    chunk re-bases its offsets.
    """
    import pyarrow as pa

    idx_type = sparse_index_type(csr.shape[1])
    fields = [pa.field("index", idx_type), pa.field("value", pa.float32())]
    n = csr.shape[0]
    step = n if not rows_per_chunk else max(1, int(rows_per_chunk))
    indptr = np.asarray(csr.indptr, dtype=np.int64)
    out = []
    for lo in range(0, max(n, 1), max(step, 1)):
        hi = min(n, lo + step)
        a, b = int(indptr[lo]), int(indptr[hi])
        elems = pa.StructArray.from_arrays(
            [
                pa.ExtensionArray.from_storage(idx_type, pa.array(csr.indices[a:b], type=pa.int32())),
                pa.array(csr.values[a:b], type=pa.float32()),
            ],
            fields=fields,
        )
        out.append(pa.LargeListArray.from_arrays(pa.array(indptr[lo : hi + 1] - a, type=pa.int64()), elems))
        if hi >= n:
            break
    return out


# device copies and plans of the host matrices the caller keeps passing in (one per epoch half):
# keyed by object identity, a few entries, oldest evicted first
_cache_keep: dict[tuple[int, str], tuple[Any, Any]] = {}
_CACHE_LIMIT = 8
# The cached plans / scorer states carry mutable device state (status word, work counter, Σ‖Δ‖²,
# contribution pool): calls into this mirror are serialised per process.  The reference's score_*
# are re-entrant on CPU threads; here concurrent callers queue on the one GPU stream anyway.
_engine_lock = threading.RLock()


def _cached(obj: Any, tag: str, make: Callable[[], Any]) -> Any:
    key = (id(obj), tag)
    with _engine_lock:
        ent = _cache_keep.get(key)
        if ent is not None and ent[0] is obj:
            return ent[1]
        val = make()
        if len(_cache_keep) >= _CACHE_LIMIT:
            _cache_keep.pop(next(iter(_cache_keep)))
        _cache_keep[key] = (obj, val)
        return val


def clear_cache() -> None:
    _cache_keep.clear()


def _check_factor(name: str, a: Any, writable: bool = False) -> np.ndarray:
    if not isinstance(a, np.ndarray) or a.dtype != np.float32 or a.ndim != 2:
        raise TypeError(f"{name} must be a 2-D float32 ndarray")
    if not a.flags.c_contiguous:
        raise TypeError(f"{name} must be C-contiguous")
    if writable and not a.flags.writeable:
        raise TypeError(f"{name} must be writable")
    return a


def _als_task(mode: int, matrix: Any, this: np.ndarray, other: np.ndarray, otor, reg: float) -> AccelTask[float]:
    this = _check_factor("this", this, writable=True)
    other = _check_factor("other", other)
    if np.shares_memory(this, other):
        raise TypeError("this and other alias")  # numpy borrow check, implicit.rs:57-64
    n_rows, k = this.shape
    csr = as_host_csr(matrix)
    if csr.shape[0] != n_rows or csr.shape[1] != other.shape[0] or other.shape[1] != k:
        raise ValueError("matrix / factor shapes do not agree")
    if otor is not None:
        otor = _check_factor("otor", otor)
        if otor.shape != (k, k):
            raise ValueError("otor must be k x k")

    def run(task: AccelTask) -> float:
        with _engine_lock:
            return run_locked(task)

    def run_locked(task: AccelTask) -> float:
        dev = _lib.require_device()
        dm = _cached(matrix, "csr", lambda: engine.DeviceCSR.from_host(csr, dev))
        # host arrays are fp32 rows: the tf32 tensor-core paths at k = 64 / 128
        chunk = {64: engine.TF32_CHUNK_NNZ, 128: engine.TF32_CHUNK_NNZ_K128}.get(k, engine.DEFAULT_CHUNK_NNZ)
        plan = _cached(matrix, f"plan{k}", lambda: engine.ALSHalfPlan.create(dm, k, chunk))
        d_this = torch.from_numpy(this).to(dev)
        d_other = torch.from_numpy(other).to(dev)
        d_otor = torch.from_numpy(otor).to(dev) if otor is not None else None
        plan.sqdelta.zero_()
        plan.status.zero_()
        # work counter ticks: groups of 4 row chunks on the tensor-core kernels, single chunks otherwise
        per_tick = 4 if (k == 64 and _lib.get_option("LK_ALS_TC") != 0 and _lib.get_option("LK_ALS_TF32") != 0) else 1
        flag = task._attach(plan.work_counter, -(-plan.n_chunks // per_tick))
        engine.als_half_epoch(plan, mode, d_this, d_other, otor=d_otor, reg=reg, cancel=flag)
        this[...] = d_this.cpu().numpy()  # rows finished before a cancel keep their new values (in place, like the reference)
        task._check_cancelled()
        st = int(plan.status.item())
        if st != 0:
            # solve.rs:99-105 → implicit.rs:79
            raise RuntimeError(f"ALS solve error: array minor of row {st - 1} is not positive")
        return float(np.sqrt(plan.sqdelta.item()))

    return AccelTask(run, total=n_rows)


def train_implicit_matrix(matrix: Any, this: np.ndarray, other: np.ndarray, otor: np.ndarray) -> AccelTask[float]:
    """``_accel.als.train_implicit_matrix`` (src/accel/als/implicit.rs:35-53)."""
    return _als_task(_lib.LK_ALS_IMPLICIT, matrix, this, other, otor, 0.0)


def train_explicit_matrix(matrix: Any, this: np.ndarray, other: np.ndarray, reg: float) -> AccelTask[float]:
    """``_accel.als.train_explicit_matrix`` (src/accel/als/explicit.rs:35-52)."""
    return _als_task(_lib.LK_ALS_EXPLICIT, matrix, this, other, None, float(reg))


def compute_similarities(
    ui_ratings: Any, iu_ratings: Any, shape: tuple[int, int], min_sim: float, save_nbrs: int | None
) -> AccelTask[list[InteractionCSR]]:
    """
    ``_accel.knn.compute_similarities`` (src/accel/knn/item_train.rs:32-93): returns, like the
    reference, a list of ``LargeListArray<Struct{index:int32, value:float32}>`` chunks in row order
    (``RESULT_CHUNK_ROWS`` rows each) for ``pa.chunked_array(...).combine_chunks()``.
    """
    nu, ni = shape
    ui = as_host_csr(ui_ratings, ni)
    iu = as_host_csr(iu_ratings, nu)
    if ui.shape != (nu, ni) or iu.shape != (ni, nu):  # asserts at item_train.rs:51-54
        raise AssertionError("matrix shapes do not match `shape`")

    def run(task: AccelTask) -> list[InteractionCSR]:
        with _engine_lock:
            return run_locked(task)

    def run_locked(task: AccelTask) -> list[InteractionCSR]:
        dev = _lib.require_device()
        d_ui = _cached(ui_ratings, "csr", lambda: engine.DeviceCSR.from_host(ui, dev))
        d_iu = _cached(iu_ratings, "csr", lambda: engine.DeviceCSR.from_host(iu, dev))
        plan = engine.KnnBuildPlan.create(d_ui, d_iu)
        truncated = save_nbrs is not None and save_nbrs > 0
        plan.cancel = task._attach(plan.work_counter, plan.units(split_hot=truncated)["n_units"])
        if truncated:
            cols, vals, cnt = plan.build_topk(min_sim, int(save_nbrs))
            indptr, c, v = engine.topk_rows_to_csr(cols, vals, cnt)
        else:
            indptr, c, v = plan.build_unbounded(min_sim)
        torch.cuda.current_stream().synchronize()
        task._check_cancelled()
        out = InteractionCSR(indptr.cpu().numpy(), c.cpu().numpy(), v.cpu().numpy(), (ni, ni))
        return csr_to_arrow_chunks(out, RESULT_CHUNK_ROWS)

    return AccelTask(run, total=ni)


def _null_to_neg(a: Any) -> np.ndarray:
    """Int32 item numbers with Arrow nulls (or masked entries) as -1."""
    if hasattr(a, "to_numpy") and hasattr(a, "null_count"):  # pyarrow
        import pyarrow.compute as pc

        return pc.fill_null(a, -1).to_numpy(zero_copy_only=False).astype(np.int32)
    return np.asarray(a, dtype=np.int32)


def _to_f32(a: Any) -> np.ndarray:
    if hasattr(a, "to_numpy") and hasattr(a, "null_count"):
        import pyarrow.compute as pc

        return pc.fill_null(a, 0.0).to_numpy(zero_copy_only=False).astype(np.float32)
    return np.asarray(a, dtype=np.float32)


def _score(sims: Any, ref_items, ref_rates, tgt_items, max_nbrs: int, min_nbrs: int):
    import pyarrow as pa

    s = as_host_csr(sims, n_cols=len(sims) if hasattr(sims, "__len__") and not hasattr(sims, "shape") else None)
    if s.shape[0] != s.shape[1]:
        raise AssertionError("similarity matrix must be square")  # item_score.rs:116
    dev = _lib.require_device()
    st = _cached(
        sims, "score", lambda: engine.KnnScorerState.create(s.shape[0], s.indptr, s.indices, s.values, dev)
    )
    ri = _null_to_neg(ref_items)
    ti = _null_to_neg(tgt_items)
    rv = None if ref_rates is None else _to_f32(ref_rates)
    i64 = torch.int64
    # (KnnScorerState.score holds the state's own lock around its mutable device scratch)
    scores, counts = st.score(
        torch.tensor([0, len(ri)], dtype=i64, device=dev),
        torch.from_numpy(ri).to(dev),
        None if rv is None else torch.from_numpy(rv).to(dev),
        torch.tensor([0, len(ti)], dtype=i64, device=dev),
        torch.from_numpy(ti).to(dev),
        max_nbrs,
        min_nbrs,
    )
    sc = scores.cpu().numpy()
    ct = counts.cpu().numpy()
    return pa.array(sc, mask=np.isnan(sc)), pa.array(ct, mask=ct < 0)


def score_explicit(sims, ref_items, ref_rates, tgt_items, max_nbrs: int, min_nbrs: int):
    """``_accel.knn.score_explicit`` (src/accel/knn/item_score.rs:22-68)."""
    return _score(sims, ref_items, ref_rates, tgt_items, max_nbrs, min_nbrs)


def score_implicit(sims, ref_items, tgt_items, max_nbrs: int, min_nbrs: int):
    """``_accel.knn.score_implicit`` (src/accel/knn/item_score.rs:71-111)."""
    return _score(sims, ref_items, None, tgt_items, max_nbrs, min_nbrs)


def _user_score(tgt_items, nbr_rows, nbr_sims, ratings, max_nbrs: int, min_nbrs: int, explicit: bool):
    import pyarrow as pa

    r = as_host_csr(ratings)
    dev = _lib.require_device()
    st = _cached(
        ratings, "uscore" + ("e" if explicit else "i"),
        lambda: engine.KnnScorerState.create(
            r.shape[1], r.indptr, r.indices, r.values if explicit else None, dev, user_mode=True
        ),
    )  # fmt: skip
    ti = _null_to_neg(tgt_items)
    # null neighbours / similarities are dropped pairwise (user_score.rs:41-44)
    ni, ns = _null_to_neg(nbr_rows), _to_f32_nan(nbr_sims)
    keep = (ni >= 0) & ~np.isnan(ns)
    ni, ns = np.ascontiguousarray(ni[keep]), np.ascontiguousarray(ns[keep])
    i64 = torch.int64
    scores, _counts = st.score(
        torch.tensor([0, len(ni)], dtype=i64, device=dev), torch.from_numpy(ni).to(dev), torch.from_numpy(ns).to(dev),
        torch.tensor([0, len(ti)], dtype=i64, device=dev), torch.from_numpy(ti).to(dev), max_nbrs, min_nbrs,
    )  # fmt: skip
    sc = scores.cpu().numpy()
    return pa.array(sc, mask=np.isnan(sc))


def _to_f32_nan(a: Any) -> np.ndarray:
    """Float32 values with Arrow nulls as NaN."""
    if hasattr(a, "to_numpy") and hasattr(a, "null_count"):
        import pyarrow.compute as pc

        return pc.fill_null(a, float("nan")).to_numpy(zero_copy_only=False).astype(np.float32)
    return np.asarray(a, dtype=np.float32)


def user_score_items_explicit(tgt_items, nbr_rows, nbr_sims, ratings, max_nbrs: int, min_nbrs: int):
    """``_accel.knn.user_score_items_explicit`` (src/accel/knn/user_score.rs:21-59)."""
    return _user_score(tgt_items, nbr_rows, nbr_sims, ratings, max_nbrs, min_nbrs, True)


def user_score_items_implicit(tgt_items, nbr_rows, nbr_sims, ratings, max_nbrs: int, min_nbrs: int):
    """``_accel.knn.user_score_items_implicit`` (src/accel/knn/user_score.rs:61-98)."""
    return _user_score(tgt_items, nbr_rows, nbr_sims, ratings, max_nbrs, min_nbrs, False)


def argtopn(scores: Any, n: int):
    """
    ``_accel.data.argtopn`` (src/accel/data/sorting.rs:131-170): indices of the ``n`` largest non-NaN
    (and non-null) scores, in the reference's order.  One vector is one thread's work for
    ``lk_topn_columns`` — this entry point exists for interface parity; batches go through
    ``argtopn_batch`` / ``ALSBase.recommend_batch``.
    """
    s = _to_f32_nan(scores)  # Arrow nulls are skipped like NaNs (`scores.is_valid(i) && accept(...)`, sorting.rs:163-167)
    idx = argtopn_batch(s[None, :], n)[0]
    if hasattr(scores, "null_count") and hasattr(scores, "to_numpy"):  # Arrow in, Arrow Int32Array out, like the reference
        import pyarrow as pa

        return pa.array(idx, type=pa.int32())
    return idx


def argtopn_batch(scores: Any, n: int) -> list[np.ndarray]:
    """``argtopn`` for every row of a host matrix ``scores`` [n_vectors, n_items] in one launch."""
    dev = _lib.require_device()
    s = np.ascontiguousarray(scores, dtype=np.float32)
    if s.ndim != 2:
        raise TypeError("scores must be 2-dimensional")
    n = int(min(n, s.shape[1]))
    if n <= 0 or s.shape[0] == 0:
        return [np.empty(0, dtype=np.int32) for _ in range(s.shape[0])]
    d = torch.from_numpy(s).to(dev).T.contiguous()  # item-major: the kernel scans a column per thread
    idx, _val, cnt = engine.topn_columns(d, n, with_values=False)
    idx, cnt = idx.cpu().numpy(), cnt.cpu().numpy()
    return [idx[b, : cnt[b]].copy() for b in range(s.shape[0])]


#: ``from lkpy_b200.accel import als, knn`` mirrors ``from lenskit._accel import als, knn``
data = SimpleNamespace(argtopn=argtopn, argtopn_batch=argtopn_batch)
als = SimpleNamespace(
    train_implicit_matrix=train_implicit_matrix, train_explicit_matrix=train_explicit_matrix
)
knn = SimpleNamespace(
    compute_similarities=compute_similarities, score_explicit=score_explicit, score_implicit=score_implicit,
    user_score_items_explicit=user_score_items_explicit, user_score_items_implicit=user_score_items_implicit,
)
