"""
ctypes binding of the C ABI declared in ``include/lkpy_b200.h``.

Loading fails loudly: there is no CPU or PyTorch fallback behind these entry
points.  ``lib()`` needs the built ``.so`` (``python -m lkpy_b200._build``);
``require_device()`` additionally needs a CUDA device.
"""

from __future__ import annotations

import ctypes as C
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "csrc" / "liblkpy_b200.so"

LK_OK = 0
LK_DTYPE_F32, LK_DTYPE_BF16 = 0, 1
LK_ALS_IMPLICIT, LK_ALS_EXPLICIT = 0, 1
LK_MAX_REPLICAS = 8

i32p = C.POINTER(C.c_int32)
i64p = C.POINTER(C.c_int64)
f32p = C.POINTER(C.c_float)
f64p = C.POINTER(C.c_double)
u64p = C.POINTER(C.c_uint64)
vp = C.c_void_p


class EngineError(RuntimeError):
    """An error reported by the CUDA library."""


class LkAlsArgs(C.Structure):
    _fields_ = [
        ("mode", C.c_int32),
        ("k", C.c_int32),
        ("n_rows", C.c_int64),
        ("n_other", C.c_int64),
        ("d_indptr", vp),
        ("d_cols", vp),
        ("d_vals", vp),
        ("d_this", vp),
        ("d_other", vp),
        ("other_dtype", C.c_int32),
        ("n_replicas", C.c_int32),
        ("d_replicas", vp * LK_MAX_REPLICAS),
        ("replica_row0", C.c_int64),
        ("d_otor", vp),
        ("reg", C.c_float),
        ("d_chunks", vp),
        ("n_chunks", C.c_int64),
        ("d_partials", vp),
        ("d_split_counters", vp),
        ("n_split_rows", C.c_int64),
        ("d_work_counter", vp),
        ("d_sqdelta", vp),
        ("d_status", vp),
        ("vals_uniform", C.c_int32),
        ("uniform_val", C.c_float),
        ("d_prof", vp),
        ("d_cancel", vp),
    ]


class LkKnnGeom(C.Structure):
    _fields_ = [
        ("n_users", C.c_int32),
        ("n_items", C.c_int32),
        ("warps", C.c_int32),
        ("tile_cols", C.c_int32),
        ("n_halves", C.c_int32),
        ("n_subtiles", C.c_int32),
        ("smem_bytes", C.c_int32),
        ("ctas_per_sm", C.c_int32),
    ]


class LkKnnBuildArgs(C.Structure):
    _fields_ = [
        ("geom", LkKnnGeom),
        ("d_ui_indptr", vp),
        ("d_ui_cols", vp),
        ("d_ui_vals", vp),
        ("d_iu_indptr", vp),
        ("d_iu_cols", vp),
        ("d_iu_vals", vp),
        ("d_tile_ptr", vp),
        ("d_units", vp),
        ("d_unit_ptr", vp),
        ("max_units_per_item", C.c_int32),
        ("d_sched", vp),
        ("n_work", C.c_int64),
        ("min_sim", C.c_float),
        ("save_nbrs", C.c_int32),
        ("d_part_cols", vp),
        ("d_part_vals", vp),
        ("d_part_cnt", vp),
        ("d_pool_cols", vp),
        ("d_pool_vals", vp),
        ("pool_capacity", C.c_int64),
        ("d_pool_off", vp),
        ("d_pool_cursor", vp),
        ("d_tie_scratch", vp),
        ("d_work_counter", vp),
        ("d_status", vp),
        ("d_cancel", vp),
    ]


class LkKnnScoreArgs(C.Structure):
    _fields_ = [
        ("n_items", C.c_int32),
        ("d_sim_indptr", vp),
        ("d_sim_cols", vp),
        ("d_sim_vals", vp),
        ("n_queries", C.c_int32),
        ("d_ref_indptr", vp),
        ("d_ref_items", vp),
        ("d_ref_vals", vp),
        ("d_tgt_indptr", vp),
        ("d_tgt_items", vp),
        ("max_nbrs", C.c_int32),
        ("min_nbrs", C.c_int32),
        ("d_slotmap", vp),
        ("slotmap_warps", C.c_int64),
        ("d_acc_ws", vp),
        ("d_acc_tw", vp),
        ("d_acc_cnt", vp),
        ("d_scores", vp),
        ("d_counts", vp),
        ("d_work_counter", vp),
        ("d_status", vp),
        ("d_heap_scratch", vp),
        ("heap_floats_per_warp", C.c_int64),
        ("d_pool", vp),
        ("pool_entries", C.c_int64),
        ("d_pool_cursor", vp),
        ("user_mode", C.c_int32),
        ("n_matrix_rows", C.c_int32),
        ("d_deferred", vp),
        ("d_n_deferred", vp),
    ]


#: every symbol ``include/lkpy_b200.h`` declares: name -> (restype, argtypes)
SYMBOLS: dict[str, tuple] = {
    "lk_version": (C.c_int, []),
    "lk_last_error": (C.c_char_p, []),
    "lk_device_info": (C.c_int, [C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "lk_set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "lk_get_option": (C.c_int, [C.c_char_p, C.POINTER(C.c_int)]),
    "lk_als_max_features": (C.c_int, []),
    "lk_als_plan_size": (C.c_int, [vp, C.c_int64, C.c_int32, i64p, i64p, i64p]),
    "lk_als_plan_fill": (C.c_int, [vp, C.c_int64, C.c_int32, vp]),
    "lk_als_slot_floats": (C.c_int64, [C.c_int32]),
    "lk_als_half_epoch": (C.c_int, [C.POINTER(LkAlsArgs), vp]),
    "lk_als_otor_scratch_floats": (C.c_int64, [C.c_int32]),
    "lk_als_otor": (C.c_int, [vp, C.c_int64, C.c_int32, C.c_float, vp, vp, vp, vp]),
    "lk_knn_geometry": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(LkKnnGeom)]),
    "lk_knn_tile_pointers": (C.c_int, [C.POINTER(LkKnnGeom), vp, vp, vp, vp]),
    "lk_knn_row_cost": (C.c_int, [C.POINTER(LkKnnGeom), vp, vp, vp, vp, vp]),
    "lk_knn_tie_scratch_ints": (C.c_int64, [C.POINTER(LkKnnGeom)]),
    "lk_knn_build": (C.c_int, [C.POINTER(LkKnnBuildArgs), vp]),
    "lk_knn_merge_topk": (C.c_int, [C.POINTER(LkKnnBuildArgs), vp, vp, vp, vp]),
    "lk_knn_pool_to_csr": (C.c_int, [C.POINTER(LkKnnBuildArgs), vp, vp, vp, vp]),
    "lk_knn_prep_columns": (C.c_int, [vp, vp, C.c_int32, C.c_int32, vp, vp, vp]),
    "lk_knn_score_warps": (C.c_int64, []),
    "lk_knn_score_dense_ctas": (C.c_int64, []),
    "lk_knn_score_batch": (C.c_int, [C.POINTER(LkKnnScoreArgs), vp]),
    "lk_topn_max": (C.c_int, []),
    "lk_topn_columns": (C.c_int, [vp, C.c_int64, C.c_int64, C.c_int64, C.c_int32, vp, vp, vp, vp]),
}

_lib = None


def lib():
    """Load the CUDA library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise EngineError(
                f"{LIB_PATH} is missing: build it with `python -m lkpy_b200._build` "
                "(there is no CPU fallback for the lkpy_b200 engines)"
            )
        L = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def set_option(name: str, value: int) -> None:
    """Switch a diagnostic kernel variant (``lk_set_option``; the LK_* environment is read once at load)."""
    check(lib().lk_set_option(name.encode(), int(value)), "lk_set_option")


def get_option(name: str) -> int:
    v = C.c_int()
    check(lib().lk_get_option(name.encode(), C.byref(v)), "lk_get_option")
    return int(v.value)


def check(rc: int, what: str = "") -> None:
    if rc != LK_OK:
        msg = lib().lk_last_error().decode("utf-8", "replace")
        raise EngineError(f"{what or 'lkpy_b200'} failed (code {rc}): {msg}")


def require_device():
    """The torch CUDA device the engines run on; raises without one."""
    import torch

    if not torch.cuda.is_available():
        raise EngineError(
            "lkpy_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback"
        )
    return torch.device("cuda", torch.cuda.current_device())


def ptr(t) -> int | None:
    """Device (or host) address of a torch tensor / NumPy array, None for None."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data


def stream_ptr() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream
