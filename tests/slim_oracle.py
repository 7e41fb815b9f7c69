"""
The SLIM restatements the tests compare against: ``train`` runs ``slim_oracle.c`` (compiled on first use into a
temporary directory with ``-O2 -ffp-contract=off -fopenmp``, OpenMP over the columns), ``score`` restates
``SLIMScorer.__call__``'s ``x @ weights`` (a 0/1 row of the known history items in query order, repeats kept).
"""

from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import scipy.sparse as sps

SRC = Path(__file__).resolve().parent / "slim_oracle.c"
_lib = None


def _compiler() -> str:
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or shutil.which("cc"))
    if not cc:
        raise RuntimeError("a C compiler is needed for the SLIM restatement")
    return cc


def lib():
    global _lib
    if _lib is None:
        src = SRC.read_bytes()
        out = Path(tempfile.gettempdir()) / f"lkpy_slim_oracle_{os.getuid()}_{hashlib.sha256(src).hexdigest()[:16]}.so"
        if not out.exists():
            tmp = out.with_suffix(f".{os.getpid()}.tmp")
            subprocess.run([_compiler(), "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared", "-o", str(tmp),
                            str(SRC), "-lm"], check=True)  # fmt: skip
            os.replace(tmp, out)
        L = C.CDLL(str(out))
        vp = C.c_void_p
        L.slim_train.restype = vp
        L.slim_train.argtypes = [C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_float, C.c_float, C.c_int32, C.c_int64,
                                 vp, C.c_int32]  # fmt: skip
        for name in ("slim_counts", "slim_fetch", "slim_free"):
            getattr(L, name).restype = None
        L.slim_counts.argtypes = [vp, vp]
        L.slim_fetch.argtypes = [vp, vp, vp]
        L.slim_free.argtypes = [vp]
        _lib = L
    return _lib


def structure(n_rows: int, rows: np.ndarray, cols: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """CSR structure (int64 offsets, int32 indices) of (row, col) pairs, keeping their order inside each row."""
    o = np.argsort(rows, kind="stable")
    ip = np.zeros(n_rows + 1, np.int64)
    np.cumsum(np.bincount(rows, minlength=n_rows), out=ip[1:])
    return ip, np.ascontiguousarray(cols[o], dtype=np.int32)


def train(n_users: int, n_items: int, ui, iu, l1: float, l2: float, max_iters: int, max_nbrs: int | None,
          columns=None) -> sps.csr_array:  # fmt: skip
    """The weight rows (row i = the weight column of target item i) of ``columns`` (all items by default) as a
    SciPy CSR with f32 values; ``ui`` / ``iu`` are (offsets, indices) pairs walked in stored order."""
    L = lib()
    ui_p, ui_c = (np.ascontiguousarray(a, dtype=t) for a, t in zip(ui, (np.int64, np.int32)))
    iu_p, iu_c = (np.ascontiguousarray(a, dtype=t) for a, t in zip(iu, (np.int64, np.int32)))
    cols = np.arange(n_items, dtype=np.int32) if columns is None else np.unique(np.asarray(columns, np.int32))
    k = -1 if max_nbrs is None or max_nbrs >= n_items else int(max_nbrs)
    h = L.slim_train(n_users, n_items, ui_p.ctypes.data, ui_c.ctypes.data, iu_p.ctypes.data, iu_c.ctypes.data,
                     float(np.float32(l1)), float(np.float32(l2)), int(max_iters), k, cols.ctypes.data, len(cols))  # fmt: skip
    try:
        cnt = np.zeros(len(cols), np.int64)
        L.slim_counts(h, cnt.ctypes.data)
        items = np.zeros(max(int(cnt.sum()), 1), np.int32)
        vals = np.zeros(max(int(cnt.sum()), 1), np.float32)
        L.slim_fetch(h, items.ctypes.data, vals.ctypes.data)
    finally:
        L.slim_free(h)
    row_len = np.zeros(n_items, np.int64)
    row_len[cols] = cnt
    indptr = np.concatenate([[0], np.cumsum(row_len)]).astype(np.int64)
    nnz = int(indptr[-1])
    return sps.csr_array((vals[:nnz], items[:nnz], indptr), shape=(n_items, n_items))


def score(weights_t: sps.csr_array, hist: np.ndarray) -> np.ndarray:
    """``x @ weights`` for one query: the f32 sum of the rows of ``weights_t`` (history items on rows) of the known
    history items ``hist``, in query order from +0.0."""
    s = np.zeros(weights_t.shape[1], np.float32)
    for r in np.asarray(hist, dtype=np.int64):
        lo, hi = weights_t.indptr[r], weights_t.indptr[r + 1]
        s[weights_t.indices[lo:hi]] += weights_t.data[lo:hi]
    return s
