"""
CPU tests of the C-ABI library: it loads, exports every symbol the header
declares, and its host-side planning logic is right.  No device calls here.
"""

import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from lkpy_b200 import _build, _lib, data

from helpers import small_synth

ROOT = Path(__file__).resolve().parent.parent


def test_header_symbols_exported(cuda_lib):
    header = (ROOT / "include" / "lkpy_b200.h").read_text()
    declared = set(re.findall(r"LK_API\s+[\w\s\*]+?\b(lk_\w+)\s*\(", header))
    assert declared, "no declarations found"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    nm = subprocess.run(["nm", "-D", "--defined-only", str(_build.LIB)], capture_output=True, text=True, check=True)
    exported = set(re.findall(r"\bT (lk_\w+)", nm.stdout))
    assert declared <= exported, declared - exported
    assert cuda_lib.lk_version() >= 100
    assert cuda_lib.lk_als_max_features() == 128


def test_library_is_sm90a():
    _build.build()
    out = subprocess.run(["cuobjdump", "-lelf", str(_build.LIB)], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout


def test_no_fallback_without_device():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    with pytest.raises(_lib.EngineError):
        _lib.require_device()
    from lkpy_b200 import accel

    inter = small_synth(50, 40, 300, seed=3)
    ui, _ = data.als_implicit_matrices(inter)
    p = np.zeros((50, 8), np.float32)
    q = np.zeros((40, 8), np.float32)
    with pytest.raises(RuntimeError):  # the task fails loudly, nothing is computed on the host
        accel.run_accel_task(accel.als.train_implicit_matrix(ui, p, q, np.eye(8, dtype=np.float32)))


@pytest.mark.parametrize("chunk", [32, 64, 4096])
def test_als_plan_covers_every_nonzero_once(cuda_lib, chunk):
    inter = small_synth(3000, 500, 80000, seed=8)
    _ui, iu = data.als_implicit_matrices(inter)
    hp = iu.indptr
    nc, ns, nslot = C.c_int64(), C.c_int64(), C.c_int64()
    _lib.check(cuda_lib.lk_als_plan_size(hp.ctypes.data, iu.shape[0], chunk, C.byref(nc), C.byref(ns), C.byref(nslot)))
    ch = np.empty((nc.value, 8), dtype=np.int32)
    _lib.check(cuda_lib.lk_als_plan_fill(hp.ctypes.data, iu.shape[0], chunk, ch.ctypes.data))
    row, begin, ln, parts, slot0, part, split = (ch[:, i] for i in range(7))
    assert ln.max() <= max(chunk, 32) and ln.min() >= 0
    cover = np.zeros(iu.nnz, dtype=np.int32)
    for b, l in zip(begin, ln):
        cover[b : b + l] += 1
    assert np.all(cover == 1)
    assert np.all(begin >= hp[row]) and np.all(begin + ln <= hp[row + 1])
    nnz_row = np.diff(hp)
    # every row appears; split rows have consistent part numbering and disjoint slots
    assert set(row.tolist()) == set(range(iu.shape[0]))
    whole = parts == 1
    assert np.all(ln[whole] == nnz_row[row[whole]])
    sp = ~whole
    assert len(set(split[sp].tolist())) == ns.value
    slots = slot0[sp] + part[sp]
    assert len(set(slots.tolist())) == nslot.value == sp.sum()
    # longest rows first
    first_of_row = {}
    for i, r in enumerate(row):
        first_of_row.setdefault(int(r), i)
    order = sorted(first_of_row, key=first_of_row.get)
    assert np.all(np.diff(nnz_row[order]) <= 0)
    with pytest.raises(_lib.EngineError):
        _lib.check(cuda_lib.lk_als_plan_size(hp.ctypes.data, iu.shape[0], 8, C.byref(nc), C.byref(ns), C.byref(nslot)))


def test_knn_geometry(cuda_lib, lk_options):
    g = _lib.LkKnnGeom()
    for n_items in (4, 9066, 59047, 500_000):
        _lib.check(cuda_lib.lk_knn_geometry(1000, n_items, C.byref(g)))
        assert g.warps * g.tile_cols * g.n_halves >= n_items
        assert g.tile_cols % 32 == 0 and g.n_subtiles == g.n_halves * g.warps
        assert g.smem_bytes * g.ctas_per_sm <= 227 * 1024
    lk_options("LK_KNN_WARPS", 7)
    assert cuda_lib.lk_knn_geometry(10, 10, C.byref(g)) == _lib.LK_OK - 1
    assert b"LK_KNN_WARPS" in cuda_lib.lk_last_error()
    assert cuda_lib.lk_set_option(b"LK_NO_SUCH_SWITCH", 1) != _lib.LK_OK


def test_component_configs():
    from lkpy_b200.als import BiasedMFScorer, ImplicitMFScorer
    from lkpy_b200.knn import ItemKNNConfig, ItemKNNScorer

    m = ItemKNNScorer(k=30)
    cfg = m.dump_config()
    assert cfg["feedback"] == "explicit" and cfg["max_nbrs"] == 30  # test_knn_item_item.py:98-103
    assert ItemKNNConfig(nnbrs=5).max_nbrs == 5
    assert ItemKNNConfig(min_sim=1e-320).min_sim == float(np.finfo(np.float64).smallest_normal)
    with pytest.raises(Exception):
        ItemKNNConfig(bogus=1)
    a = ImplicitMFScorer(features=32, regularization=(0.1, 0.2))
    assert a.config.embedding_size == 32 and a.config.user_reg == 0.1 and a.config.item_reg == 0.2
    assert a.config.weight == 40 and not a.config.use_ratings
    assert BiasedMFScorer().config.damping == 5.0 and not a.is_trained()
