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
    assert cuda_lib.lk_version() >= 101
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


def _boundary_lengths(chunk: int) -> list[int]:
    """Row lengths where the ALS kernels change behaviour (32-row stages, 16 / 8-row MMA steps, part cuts)."""
    base = [0, 1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 481]
    return base + [chunk - 1, chunk, chunk + 1, 2 * chunk, 2 * chunk + 1, 3 * chunk - 1, 40 * chunk + 1]


@pytest.mark.parametrize("chunk", [32, 64, 96, 256, 1024, 4096])
def test_als_plan_covers_every_nonzero_once(cuda_lib, chunk):
    inter = small_synth(3000, 500, 80000, seed=8)
    _ui, iu = data.als_implicit_matrices(inter)
    _check_plan(cuda_lib, iu.indptr, chunk)


@pytest.mark.parametrize("chunk", [32, 64, 96, 256, 1024, 4096])
def test_als_plan_boundary_lengths(cuda_lib, chunk):
    """The same plan checks on rows of the lengths where the kernels change behaviour: every boundary length of
    every chunk size under test (so each plan also sees the others' cut points), then this chunk size's own."""
    lens = sorted({n for c in (32, 33, 40, 48, 50, 64, 96, 100, 256, 1024) for n in _boundary_lengths(c)})
    lens += _boundary_lengths(chunk)
    _check_plan(cuda_lib, np.concatenate([[0], np.cumsum(lens)]).astype(np.int32), chunk)


def _check_plan(cuda_lib, hp, chunk):
    n_rows = len(hp) - 1
    nnz = int(hp[-1])
    nc, ns, nslot = C.c_int64(), C.c_int64(), C.c_int64()
    _lib.check(cuda_lib.lk_als_plan_size(hp.ctypes.data, n_rows, chunk, C.byref(nc), C.byref(ns), C.byref(nslot)))
    ch = np.empty((nc.value, 8), dtype=np.int32)
    _lib.check(cuda_lib.lk_als_plan_fill(hp.ctypes.data, n_rows, chunk, ch.ctypes.data))
    row, begin, ln, parts, slot0, part, split = (ch[:, i] for i in range(7))
    assert ln.max() <= chunk
    # every part of a split row holds 1 .. chunk nonzeros, and a row has exactly ceil(n / chunk) parts
    assert np.all(ln[parts > 1] >= 1)
    assert np.all(parts == np.maximum(1, -(-np.diff(hp)[row] // chunk)))
    np.testing.assert_array_equal(np.bincount(row, minlength=n_rows)[row], parts)
    cover = np.zeros(nnz, dtype=np.int32)
    for b, l in zip(begin, ln):
        cover[b : b + l] += 1
    assert np.all(cover == 1)
    assert np.all(begin >= hp[row]) and np.all(begin + ln <= hp[row + 1])
    nnz_row = np.diff(hp)
    # every row appears; split rows have consistent part numbering and disjoint slots
    assert set(row.tolist()) == set(range(n_rows))
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
        _lib.check(cuda_lib.lk_als_plan_size(hp.ctypes.data, n_rows, 8, C.byref(nc), C.byref(ns), C.byref(nslot)))


@pytest.mark.parametrize("chunk", [8, 31, 33, 40, 48, 50, 100, 4095])
def test_als_plan_rejects_chunk_not_multiple_of_32(cuda_lib, chunk):
    """Equal parts rounded up to 32 nonzeros only stay within 1 .. chunk_nnz when chunk_nnz is a multiple of 32:
    at 40 a row of 97 would be cut 64 + 33 + 0 (also 97 at 33 or 48, 101 at 50, 481 at 100).  Such sizes are
    refused by both calls rather than planned with an empty or overlong part."""
    lens = _boundary_lengths(32) + [97, 101, 481]
    hp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    nc, ns, nslot = C.c_int64(), C.c_int64(), C.c_int64()
    with pytest.raises(_lib.EngineError, match="multiple of 32"):
        _lib.check(cuda_lib.lk_als_plan_size(hp.ctypes.data, len(lens), chunk, C.byref(nc), C.byref(ns), C.byref(nslot)))
    out = np.zeros((4096, 8), dtype=np.int32)
    with pytest.raises(_lib.EngineError, match="multiple of 32"):
        _lib.check(cuda_lib.lk_als_plan_fill(hp.ctypes.data, len(lens), chunk, out.ctypes.data))
    assert not out.any()


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


# (n_users, n_items) -> every lk_knn_geom field (n_users, n_items, warps, tile_cols, n_halves, n_subtiles,
# smem_bytes, ctas_per_sm) of lk_knn_geometry(n_users, n_items), lk_uknn_geometry(n_users, n_items, ctas) for
# ctas 0, 1, 2, and lk_cooc_geometry(n_users, n_items), from one to a few hundred column tiles
GEOMETRIES = {
    (1_000, 1): (
        [1000, 1, 16, 32, 1, 16, 10384, 2],
        [[1, 1000, 16, 64, 1, 16, 8272, 2], [1, 1000, 16, 64, 1, 16, 8272, 1], [1, 1000, 16, 64, 1, 16, 8272, 2]],
        [1000, 1, 16, 32, 1, 16, 10320, 2],
    ),
    (610, 9_724): (
        [610, 9724, 16, 608, 1, 16, 47248, 2],
        [[9724, 610, 16, 64, 1, 16, 8272, 2], [9724, 610, 16, 64, 1, 16, 8272, 1], [9724, 610, 16, 64, 1, 16, 8272, 2]],
        [610, 9724, 16, 608, 1, 16, 47184, 2],
    ),
    (162_541, 59_047): (
        [162541, 59047, 16, 1248, 3, 48, 88208, 2],
        [
            [59047, 162541, 16, 864, 12, 192, 110672, 2],
            [59047, 162541, 16, 1696, 6, 96, 217168, 1],
            [59047, 162541, 16, 864, 12, 192, 110672, 2],
        ],
        [162541, 59047, 16, 1248, 3, 48, 88144, 2],
    ),
    (100, 28_000): (
        [100, 28000, 16, 896, 2, 32, 65680, 2],
        [
            [28000, 100, 16, 32, 1, 16, 4176, 2],
            [28000, 100, 16, 32, 1, 16, 4176, 1],
            [28000, 100, 16, 32, 1, 16, 4176, 2],
        ],
        [100, 28000, 16, 896, 2, 32, 65616, 2],
    ),
    (59_047, 162_541): (
        [59047, 162541, 16, 1472, 7, 112, 102544, 2],
        [
            [162541, 59047, 16, 768, 5, 80, 98384, 2],
            [162541, 59047, 16, 1248, 3, 48, 159824, 1],
            [162541, 59047, 16, 768, 5, 80, 98384, 2],
        ],
        [59047, 162541, 16, 1472, 7, 112, 102480, 2],
    ),
    (5_000, 500_000): (
        [5000, 500000, 16, 1664, 19, 304, 114832, 2],
        [
            [500000, 5000, 16, 320, 1, 16, 41040, 2],
            [500000, 5000, 16, 320, 1, 16, 41040, 1],
            [500000, 5000, 16, 320, 1, 16, 41040, 2],
        ],
        [5000, 500000, 16, 1664, 19, 304, 114768, 2],
    ),
    (7, 3_000_000): (
        [7, 3000000, 16, 1664, 113, 1808, 114832, 2],
        [
            [3000000, 7, 16, 32, 1, 16, 4176, 2],
            [3000000, 7, 16, 32, 1, 16, 4176, 1],
            [3000000, 7, 16, 32, 1, 16, 4176, 2],
        ],
        [7, 3000000, 16, 1664, 113, 1808, 114768, 2],
    ),
    (3_000_000, 20): (
        [3000000, 20, 16, 32, 1, 16, 10384, 2],
        [
            [20, 3000000, 16, 896, 210, 3360, 114768, 2],
            [20, 3000000, 16, 1792, 105, 1680, 229456, 1],
            [20, 3000000, 16, 896, 210, 3360, 114768, 2],
        ],
        [3000000, 20, 16, 32, 1, 16, 10320, 2],
    ),
}


@pytest.mark.parametrize("shape", list(GEOMETRIES))
def test_tile_geometries_are_pinned(cuda_lib, lk_options, shape):
    lk_options("LK_KNN_WARPS", -1)  # the built-in choices, whatever the environment says
    lk_options("LK_KNN_CTAS", -1)
    n_users, n_items = shape
    want_knn, want_uknn, want_cooc = GEOMETRIES[shape]
    g = _lib.LkKnnGeom()

    def fields():
        return [getattr(g, f) for f, _ in _lib.LkKnnGeom._fields_]

    _lib.check(cuda_lib.lk_knn_geometry(n_users, n_items, C.byref(g)))
    assert fields() == want_knn
    for ctas, want in enumerate(want_uknn):
        _lib.check(cuda_lib.lk_uknn_geometry(n_users, n_items, ctas, C.byref(g)))
        assert fields() == want, ctas
    _lib.check(cuda_lib.lk_cooc_geometry(n_users, n_items, C.byref(g)))
    assert fields() == want_cooc


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
