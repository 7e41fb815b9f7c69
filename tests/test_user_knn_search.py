"""
User-kNN neighbour search, CPU side: the ordered-f64 restatement the device search implements equals
SciPy's ``user_vectors @ x`` bit for bit (the exactness claim of ``knn_user.cu``), the ctypes mirror of
``lk_uknn_search_args`` has the header's layout, and provided histories become queries with the
reference's rules.
"""

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import scipy.sparse as sps

from lkpy_b200 import _lib, engine
from lkpy_b200.components import Dataset, ItemList
from lkpy_b200.knn_user import UserKNNScorer

ROOT = Path(__file__).resolve().parent.parent


def ordered_sims(vt: sps.csr_array, n_users: int, items: np.ndarray, vals: np.ndarray) -> np.ndarray:
    """sim = sum over the query's items in ascending order of VT[i, v] * x[i]: one f64 multiply and one f64
    add per step (NumPy's elementwise ops are never fused), from +0.0."""
    acc = np.zeros(n_users, dtype=np.float64)
    for i, x in zip(items, vals):
        lo, hi = vt.indptr[i], vt.indptr[i + 1]
        users = vt.indices[lo:hi]
        acc[users] = acc[users] + vt.data[lo:hi] * np.float64(x)
    return acc


def _bits_match_nonzero(got: np.ndarray, ref: np.ndarray) -> int:
    """Equal bits wherever either side is nonzero (a zero sum may differ only in its sign)."""
    nz = (ref != 0) | (got != 0)
    assert np.array_equal(got[nz].view(np.int64), ref[nz].view(np.int64))
    return int(nz.sum())


@pytest.mark.parametrize("feedback", ["explicit", "implicit"])
def test_ordered_f64_restatement_equals_scipy(ml_small, feedback):
    m = UserKNNScorer(feedback=feedback)
    m.train(Dataset(ml_small))
    V = m.user_vectors
    assert V.dtype == np.float64
    vt = sps.csr_array(V.T)
    vt.sort_indices()
    n_users = V.shape[0]
    checked = 0
    for u in range(0, n_users, 7):
        lo, hi = V.indptr[u], V.indptr[u + 1]
        x = V[[u], :].toarray()[0]
        checked += _bits_match_nonzero(ordered_sims(vt, n_users, V.indices[lo:hi], V.data[lo:hi]), V @ x)
    assert checked > 50_000
    # provided histories: f32 query values widened to f64, as the reference's f32 rating vector
    rng = np.random.default_rng(11)
    for _ in range(20):
        nums = rng.choice(V.shape[1], int(rng.integers(1, 80)), replace=False).astype(np.int32)
        r = (rng.integers(1, 11, len(nums)) * 0.5).astype(np.float32)
        items, vals, _ = engine.history_query(nums, r if feedback == "explicit" else None)
        dense = np.zeros(V.shape[1], dtype=np.float32)
        dense[items] = vals.astype(np.float32)
        _bits_match_nonzero(ordered_sims(vt, n_users, items, vals), V @ dense)


def test_uknn_struct_matches_header(tmp_path):
    cls, cname = _lib.LkUknnSearchArgs, "lk_uknn_search_args"
    expected, lines = [], []
    for field in cls._fields_:
        name = field[0]
        expected.append((f"{cname}.{name}", getattr(cls, name).offset))
        lines.append(f'    printf("{cname}.{name} %zu\\n", offsetof({cname}, {name}));')
    expected.append((f"sizeof {cname}", C.sizeof(cls)))
    lines.append(f'    printf("sizeof {cname} %zu\\n", sizeof({cname}));')
    src = tmp_path / "layout.c"
    src.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "lkpy_b200.h"\n\nint main(void)\n{\n'
        + "\n".join(lines)
        + "\n    return 0;\n}\n"
    )
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    got = [(line.rsplit(" ", 1)[0], int(line.rsplit(" ", 1)[1])) for line in out]
    assert got == expected
    for name in ("lk_uknn_geometry", "lk_uknn_query_cost", "lk_uknn_search", "lk_uknn_pool_to_csr"):
        assert name in _lib.SYMBOLS


def _reference_dense(nums: np.ndarray, urv: np.ndarray | None, n_items: int) -> tuple[np.ndarray, float]:
    """The reference's dense f32 rating vector of a provided history (user.py:281-298)."""
    ratings = np.zeros(n_items, dtype=np.float32)
    mask = nums >= 0
    if urv is None:
        ratings[nums[mask]] = 1.0
        return ratings, 0.0
    urv = np.require(urv, dtype=np.float32)
    umean = float(urv.mean())
    ratings[nums[mask]] = urv[mask] - umean
    return ratings, umean


@pytest.mark.parametrize("explicit", [True, False])
def test_history_query_rules(explicit):
    nums = np.array([7, 3, -1, 7, 12, 3, -1, 0, 7], dtype=np.int32)
    r = np.array([4.0, 2.5, 5.0, 1.0, 3.5, 0.5, 2.0, 4.5, 3.0], dtype=np.float32)
    items, vals, umean = engine.history_query(nums, r if explicit else None)
    assert items.dtype == np.int32 and vals.dtype == np.float64
    assert items.tolist() == [0, 3, 7, 12]  # unknown items dropped, duplicates merged, ascending
    dense, ref_mean = _reference_dense(nums, r if explicit else None, 16)
    assert umean == ref_mean
    assert np.array_equal(vals.view(np.int64), dense[items].astype(np.float64).view(np.int64))
    assert np.count_nonzero(dense) == np.count_nonzero(vals)
    if explicit:
        mean = np.float32(r.mean())  # over the whole history, unknown items included
        assert umean == float(mean)
        assert vals[2] == np.float64(np.float32(3.0) - mean)  # item 7: the LAST of its three ratings
        assert vals[1] == np.float64(np.float32(0.5) - mean)  # item 3: last of two
    else:
        assert np.all(vals == 1.0)


def test_history_query_random_matches_reference_dense():
    rng = np.random.default_rng(4)
    for _ in range(50):
        n = int(rng.integers(1, 40))
        nums = rng.integers(-1, 25, n).astype(np.int32)
        r = (rng.integers(1, 11, n) * 0.5).astype(np.float32)
        items, vals, umean = engine.history_query(nums, r)
        dense, ref_mean = _reference_dense(nums, r, 25)
        assert umean == ref_mean
        assert np.all(np.diff(items) > 0)
        got = np.zeros(25, dtype=np.float64)
        got[items] = vals
        assert np.array_equal(got, dense.astype(np.float64))
    items, vals, _ = engine.history_query(np.array([-1, -1], np.int32), None)
    assert items.size == 0 and vals.size == 0


def test_component_history_is_item_list_rules(ml_small):
    """``UserKNNScorer._query`` feeds ItemList ids through the same rules: unknown ids negative, ratings kept."""
    m = UserKNNScorer()
    ds = Dataset(ml_small)
    m.train(ds)
    ids = ds.items.ids([5, 9, 5])
    hist = ItemList(item_ids=np.concatenate([ids, [-12345]]), rating=np.array([1.0, 2.0, 4.0, 5.0], np.float32))
    from lkpy_b200.components import RecQuery

    (items, vals, self_), umean = m._query(RecQuery(user_id=None, query_items=hist))
    assert self_ is None and items.tolist() == [5, 9]
    mean = np.float32(np.array([1.0, 2.0, 4.0, 5.0], np.float32).mean())
    assert umean == float(mean) and vals[0] == np.float64(np.float32(4.0) - mean)
    assert m._query(RecQuery(user_id=None, query_items=ItemList(item_ids=ids))) is None  # explicit without ratings
    assert m._query(RecQuery(user_id=ds.users.id(3))) == (3, float(m.user_means[3]))
