"""
Co-occurrence counting and association scoring, host side (no GPU): the oracle in ``tests/cooc_oracle.py``
against SciPy and NumPy, the input validation of ``accel.data.count_cooc`` / ``dense_cooc``, and the layout of
the new C ABI structs.
"""

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

from lkpy_b200 import _lib, accel
import cooc_oracle as co

ROOT = Path(__file__).resolve().parent.parent


def test_oracle_matches_xtx_on_ml_small(ml_small):
    it = ml_small
    X = co.count_matrix(it.n_users, it.n_items, it.users, it.items)
    G = (X.T @ X).toarray()
    dense = co.dense_cooc(it.n_users, it.n_items, it.users, it.items, diagonal=True)
    assert np.array_equal(dense, G.astype(np.float32))
    diag, upper, lower = co.count_cooc(it.n_users, it.n_items, it.users, it.items)
    assert np.array_equal(diag[2], np.diag(G))
    iu = np.triu_indices(it.n_items, 1)
    nz = G[iu] > 0
    assert np.array_equal(upper[0], iu[0][nz]) and np.array_equal(upper[1], iu[1][nz])
    assert np.array_equal(upper[2], G[iu][nz])
    assert np.array_equal(lower[0], upper[1]) and np.array_equal(lower[1], upper[0])
    # ml-latest-small is 27 % dense: 21,983,224 entries including the diagonal
    assert int((G > 0).sum()) == 21_983_224


def test_oracle_duplicates_and_empty_groups():
    # group 0: [3, 1, 3]; group 1 empty; group 2: [1, 1, 1, 2]; item 0 and 4 never occur
    groups = np.array([0, 0, 0, 2, 2, 2, 2], np.int32)
    items = np.array([3, 1, 3, 1, 1, 1, 2], np.int32)
    diag, upper, lower = co.count_cooc(3, 5, groups, items)
    assert diag[2].tolist() == [0, 7, 1, 3, 0]  # #i (#i + 1) / 2: item 1 -> 1 + 6, item 3 -> 3
    assert list(zip(upper[0].tolist(), upper[1].tolist(), upper[2].tolist())) == [(1, 2, 3), (1, 3, 2)]
    X = co.count_matrix(3, 5, groups, items)
    G = (X.T @ X).toarray()
    d = co.dense_cooc(3, 5, groups, items, diagonal=False)
    off = ~np.eye(5, dtype=bool)
    assert np.array_equal(d[off], G[off].astype(np.float32)) and not d.diagonal().any()


def test_value_chain_matches_the_stated_roundings(ml_small):
    it = ml_small
    (row, col, cnt), _l = co.count_cooc(it.n_users, it.n_items, it.users, it.items, diagonal=False)
    ic = np.bincount(it.items, minlength=it.n_items).astype(np.int32)
    for method, kappa in (("probability", 0.0), ("lift", 0.0), ("lift", 0.1)):
        got = co.assoc_values(row, col, cnt, ic, it.n_users, method, kappa)
        v = (cnt.astype(np.float32).astype(np.float64) / (ic[row].astype(np.float64) + kappa)).astype(np.float32)
        if method == "lift":
            v = (v * np.float32(it.n_users)).astype(np.float32)
            v = (v.astype(np.float64) / (ic[col].astype(np.float64) + kappa)).astype(np.float32)
        assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), v.view(np.int32)), method


@pytest.mark.parametrize("R", [1, 2, 9, 64, 333])
def test_np_mean_is_a_sequential_sum_in_row_order(R):
    rng = np.random.default_rng(R)
    rows = rng.random((R, 4000)).astype(np.float32) * (rng.random((R, 4000)) < 0.5)
    rows *= np.float32(10.0) ** rng.integers(-3, 4, size=(R, 1)).astype(np.float32)
    want = np.mean(rows, axis=0)
    assert want.dtype == np.float32
    assert np.array_equal(co.score_sequential(rows).view(np.int32), want.view(np.int32))


def test_count_cooc_validates_input_without_a_device():
    g = pa.array([0, 0, 1], pa.int32())
    i = pa.array([1, 2, 0], pa.int32())
    with pytest.raises(ValueError, match="array length mismatch"):
        accel.data.count_cooc(2, 3, g, pa.array([1, 2], pa.int32()))
    with pytest.raises(ValueError):
        accel.data.count_cooc(2, 3, pa.array([1, 0, 1], pa.int32()), i)  # not ascending
    with pytest.raises(ValueError):
        accel.data.count_cooc(1, 3, g, i)  # group out of range
    with pytest.raises(ValueError):
        accel.data.dense_cooc(2, 2, g, i)  # item out of range
    with pytest.raises(ValueError):
        accel.data.count_cooc(2, 3, g, pa.array([1, -1, 0], pa.int32()))
    with pytest.raises(ValueError):
        accel.data.count_cooc(2, 3, g, pa.array([1, None, 0], pa.int32()))
    with pytest.raises(NotImplementedError):
        accel.data.count_cooc(2, 3, g, i, ordered=True)


def test_cooc_structs_match_header(tmp_path):
    structs = {"lk_cooc_args": _lib.LkCoocArgs, "lk_assoc_score_args": _lib.LkAssocScoreArgs}
    expected, lines = [], []
    for cname, cls in structs.items():
        for field in cls._fields_:
            expected.append((f"{cname}.{field[0]}", getattr(cls, field[0]).offset))
            lines.append(f'    printf("{cname}.{field[0]} %zu\\n", offsetof({cname}, {field[0]}));')
        expected.append((f"sizeof {cname}", C.sizeof(cls)))
        lines.append(f'    printf("sizeof {cname} %zu\\n", sizeof({cname}));')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"lkpy_b200.h\"\n\nint main(void)\n{\n"
                   + "\n".join(lines) + "\n    return 0;\n}\n")  # fmt: skip
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert [(ln.rsplit(" ", 1)[0], int(ln.rsplit(" ", 1)[1])) for ln in out] == expected


def test_association_config():
    from lkpy_b200.association import AssociationConfig, AssociationScorer

    assert AssociationScorer().config == AssociationConfig()
    with pytest.raises(ValueError):
        AssociationConfig(damping=-1.0)
    with pytest.raises(ValueError):
        AssociationConfig(method="cosine")
    AssociationScorer(max_nbrs=5)  # accepted at configuration; scoring raises NotImplementedError
