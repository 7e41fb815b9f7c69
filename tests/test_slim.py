"""
SLIM, host side (no GPU): the C restatement (``tests/slim_oracle.c``) against hand-worked columns and a Python
restatement of the same statements, the ``x @ weights`` restatement against SciPy, the input validation of
``accel.slim.train_slim``, the layout of ``lk_slim_args``, and the reference's own ``SLIMScorer`` run over the
mirror (with the restatement as its device part).
"""

import ctypes as C
import math
import shutil
import subprocess
import sys
import warnings
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest
import scipy.sparse as sps

import ref_sandbox
import slim_oracle as so
from lkpy_b200 import _lib, accel, data

ROOT = Path(__file__).resolve().parent.parent
f32 = np.float32


def py_column(item, ui, iu, n_items, l1, l2, max_iters, k):
    """The five contract steps for one target item in Python, every f32 operation on NumPy f32 scalars."""
    (ui_p, ui_c), (iu_p, iu_c) = ui, iu
    U = list(iu_c[iu_p[item] : iu_p[item + 1]])
    resid = {u: f32(1.0) for u in U}
    pc, active = {}, []
    for u in U:
        for j in ui_c[ui_p[u] : ui_p[u + 1]]:
            if j != item:
                if pc.get(j, 0) == 0:
                    active.append(j)
                pc[j] = pc.get(j, 0) + 1
    if k is not None and k < len(active):
        i_norm = math.sqrt(float(len(U)))
        active = sorted(active, key=lambda j: -float(pc[j]) / (i_norm * math.sqrt(float(iu_p[j + 1] - iu_p[j]))))[:k]
    W = {}
    for _it in range(max_iters):
        dmax = f32(0.0)
        for j in active:
            Uj = iu_c[iu_p[j] : iu_p[j + 1]]
            w = W.get(j, f32(0.0))
            upd = f32(0.0)
            for u in Uj:
                upd = f32(upd + f32(resid.get(u, f32(0.0)) + w))
            new = f32((upd - f32(l1)) / f32(f32(len(Uj)) + f32(l2))) if upd >= f32(l1) else f32(0.0)
            diff = f32(new - w)
            W[j] = new
            for u in Uj:
                resid[u] = f32(resid.get(u, f32(0.0)) - diff)
            if abs(diff) > dmax:
                dmax = abs(diff)
        if dmax <= f32(1e-3):
            break
    return [(j, W[j]) for j in sorted(W) if W[j] >= f32(1e-12)]


def _rows(W, i):
    lo, hi = W.indptr[i], W.indptr[i + 1]
    return list(zip(W.indices[lo:hi].tolist(), W.data[lo:hi].tolist()))


def _pairs_structs(n_users, n_items, rows):
    """UI and IU structures of per-user item lists given in stored order (IU users ascending)."""
    u = np.concatenate([[k] * len(r) for k, r in enumerate(rows)]).astype(np.int32)
    i = np.concatenate(rows).astype(np.int32)
    return so.structure(n_users, u, i), so.structure(n_items, i, u)


def test_hand_worked_column():
    # u0: {0, 1}, u1: {0, 1, 2}, u2: {1, 2}.  Target 0: resid = (1, 1, 0), active = [1, 2].
    # Round 1: j = 1: upd = 1 + 1 + 0 = 2 >= 1, w = (2 - 1) / (3 + 1) = 0.25, resid = (.75, .75, -.25);
    #          j = 2: upd = .75 - .25 = .5 < 1, w = 0.  Round 2 changes nothing: converged.
    ui, iu = _pairs_structs(3, 4, [[0, 1], [0, 1, 2], [1, 2]])
    for iters in (1, 100):
        W = so.train(3, 4, ui, iu, 1.0, 1.0, iters, None)
        assert _rows(W, 0) == [(1, 0.25)]
        assert _rows(W, 3) == []  # an item nobody rated
        assert W.indptr[4] == W.indptr[3]


def test_fsslim_ties_keep_first_encounter_order():
    # UI rows not sorted by item: u0 = [0, 2, 1], u1 = [0, 1, 2].  Target 0: active = [2, 1], both with pc = 2 and
    # 2 users, so their keys tie; k = 1 keeps item 2, first encountered.  w = (2 - 1) / (2 + 1).
    ui, iu = _pairs_structs(2, 3, [[0, 2, 1], [0, 1, 2]])
    W = so.train(2, 3, ui, iu, 1.0, 1.0, 100, 1)
    assert _rows(W, 0) == [(2, float(f32(1.0) / f32(3.0)))]
    # k >= |active| is plain SLIM
    assert _rows(so.train(2, 3, ui, iu, 1.0, 1.0, 100, 2), 0) == _rows(so.train(2, 3, ui, iu, 1.0, 1.0, 100, None), 0)
    ui2, iu2 = _pairs_structs(2, 3, [[0, 1, 2], [0, 1, 2]])
    assert [j for j, _ in _rows(so.train(2, 3, ui2, iu2, 1.0, 1.0, 100, 1), 0)] == [1]


@pytest.mark.parametrize("seed,l1,l2,iters,k", [(1, 1.0, 1.0, 100, None), (2, 0.1, 0.3, 1, None), (3, 0.05, 0.1, 3, 4),
                                                (4, 0.01, 0.01, 2, None), (5, 0.2, 0.7, 100, 2)])  # fmt: skip
def test_restatement_matches_python_statements(seed, l1, l2, iters, k):
    """Random small problems with shuffled UI rows (first-encounter order differs from item order), coupled
    coordinates that do not converge in 1-3 rounds, fsSLIM ties and an item nobody rated."""
    rng = np.random.default_rng(seed)
    n_users, n_items = 25, 12
    rows = [rng.permutation(rng.choice(n_items - 1, size=rng.integers(1, 8), replace=False)) for _ in range(n_users)]
    ui, iu = _pairs_structs(n_users, n_items, rows)
    W = so.train(n_users, n_items, ui, iu, l1, l2, iters, k)
    for i in range(n_items):
        want = py_column(i, ui, iu, n_items, l1, l2, iters, k)
        got = _rows(W, i)
        assert [j for j, _ in got] == [j for j, _ in want], i
        assert np.array_equal(np.array([v for _, v in got], f32).view(np.int32),
                              np.array([v for _, v in want], f32).view(np.int32)), i  # fmt: skip
    assert _rows(W, n_items - 1) == []


def test_non_convergence_stops_at_max_iters():
    ui, iu = _pairs_structs(4, 3, [[0, 1, 2], [0, 1], [0, 2], [1, 2]])
    outs = [_rows(so.train(4, 3, ui, iu, 0.01, 0.01, n, None), 0) for n in (1, 2, 3, 100)]
    assert outs[0] != outs[1] != outs[2]  # each round still moves the weights
    assert outs[3] == py_column(0, ui, iu, 3, 0.01, 0.01, 100, None)


def test_score_restatement_matches_scipy(ml_small):
    it = ml_small
    ui = so.structure(it.n_users, it.users, it.items)
    iu = so.structure(it.n_items, it.items, it.users)
    Wt = so.train(it.n_users, it.n_items, ui, iu, 1.0, 1.0, 100, 20).T.tocsr()
    rng = np.random.default_rng(3)
    for u in (0, 7, 100, 414, 670):
        h = rng.permutation(it.items[it.users == u])
        h = np.concatenate([h, h[:4], h[:1]])  # unsorted and repeated
        x = sps.csr_array((np.ones(len(h), np.float32), h, [0, len(h)]), shape=(1, it.n_items))
        want = (x @ Wt).toarray()[0]
        assert want.dtype == np.float32
        assert np.array_equal(so.score(Wt, h).view(np.int32), want.view(np.int32))


def _srows(ip, cols, dim):
    csr = data.InteractionCSR(np.asarray(ip), np.asarray(cols, np.int32), np.ones(len(cols), np.float32),
                              (len(ip) - 1, dim))  # fmt: skip
    return pa.chunked_array(accel.csr_to_arrow_chunks(csr)).combine_chunks()


def test_train_slim_validates_input_without_a_device():
    ui = _srows([0, 2, 3], [0, 1, 1], 3)  # 2 users x 3 items
    iu = _srows([0, 1, 3, 3], [0, 0, 1], 2)
    accel.slim.train_slim(ui, iu, 1.0, 1.0, 10, None)  # valid: nothing runs before invoke
    with pytest.raises(ValueError, match="user count mismatch"):
        accel.slim.train_slim(ui, _srows([0, 1, 3, 3], [0, 0, 1], 3), 1.0, 1.0, 10, None)
    with pytest.raises(ValueError, match="item count mismatch"):
        accel.slim.train_slim(ui, _srows([0, 1, 3], [0, 0, 1], 2), 1.0, 1.0, 10, None)
    with pytest.raises(ValueError, match="rating count mismatch"):
        accel.slim.train_slim(ui, _srows([0, 1, 2, 2], [0, 0], 2), 1.0, 1.0, 10, None)
    with pytest.raises(OverflowError):
        accel.slim.train_slim(ui, iu, 1.0, 1.0, -1, None)
    with pytest.raises(OverflowError):
        accel.slim.train_slim(ui, iu, 1.0, 1.0, 10, -2)
    with pytest.raises(TypeError):
        accel.slim.train_slim(ui, iu, 1.0, 1.0, 1.5, None)


def test_slim_struct_matches_header(tmp_path):
    cls = _lib.LkSlimArgs
    expected = [(f"lk_slim_args.{f[0]}", getattr(cls, f[0]).offset) for f in cls._fields_]
    expected.append(("sizeof lk_slim_args", C.sizeof(cls)))
    lines = [f'    printf("lk_slim_args.{f[0]} %zu\\n", offsetof(lk_slim_args, {f[0]}));' for f in cls._fields_]
    lines.append('    printf("sizeof lk_slim_args %zu\\n", sizeof(lk_slim_args));')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"lkpy_b200.h\"\n\nint main(void)\n{\n"
                   + "\n".join(lines) + "\n    return 0;\n}\n")  # fmt: skip
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert [(ln.rsplit(" ", 1)[0], int(ln.rsplit(" ", 1)[1])) for ln in out] == expected
    assert {"lk_slim_workspace_bytes", "lk_slim_train", "lk_slim_pool_to_csr"} <= set(_lib.SYMBOLS)


def test_slim_config():
    from lkpy_b200.slim import SLIMConfig, SLIMScorer

    assert SLIMScorer().config == SLIMConfig()
    assert SLIMConfig().model_dump() == {"l1_reg": 1.0, "l2_reg": 1.0, "max_iters": 100, "max_nbrs": None}
    for bad in ({"l1_reg": 0.0}, {"l2_reg": -1.0}, {"max_iters": 0}, {"max_nbrs": 0}):
        with pytest.raises(ValueError):
            SLIMConfig(**bad)


# --- the reference's SLIMScorer over the mirror ----------------------------------------------------------------


def _transpose_csr(structure, has_values):
    """``_accel.data.transpose_csr`` (src/accel/data/transpose.rs): counting-sort transpose of a sparse-row array's
    structure, rows of the result ascending; (offsets, indices, permutation of the values or None)."""
    off = structure.offsets.to_numpy(zero_copy_only=False).astype(np.int64)
    idx = structure.indices.to_numpy(zero_copy_only=False)
    rows = np.repeat(np.arange(len(off) - 1), np.diff(off))
    perm = np.argsort(idx, kind="stable")
    t_off = np.zeros(structure.dimension + 1, np.int64)
    np.cumsum(np.bincount(idx, minlength=structure.dimension), out=t_off[1:])
    return pa.array(t_off), pa.array(rows[perm].astype(np.int32)), (pa.array(perm) if has_values else None)


class _SlimMatrix(ref_sandbox._MatrixView):
    def csr_structure(self, *, format="numpy"):
        assert format == "arrow"
        it = self._inter
        m = sps.csr_array((np.ones(it.nnz, np.float32), (it.users, it.items)), shape=(it.n_users, it.n_items))
        SparseRowArray = sys.modules["lenskit.data.matrix"].SparseRowArray
        return SparseRowArray.from_scipy(m, values=False)


class _SlimRelationship(ref_sandbox._Relationship):
    def matrix(self, **_kw):
        return _SlimMatrix(self._inter)


class SlimDataset(ref_sandbox.FakeDataset):
    def interactions(self, *_a, **_kw):
        return _SlimRelationship(self._inter)


@pytest.fixture(scope="module")
def slim_ref(monkeypatch_module):
    if not ref_sandbox.available():
        pytest.skip("needs a lenskit/lkpy checkout for the reference's SLIMScorer")
    with ref_sandbox.reference_modules() as mods, warnings.catch_warnings():
        warnings.simplefilter("ignore")
        acc = sys.modules["lenskit._accel"]
        acc.slim = accel.slim
        acc.data.transpose_csr = _transpose_csr
        sys.modules["lenskit._accel.slim"] = accel.slim
        mods["lenskit.knn.slim"] = ref_sandbox._load("lenskit.knn.slim", "knn/slim.py")
        yield mods


@pytest.fixture(scope="module")
def monkeypatch_module():
    with pytest.MonkeyPatch.context() as mp:
        yield mp


def test_reference_slim_scorer_through_the_mirror(slim_ref, monkeypatch_module, ml_small):
    """``SLIMScorer.train`` (knn/slim.py:121-140) through ``_accel.slim.train_slim`` — its device part the
    restatement when there is no GPU — and ``__call__`` (slim.py:142-170): the transposed weights and the scores
    equal the restatements', and the NaN / zero rules hold."""
    import torch

    if not torch.cuda.is_available():

        def rows(ui, iu, l1, l2, iters, nbrs, task):
            W = so.train(ui.shape[0], ui.shape[1], (ui.indptr, ui.indices), (iu.indptr, iu.indices), l1, l2, iters,
                         nbrs)  # fmt: skip
            task._check_cancelled()
            return data.InteractionCSR(W.indptr, W.indices, W.data, W.shape)

        monkeypatch_module.setattr(accel, "_slim_rows", rows)
    it = ml_small
    mod, items_mod, query_mod = (slim_ref[k] for k in ("lenskit.knn.slim", "lenskit.data._items", "lenskit.data._query"))
    m = mod.SLIMScorer(max_nbrs=20)
    m.train(SlimDataset(it))
    ui = so.structure(it.n_users, it.users, it.items)
    iu = so.structure(it.n_items, it.items, it.users)
    Wt = so.train(it.n_users, it.n_items, ui, iu, 1.0, 1.0, 100, 20).T.tocsr()
    assert m.weights.shape == Wt.shape
    assert np.array_equal(m.weights.indptr, Wt.indptr) and np.array_equal(m.weights.indices, Wt.indices)
    assert np.array_equal(m.weights.data.view(np.int32), Wt.data.view(np.int32))
    tgt = items_mod.ItemList(item_ids=np.concatenate([it.item_ids[::11], [-1]]))
    rng = np.random.default_rng(5)
    for u in (0, 200):
        h = rng.permutation(it.items[it.users == u])
        h = np.concatenate([h, h[:2]])
        q = query_mod.RecQuery.create(items_mod.ItemList(item_ids=it.item_ids[h]))
        s = m(q, tgt).scores("numpy").astype(np.float32)
        assert np.array_equal(s[:-1].view(np.int32), so.score(Wt, h)[::11].view(np.int32)) and np.isnan(s[-1])
    unknown = query_mod.RecQuery.create(items_mod.ItemList(item_ids=np.array([-5])))
    assert np.all(m(unknown, tgt).scores("numpy")[:-1] == 0)
    empty = query_mod.RecQuery.create(items_mod.ItemList(item_ids=np.array([], np.int64)))
    assert np.all(np.isnan(m(empty, tgt).scores("numpy")))
