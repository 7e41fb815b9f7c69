"""
EASE without a GPU: the config and ``LK_EASE_SOLVER`` handling, the OOM fallback, the C struct layout, the oracle's
score order against an f64 sum, and the reference's own ``EASEScorer`` (``knn/ease.py``) run in the sandbox of
``tests/ref_sandbox.py`` with ``co_occurrences(dense=True)`` bound to this package's ``dense_cooc`` mirror.

As in ``test_reference_association.py``, the reference's side is computed live when a lenskit/lkpy checkout is there
(``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites the golden file) and otherwise read from
``tests/golden/reference_classes/ease_ml_small.npz``.  This package's side is the GPU scorer when there is a device,
the oracle's statements with the torch inverse on the CPU otherwise.
"""

import ctypes as C
import os
import shutil
import subprocess
import sys
import types
import warnings
from pathlib import Path

import numpy as np
import pytest
import pyarrow as pa
import torch

import cooc_oracle as co
import ease_oracle as eo
import ref_sandbox
from lkpy_b200 import _lib, accel, ease
from lkpy_b200.ease import EASEConfig, EASEScorer

ROOT = Path(__file__).resolve().parent.parent
GOLD = Path(__file__).resolve().parent / "golden" / "reference_classes" / "ease_ml_small.npz"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"


def test_config():
    assert EASEScorer().config == EASEConfig() and EASEConfig().regularization == 1
    assert EASEScorer(regularization=0.5).config.regularization == 0.5
    for bad in (0, -1.0):
        with pytest.raises(ValueError):
            EASEConfig(regularization=bad)
    with pytest.raises(ValueError):
        EASEConfig(damping=1.0)
    m = EASEScorer()
    assert not m.is_trained() and not hasattr(m, "weights")


def test_solver_variable(monkeypatch, ml_small):
    from lkpy_b200.components import Dataset

    for ok in (None, "", "torch", "scipy"):
        ease._check_solver(ok)
    monkeypatch.setenv("LK_EASE_SOLVER", "cholmod")
    with pytest.raises(ValueError, match="unsupported option: LK_EASE_SOLVER=cholmod"):
        EASEScorer().train(Dataset(ml_small))  # rejected before any device work


def _spd(n=40, seed=0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    X = (rng.random((3 * n, n)) < 0.2).astype(np.float32)
    G = X.T @ X
    G[np.diag_indices(n)] += 1.0
    return G


def test_torch_inverse_and_normalise_are_the_reference_statements():
    G = _spd()
    got = ease._normalise(ease._invert(lambda: torch.from_numpy(G.copy()), None)).numpy()
    want = eo.normalise(eo.invert_torch(G.copy(), "cpu"))
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_out_of_memory_falls_back_to_scipy(monkeypatch):
    G = _spd()
    tried, built = [], []

    def no_memory(gram):
        tried.append(1)
        raise torch.OutOfMemoryError("CUDA out of memory (test)")

    def gram():
        built.append(1)
        return torch.from_numpy(G.copy())

    monkeypatch.setattr(ease, "_chol_invert_torch", no_memory)
    with pytest.warns(RuntimeWarning, match="falling back to SciPy"):
        got = ease._invert(gram, None)
    assert got.dtype == torch.float32 and len(tried) == 1 and len(built) == 2  # the Gram is built again
    want = eo.invert_scipy(G.copy())
    assert np.array_equal(got.numpy().view(np.int32), want.view(np.int32))
    with pytest.raises(torch.OutOfMemoryError):  # a requested solver is not replaced
        ease._invert(gram, "torch")
    tried.clear()
    got = ease._invert(gram, "scipy")
    assert not tried and np.array_equal(got.numpy().view(np.int32), want.view(np.int32))


def test_ease_struct_matches_header(tmp_path):
    cls, cname = _lib.LkEaseScoreArgs, "lk_ease_score_args"
    expected = [(f"{cname}.{f[0]}", getattr(cls, f[0]).offset) for f in cls._fields_] + [(f"sizeof {cname}", C.sizeof(cls))]
    lines = [f'    printf("{cname}.{f[0]} %zu\\n", offsetof({cname}, {f[0]}));' for f in cls._fields_]
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


def test_score_order_against_f64_sum():
    """The sequential f32 sum is within the textbook bound of the exact sum: |s - S| <= gamma_{R-1} sum |W[h, j]|,
    gamma_k = k u / (1 - k u), u = 2^-24 (the first add, to +0.0, is exact)."""
    rng = np.random.default_rng(3)
    W = rng.standard_normal((3000, 500)).astype(np.float32)
    for hist in (np.array([7]), np.array([5, 5, 2, 9, 2]), rng.choice(3000, 2000, replace=False), np.zeros(0)):
        s = eo.score(W, hist)
        h = eo.history(hist)
        if len(h) == 0:
            assert np.isnan(s).all()
            continue
        exact = W[h].astype(np.float64).sum(axis=0)
        k, u = len(h) - 1, 2.0**-24
        bound = k * u / (1 - k * u) * np.abs(W[h]).astype(np.float64).sum(axis=0)
        assert np.all(np.abs(s - exact) <= bound)
        if len(h) == 1:
            assert np.array_equal(s, W[h[0]])


# ---------------------------------------------------------------------------
# the reference's own EASEScorer
# ---------------------------------------------------------------------------

ROWS = np.array([0, 1, 17, 314, 2224, 9065])  # sampled weight rows (row 0 is the most rated item)
TARGETS = np.arange(0, 9066, 37)
#: norm-wise tolerance for weights and scores.  The two sides differ by the f32 inverse only (torch on a CPU, or
#: cuSOLVER, against the same on another machine).  The Gram of ml-latest-small with regularization 1 has
#: lambda_max / lambda_min = 19,888 (lambda_min = 1.0, the regularisation; lambda_max = 19,887.7; measured in f64
#: with numpy.linalg.eigvalsh); a backward-stable f32 inverse has a norm-wise relative error of order
#: kappa * eps_f32 = 19,888 * 2^-23 = 2.37e-3, and the tolerance is that figure.
KAPPA = 19_888
TOL = KAPPA * float(np.finfo(np.float32).eps)


def _oracle_device(monkeypatch):
    """No GPU: keep the mirror's own ``dense_cooc`` and swap its device part for ``cooc_oracle``."""

    class CpuPlan:
        def dense(self, indptr, cols, counts, diag):
            n = len(indptr) - 1
            rows = np.repeat(np.arange(n), np.diff(indptr.numpy()))
            m = np.zeros((n, n), np.float32)
            m[rows, cols.numpy()] = counts.numpy().astype(np.float32)
            m[cols.numpy(), rows] = counts.numpy().astype(np.float32)
            if diag is not None:
                m[np.arange(n), np.arange(n)] = diag.numpy().astype(np.float32)
            return torch.from_numpy(m)

    def cooc_upper(n_groups, n_items, g, i, task, diagonal):
        diag, row, col, cnt = co._tally(n_items, *co._pairs(n_groups, n_items, g, i))
        indptr = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n_items))]).astype(np.int64)
        t = torch.from_numpy
        return CpuPlan(), t(indptr), t(col), t(cnt.astype(np.int32)), t(diag.astype(np.int32)) if diagonal else None

    monkeypatch.setattr(accel, "_cooc_upper", cooc_upper)


class _EaseRelationship(ref_sandbox._Relationship):
    def co_occurrences(self, entity, *, group=None, order=None, include_self=False, dense=False):
        """``RelationshipSet.co_occurrences`` (data/_relationships.py) for the user-item relationship: the table
        sorted by user, then the reference's ``fast_col_cooc``."""
        assert entity == "item" and group is None and order is None
        it = self._inter
        o = np.argsort(it.users, kind="stable")
        fcc = sys.modules["lenskit.data.matrix"].fast_col_cooc
        return fcc(pa.array(it.users[o]), pa.array(it.items[o]), (it.n_users, it.n_items),
                   include_diagonal=include_self, ordered=False, dense=dense, progress=ref_sandbox._Progress())  # fmt: skip


class _EaseDataset(ref_sandbox.FakeDataset):
    def interactions(self, *_a, **_kw):
        return _EaseRelationship(self._inter)


def _queries(ml_small):
    """Two users' histories with repeats, one with an unknown item, one of unknown items only, and an empty one."""
    ids = ml_small.item_ids
    unknown = int(ids.max()) + 1
    out = []
    for u in (3, 100):
        nums = ml_small.items[ml_small.users == u]
        out.append(ids[np.concatenate([nums, nums[:5]])])
    out.append(np.concatenate([ids[ml_small.items[ml_small.users == 414]], [unknown]]))
    out.append(np.array([unknown, unknown + 1]))
    out.append(ids[:0])
    return out


@pytest.fixture(scope="module")
def ref():
    if not ref_sandbox.available():
        yield None
        return
    with ref_sandbox.reference_modules() as mods, warnings.catch_warnings(), pytest.MonkeyPatch.context() as mp:
        warnings.simplefilter("ignore")
        if not torch.cuda.is_available():
            _oracle_device(mp)
        # what knn/ease.py imports beyond the sandbox: humanize's naturalsize (log text only)
        mp.setitem(sys.modules, "humanize", types.SimpleNamespace(naturalsize=lambda n: f"{n} B"))
        shim = sys.modules["lenskit._accel"].data
        shim.count_cooc, shim.dense_cooc = accel.data.count_cooc, accel.data.dense_cooc
        mods["lenskit.knn.ease"] = ref_sandbox._load("lenskit.knn.ease", "knn/ease.py")
        yield mods


def _rel(a, b) -> float:
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def test_reference_ease_scorer_through_the_mirror(ref, ml_small):
    """``EASEScorer.train`` and ``__call__`` (knn/ease.py): sampled weight rows and the scores of queries with
    repeats, unknown items, only unknown items and no items, against this package's within ``TOL``."""
    qs = _queries(ml_small)
    tgt_ids = np.concatenate([ml_small.item_ids[TARGETS], [int(ml_small.item_ids.max()) + 1]])

    if ref is not None:
        mod, items_mod, query_mod = ref["lenskit.knn.ease"], ref["lenskit.data._items"], ref["lenskit.data._query"]
        m = mod.EASEScorer()
        m.train(_EaseDataset(ml_small))
        assert m.is_trained() and m.weights.dtype == np.float32
        theirs = {"rows": m.weights[ROWS]}
        tgt = items_mod.ItemList(item_ids=tgt_ids)
        for k, q in enumerate(qs):
            query = query_mod.RecQuery.create(items_mod.ItemList(item_ids=q))
            theirs[f"scores_{k}"] = m(query, tgt).scores("numpy").astype(np.float32)
        if RECORD:
            np.savez_compressed(GOLD, **theirs)
    else:
        with np.load(GOLD) as z:
            theirs = {k: z[k] for k in z.files}

    if torch.cuda.is_available():
        from lkpy_b200.components import Dataset, ItemList

        ours = EASEScorer()
        ours.train(Dataset(ml_small))
        W = ours.weights
        mine = [ours(ItemList(item_ids=q), ItemList(item_ids=tgt_ids)).scores() for q in qs]
    else:
        W = eo.train(ml_small.n_users, ml_small.n_items, ml_small.users, ml_small.items, 1.0, "cpu")
        num = {v: i for i, v in enumerate(ml_small.item_ids.tolist())}
        mine = []
        for q in qs:
            h = np.array([num.get(int(v), -1) for v in q], dtype=np.int64)
            s = eo.score(W, h)[TARGETS] if (h >= 0).any() else np.full(len(TARGETS), np.nan, np.float32)
            mine.append(np.concatenate([s, [np.nan]]).astype(np.float32))

    assert _rel(W[ROWS], theirs["rows"]) <= TOL
    for k, s in enumerate(mine):
        want = theirs[f"scores_{k}"]
        assert np.array_equal(np.isnan(s), np.isnan(want)), k
        assert np.isnan(want[-1])  # the unknown target
        if k >= 3:  # no usable history: NaN everywhere
            assert np.isnan(want).all()
        else:
            ok = ~np.isnan(want)
            assert _rel(s[ok], want[ok]) <= TOL, k
