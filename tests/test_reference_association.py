"""
The reference's own co-occurrence and association classes over this package's mirror: ``lenskit.data.matrix.
fast_col_cooc`` and ``lenskit.knn.association.AssociationScorer`` (``train`` and ``__call__``) run in the sandbox of
``tests/ref_sandbox.py`` with ``_accel.data.count_cooc`` / ``dense_cooc`` bound to ``lkpy_b200.accel`` (INTEGRATION.md
§3c), and what they produce — the COO matrix and dense array, ``item_freqs``, ``assoc_scores`` and the scores — is
compared with what this package computes on the same inputs.  Also: the mirror's signatures against the stub
``_accel/data.pyi`` (recorded in ``tests/golden/accel_data_cooc_signatures.json``).

As in ``test_reference_classes.py``, the reference's side is computed live from a lenskit/lkpy checkout when there
is one (``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites the goldens) and otherwise read from
``tests/golden/reference_classes/``, recorded on a machine without a GPU, where the device part of the two entry
points is ``tests/cooc_oracle.py``.  This package's side is the GPU when there is one, the oracle otherwise.
"""

import ast
import inspect
import json
import os
import sys
import warnings
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest
import scipy.sparse as sps
import torch

import cooc_oracle as co
import ref_sandbox
from lkpy_b200 import accel, data

GOLD = Path(__file__).resolve().parent / "golden" / "reference_classes"
SIGS = Path(__file__).resolve().parent / "golden" / "accel_data_cooc_signatures.json"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"
ROWS = np.array([0, 1, 17, 314, 2224, 9065])  # sampled rows of the association matrix (row 0 is the most rated)
CONFIGS = [("probability", 0.0), ("lift", 0.0), ("lift", 0.1)]


def _theirs(name: str, ref, live) -> dict:
    if ref is None:
        with np.load(GOLD / f"{name}.npz") as z:
            return {k: z[k] for k in z.files}
    vals = {k: np.asarray(v) for k, v in live().items()}
    if RECORD:
        np.savez_compressed(GOLD / f"{name}.npz", **vals)
    return vals


def _oracle_device(monkeypatch):
    """No GPU: keep the mirror's own validation and result layout, swap its device part for the oracle."""

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


@pytest.fixture(scope="module")
def ref():
    if not ref_sandbox.available():
        with pytest.MonkeyPatch.context() as mp:
            if not torch.cuda.is_available():
                _oracle_device(mp)
            yield None
        return
    with ref_sandbox.reference_modules() as mods, warnings.catch_warnings(), pytest.MonkeyPatch.context() as mp:
        warnings.simplefilter("ignore")
        if not torch.cuda.is_available():
            _oracle_device(mp)
        shim = sys.modules["lenskit._accel"].data  # the module data/matrix.py imported as _data_accel
        shim.count_cooc, shim.dense_cooc = accel.data.count_cooc, accel.data.dense_cooc
        mods["lenskit.knn.association"] = ref_sandbox._load("lenskit.knn.association", "knn/association.py")
        yield mods


@pytest.fixture(scope="module")
def ml_small():
    return data.load_ml_small()


def _dup_input():
    """Groups ascending, items in any order inside a group, repeats, an empty group and unused items."""
    rng = np.random.default_rng(11)
    g = np.sort(rng.integers(0, 60, 1500)).astype(np.int32)
    g[g == 5] = 6
    i = (rng.zipf(1.4, 1500) % 110).astype(np.int32)  # items 110..119 never occur
    return 60, 120, g, i


def test_reference_fast_col_cooc_through_the_mirror(ref):
    """``fast_col_cooc`` (data/matrix.py:596-640), the function ``co_occurrences`` calls, with the unordered
    sparse and dense counts from the mirror: its COO matrix with and without the diagonal and its dense array."""
    m, n, g, i = _dup_input()

    def live():
        fcc = ref["lenskit.data.matrix"].fast_col_cooc
        out = {}
        for diag in (True, False):
            coo = fcc(pa.array(g), pa.array(i), (m, n), include_diagonal=diag)
            assert isinstance(coo, sps.coo_array) and coo.shape == (n, n)
            out[f"row{int(diag)}"], out[f"col{int(diag)}"], out[f"val{int(diag)}"] = coo.row, coo.col, coo.data
            out[f"dense{int(diag)}"] = fcc(pa.array(g), pa.array(i), (m, n), include_diagonal=diag, dense=True)
        return out

    theirs = _theirs("fast_col_cooc", ref, live)
    for diag in (True, False):
        want = co.count_cooc(m, n, g, i, diagonal=diag)
        for k, name in enumerate(("row", "col", "val")):
            assert np.array_equal(theirs[f"{name}{int(diag)}"], np.concatenate([b[k] for b in want])), (name, diag)
        assert theirs[f"dense{int(diag)}"].dtype == np.float32
        assert np.array_equal(theirs[f"dense{int(diag)}"], co.dense_cooc(m, n, g, i, diagonal=diag))


class _AssocMatrix(ref_sandbox._MatrixView):
    @property
    def n_rows(self) -> int:
        return self._inter.n_users


class _AssocRelationship(ref_sandbox._Relationship):
    def matrix(self, **_kw):
        return _AssocMatrix(self._inter)

    def co_occurrences(self, entity, *, group=None, order=None, include_self=False, dense=False):
        """``RelationshipSet.co_occurrences`` (data/_relationships.py:216-247) for the user-item relationship: the
        table sorted by user, then the reference's ``fast_col_cooc``."""
        assert entity == "item" and group is None and order is None
        it = self._inter
        o = np.argsort(it.users, kind="stable")
        fcc = sys.modules["lenskit.data.matrix"].fast_col_cooc
        return fcc(pa.array(it.users[o]), pa.array(it.items[o]), (it.n_users, it.n_items),
                   include_diagonal=include_self, ordered=False, dense=dense, progress=ref_sandbox._Progress())  # fmt: skip


class AssocDataset(ref_sandbox.FakeDataset):
    """``FakeDataset`` plus what ``AssociationScorer.train`` reads: ``co_occurrences`` and ``item_stats``."""

    def interactions(self, *_a, **_kw):
        return _AssocRelationship(self._inter)

    def item_stats(self):
        import pandas as pd

        # the record count per item of data/_relationships.py:877-908 (an Arrow group_by count: int64)
        return pd.DataFrame({"count": np.bincount(self._inter.items, minlength=self._inter.n_items).astype(np.int64)})


def _queries(ml_small):
    rng = np.random.default_rng(4)
    out = []
    for u in (3, 100, 414):
        nums = ml_small.items[ml_small.users == u]
        out.append(np.concatenate([nums, nums[:5]]))  # repeated reference items
    out.append(rng.integers(0, ml_small.n_items, 2))
    return out


TARGETS = np.arange(0, 9066, 37)


@pytest.mark.parametrize("method,damping", CONFIGS)
def test_reference_association_scorer_through_the_mirror(ref, ml_small, method, damping):
    """``AssociationScorer.train`` (knn/association.py:91-130) counts through ``fast_col_cooc`` and the mirror, and
    ``__call__`` (association.py:132-163) scores with ``max_nbrs`` None and 1: its ``item_freqs``, sampled rows of
    ``assoc_scores`` and scores equal this package's."""
    qs = _queries(ml_small)

    def live():
        mod, items_mod, query_mod = ref["lenskit.knn.association"], ref["lenskit.data._items"], ref["lenskit.data._query"]
        m = mod.AssociationScorer(method=method, damping=damping)
        m.train(AssocDataset(ml_small))
        A = m.assoc_scores
        assert isinstance(A, sps.csr_array) and A.has_sorted_indices
        out = {"item_freqs": np.asarray(m.item_freqs), "nnz": np.int64(A.nnz), "row_len": np.diff(A.indptr)[ROWS]}
        sub = A[ROWS, :]
        out["row_cols"], out["row_vals"] = sub.indices, sub.data
        tgt = items_mod.ItemList(item_ids=ml_small.item_ids[TARGETS])
        for mx in (None, 1):
            m.config.max_nbrs = mx
            for k, q in enumerate(qs):
                query = query_mod.RecQuery.create(items_mod.ItemList(item_ids=ml_small.item_ids[q]))
                out[f"scores{mx}_{k}"] = m(query, tgt).scores("numpy").astype(np.float32)
        return out

    theirs = _theirs(f"association_{method}_{damping}", ref, live)
    assert theirs["item_freqs"].dtype == np.int64
    if torch.cuda.is_available():
        from lkpy_b200.association import AssociationScorer
        from lkpy_b200.components import Dataset

        ours = AssociationScorer(method=method, damping=damping)
        ours.train(Dataset(ml_small))
        A = ours.assoc_scores
        assert ours.item_freqs.dtype == np.int64 and np.array_equal(ours.item_freqs, theirs["item_freqs"])
    else:
        A = co.assoc_matrix(ml_small.n_users, ml_small.n_items, ml_small.users, ml_small.items, method, damping)
    assert A.nnz == int(theirs["nnz"])
    assert np.array_equal(np.diff(A.indptr)[ROWS], theirs["row_len"])
    sub = A[ROWS, :]
    assert np.array_equal(sub.indices, theirs["row_cols"])
    assert np.array_equal(sub.data.view(np.int32), theirs["row_vals"].view(np.int32))
    for mx in (None, 1):
        for k, q in enumerate(qs):
            want = co.score(A, q, mx)[TARGETS]
            got = theirs[f"scores{mx}_{k}"]
            assert np.array_equal(got.view(np.int32), want.view(np.int32)), (mx, k)
            if torch.cuda.is_available():
                from lkpy_b200.components import ItemList

                ours.config = ours.config.model_copy(update={"max_nbrs": mx})
                mine = ours(ItemList(item_ids=ml_small.item_ids[q]), ItemList(item_ids=ml_small.item_ids[TARGETS]))
                assert np.array_equal(mine.scores().view(np.int32), got.view(np.int32)), (mx, k)


def _stub_signatures(pyi: Path) -> dict:
    """Parameter names and kinds (positional / keyword-only) and defaults of the co-occurrence stubs."""
    tree = ast.parse(pyi.read_text())
    out = {}
    for fn in tree.body:
        if isinstance(fn, ast.FunctionDef) and fn.name in ("count_cooc", "dense_cooc"):
            a = fn.args
            pos = [p.arg for p in a.posonlyargs + a.args]
            kw = {p.arg: ast.literal_eval(d) for p, d in zip(a.kwonlyargs, a.kw_defaults)}
            out[fn.name] = {"positional": pos, "keyword_only": kw}
    return out


def test_cooc_mirror_signatures_match_the_data_stub():
    """``_accel/data.pyi:23-39`` (recorded in the golden JSON; checked against the stub when the checkout is there):
    the mirror takes the same positional names in the same order and the same keyword-only flags and defaults."""
    want = json.loads(SIGS.read_text())
    if ref_sandbox.available():
        live = _stub_signatures(ref_sandbox.REF_SRC / "_accel" / "data.pyi")
        if RECORD:
            SIGS.write_text(json.dumps(live, indent=1, sort_keys=True) + "\n")
            want = live
        assert live == want
    assert set(want) == {"count_cooc", "dense_cooc"}
    for name, sig in want.items():
        params = inspect.signature(getattr(accel.data, name)).parameters.values()
        pos = [p.name for p in params if p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD]
        kw = {p.name: p.default for p in params if p.kind is inspect.Parameter.KEYWORD_ONLY}
        assert pos == sig["positional"] and kw == sig["keyword_only"], name
