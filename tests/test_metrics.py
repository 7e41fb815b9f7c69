"""
The ranking metrics without a GPU: the host restatements of lkpy_b200/metrics.py against recordings of the
reference's own metric classes (``tests/golden/reference_classes/metrics_*.npz``, which
``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites from a reference checkout through tests/metrics_ref_sandbox.py), the
options that are not covered, the rank-weight tables the device reads, the ABI, and the argument checks made before
any launch.
"""

import ctypes as C
import os
import warnings
from pathlib import Path

import numpy as np
import pandas as pd
import pytest

import metrics_ref_sandbox as mrs
from lkpy_b200 import _lib
from lkpy_b200 import metrics as lm
from lkpy_b200.components import ItemList, Vocabulary
from lkpy_b200.data import Interactions
from test_flexmf import test_ctypes_structs_match_header as _layout_check

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"

_recorded: list[bool] = []

#: this package's classes, by the reference's class names
CLASSES = {name: getattr(lm, name) for name in (
    "Hit", "Precision", "Recall", "RecipRank", "DCG", "NDCG", "RBP", "AveragePrecision", "MeanPopRank", "ListGini",
    "ExposureGini", "LogRankWeight", "GeometricRankWeight",
)}  # fmt: skip


def reference_golden(name: str) -> dict:
    """The reference's recording ``name`` (metrics_ref_sandbox.record): recorded live when asked to, else read."""
    if RECORD and not _recorded:
        import ref_sandbox

        assert ref_sandbox.available(), "recording needs the reference checkout"
        for n, d in mrs.record().items():
            np.savez_compressed(GOLD / f"{n}.npz", **d)
        _recorded.append(True)
    with np.load(GOLD / f"{name}.npz") as z:
        return {k: z[k] for k in z.files}


def cases():
    """``(recs, tests, vocabulary, stats)``: the recorded lists as ordered ``ItemList``s, the test lists, the Gini
    metrics' item vocabulary and MeanPopRank's item statistics."""
    g = reference_golden("metrics_cases")
    rp, tp = g["rec_ptr"], g["test_ptr"]
    recs = [ItemList(item_ids=g["recs"][rp[b] : rp[b + 1]], ordered=True) for b in range(len(rp) - 1)]
    tests = [ItemList(item_ids=g["tests"][tp[b] : tp[b + 1]]) for b in range(len(tp) - 1)]
    stats = pd.DataFrame({"user_count": g["user_count"], "count": g["count"]},
                         index=pd.Index(mrs.item_ids(), name="item_id"))  # fmt: skip
    return recs, tests, Vocabulary(mrs.item_ids(), "item"), stats


def metric(name: str, vocab, stats):
    return mrs.build(CLASSES, name, vocab, stats)


def same_bits(a, b) -> bool:
    """Equal f64 bits, with NaN in the same places (any NaN payload)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64)))


def test_recording_covers_the_cases():
    recs, tests, _v, _s = cases()
    lens = {len(r) for r in recs}
    assert {0, 1, 7, 8, 9, 127, 128, 129, 1024} <= lens
    assert any(len(t) == 0 and len(r) > 0 for r, t in zip(recs, tests))
    assert any(len(t) > len(r) > 0 for r, t in zip(recs, tests))
    assert any(mrs.UNKNOWN in t.ids() for t in tests) and any(len(np.unique(t.ids())) < len(t) for t in tests)
    assert not mrs.known([r.ids() for r in recs]).all()
    assert set(mrs.CONFIGS) == {k for k in reference_golden("metrics_values") if k in mrs.CONFIGS} | {
        k for k, (c, _kw) in mrs.CONFIGS.items() if c in mrs.GINI
    }


@pytest.mark.parametrize("name", [k for k, (c, _kw) in mrs.CONFIGS.items() if c not in mrs.GINI])
def test_list_metrics_are_the_reference(name):
    """Every list's ``measure_list`` bit for bit, NaN where the reference gives NaN, and ``ZeroDivisionError`` where
    it raises it."""
    g = reference_golden("metrics_values")
    recs, tests, vocab, stats = cases()
    m = metric(name, vocab, stats)
    got = np.full(len(recs), np.nan)
    for b, (r, t) in enumerate(zip(recs, tests)):
        if g[f"raised_{name}"][b]:
            with pytest.raises(ZeroDivisionError):
                m.measure_list(r, t)
            continue
        got[b] = m.measure_list(r, t)
    assert same_bits(got, g[name]), name


@pytest.mark.parametrize("name", [k for k, (c, _kw) in mrs.CONFIGS.items() if c in mrs.GINI])
def test_gini_metrics_are_the_reference(name):
    g = reference_golden("metrics_values")
    recs, tests, vocab, stats = cases()
    m = metric(name, vocab, stats)
    acc = m.create_accumulator()
    for r, t, k in zip(recs, tests, mrs.known([r.ids() for r in recs])):
        if k:
            acc.add(m.measure_list(r, t))
    assert same_bits(acc.totals, g[f"totals_{name}"])
    assert acc.accumulate() == float(g[f"gini_{name}"])


def test_labels_and_arguments():
    vocab = Vocabulary(np.arange(5))
    assert lm.NDCG().label == "NDCG" and lm.NDCG(10).label == "NDCG@10" and lm.Hit(n=3).label == "Hit@3"
    assert lm.AveragePrecision(5).label == "AveragePrecision@5" and lm.RBP().label == "RBP"
    assert lm.ListGini(4, items=vocab).label == "ListGini@4" and lm.ExposureGini(items=vocab).label == "ExposureGini"
    with pytest.warns(DeprecationWarning):
        assert lm.Recall(k=7).n == 7
    with pytest.raises(ValueError, match="positive"):
        lm.Precision(-1)
    with pytest.raises(ValueError):
        lm.GeometricRankWeight(1.0)
    with pytest.raises(ValueError):
        lm.LogRankWeight(offset=-1)
    assert lm.RBP(patience=0.5).weight.series_sum() == 2.0 and lm.LogRankWeight().series_sum() is None


def test_excluded_options_raise():
    with pytest.raises(ValueError, match="gain"):
        lm.NDCG(gain="rating")
    with pytest.raises(ValueError, match="gain"):
        lm.DCG(5, gain="rating")
    with pytest.raises(ValueError, match="weight_field"):
        lm.RBP(weight_field="w")


def test_unordered_lists_raise_as_the_reference():
    recs, test = ItemList(item_ids=[1, 2, 3]), ItemList(item_ids=[2])
    with pytest.raises(ValueError, match="ordered"):
        lm.Precision(2).measure_list(recs, test)
    with pytest.raises(TypeError, match="not ordered"):
        lm.DCG().measure_list(recs, test)
    assert lm.Precision().measure_list(recs, test) == 1 / 3


@pytest.mark.parametrize("weight", [lm.LogRankWeight(), lm.LogRankWeight(base=10, offset=3), lm.GeometricRankWeight(),
                                    lm.GeometricRankWeight(0.37), lm.DiscountWeight(np.log2)])  # fmt: skip
def test_weight_tables_are_elementwise(weight):
    """The device reads rank weights from one table per metric, ``weight(1 .. K)``: each entry must be what the
    reference's call on any subset of ranks, or a shorter range, gives for that rank."""
    rng = np.random.default_rng(3)
    table = weight.weight(np.arange(1, 1025, dtype=np.int32))
    for _ in range(50):
        K = int(rng.integers(0, 1025))
        ranks = np.arange(1, K + 1, dtype=np.int32)
        assert same_bits(weight.weight(ranks), table[:K])
        sub = ranks[rng.random(K) < rng.random()]
        assert same_bits(weight.weight(sub), table[sub - 1])


def test_item_counts_match_pandas():
    rng = np.random.default_rng(2)
    pairs = np.unique(rng.integers(0, 30, 400) * 50 + rng.integers(0, 50, 400))
    users, items = (pairs // 50).astype(np.int32), (pairs % 50).astype(np.int32)
    inter = Interactions(users, items, np.ones(len(users), np.float32), 30, 50)
    got = lm.item_counts(inter)
    df = pd.DataFrame({"u": users, "i": items})
    want = df.groupby("i")["u"].nunique().reindex(range(50), fill_value=0).to_numpy()
    assert np.array_equal(got["user_count"].to_numpy(), want) and np.array_equal(got["count"].to_numpy(), want)
    m = lm.MeanPopRank(inter)
    assert m.measure_list(ItemList(item_ids=[3, 4], ordered=True), ItemList(item_ids=[])) == (
        m.item_ranks[3] + m.item_ranks[4]) / 2  # fmt: skip


def test_host_summary_is_the_collector():
    """``measure_lists_host``'s summary: ``ValueStatAccumulator`` over the non-NaN values, and the Gini coefficient."""
    recs, tests, vocab, stats = cases()
    ms = [lm.NDCG(10), lm.Precision(), lm.ListGini(items=vocab)]
    keep = mrs.known([r.ids() for r in recs])
    recs = [r for r, k in zip(recs, keep) if k]
    tests = [t for t, k in zip(tests, keep) if k]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s, df = lm.measure_lists_host(ms, recs, tests)
    v = df["NDCG@10"].to_numpy()
    v = v[~np.isnan(v)]
    assert s["NDCG@10.n"] == len(v) and s["NDCG@10.mean"] == np.mean(v) and s["NDCG@10.median"] == np.median(v)
    assert s["NDCG@10.std"] == np.std(v) and "ListGini" in s and list(df.columns) == ["NDCG@10", "Precision"]


def test_ctypes_structs_match_header(tmp_path, monkeypatch):
    import test_flexmf

    monkeypatch.setattr(test_flexmf, "STRUCTS", {"lk_metric_spec": _lib.LkMetricSpec,
                                                 "lk_rank_metrics_args": _lib.LkRankMetricsArgs,
                                                 "lk_item_exposure_args": _lib.LkItemExposureArgs})  # fmt: skip
    _layout_check(tmp_path)


def test_entry_points_check_arguments_on_the_host(cuda_lib):
    a = _lib.LkRankMetricsArgs()
    a.n_lists, a.n_metrics = 4, 33
    assert cuda_lib.lk_rank_metrics(C.byref(a), None) == -1 and b"n_metrics" in cuda_lib.lk_last_error()
    a.n_metrics = 1
    a.metrics[0].kind = 9
    assert cuda_lib.lk_rank_metrics(C.byref(a), None) == -1 and b"kind" in cuda_lib.lk_last_error()
    a.metrics[0].kind, a.metrics[0].n = _lib.LK_METRIC_RBP, -2
    assert cuda_lib.lk_rank_metrics(C.byref(a), None) == -1 and b"truncation" in cuda_lib.lk_last_error()
    a.metrics[0].n, a.metrics[0].norm_mode = 5, 3
    assert cuda_lib.lk_rank_metrics(C.byref(a), None) == -1 and b"RBP" in cuda_lib.lk_last_error()
    a.metrics[0].norm_mode = _lib.LK_RBP_NORM_PREFIX
    assert cuda_lib.lk_rank_metrics(C.byref(a), None) == -1 and b"null list" in cuda_lib.lk_last_error()
    # never dereferenced: every check comes before a launch
    a.d_rec_indptr = a.d_rec_items = a.d_test_indptr = a.d_test_items = a.d_nrel = 8
    assert cuda_lib.lk_rank_metrics(C.byref(a), None) == -1 and b"tables" in cuda_lib.lk_last_error()
    z = _lib.LkRankMetricsArgs()
    assert cuda_lib.lk_rank_metrics(C.byref(z), None) == 0  # an empty batch does nothing
    e = _lib.LkItemExposureArgs()
    e.n_items, e.n_entries = -1, 0
    assert cuda_lib.lk_item_exposure(C.byref(e), None) == -1
    e.n_items, e.n_entries = 10, 5
    assert cuda_lib.lk_item_exposure(C.byref(e), None) == -1 and b"totals" in cuda_lib.lk_last_error()
    e.d_totals = 8
    assert cuda_lib.lk_item_exposure(C.byref(e), None) == -1 and b"entries" in cuda_lib.lk_last_error()
    e.d_sorted_items = e.d_order = e.d_entry_list = e.d_weights = 8
    assert cuda_lib.lk_item_exposure(C.byref(e), None) == -1 and b"d_entry_rank" in cuda_lib.lk_last_error()
    assert cuda_lib.lk_item_exposure(C.byref(_lib.LkItemExposureArgs()), None) == 0


def test_batch_checks_before_the_device(cuda_lib):
    """What ``measure_batch`` refuses before it needs a device."""
    with pytest.raises(TypeError, match="not a metric"):
        lm.measure_batch([object()], [], [])
