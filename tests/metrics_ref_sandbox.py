"""
The reference's own ranking metrics (``metrics/ranking/*.py``, their rank weights ``_weighting.py``, the metric base
classes ``metrics/_base.py``, ``data/accum`` and ``stats.gini``) on top of the sandbox of ``ref_sandbox``; and the
recording of their values on crafted lists that ``tests/golden/reference_classes/metrics_*.npz`` holds.

MeanPopRank reads ``Dataset.item_stats()``; ``_Stats`` below is that one call over recorded per-item counts.
Everything else, from the constructors to ``measure_list`` and the accumulators, is the reference's code.
"""

from __future__ import annotations

import contextlib
import warnings

import numpy as np

import ref_sandbox

#: the item vocabulary: ids 3, 10, 17, ...
N_ITEMS = 1500
#: an id outside the vocabulary (and outside every list)
UNKNOWN = -5


def item_ids() -> np.ndarray:
    return np.arange(N_ITEMS, dtype=np.int64) * 7 + 3


def item_stats() -> tuple[np.ndarray, np.ndarray]:
    """``(user_count, count)`` of every item: about a tenth of the items without any, ties among the rest."""
    rng = np.random.default_rng(11)
    users = rng.integers(0, 40, N_ITEMS)
    users[rng.random(N_ITEMS) < 0.1] = 0
    return users, users + rng.integers(0, 3, N_ITEMS) * (users > 0)


#: the metrics recorded, by name: (class name, constructor arguments); "weight" is a (class name, arguments) pair
CONFIGS: dict[str, tuple[str, dict]] = {
    "hit": ("Hit", {}), "hit_5": ("Hit", {"n": 5}), "hit_0": ("Hit", {"n": 0}),
    "precision": ("Precision", {}), "precision_3": ("Precision", {"n": 3}), "precision_130": ("Precision", {"n": 130}),
    "recall": ("Recall", {}), "recall_5": ("Recall", {"n": 5}), "recall_0": ("Recall", {"n": 0}),
    "recall_128": ("Recall", {"k": 128}),
    "recip": ("RecipRank", {}), "recip_10": ("RecipRank", {"n": 10}),
    "dcg": ("DCG", {}), "dcg_10": ("DCG", {"n": 10}),
    "dcg_log3_off1": ("DCG", {"weight": ("LogRankWeight", {"base": 3, "offset": 1})}),
    "ndcg": ("NDCG", {}), "ndcg_10": ("NDCG", {"n": 10}), "ndcg_0": ("NDCG", {"n": 0}),
    "ndcg_1000": ("NDCG", {"n": 1000}), "ndcg_129": ("NDCG", {"k": 129}),
    "ndcg_log10_off2": ("NDCG", {"n": 50, "weight": ("LogRankWeight", {"base": 10, "offset": 2})}),
    "ndcg_discount": ("NDCG", {"discount": "log2"}),
    "rbp": ("RBP", {}), "rbp_p5": ("RBP", {"patience": 0.5}), "rbp_20": ("RBP", {"n": 20, "patience": 0.95}),
    "rbp_norm": ("RBP", {"normalize": True}), "rbp_norm_8": ("RBP", {"n": 8, "normalize": True}),
    "rbp_log": ("RBP", {"weight": ("LogRankWeight", {})}),
    "rbp_log_norm": ("RBP", {"n": 100, "normalize": True, "weight": ("LogRankWeight", {"offset": 1})}),
    "rbp_geo_weight": ("RBP", {"weight": ("GeometricRankWeight", {"patience": 0.3})}),
    "ap": ("AveragePrecision", {}), "ap_10": ("AveragePrecision", {"n": 10}),
    "ap_129": ("AveragePrecision", {"n": 129}),
    "meanpop": ("MeanPopRank", {}), "meanpop_10": ("MeanPopRank", {"n": 10}),
    "meanpop_inter": ("MeanPopRank", {"count": "interactions"}),
    "listgini": ("ListGini", {}), "listgini_10": ("ListGini", {"n": 10}),
    "expgini": ("ExposureGini", {}), "expgini_5": ("ExposureGini", {"n": 5}),
    "expgini_p7": ("ExposureGini", {"weight": ("GeometricRankWeight", {"patience": 0.7})}),
    "expgini_log": ("ExposureGini", {"n": 200, "weight": ("LogRankWeight", {"base": 3})}),
}  # fmt: skip

GINI = ("ListGini", "ExposureGini")
LENGTHS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 31, 32, 33, 64, 127, 128, 129, 200, 511, 1024]


def lists() -> tuple[list[np.ndarray], list[np.ndarray]]:
    """``(recs, tests)``: for every length of ``LENGTHS``, lists of distinct known items with test sets that are
    empty, a random part of the list plus items outside it, the whole list, the whole list and 300 more items (test
    sets longer than the list), and a part with unknown and repeated ids; and lists holding unknown items."""
    rng = np.random.default_rng(5)
    ids = item_ids()
    recs, tests = [], []
    for L in LENGTHS:
        for variant in range(5):
            r = rng.permutation(ids)[:L]
            if variant == 0:
                t = np.zeros(0, np.int64)
            elif variant == 1:
                t = np.concatenate([rng.choice(r, int(rng.integers(0, L + 1)), replace=False) if L else r,
                                    rng.choice(np.setdiff1d(ids, r), 3, replace=False)])  # fmt: skip
            elif variant == 2:
                t = rng.permutation(r)
            elif variant == 3:
                t = np.concatenate([r, rng.choice(np.setdiff1d(ids, r), 300, replace=False)])
            else:
                part = r[rng.random(L) < 0.4]
                t = np.concatenate([part, part[: len(part) // 2], [UNKNOWN, UNKNOWN - 1, UNKNOWN]])
            recs.append(r)
            tests.append(rng.permutation(t))
    for L in (3, 40, 130):  # an unknown item in the list, in the test set too or not
        r = rng.permutation(ids)[:L].copy()
        r[L // 3] = UNKNOWN
        r[-1] = UNKNOWN - 7
        t = np.concatenate([r[: L // 2], [UNKNOWN - 7]])
        recs.append(r)
        tests.append(t)
    return recs, tests


def known(recs: list[np.ndarray]) -> np.ndarray:
    """The lists the Gini metrics can measure: every item known."""
    ids = item_ids()
    return np.array([np.isin(r, ids).all() for r in recs])


class _Stats:
    """``Dataset.item_stats()`` as MeanPopRank reads it."""

    def __init__(self, user_count, count):
        import pandas as pd

        self._df = pd.DataFrame({"user_count": user_count, "count": count}, index=pd.Index(item_ids(), name="item_id"))

    def item_stats(self):
        return self._df


def build(mods: dict, name: str, vocab, stats):
    """Metric ``name`` of ``CONFIGS`` from the classes in ``mods`` (``{class name: class}``): this package's or the
    reference's.  ``vocab`` is the Gini metrics' item vocabulary and ``stats`` MeanPopRank's data."""
    cls, kw = CONFIGS[name]
    kw = dict(kw)
    if "weight" in kw:
        wc, wkw = kw["weight"]
        kw["weight"] = mods[wc](**wkw)
    if "discount" in kw:
        kw["discount"] = getattr(np, kw["discount"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        if cls in GINI:
            return mods[cls](items=vocab, **kw)
        if cls == "MeanPopRank":
            return mods[cls](stats, **kw)
        return mods[cls](**kw)


@contextlib.contextmanager
def metric_modules():
    """``ref_sandbox.reference_modules()`` plus the ranking metrics; yields ``{class name: class}``."""
    with ref_sandbox.reference_modules() as mods:
        for pkg in ("lenskit.metrics", "lenskit.metrics.ranking", "lenskit.data.accum"):
            ref_sandbox._module(pkg, package=True)
        for name, rel in (
            ("lenskit.stats", "stats.py"),
            ("lenskit.data.accum._proto", "data/accum/_proto.py"),
            ("lenskit.data.accum._value", "data/accum/_value.py"),
        ):
            mods[name] = ref_sandbox._load(name, rel)
        acc = __import__("sys").modules["lenskit.data.accum"]
        acc.Accumulator, acc.AccumulatorFactory = mods["lenskit.data.accum._proto"].Accumulator, mods["lenskit.data.accum._proto"].AccumulatorFactory
        acc.ValueStatAccumulator = mods["lenskit.data.accum._value"].ValueStatAccumulator
        acc.ValueStatistics = mods["lenskit.data.accum._value"].ValueStatistics
        mods["lenskit.metrics._base"] = ref_sandbox._load("lenskit.metrics._base", "metrics/_base.py")
        classes = {}
        for leaf in ("_base", "_weighting", "_dcg", "_rbp", "_hit", "_pr", "_recip", "_map", "_pop", "_gini"):
            m = ref_sandbox._load(f"lenskit.metrics.ranking.{leaf}", f"metrics/ranking/{leaf}.py")
            classes.update({k: v for k, v in vars(m).items() if isinstance(v, type)})
        yield classes


def record() -> dict[str, dict]:
    """``metrics_cases``: the lists, test sets and item statistics.  ``metrics_values``: for every ``CONFIGS``
    entry, each list's ``measure_list`` value (NaN where it raises, with ``raised_<name>`` marking those), or for the
    Gini metrics the accumulator's totals and coefficient over the ``known`` lists."""
    recs, tests = lists()
    uc, cnt = item_stats()
    cases = {
        "rec_ptr": np.cumsum([0] + [len(r) for r in recs]), "recs": np.concatenate(recs).astype(np.int64),
        "test_ptr": np.cumsum([0] + [len(t) for t in tests]), "tests": np.concatenate(tests).astype(np.int64),
        "user_count": uc, "count": cnt,
    }  # fmt: skip
    values = {}
    with metric_modules() as ref:
        import sys

        ItemList, Vocabulary = sys.modules["lenskit.data"].ItemList, sys.modules["lenskit.data"].Vocabulary
        vocab = Vocabulary(item_ids(), "item")
        stats = _Stats(uc, cnt)
        outs = [ItemList(item_ids=r, ordered=True) for r in recs]
        tls = [ItemList(item_ids=t) for t in tests]
        ok = known(recs)
        for name, (cls, _kw) in CONFIGS.items():
            m = build(ref, name, vocab, stats)
            if cls in GINI:
                acc = m.create_accumulator()
                for o, t, k in zip(outs, tls, ok):
                    if k:
                        acc.add(m.measure_list(o, t))
                values[f"totals_{name}"] = acc.totals.copy()
                values[f"gini_{name}"] = np.array(acc.accumulate())
                continue
            v, raised = np.full(len(outs), np.nan), np.zeros(len(outs), bool)
            for b, (o, t) in enumerate(zip(outs, tls)):
                try:
                    with warnings.catch_warnings():
                        warnings.simplefilter("ignore")
                        v[b] = m.measure_list(o, t)
                except ZeroDivisionError:
                    raised[b] = True
            values[name], values[f"raised_{name}"] = v, raised
    return {"metrics_cases": cases, "metrics_values": values}
