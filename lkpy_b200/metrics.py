"""
Ranking metrics on the H100 engine — the metric classes of ``lenskit.metrics.ranking`` (``src/lenskit/metrics/
ranking/*.py``) and their rank weights (``_weighting.py``), with batched measurement of many lists on the device.

Each metric class keeps the reference's constructor arguments, ``label`` and a host ``measure_list(recs, test)``
that restates the reference's statements for one list.  :func:`measure_batch` measures many lists against their test
sets in one launch per call (``lk_rank_metrics``) and returns what ``MeasurementCollector.measure_run`` returns;
:func:`measure_topn` does the same from a top-n kernel's ``idx`` / ``cnt`` output without building ``ItemList``s.

What the device is given: the rank weights (``RankWeight.weight`` on the host, once per metric and batch), every
normaliser that depends only on a length (NDCG's ``fixed_dcg(m)`` for each distinct m, RBP's prefix sums), and
MeanPopRank's quantile per item.  It computes set membership, counts, and NumPy-order pairwise sums of those table
entries, bit for bit with ``measure_list``.  ListGini's and ExposureGini's per-item totals are summed on the device
in list order (``lk_item_exposure``); the Gini coefficient of the totals, and the summary statistics of the per-list
values, are the reference's host statements.

Not covered (``ValueError`` naming the option): graded gains (``gain=``, whose ``np.dot`` and pandas ``align`` order
is not reproduced) and RBP's ``weight_field=``.
"""

from __future__ import annotations

import warnings
from abc import ABC, abstractmethod
from collections.abc import Callable, Mapping
from typing import Annotated, Any, Literal, NamedTuple

import numpy as np
import pandas as pd
import torch
from annotated_types import Gt, Lt
from pydantic import NonNegativeInt, PositiveFloat, validate_call

from . import _lib, engine
from .batch import take
from .components import ItemList, Vocabulary, _as_dataset

# ---------------------------------------------------------------------------
# rank weights (_weighting.py)
# ---------------------------------------------------------------------------


class RankWeight(ABC):
    """Multiplicative weights of ranks (starting at 1)."""

    @abstractmethod
    def weight(self, ranks) -> np.ndarray: ...

    def log_weight(self, ranks) -> np.ndarray:
        return np.log(self.weight(ranks))

    def series_sum(self) -> float | None:
        """The sum of the infinite series of weights, where it is known."""
        return None


class GeometricRankWeight(RankWeight):
    """``patience ** (rank - 1)``, computed as ``exp(log(patience) * (rank - 1))``; its series sums to
    ``1 / (1 - patience)``."""

    @validate_call
    def __init__(self, patience: Annotated[float, Gt(0.0), Lt(1.0)] = 0.85):
        self.patience = patience

    def weight(self, ranks) -> np.ndarray:
        return np.exp(self.log_weight(ranks))

    def log_weight(self, ranks) -> np.ndarray:
        return np.log(self.patience) * (ranks - 1)

    def series_sum(self) -> float:
        return 1 / (1 - self.patience)


class LogRankWeight(RankWeight):
    """``log(base) / log(rank + offset)``, or with ``offset = 0`` the rank clipped below at 2."""

    @validate_call
    def __init__(self, *, base: PositiveFloat = 2, offset: NonNegativeInt = 0):
        self.base = base
        self.offset = offset

    def weight(self, ranks) -> np.ndarray:
        if self.offset > 0:
            return np.log(self.base) / np.log(ranks + self.offset)
        return np.log(self.base) / np.log(np.maximum(ranks, 2))


class DiscountWeight(RankWeight):
    """The weight of NDCG's and DCG's deprecated ``discount=``: ``1 / max(discount(ranks), 1)``."""

    def __init__(self, discount: Callable[[np.ndarray], np.ndarray]):
        self.discount = discount

    def weight(self, ranks) -> np.ndarray:
        return np.reciprocal(np.maximum(self.discount(ranks), 1))


# ---------------------------------------------------------------------------
# metric classes
# ---------------------------------------------------------------------------


def _ranks(items: ItemList) -> np.ndarray | None:
    """``ItemList.ranks()``: 1 .. len as int32 for an ordered list, None otherwise."""
    return np.arange(1, len(items) + 1, dtype=np.int32) if items.ordered else None


def _isin(recs: ItemList, test: ItemList) -> np.ndarray:
    """``recs.isin(test)``: which entries of ``recs`` have an id among ``test``'s."""
    return np.isin(recs.ids(), test.ids())


class Metric(ABC):
    @property
    def label(self) -> str:
        return self.__class__.__name__

    def __str__(self):
        return f"Metric {self.label}"

    @abstractmethod
    def measure_list(self, output: ItemList, test: ItemList, /) -> Any: ...


class RankingMetricBase(Metric):
    """The ``n`` truncation (``k=`` its deprecated alias) and the ``Name@n`` label."""

    n: int | None = None

    def __init__(self, n: int | None = None, *, k: int | None = None):
        if n is None and k is not None:
            warnings.warn("k= is deprecated, use n=", DeprecationWarning)
            n = k
        if n is not None and n < 0:
            raise ValueError("n must be positive or None")
        self.n = n

    @property
    def k(self):
        return self.n

    @property
    def label(self):
        name = self.__class__.__name__
        return f"{name}@{self.n}" if self.n is not None else name

    def truncate(self, items: ItemList) -> ItemList:
        if self.n is not None:
            if not items.ordered:
                raise ValueError("top-n filtering requires ordered list")
            if len(items) > self.n:
                return take(items, np.arange(self.n), ordered=items.ordered)
        return items


class ListMetric(Metric):
    """A metric with one value per list, summarised by :func:`value_statistics`."""


def _no_gain(gain):
    if gain is not None:
        raise ValueError(f"gain={gain!r}: graded gains are not supported by lkpy_b200.metrics")


class NDCG(ListMetric, RankingMetricBase):
    def __init__(self, n: int | None = None, *, k: int | None = None, weight: RankWeight = LogRankWeight(),
                 discount: Callable | None = None, gain: str | None = None):  # fmt: skip
        super().__init__(n, k=k)
        _no_gain(gain)
        self.weight = weight
        self.discount = discount
        if discount is not None:
            self.weight = DiscountWeight(discount)
        self.gain = gain

    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        recs = self.truncate(recs)
        if len(test) == 0:
            return np.nan
        realized = binary_dcg(recs, test, self.weight)
        n = len(test)
        if self.n and self.n < n:
            n = self.n
        return realized / fixed_dcg(n, self.weight)


class DCG(ListMetric, RankingMetricBase):
    def __init__(self, n: int | None = None, *, k: int | None = None, weight: RankWeight = LogRankWeight(),
                 discount: Callable | None = None, gain: str | None = None):  # fmt: skip
        super().__init__(n, k=k)
        _no_gain(gain)
        self.weight = weight
        self.discount = discount
        if discount is not None:
            self.weight = DiscountWeight(discount)
        self.gain = gain

    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        recs = self.truncate(recs)
        if len(test) == 0:
            return np.nan
        return binary_dcg(recs, test, self.weight)


def binary_dcg(recs: ItemList, test: ItemList, weight: RankWeight = LogRankWeight()) -> float:
    """The sum, in rank order, of the weights of the good ranks."""
    good = _isin(recs, test)
    ranks = _ranks(recs)
    if ranks is None:
        raise TypeError("item list is not ordered")
    return np.sum(weight.weight(ranks[good])).item()


def fixed_dcg(n: int, weight: RankWeight = LogRankWeight()) -> float:
    """The DCG of ``n`` good items: the sum of the weights of ranks 1 .. n."""
    return np.sum(weight.weight(np.arange(1, n + 1))).item()


class RBP(ListMetric, RankingMetricBase):
    def __init__(self, n: int | None = None, *, k: int | None = None, weight: RankWeight | None = None,
                 patience: float = 0.85, normalize: bool = False, weight_field: str | None = None):  # fmt: skip
        super().__init__(n, k=k)
        if weight_field is not None:
            raise ValueError(f"weight_field={weight_field!r}: field weights are not supported by lkpy_b200.metrics")
        self.patience = patience
        if weight is None:
            weight = GeometricRankWeight(patience)
        self.weight = weight
        self.normalize = normalize
        self.weight_field = weight_field

    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        recs = self.truncate(recs)
        k = len(recs)
        nrel = len(test)
        if nrel == 0:
            return np.nan
        good = _isin(recs, test)
        ranks = _ranks(recs)
        if ranks is None:
            raise TypeError("item list is not ordered")
        weights = self.weight.weight(ranks)
        wmax = self.weight.series_sum()
        if self.normalize:
            normalization = np.sum(weights[: min(nrel, k)]).item()
        elif wmax is not None:
            normalization = wmax
        else:
            normalization = np.sum(weights).item()
        return np.sum(weights[good]).item() / normalization


class RecipRank(ListMetric, RankingMetricBase):
    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        if len(test) == 0:
            return np.nan
        recs = self.truncate(recs)
        (npz,) = np.nonzero(_isin(recs, test))
        return 1.0 / (npz[0] + 1.0) if len(npz) else 0.0


class Hit(ListMetric, RankingMetricBase):
    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        if len(test) == 0:
            return np.nan
        recs = self.truncate(recs)
        return 1 if np.any(_isin(recs, test)) else 0


class Precision(ListMetric, RankingMetricBase):
    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        recs = self.truncate(recs)
        nrecs = len(recs)
        if nrecs == 0:
            return np.nan
        return _isin(recs, test).sum() / nrecs


class Recall(ListMetric, RankingMetricBase):
    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        recs = self.truncate(recs)
        ngood = _isin(recs, test).sum()
        nrel = len(test)
        if self.n is not None and self.n < nrel:
            nrel = self.n
        with np.errstate(invalid="ignore"):
            return ngood / nrel


class AveragePrecision(ListMetric, RankingMetricBase):
    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        recs = self.truncate(recs)
        nrecs = len(recs)
        if nrecs == 0:
            return np.nan
        good = _isin(recs, test)
        ranks = _ranks(recs)
        if ranks is None:
            raise TypeError("item list is not ordered")
        ap_sum = np.sum(np.cumsum(good)[good] / ranks[good]).item()
        return ap_sum / min(len(test), len(recs))


def item_counts(data) -> pd.DataFrame:
    """The ``user_count`` (distinct users) and ``count`` (interactions) of every item of ``data`` (this package's
    ``Dataset`` or ``Interactions``), indexed by item id in vocabulary order: the two columns of
    ``Dataset.item_stats()`` that MeanPopRank reads."""
    ds = _as_dataset(data)
    it = ds.interactions
    n = len(ds.items)
    items = np.asarray(it.items, dtype=np.int64)
    pairs = np.unique(items * max(int(it.n_users), 1) + np.asarray(it.users, dtype=np.int64))
    return pd.DataFrame({"count": np.bincount(items, minlength=n),
                         "user_count": np.bincount(pairs // max(int(it.n_users), 1), minlength=n)},
                        index=pd.Index(ds.items.ids(), name="item_id"))  # fmt: skip


class MeanPopRank(ListMetric, RankingMetricBase):
    """The mean popularity quantile of a list's items; ``data`` is this package's ``Dataset`` (or ``Interactions``),
    or a data frame of item statistics indexed by item id (``Dataset.item_stats()``)."""

    def __init__(self, data, *, n: int | None = None, k: int | None = None,
                 count: Literal["users", "interactions"] = "users"):  # fmt: skip
        super().__init__(n, k=k)
        stats = data if isinstance(data, pd.DataFrame) else item_counts(data)
        match count:
            case "users":
                counts = stats["user_count"]
            case "interactions":
                counts = stats["count"]
            case _:
                raise ValueError(f"invalid count {count}")
        pos = counts[counts > 0]
        ranks = pos.rank(method="average", ascending=True)
        ranks /= len(pos)
        self.item_ranks = ranks.reindex(counts.index, fill_value=0)

    def measure_list(self, recs: ItemList, test: ItemList) -> float:
        recs = self.truncate(recs)
        if len(recs) == 0:
            return np.nan
        return self.item_ranks.reindex(recs.ids(), fill_value=0).mean()


class GiniBase(RankingMetricBase):
    """A Gini coefficient over per-item totals of every list; ``items`` is the item vocabulary or a ``Dataset``."""

    def __init__(self, n: int | None = None, *, k: int | None = None, items):
        super().__init__(n, k=k)
        self.item_vocab = items.items if hasattr(items, "items") and isinstance(items.items, Vocabulary) else items

    def create_accumulator(self) -> GiniAccumulator:
        return GiniAccumulator(len(self.item_vocab))


class ListGini(GiniBase):
    """The Gini coefficient of the number of lists each item appears in."""

    def measure_list(self, output: ItemList, test) -> tuple[np.ndarray, float]:
        recs = self.truncate(output)
        return recs.numbers(vocabulary=self.item_vocab), 1.0


class ExposureGini(GiniBase):
    """The Gini coefficient of each item's total rank weight (exposure) over the lists."""

    def __init__(self, n: int | None = None, *, k: int | None = None, items, weight: RankWeight = GeometricRankWeight()):
        super().__init__(n=n, k=k, items=items)
        self.weight = weight

    def measure_list(self, output: ItemList, test) -> tuple[np.ndarray, np.ndarray]:
        recs = self.truncate(output)
        return recs.numbers(vocabulary=self.item_vocab), self.weight.weight(np.arange(1, len(recs) + 1, dtype=np.int32))


def gini(xs) -> float:
    """The Gini coefficient of ``xs`` (``lenskit.stats.gini``)."""
    xs = np.asarray(xs)
    n = len(xs)
    xs = np.sort(xs)
    ranks = np.arange(1, n + 1, dtype=np.float64)
    ranks *= 2
    ranks -= n + 1
    num = np.sum(xs * ranks)
    denom = n * np.sum(xs, dtype=np.float64)
    return max(num / denom, 0)


class GiniAccumulator:
    """Per-item totals, added to one list at a time, and their Gini coefficient."""

    def __init__(self, n: int):
        self.n_items = n
        self.totals = np.zeros(n)

    def add(self, value) -> None:
        items, values = value
        self.totals[items] += values

    def accumulate(self) -> float:
        with np.errstate(invalid="ignore", divide="ignore"):
            return gini(self.totals / self.totals.sum())


def value_statistics(values: np.ndarray) -> dict[str, float | int]:
    """``ValueStatAccumulator.accumulate`` over the non-NaN ``values``, in list order."""
    v = np.asarray(values, dtype=np.float64)
    v = v[~np.isnan(v)]
    n = len(v)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return {"n": n, "mean": np.mean(v).item(), "median": np.median(v).item(), "std": np.std(v).item()}


class RunMetrics(NamedTuple):
    """What ``MeasurementCollector.measure_run`` returns: flattened summaries, and one row of values per list."""

    summary_metrics: Mapping[str, Any]
    list_metrics: pd.DataFrame


_KINDS = {Hit: _lib.LK_METRIC_HIT, Precision: _lib.LK_METRIC_PRECISION, Recall: _lib.LK_METRIC_RECALL,
          RecipRank: _lib.LK_METRIC_RECIP_RANK, DCG: _lib.LK_METRIC_DCG, NDCG: _lib.LK_METRIC_NDCG,
          RBP: _lib.LK_METRIC_RBP, AveragePrecision: _lib.LK_METRIC_AP, MeanPopRank: _lib.LK_METRIC_MEAN_POP_RANK}  # fmt: skip
#: the metrics that read ranks (an unordered list raises even without a truncation)
_RANKED = (DCG, NDCG, RBP, AveragePrecision)


def measure_lists_host(metrics, outputs: list[ItemList], tests: list[ItemList]) -> RunMetrics:
    """The reference's per-list path: every metric's ``measure_list`` on every list, accumulated as
    ``MeasurementCollector`` does.  The oracle of :func:`measure_batch`."""
    values = {m.label: [] for m in metrics if not isinstance(m, GiniBase)}
    accs = {m.label: m.create_accumulator() for m in metrics if isinstance(m, GiniBase)}
    for out, test in zip(outputs, tests, strict=True):
        for m in metrics:
            v = m.measure_list(out, test)
            if isinstance(m, GiniBase):
                accs[m.label].add(v)
            else:
                values[m.label].append(v)
    return _run_metrics(metrics, {k: np.asarray(v, dtype=np.float64) for k, v in values.items()},
                        {k: a.accumulate() for k, a in accs.items()}, len(outputs))  # fmt: skip


def _run_metrics(metrics, values: dict, ginis: dict, B: int) -> RunMetrics:
    summary: dict[str, Any] = {}
    for m in metrics:
        if isinstance(m, GiniBase):
            summary[m.label] = ginis[m.label]
        else:
            for k, v in value_statistics(values[m.label]).items():
                summary[f"{m.label}.{k}"] = v
    df = pd.DataFrame({k: v for k, v in values.items()}, index=pd.RangeIndex(B))
    return RunMetrics(summary, df)


# ---------------------------------------------------------------------------
# batched measurement
# ---------------------------------------------------------------------------


def _check_metrics(metrics) -> None:
    for m in metrics:
        if type(m) not in _KINDS and not isinstance(m, GiniBase):
            raise TypeError(f"{m!r} is not a metric of lkpy_b200.metrics")


def _test_csr(tests: list[ItemList], vocabulary: Vocabulary, dev):
    """The test sets as a device CSR of ascending unique known item numbers, and ``nrel`` (each test list's
    length, unknown and repeated ids included).  Integer ids are numbered, and each set sorted, on the device."""
    B, V = len(tests), max(len(vocabulary), 1)
    nrel = np.array([len(t) for t in tests], dtype=np.int64)
    ids = [t.ids() for t in tests if len(t)]
    ids = np.concatenate(ids) if ids else np.zeros(0, np.int64)
    vids = vocabulary.ids()
    if vocabulary._sorted and len(vids) and ids.dtype.kind in "iu" and vids.dtype.kind in "iu":
        vid = torch.from_numpy(vids.astype(np.int64)).to(dev)
        q = torch.from_numpy(ids.astype(np.int64)).to(dev)
        pos = torch.searchsorted(vid, q).clamp_max(len(vids) - 1)
        nums = torch.where(vid[pos] == q, pos, -1)
    else:
        nums = torch.from_numpy(vocabulary.numbers(ids, missing="negative").astype(np.int64)).to(dev)
    d_nrel = torch.from_numpy(nrel).to(dev)
    owner = torch.repeat_interleave(torch.arange(B, dtype=torch.int64, device=dev), d_nrel, output_size=len(ids))
    keep = nums >= 0
    key = torch.unique(owner[keep] * V + nums[keep], sorted=True)
    owner, items = key // V, key % V
    indptr = torch.zeros(B + 1, dtype=torch.int64, device=dev)
    torch.cumsum(torch.bincount(owner, minlength=B), 0, out=indptr[1:])
    return indptr, items.to(torch.int32), d_nrel, nrel


def _lengths(m, lens: np.ndarray) -> np.ndarray:
    return lens if m.n is None else np.minimum(lens, m.n)


def _measure(metrics, vocabulary: Vocabulary, rec_indptr: torch.Tensor, rec_items: torch.Tensor, lens: np.ndarray,
             ordered: np.ndarray, tests: list[ItemList]) -> RunMetrics:  # fmt: skip
    """The shared core: the lists as a device CSR of item numbers of ``vocabulary`` (``lens`` on the host)."""
    B = len(lens)
    if len(tests) != B:
        raise ValueError(f"{B} lists but {len(tests)} test lists")
    dev = rec_indptr.device
    n_max = int(_lib.lib().lk_topn_max())
    for m in metrics:
        if m.n is not None and not ordered.all():
            raise ValueError("top-n filtering requires ordered list")
        if isinstance(m, _RANKED) and not ordered.all():
            raise TypeError("item list is not ordered")
        if B and _lengths(m, lens).max() > n_max:
            raise ValueError(f"{m.label}: lists of more than {n_max} items are not supported")
    test_indptr, test_items, d_nrel, nrel = _test_csr(tests, vocabulary, dev)

    specs, weights, norms = [], [np.zeros(0)], [np.zeros(0)]
    w_off = n_off = 0
    list_metrics = [m for m in metrics if not isinstance(m, GiniBase)]
    for m in list_metrics:
        k = _lengths(m, lens)
        sp = {"kind": _KINDS[type(m)], "n": -1 if m.n is None else int(m.n), "weight_offset": w_off,
              "norm_offset": n_off, "norm_mode": 0, "series_sum": 0.0}  # fmt: skip
        w = norm = np.zeros(0)
        if isinstance(m, (DCG, NDCG, RBP)):
            w = m.weight.weight(np.arange(1, int(k.max(initial=0)) + 1, dtype=np.int32))
        if isinstance(m, NDCG):
            mm = np.where((nrel > m.n) if m.n else np.zeros(B, bool), m.n or 0, nrel)[nrel > 0]
            norm = np.zeros(int(mm.max(initial=0)) + 1)
            for v in np.unique(mm):
                norm[v] = fixed_dcg(int(v), m.weight)
            if np.any(norm[mm] == 0):
                raise ZeroDivisionError("float division by zero")
        elif isinstance(m, RBP):
            wmax = m.weight.series_sum()
            if m.normalize or wmax is None:
                sp["norm_mode"] = _lib.LK_RBP_NORM_PREFIX if m.normalize else _lib.LK_RBP_NORM_LIST
                norm = np.array([np.sum(w[:j]).item() for j in range(len(w) + 1)])
                idx = np.minimum(k, nrel) if m.normalize else k
                if np.any(norm[idx[nrel > 0]] == 0):
                    raise ZeroDivisionError("float division by zero")
            else:
                sp["series_sum"] = float(wmax)
        elif isinstance(m, AveragePrecision):
            if np.any((k > 0) & (nrel == 0)):
                raise ZeroDivisionError("division by zero")
        elif isinstance(m, MeanPopRank):
            w = m.item_ranks.reindex(vocabulary.ids(), fill_value=0).to_numpy(dtype=np.float64)
        specs.append(sp)
        weights.append(np.asarray(w, np.float64))
        norms.append(np.asarray(norm, np.float64))
        w_off += len(w)
        n_off += len(norm)
    out = engine.rank_metrics(specs, rec_indptr, rec_items, test_indptr, test_items, d_nrel,
                              np.concatenate(weights), np.concatenate(norms))  # fmt: skip
    out = out.cpu().numpy()
    values = {m.label: out[j] for j, m in enumerate(list_metrics)}
    ginis = {m.label: _gini_totals(m, vocabulary, rec_indptr, rec_items, lens).accumulate()
             for m in metrics if isinstance(m, GiniBase)}  # fmt: skip
    return _run_metrics(metrics, values, ginis, B)


def _gini_totals(m: GiniBase, vocabulary: Vocabulary, rec_indptr, rec_items, lens) -> GiniAccumulator:
    """The metric's accumulator with its per-item totals summed on the device."""
    dev = rec_items.device
    B = len(lens)
    d_lens = torch.from_numpy(lens.astype(np.int64)).to(dev)
    lists = torch.repeat_interleave(torch.arange(B, dtype=torch.int32, device=dev), d_lens, output_size=int(lens.sum()))
    ranks = (torch.arange(rec_items.numel(), dtype=torch.int64, device=dev) - rec_indptr[:-1].repeat_interleave(d_lens)).int()
    keep = ranks < (m.n if m.n is not None else np.iinfo(np.int32).max)
    items = rec_items
    if not (m.item_vocab is vocabulary or m.item_vocab == vocabulary):
        remap = torch.from_numpy(m.item_vocab.numbers(vocabulary.ids(), missing="negative").astype(np.int32)).to(dev)
        items = torch.where(items >= 0, remap[items.clamp_min(0).long()], -1)
    items, lists, ranks = items[keep], lists[keep], ranks[keep]
    if bool((items < 0).any()):
        raise KeyError("unknown ids")
    acc = m.create_accumulator()
    w = None
    if isinstance(m, ExposureGini):
        w = m.weight.weight(np.arange(1, int(_lengths(m, lens).max(initial=0)) + 1, dtype=np.int32))
    acc.totals = engine.item_exposure(len(m.item_vocab), items.int(), lists, ranks, w).cpu().numpy()
    return acc


def _shared_vocabulary(outputs: list[ItemList]) -> Vocabulary | None:
    v = outputs[0]._vocab if outputs else None
    if v is None or any(o._vocab is not v and o._vocab != v for o in outputs):
        return None
    return v


def measure_batch(metrics, outputs: list[ItemList], tests: list[ItemList]) -> RunMetrics:
    """
    Every metric of ``metrics`` on every list of ``outputs`` against the test list of the same index, on the device:
    ``RunMetrics(summary, list_metrics)`` as ``MeasurementCollector.measure_run`` returns it (a missing test set is
    an empty ``ItemList``).  The per-list values are bit for bit those of ``measure_list``, and the summaries are the
    reference's statements over them: ``n``, ``mean``, ``median`` and ``std`` of the non-NaN values of a list metric
    (``"{label}.mean"`` ...), and the Gini coefficient of ListGini's and ExposureGini's totals (``label``).

    Items are numbered by the lists' shared vocabulary, or by the union of their ids when they have none.  Where the
    reference divides a Python float by zero (AveragePrecision of a list with an empty test set, RBP normalised over
    an empty list) this raises ``ZeroDivisionError`` as it does.
    """
    _check_metrics(metrics)
    dev = _lib.require_device()
    vocab = _shared_vocabulary(outputs)
    lens = np.array([len(o) for o in outputs], dtype=np.int64)
    if vocab is not None:
        nums = [o.numbers(vocabulary=vocab) for o in outputs]
        items = np.concatenate(nums).astype(np.int32) if nums else np.zeros(0, np.int32)
    else:
        ids = np.concatenate([o.ids() for o in outputs]) if outputs else np.zeros(0, np.int64)
        vocab = Vocabulary(np.unique(ids))
        items = vocab.numbers(ids).astype(np.int32)
    indptr = np.zeros(len(outputs) + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(lens)
    ordered = np.array([o.ordered for o in outputs], dtype=bool)
    return _measure(metrics, vocab, torch.from_numpy(indptr).to(dev), torch.from_numpy(items).to(dev), lens, ordered,
                    tests)  # fmt: skip


def measure_topn(metrics, vocabulary: Vocabulary, idx: torch.Tensor, cnt: torch.Tensor,
                 tests: list[ItemList]) -> RunMetrics:  # fmt: skip
    """
    :func:`measure_batch` of the ranked lists a top-n kernel returned (``batch.py``: ``idx [B, n]`` item numbers of
    ``vocabulary``, ``cnt [B]`` their counts, on the device), without building an ``ItemList`` per list.
    """
    _check_metrics(metrics)
    _lib.require_device()
    if idx.dim() != 2 or cnt.dim() != 1 or cnt.shape[0] != idx.shape[0]:
        raise ValueError("idx must be [B, n] and cnt [B]")
    dev = idx.device
    cnt64 = cnt.to(torch.int64)
    indptr = torch.zeros(idx.shape[0] + 1, dtype=torch.int64, device=dev)
    torch.cumsum(cnt64, 0, out=indptr[1:])
    keep = torch.arange(idx.shape[1], device=dev)[None, :] < cnt64[:, None]
    items = idx.to(torch.int32)[keep].contiguous()
    lens = cnt64.cpu().numpy()
    return _measure(metrics, vocabulary, indptr, items, lens, np.ones(len(lens), dtype=bool), tests)
