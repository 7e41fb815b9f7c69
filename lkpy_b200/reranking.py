"""
FA*IR re-ranking on the H100 engine — the component surface of ``lenskit.reranking.FAIRReranker``
(``src/lenskit/reranking/fair.py``; Zehlike et al. 2017, https://doi.org/10.1145/3132847.3132938).

Same config (:class:`FAIRRerankerConfig`: ``n``, ``p``, ``alpha``, ``protected_attribute``), the same ``train`` and
the same ``__call__``; plus ``rerank_batch`` for many ranked lists and ``rank_scores``, which selects each query's top
``candidates`` from a device score matrix and re-ranks them in one kernel (``lk_fair_rerank``).

Training is host code of at most ``n`` steps per probe: the corrected significance ``alpha_c`` is found by bisection
on [0, 1] (at most 100 probes, tolerance 1e-10 on both stopping tests, the midpoint of the last bracket), each probe
taking the rejection probability of ``m(i) = clip(binom.ppf(alpha_c, i, p), 0, i)``: one binomial pmf convolved in
per block of positions ending where ``m`` steps up, the bucket of the block's rank zeroed after each.  ``m_list`` is
``m(1..n)`` at ``alpha_c``.

The merge reads only positions: with the list split into a protected and an unprotected queue in list order, step i
takes the protected head while fewer than ``m_list[i]`` protected items have been taken, else the earlier head.
Items outside the trained vocabulary count as unprotected.
"""

from __future__ import annotations

import logging
from typing import Literal

import numpy as np
import torch
from pydantic import BaseModel, Field, PositiveInt
from scipy.stats import binom

from . import _lib, engine
from .batch import check_exclude, history_csr, take
from .components import Component, ItemList, RecQuery, Trainable, TrainingOptions, _as_dataset

_log = logging.getLogger(__name__)


class FAIRRerankerConfig(BaseModel, extra="forbid"):
    n: PositiveInt
    "The length of the re-ranked lists the thresholds are computed for."
    p: float = Field(0.5, gt=0.0, lt=1.0)
    "The target proportion of protected items."
    alpha: float = Field(0.1, gt=0.0, lt=1.0)
    "The significance of the test across all prefixes."
    protected_attribute: str = "protected"
    "The item attribute that is True for protected items."


# ---------------------------------------------------------------------------
# training: alpha_c and m_list
# ---------------------------------------------------------------------------


def minimum_protected(n: int, p: float, alpha: float) -> np.ndarray:
    """``m(i)`` for i = 1..n: the largest protected count of an i-prefix that a binomial test at ``alpha`` rejects
    (``binom.ppf``), clipped to 0..i."""
    i = np.arange(1, n + 1)
    return np.clip(binom.ppf(alpha, i, p), 0, i).astype(int)


def rejection_probability(n: int, p: float, alpha_c: float, pmfs: dict) -> float:
    """The probability that a fair ranking of ``n`` fails one of the prefix tests at ``alpha_c``.  The blocks are the
    runs of positions between the steps of ``m``; after convolving block j's ``Bin(size, p)`` pmf into the
    distribution of protected counts, the count ``j - 1`` fails and its bucket is zeroed.  ``pmfs`` caches the pmfs
    by block size."""
    m = minimum_protected(n, p, alpha_c)
    dist = np.array([1.0])
    if m[-1] > 0:
        steps = np.flatnonzero(np.diff(m, prepend=0)) + 1
        for j, size in enumerate(np.diff(steps, prepend=0)):
            if size not in pmfs:
                pmfs[size] = binom.pmf(np.arange(size + 1), size, p)
            dist = np.convolve(pmfs[size], dist)
            dist[j] = 0
    return float(1 - dist.sum())


def adjusted_significance(n: int, p: float, alpha: float, tolerance: float = 1e-10, max_iter: int = 100) -> float:
    """``alpha_c``: bisection on [0, 1] for the significance whose rejection probability is ``alpha``."""
    lo, hi = 0, 1
    pmfs: dict = {}
    for _ in range(max_iter):
        mid = (lo + hi) / 2
        r = rejection_probability(n, p, mid, pmfs)
        if r > alpha:
            hi = mid
        else:
            lo = mid
        if abs(r - alpha) < tolerance or hi - lo < tolerance:
            break
    return (lo + hi) / 2


# ---------------------------------------------------------------------------
# the merge
# ---------------------------------------------------------------------------


def fair_merge(protected: np.ndarray, m_list, length: int) -> np.ndarray:
    """The positions the FA*IR merge picks from a list with flags ``protected``, ``length`` of them (at most the
    list's length)."""
    prot, unprot = np.flatnonzero(protected), np.flatnonzero(~np.asarray(protected, dtype=bool))
    a = b = 0  # heads of the two queues
    out = np.empty(max(length, 0), dtype=np.int64)
    for i in range(len(out)):
        if a < len(prot) and (a < m_list[i] or b == len(unprot) or prot[a] < unprot[b]):
            out[i] = prot[a]
            a += 1
        else:
            out[i] = unprot[b]
            b += 1
    return out


class FAIRReranker(Component, Trainable):
    """
    ``FAIRReranker``: ``__call__(items, n)`` re-ranks one sorted list so that every prefix holds at least
    ``m_list`` protected items.  :meth:`rerank_batch` re-ranks many lists in one launch, and :meth:`rank_scores`
    takes each query's top ``candidates`` from a device score matrix and re-ranks them in the same kernel.
    """

    CONFIG_CLASS = FAIRRerankerConfig
    config: FAIRRerankerConfig

    alpha_c: float
    m_list: np.ndarray
    protected_attributes: np.ndarray
    "One bool per item of ``vocab``."

    def is_trained(self) -> bool:
        return hasattr(self, "alpha_c")

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        """``alpha_c`` and ``m_list`` for the configured ``(n, p, alpha)``, and the protected flag of every item:
        the item attribute ``protected_attribute`` equal to True.  ``data`` is this package's ``Dataset`` (its
        ``item_attributes``) or a LensKit ``Dataset`` (``entities("item").attribute(name)``)."""
        c = self.config
        self.alpha_c = adjusted_significance(c.n, c.p, c.alpha)
        self.m_list = minimum_protected(c.n, c.p, self.alpha_c)
        name = c.protected_attribute
        missing = ValueError(f"Dataset is missing required '{name}' attribute for item entities")
        if hasattr(data, "entities"):
            items = data.entities("item")
            if name not in items.attributes:
                raise missing
            values, self.vocab = items.attribute(name).numpy(), items.vocabulary
        else:
            ds = _as_dataset(data)
            if name not in ds.item_attributes:
                raise missing
            values, self.vocab = np.asarray(ds.item_attributes[name]), ds.items
            if len(values) != len(self.vocab):
                raise ValueError(f"attribute '{name}' has {len(values)} values for {len(self.vocab)} items")
        self.protected_attributes = np.equal(values, True)

    def _flags(self, items: ItemList) -> np.ndarray:
        """One protected flag per position of ``items``; unknown items are unprotected."""
        nums = np.asarray(items.numbers(vocabulary=self.vocab, missing="negative"))
        flags = np.zeros(len(items), dtype=bool)
        known = nums >= 0
        flags[known] = self.protected_attributes[nums[known]]
        return flags

    def _item_flags(self, vocabulary) -> np.ndarray:
        """One protected flag per item of ``vocabulary``."""
        if vocabulary is self.vocab or vocabulary == self.vocab:
            return self.protected_attributes
        nums = np.asarray(self.vocab.numbers(vocabulary.ids(), missing="negative"))
        flags = np.zeros(len(vocabulary), dtype=bool)
        flags[nums >= 0] = self.protected_attributes[nums[nums >= 0]]
        return flags

    def _n(self, n: int | None) -> int:
        """The call's ``n`` (0 or None: the config's); larger than the config's is an error, smaller a warning."""
        nc = self.config.n
        if n is not None:
            if n > nc:
                raise ValueError(f"The requested rerank length n={n}, exceeds configured n={nc}.")
            if n < nc:
                _log.warning("FA*IR: model trained for n=%d used on n=%d; fairness test might be violated.", nc, n)
        return n or nc

    def __call__(self, items: ItemList, n: int | None = None) -> ItemList:
        """The first ``min(n, len(items))`` entries of the merge, with every field of ``items``, marked ordered.  One
        list is at most ``n`` host steps; :meth:`rerank_batch` runs many on the device."""
        pos = fair_merge(self._flags(items), self.m_list, min(self._n(n), len(items)))
        return take(items, pos, ordered=True)

    def rerank_batch(self, lists: list[ItemList], n: int | None = None) -> list[ItemList]:
        """``[self(items, n) for items in lists]`` in one launch (the ``n`` rules and warning apply once).  The length
        is at most ``lk_topn_max()``; a longer one raises ``ValueError``."""
        k = self._n(n)
        lens = np.array([max(min(k, len(it)), 0) for it in lists], dtype=np.int32)
        width = int(lens.max(initial=0))
        if width == 0:
            return [take(it, np.zeros(0, np.int64), ordered=True) for it in lists]
        n_max = int(_lib.lib().lk_topn_max())
        if width > n_max:
            raise ValueError(f"n={width} exceeds the engine limit of {n_max}")
        flags = [self._flags(it) for it in lists]
        indptr = np.zeros(len(lists) + 1, dtype=np.int64)
        indptr[1:] = np.cumsum([len(f) for f in flags])
        idx, _val, _cnt = engine.fair_rerank(self.m_list, width, np.concatenate(flags), indptr=indptr, lengths=lens)
        idx = idx.cpu().numpy()
        return [take(it, idx[b, : lens[b]].astype(np.int64), ordered=True) for b, it in enumerate(lists)]

    def rank_scores(self, scores: torch.Tensor, queries, vocabulary, n: int | None = None, *, candidates: int,
                    exclude: Literal["query"] | None = "query") -> list[ItemList]:  # fmt: skip
        """
        ``TopNRanker(n=candidates)`` followed by ``self(list, n)`` for each query, from the device matrix ``scores``
        [B, n_items] (f32, any strides, such as ``scorer.score_matrix(queries).T``) without copying it to the host.
        Query b's candidates are argtopn's top ``candidates`` of row b over ``vocabulary``, minus its
        ``query_items`` when ``exclude="query"``; NaN scores are never candidates.  Returns ordered ``ItemList``s
        with ``score``.  ``candidates`` above ``lk_topn_max()`` raises ``ValueError``.
        """
        check_exclude(exclude)
        queries = [RecQuery.create(q) for q in queries]
        n_max = int(_lib.lib().lk_topn_max())
        if not 1 <= int(candidates) <= n_max:
            raise ValueError(f"candidates={candidates} must be in 1..{n_max}")
        if scores.dim() != 2 or scores.shape[0] != len(queries) or scores.shape[1] != len(vocabulary):
            raise ValueError(f"scores must be [{len(queries)}, {len(vocabulary)}], not {list(scores.shape)}")
        width = min(self._n(n), int(candidates))
        if width < 1:  # a negative n: every list is empty
            return [ItemList(item_ids=vocabulary.ids(np.zeros(0, np.int32)), item_nums=np.zeros(0, np.int32),
                             vocabulary=vocabulary, scores=np.zeros(0, np.float32), ordered=True) for _ in queries]  # fmt: skip
        excl = history_csr(queries, vocabulary, scores.device)[1:] if exclude == "query" else (None, None)
        idx, val, cnt = engine.fair_rerank(self.m_list, width, self._item_flags(vocabulary), scores=scores,
                                           candidates=int(candidates), excl_indptr=excl[0], excl_items=excl[1])  # fmt: skip
        idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy()
        out = []
        for b in range(len(queries)):
            c = int(cnt[b])
            nums = idx[b, :c].copy()
            out.append(ItemList(item_ids=vocabulary.ids(nums), item_nums=nums, vocabulary=vocabulary,
                                scores=val[b, :c].copy(), ordered=True))  # fmt: skip
        return out
