"""
Bias and popularity scorers on the H100 engine — the component surface of ``lenskit.basic.BiasScorer`` and
``PopScorer`` (``src/lenskit/basic/bias.py``, ``popularity.py``): the two baselines that run beside most models.

Same configs (``BiasConfig.entities`` / ``damping``, ``PopConfig.score``), the same trained attributes
(``BiasScorer.model``, a :class:`BiasModel`; ``PopScorer.items`` and ``item_scores``) and the same
``__call__``; plus ``score_batch`` and ``recommend_batch``.  :class:`BiasModel` is also the bias model of BiasedMF
and BiasedSVD.

``BiasScorer.train`` is ``BiasModel.learn`` on the device (``lk_bias_learn``), bit for bit with the host statements
on the f32 rating matrix: NumPy's pairwise mean, then each entity's ``np.add.at`` sum in COO order and the f64
quotient rounded to f32.  ``PopScorer.train`` counts on the device and runs the reference's pandas statements for
``rank`` and ``quantile`` on the host (one value per item).

Both score ``s(q, i) = f32(f64(base[i]) + offset[q])`` on ``lk_offset_score_batch``, which also ranks every item
through argtopn's heap (ties included) without a score matrix:

* ``BiasScorer``: ``base = f32(g) + ib`` (f32), the offset the user's bias, the bias of the query's ratings
  (:meth:`BiasModel.user_bias_for_items`, NaN counted as 0) or 0 for an unknown user.  That is the reference's
  ``scores += user_bias``: an f64 bias is added in f64 and rounded once, an f32 one gives the f32 sum.  An item
  the model does not know scores ``f32(g)`` plus the offset, as in the reference, not NaN.
* ``PopScorer``: ``base = item_scores`` and no offset; an unknown item scores NaN.
"""

from __future__ import annotations

from typing import Annotated, Literal

import numpy as np
import pandas as pd
import torch
from pydantic import BaseModel, NonNegativeFloat, PlainSerializer

from . import _lib, engine
from .batch import check_exclude, empty_list, history_csr, rank_size, ranked_lists, target_scores
from .components import Component, ItemList, RecQuery, Trainable, TrainingOptions, _as_dataset
from .data import Interactions
from .prep import coo_to_csr_pair

ENTITIES = frozenset({"user", "item"})


class BiasModel:
    """The part of ``lenskit.basic.BiasModel`` (basic/bias.py:84-150, 216-230) the bias, BiasedMF and BiasedSVD
    scorers need.  :meth:`learn` is the host statement of :func:`learn`, and its oracle."""

    def __init__(self, global_bias, item_biases, user_biases, damping):
        self.global_bias = global_bias
        self.item_biases = item_biases
        self.user_biases = user_biases
        self.damping = damping

    @classmethod
    def learn(cls, it: Interactions, damping, centered_dtype=np.float64, entities=("user", "item")) -> "BiasModel":
        """``damping``: one float for both, a ``(user, item)`` tuple, or a dict ``{"user": ..., "item": ...}`` in
        which a missing key means 0.  ``centered_dtype`` is the type of the centred ratings, which the reference
        takes from its rating matrix: ``np.float32`` gives its statements on an f32 matrix exactly.  ``entities``
        names the biases to learn; one left out is None."""
        if isinstance(damping, dict):
            damping = (float(damping.get("user", 0.0)), float(damping.get("item", 0.0)))
        d_user, d_item = damping if isinstance(damping, tuple) else (damping, damping)
        g = float(np.mean(it.ratings))
        centered = it.ratings.astype(centered_dtype) - g
        ib = ub = None
        if "item" in entities:
            counts = np.full(it.n_items, float(d_item))
            sums = np.zeros(it.n_items)
            np.add.at(counts, it.items, 1)
            np.add.at(sums, it.items, centered)
            ib = np.zeros(it.n_items, dtype=np.float32)
            np.divide(sums, counts, out=ib, where=counts > 0, casting="unsafe")
            centered = centered - ib[it.items]
        if "user" in entities:
            counts = np.full(it.n_users, float(d_user))
            sums = np.zeros(it.n_users)
            np.add.at(counts, it.users, 1)
            np.add.at(sums, it.users, centered)
            ub = np.zeros(it.n_users, dtype=np.float32)
            np.divide(sums, counts, out=ub, where=counts > 0, casting="unsafe")
        return cls(g, ib, ub, (d_user, d_item))

    def user_bias_for_items(self, item_nums: np.ndarray | None, ratings: np.ndarray) -> float:
        """
        The user bias ``compute_for_items`` takes from a query's rated items (basic/bias.py:216-230): the damped mean
        of ``rating - g - ib[item]``, with ``ib`` subtracted for the known items (``item_nums >= 0``; ``item_nums``
        may be None for a model without item biases).  Ratings that are not finite are left out of the count, and a
        NaN result counts as 0.  The arithmetic is in the dtype of ``ratings``, which the caller chooses.
        """
        uoff = ratings - self.global_bias
        if self.item_biases is not None:
            known = item_nums >= 0
            uoff[known] -= self.item_biases[item_nums[known]]
        ub = np.sum(uoff) / (np.sum(np.isfinite(uoff)) + self.damping[0])
        return 0.0 if np.isnan(ub) else float(ub)

    def batch_offsets(self, user_nums: np.ndarray, fold_bias: np.ndarray | None):
        """``compute_for_items`` for a batch, as score offsets: global + item bias per item (f32, the global bias
        rounded to f32 first), and per query the user's bias, or ``fold_bias`` where that is not NaN."""
        ub = np.where(user_nums >= 0, self.user_biases[np.maximum(user_nums, 0)], 0.0).astype(np.float32)
        if fold_bias is not None:
            ub = np.where(np.isnan(fold_bias), ub, fold_bias).astype(np.float32)
        return (self.item_biases + self.global_bias).astype(np.float32), ub

    def transform(self, it: Interactions) -> np.ndarray:
        return (it.ratings - self.global_bias - self.item_biases[it.items] - self.user_biases[it.users]).astype(
            np.float32
        )


def damping_pair(damping) -> tuple[float, float]:
    """``(user, item)`` damping from a float, a ``(user, item)`` tuple, or a dict in which a missing key means 0."""
    if isinstance(damping, dict):
        pair = (float(damping.get("user", 0.0)), float(damping.get("item", 0.0)))
    elif isinstance(damping, tuple):
        pair = (float(damping[0]), float(damping[1]))
    else:
        pair = (float(damping), float(damping))
    if not (pair[0] >= 0 and pair[1] >= 0):
        raise ValueError(f"damping must be non-negative, not {damping!r}")
    return pair


def learn(data, damping=0.0, *, entities=ENTITIES, centered_dtype=np.float32) -> BiasModel:
    """
    ``BiasModel.learn(data, damping, entities=...)`` on the device, bit for bit with :meth:`BiasModel.learn` on
    the same ``centered_dtype`` (``np.float32``: the reference's f32 rating matrix; ``np.float64``: BiasedMF's
    centring).  A bias left out of ``entities`` is None.
    """
    it = _as_dataset(data).interactions
    d_user, d_item = damping_pair(damping)
    unknown = set(entities) - ENTITIES
    if unknown:
        raise ValueError(f"unknown bias entities {sorted(unknown)}")
    if np.dtype(centered_dtype) not in (np.float32, np.float64):
        raise ValueError(f"centered_dtype must be float32 or float64, not {np.dtype(centered_dtype)}")
    if it.nnz == 0:
        raise ValueError("a bias model needs at least one rating")
    dev = _lib.require_device()
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    users, items = up(it.users.astype(np.int32, copy=False)), up(it.items.astype(np.int32, copy=False))
    ratings = up(np.asarray(it.ratings, dtype=np.float32))
    ui, iu, _perm = coo_to_csr_pair(users, items, ratings, it.n_users, it.n_items)
    mean, ib, ub = engine.bias_learn(
        ratings, items, ui.indptr, iu.indptr, iu.values, (d_user, d_item), item_pass="item" in entities,
        user_pass="user" in entities, centered_f64=np.dtype(centered_dtype) == np.float64,
    )  # fmt: skip
    host = lambda t: None if t is None else t.cpu().numpy()  # noqa: E731
    return BiasModel(float(mean.item()), host(ib), host(ub), (d_user, d_item))


class BiasConfig(BaseModel, extra="forbid"):
    entities: Annotated[set[Literal["user", "item"]], PlainSerializer(lambda s: sorted(s), return_type=list[str])] = {
        "user", "item",
    }  # fmt: skip
    damping: NonNegativeFloat | dict[Literal["user", "item"], NonNegativeFloat] = 0.0

    def entity_damping(self, entity: Literal["user", "item"]) -> float:
        return damping_pair(self.damping)[0 if entity == "user" else 1]


class _OffsetScorer(Component, Trainable):
    """What the two scorers share: ``score_batch`` and ``recommend_batch`` over ``base`` and per-query offsets."""

    users = None
    items = None

    def base_scores(self) -> np.ndarray:  # pragma: no cover
        raise NotImplementedError

    def query_offsets(self, queries: list[RecQuery]) -> np.ndarray | None:
        return None

    def _device_base(self) -> torch.Tensor:
        d = self.__dict__.get("_d_base")
        if d is None:
            d = torch.from_numpy(np.ascontiguousarray(self.base_scores(), dtype=np.float32)).to(_lib.require_device())
            self._d_base = d
        return d

    def score_batch(self, queries, targets: list[ItemList]) -> list[ItemList]:
        """Score ``targets[i]`` for ``queries[i]``: every item of the model in one launch, the targets picked out;
        NaN for an item the model does not know."""
        queries = [RecQuery.create(q) for q in queries]
        return self._score_targets(queries, targets, self.query_offsets(queries))

    def _score_targets(self, queries: list[RecQuery], targets: list[ItemList], off) -> list[ItemList]:
        S = engine.offset_scores(self._device_base(), len(queries), None if off is None else torch.from_numpy(off))
        return target_scores(S, targets, self.items)

    def recommend_batch(self, queries, n: int, *, exclude: Literal["query"] | None = "query") -> list[ItemList]:
        """
        Top-``n`` items for every query, scored and selected on the device in one launch: for each query the result
        of ``TrainingItemsCandidateSelector`` (every item, minus the query's items when ``exclude="query"``),
        ``__call__`` and ``TopNRanker``, bit for bit with the scores of ``score_batch``.  Every query is ranked.
        """
        check_exclude(exclude)
        queries = [RecQuery.create(q) for q in queries]
        base = self._device_base()
        n_eff = rank_size(n, base.numel())
        if n_eff == 0 or not queries:
            return [empty_list(self.items) for _ in queries]
        excl = history_csr(queries, self.items, base.device)[1:] if exclude == "query" else (None, None)
        off = self.query_offsets(queries)
        idx, val, cnt = engine.offset_scores(base, len(queries), None if off is None else torch.from_numpy(off), n_eff,
                                             *excl)  # fmt: skip
        return ranked_lists(self.items, len(queries), range(len(queries)), idx, val, cnt)

    def __getstate__(self):
        d = dict(self.__dict__)
        d.pop("_d_base", None)  # host arrays are the pickled state
        return d


class BiasScorer(_OffsetScorer):
    """
    ``BiasScorer``: ``train`` learns the bias model on the device; ``__call__`` is ``compute_for_items`` for the
    query's user or its rated items.
    """

    CONFIG_CLASS = BiasConfig
    config: BiasConfig
    model: BiasModel

    def is_trained(self) -> bool:
        return "model" in self.__dict__

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        self.model = learn(ds, self.config.damping, entities=self.config.entities)
        self.users, self.items = ds.users, ds.items
        self.__dict__.pop("_d_base", None)

    def base_scores(self) -> np.ndarray:
        """``compute_for_items`` before the user bias: ``f32(g) + ib`` (f32)."""
        scores = np.full(len(self.items), self.model.global_bias, dtype=np.float32)
        if self.model.item_biases is not None:
            scores += self.model.item_biases
        return scores

    def query_offsets(self, queries: list[RecQuery]) -> np.ndarray:
        """Each query's user bias as ``compute_for_items`` adds it (f64): from the query's ratings when it has them,
        else the known user's bias, else 0; always 0 without user biases."""
        m = self.model
        out = np.zeros(len(queries), dtype=np.float64)
        if m.user_biases is None:
            return out
        for b, q in enumerate(queries):
            rated = q.query_items
            ratings = None if rated is None else rated.field("rating")
            if ratings is not None:
                nums = None if m.item_biases is None else rated.numbers(vocabulary=self.items, missing="negative")
                out[b] = m.user_bias_for_items(nums, ratings)
            elif q.user_id is not None:
                uno = self.users.number(q.user_id, missing="none")
                if uno is not None:
                    out[b] = m.user_biases[uno]
        return out

    def score_batch(self, queries, targets: list[ItemList]) -> list[ItemList]:
        """As the reference: an item the model does not know scores the global bias plus the user bias."""
        queries = [RecQuery.create(q) for q in queries]
        off = self.query_offsets(queries)
        out = self._score_targets(queries, targets, off)
        g32 = np.float64(np.float32(self.model.global_bias))
        for b, tgt in enumerate(targets):
            unknown = tgt.numbers(vocabulary=self.items, missing="negative") < 0
            if unknown.any():
                s = out[b].scores().copy()
                s[unknown] = np.float32(g32 + off[b])
                out[b] = ItemList(tgt, scores=s)
        return out

    def __call__(self, query, items: ItemList) -> ItemList:
        return self.score_batch([query], [items])[0]


class PopConfig(BaseModel):
    score: Literal["quantile", "rank", "count"] = "quantile"


class PopScorer(_OffsetScorer):
    """``PopScorer``: popularity counts from the device, the reference's pandas statements for rank and quantile."""

    CONFIG_CLASS = PopConfig
    config: PopConfig
    item_scores: np.ndarray

    def is_trained(self) -> bool:
        return "item_scores" in self.__dict__

    def train(self, data, options: TrainingOptions = TrainingOptions()) -> None:
        if self.is_trained() and not options.retrain:
            return
        ds = _as_dataset(data)
        it = ds.interactions
        dev = _lib.require_device()
        items = torch.from_numpy(np.ascontiguousarray(it.items, dtype=np.int64)).to(dev)
        counts = torch.bincount(items, minlength=it.n_items).cpu().numpy()
        self.items = ds.items
        scores = pd.Series(counts, index=pd.Index(ds.items.ids(), name="item_id"), name="count")
        self.item_scores = np.require(self._train_internal(scores).values, np.float32)
        self.__dict__.pop("_d_base", None)

    def _train_internal(self, scores: pd.Series) -> pd.Series:
        if self.config.score == "rank":
            return scores.rank()
        elif self.config.score == "quantile":
            cmass = scores.sort_values()
            cmass = cmass.cumsum()
            cdens = cmass / scores.sum()
            return cdens.reindex(scores.index)
        elif self.config.score == "count":
            return scores
        else:
            raise ValueError("invalid scoring method " + repr(self.config.score))

    def base_scores(self) -> np.ndarray:
        return self.item_scores

    def __call__(self, items: ItemList) -> ItemList:
        """The items' popularity scores; NaN for an item the model does not know."""
        inums = items.numbers(vocabulary=self.items, missing="negative")
        mask = inums >= 0
        scores = np.full(len(items), np.nan, np.float32)
        scores[mask] = self.item_scores[inums[mask]]
        return ItemList(items, scores=scores)
