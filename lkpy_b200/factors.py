"""
The batched scoring path that the matrix-factorisation scorers (ALS, FlexMF, BiasedSVD, NMF) share: a query embedding
``x`` against the item table ``Q``, ``s(q, i) = x_q · Q_i + item_offset[i] + query_offset[q]``, scored and top-n
selected on the device by ``lk_als_recommend_batch`` with the factors resident in HBM; and the embedding-size rules of
their configurations.  A :class:`FactorScorer` subclass says how queries become embeddings (``embed_batch``) and which
offsets apply (``batch_offsets``); :class:`KnownUserScorer` embeds known users only.
"""

from __future__ import annotations

from typing import Annotated, Literal

import numpy as np
import torch
from pydantic import AfterValidator, AliasChoices, BaseModel, PositiveInt, model_validator

from . import _lib, engine
from .batch import check_exclude, empty_list, history_csr, rank_size, ranked_lists, target_scores
from .components import Component, ItemList, RecQuery


def within_engine_limit(k: int) -> int:
    """The engine's largest embedding size (the reference has none), checked when a configuration is made."""
    if k > engine.ALS_MAX_FEATURES:
        raise ValueError(f"embedding_size={k} exceeds the engine limit of {engine.ALS_MAX_FEATURES}")
    return k


#: a positive embedding size within the engine's limit
EmbeddingSize = Annotated[PositiveInt, AfterValidator(within_engine_limit)]


class EmbeddingSizeExp(BaseModel):
    """``embedding_size_exp=e`` configures ``embedding_size = 2**e`` (the reference's ``EmbeddingSizeMixin``), in
    place of the size given under any of its names."""

    @model_validator(mode="before")
    @classmethod
    def apply_aliases(cls, data):
        if isinstance(data, dict) and "embedding_size_exp" in data:
            alias = cls.model_fields["embedding_size"].validation_alias
            names = {"embedding_size_exp", "embedding_size"}
            names.update(alias.choices if isinstance(alias, AliasChoices) else ())
            size = 2 ** data["embedding_size_exp"]
            data = {k: v for k, v in data.items() if k not in names} | {"embedding_size": size}
        return data


class FactorScorer(Component):
    """User and item embeddings, and ``score_matrix`` / ``recommend_batch`` over them on the device."""

    users = None
    items = None
    user_embeddings: np.ndarray | None = None
    item_embeddings: np.ndarray | None = None

    def is_trained(self) -> bool:
        return self.item_embeddings is not None

    def _device_items(self) -> torch.Tensor:
        """The item table in HBM, uploaded again when ``item_embeddings`` is another array (a retrain)."""
        dev = _lib.require_device()
        cached = self.__dict__.get("_d_items_cache")
        if cached is None or cached[0] is not self.item_embeddings:
            t = torch.from_numpy(np.ascontiguousarray(self.item_embeddings, dtype=np.float32)).to(dev)
            self.__dict__["_d_items_cache"] = cached = (self.item_embeddings, t)
        return cached[1]

    def embed_batch(self, queries) -> tuple[torch.Tensor, np.ndarray, np.ndarray, np.ndarray | None]:
        """
        Query embeddings on the device: ``(X [B, k], scorable [B] bool, user_nums [B] (-1 unknown),
        per-query user offsets or None)``.
        """
        raise NotImplementedError  # pragma: no cover

    def batch_offsets(self, user_nums: np.ndarray, fold_bias: np.ndarray | None):
        """(per-item offset [n_items] or None, per-query offset [B] or None) added to Q · Xᵀ."""
        return None, None

    def _offsets(self, user_nums, fold_bias, dev):
        item_off, query_off = self.batch_offsets(user_nums, fold_bias)
        if item_off is not None:
            item_off = torch.from_numpy(np.ascontiguousarray(item_off, dtype=np.float32)).to(dev)
        if query_off is not None:
            query_off = torch.from_numpy(np.ascontiguousarray(query_off, dtype=np.float32)).to(dev)
        return item_off, query_off

    def score_matrix(self, queries) -> torch.Tensor:
        """
        Scores of every item for every query, item-major: [n_items, B] f32, NaN columns for unscorable queries.
        Each score is one fp32 FMA chain over ascending d, then the item offset and the query offset (f32 adds):
        ``engine.als_recommend``'s score mode.
        """
        X, scorable, user_nums, fold_bias = self.embed_batch(queries)
        item_off, query_off = self._offsets(user_nums, fold_bias, X.device)
        S = engine.als_recommend(self._device_items(), X, None, item_off, query_off)
        if not scorable.all():
            S[:, torch.from_numpy(np.flatnonzero(~scorable)).to(S.device)] = float("nan")
        return S

    def recommend_batch(self, queries, n: int, *, exclude: Literal["query"] | None = None) -> list[ItemList]:
        """
        Top-``n`` items for every query, scored and selected on the device in one launch (``engine.als_recommend``'s
        rank mode; memory O(B·n), no score matrix): for each query the result of the candidate selector, the
        scores of :meth:`score_matrix` and ``TopNRanker``, bit for bit.  ``exclude="query"`` leaves the query's
        own items (``query.query_items`` known to the model) out of the candidates, as
        ``TrainingItemsCandidateSelector`` does; the default ``None`` ranks every item.  (The kNN scorers'
        ``recommend_batch`` defaults to ``"query"``.)  An unscorable query gets an empty list.  The kernel sweeps
        every item once per 64 queries, so batch widely.
        """
        check_exclude(exclude)
        queries = [RecQuery.create(q) for q in queries]
        n_eff = rank_size(n, self.item_embeddings.shape[0])
        if n_eff == 0:
            return [empty_list(self.items) for _ in queries]
        X, scorable, user_nums, fold_bias = self.embed_batch(queries)
        at = np.flatnonzero(scorable)
        if len(at) == 0:
            return [empty_list(self.items) for _ in queries]
        dev = X.device
        item_off, query_off = self._offsets(user_nums, fold_bias, dev)
        excl = (None, None)
        if exclude == "query":
            excl = history_csr([queries[b] for b in at], self.items, dev)[1:]
        sel = torch.from_numpy(at).to(dev)
        idx, val, cnt = engine.als_recommend(
            self._device_items(), X[sel].contiguous(), n_eff, item_off,
            query_off[sel] if query_off is not None else None, *excl,
        )  # fmt: skip
        return ranked_lists(self.items, len(queries), at, idx, val, cnt)

    def __getstate__(self):
        d = dict(self.__dict__)
        d.pop("_d_items_cache", None)  # host arrays are the pickled state
        return d


class KnownUserScorer(FactorScorer):
    """Scoring for known users only (no fold-in): ``score_matrix`` / ``score_batch`` / ``__call__`` /
    ``recommend_batch``.  A query whose user is unknown scores NaN and gets an empty list."""

    def embed_batch(self, queries):
        """Known users' embeddings; a query without a known user is unscorable (flexmf/_base.py:126-133)."""
        dev = _lib.require_device()
        queries = [RecQuery.create(q) for q in queries]
        nums = [None if q.user_id is None else self.users.number(q.user_id, missing=None) for q in queries]
        user_nums = np.array([-1 if u is None else u for u in nums], dtype=np.int64)
        scorable = user_nums >= 0
        X = np.zeros((len(queries), self.item_embeddings.shape[1]), dtype=np.float32)
        X[scorable] = self.user_embeddings[user_nums[scorable]]
        return torch.from_numpy(X).to(dev), scorable, user_nums, None

    def score_batch(self, queries, targets: list[ItemList]) -> list[ItemList]:
        """Score ``targets[i]`` for ``queries[i]``: columns of :meth:`score_matrix` picked out on the device.
        Unknown items, and every item of a query without a known user, score NaN."""
        return target_scores(self.score_matrix(queries).T, targets, self.items)

    def __call__(self, query, items: ItemList) -> ItemList:
        return self.score_batch([query], [items])[0]
