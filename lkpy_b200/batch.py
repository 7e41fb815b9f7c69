"""
The scorer side of batched top-n: what every scorer's ``score_batch`` and ``recommend_batch`` share.

The kernels behind ``recommend_batch`` all return ``argtopn``'s output for a batch: ``idx [B, n]`` item numbers
padded with -1, ``val [B, n]`` scores padded with NaN, and ``cnt [B]``.  The functions here build the query
histories the kernels take, check ``n`` and ``exclude``, and turn that output, or a dense score matrix, into
``ItemList``s.
"""

from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .components import ItemList, RecQuery


def check_exclude(exclude) -> None:
    if exclude not in ("query", None):
        raise ValueError(f'exclude must be "query" or None, not {exclude!r}')


def empty_list(vocabulary) -> ItemList:
    return ItemList(
        item_ids=vocabulary.ids(np.zeros(0, np.int32)), item_nums=np.zeros(0, np.int32), vocabulary=vocabulary,
        scores=np.zeros(0, np.float32),
    )  # fmt: skip


def take(items: ItemList, pos: np.ndarray, *, ordered: bool | None = None, **extra) -> ItemList:
    """The entries ``pos`` of ``items``, with every field, plus ``extra`` fields."""
    fields = {k: v[pos] for k, v in items._fields.items()}
    fields.update(extra)
    scores = fields.pop("score", None)
    return ItemList(
        item_ids=None if items._ids is None else items._ids[pos], item_nums=None if items._nums is None else items._nums[pos],
        vocabulary=items._vocab, scores=scores, ordered=ordered, **fields,
    )  # fmt: skip


def rank_size(n: int, n_items: int) -> int:
    """The list length a kernel is asked for: ``min(n, n_items)``, or 0 when every list is empty.  Raises
    ``ValueError`` past the engine limit ``lk_topn_max()``."""
    n_eff = min(int(n), n_items)
    if n_eff <= 0:
        return 0
    n_max = int(_lib.lib().lk_topn_max())
    if n_eff > n_max:
        raise ValueError(f"n={n_eff} exceeds the engine limit of {n_max}")
    return n_eff


def history_csr(queries, vocabulary, device, *, unique: bool = False):
    """
    The queries' known history items as a device CSR: ``(has, indptr, items)`` with ``has`` a bool array (the query
    has a non-empty ``query_items``), ``indptr`` int64 and ``items`` int32.  Unknown items are dropped; the items
    keep query order and repeats (the summation order of the association and SLIM scores), or with ``unique=True``
    are ascending without repeats.
    """
    has, hists = [], []
    for q in queries:
        hist = RecQuery.create(q).query_items
        has.append(hist is not None and len(hist) > 0)
        h = np.zeros(0, np.int32)
        if has[-1]:
            h = hist.numbers(vocabulary=vocabulary, missing="negative").astype(np.int32)
            h = np.unique(h[h >= 0]) if unique else h[h >= 0]
        hists.append(h)
    indptr = np.zeros(len(hists) + 1, dtype=np.int64)
    indptr[1:] = np.cumsum([len(h) for h in hists], dtype=np.int64)
    items = np.concatenate(hists) if hists else np.zeros(0, np.int32)
    return np.array(has, dtype=bool), torch.from_numpy(indptr).to(device), torch.from_numpy(items).to(device)


def target_scores(scores: torch.Tensor, targets: list[ItemList], vocabulary, has=None) -> list[ItemList]:
    """``targets[b]`` with their scores from row b of ``scores`` [B, n_items]: NaN for unknown items, and for every
    item of a row whose ``has[b]`` is False."""
    out = []
    for b, tgt in enumerate(targets):
        tn = tgt.numbers(vocabulary=vocabulary, missing="negative").astype(np.int64)
        s = np.full(len(tn), np.nan, dtype=np.float32)
        ok = tn >= 0
        if (has is None or has[b]) and ok.any():
            s[ok] = scores[b, torch.from_numpy(tn[ok]).to(scores.device)].cpu().numpy()
        out.append(ItemList(tgt, scores=s))
    return out


def ranked_lists(vocabulary, B: int, at, idx, val, cnt, **fields) -> list[ItemList]:
    """
    ``B`` lists from a top-n kernel's output: row j of ``idx``/``val``/``cnt`` (and of each ``fields`` array, such
    as ``nbr_counts``) truncated to ``cnt[j]`` entries goes to query ``at[j]``; every other query gets an empty list.
    """
    idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy()
    fields = {k: v.cpu().numpy() for k, v in fields.items()}
    out = [None] * B
    for j, b in enumerate(at):
        c = int(cnt[j])
        out[b] = ItemList(
            item_ids=vocabulary.ids(idx[j, :c]), item_nums=idx[j, :c].copy(), vocabulary=vocabulary,
            scores=val[j, :c].copy(), **{k: v[j, :c].copy() for k, v in fields.items()},
        )  # fmt: skip
    return [empty_list(vocabulary) if r is None else r for r in out]
