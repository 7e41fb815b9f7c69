"""The scorer side of batched top-n (``lkpy_b200.batch``) and the engine's exclusion sorting, on CPU tensors."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from lkpy_b200 import _lib, batch, engine
from lkpy_b200.components import ItemList, RecQuery, Vocabulary

VOCAB = Vocabulary(np.array(["a", "b", "c", "d", "e"]))


def _hist(ids) -> ItemList:
    return ItemList(item_ids=np.array(ids), vocabulary=None)


def test_history_csr_keeps_query_order_and_drops_unknown():
    queries = [_hist(["c", "a", "x", "c"]), RecQuery(), RecQuery("u", None), _hist([]), RecQuery("u", _hist(["e", "b"]))]
    has, indptr, items = batch.history_csr(queries, VOCAB, "cpu")
    assert has.tolist() == [True, False, False, False, True]
    assert indptr.dtype == torch.int64 and items.dtype == torch.int32
    assert indptr.tolist() == [0, 3, 3, 3, 3, 5]
    assert items.tolist() == [2, 0, 2, 4, 1]


def test_history_csr_unique():
    has, indptr, items = batch.history_csr([_hist(["c", "a", "x", "c"]), _hist(["x"]), _hist(["e", "b", "e"])],
                                           VOCAB, "cpu", unique=True)  # fmt: skip
    assert has.tolist() == [True, True, True]  # a history of unknown items is still a history
    assert indptr.tolist() == [0, 2, 2, 4]
    assert items.tolist() == [0, 2, 1, 4]


def test_history_csr_empty_batch():
    has, indptr, items = batch.history_csr([], VOCAB, "cpu")
    assert has.shape == (0,) and indptr.tolist() == [0] and items.numel() == 0


def test_target_scores_nan_for_unknown_items_and_rows_without_history():
    scores = torch.arange(10, dtype=torch.float32).reshape(2, 5)
    targets = [_hist(["e", "x", "a"]), _hist(["b"])]
    out = batch.target_scores(scores, targets, VOCAB)
    assert np.array_equal(out[0].scores(), [4.0, np.nan, 0.0], equal_nan=True)
    assert out[0].ids().tolist() == ["e", "x", "a"]
    assert out[1].scores().tolist() == [6.0]
    out = batch.target_scores(scores, targets, VOCAB, has=np.array([True, False]))
    assert np.array_equal(out[0].scores(), [4.0, np.nan, 0.0], equal_nan=True)
    assert np.isnan(out[1].scores()).all()


def test_ranked_lists_maps_rows_and_truncates():
    idx = torch.tensor([[3, 1, -1], [0, -1, -1]], dtype=torch.int32)
    val = torch.tensor([[2.5, 1.5, np.nan], [0.5, np.nan, np.nan]], dtype=torch.float32)
    cnt = torch.tensor([2, 1], dtype=torch.int32)
    nbrs = torch.tensor([[7, 8, 0], [9, 0, 0]], dtype=torch.int32)
    out = batch.ranked_lists(VOCAB, 4, [3, 1], idx, val, cnt, nbr_counts=nbrs)
    assert [len(r) for r in out] == [0, 1, 0, 2]
    assert out[3].ids().tolist() == ["d", "b"] and out[3].numbers(vocabulary=VOCAB).tolist() == [3, 1]
    assert out[3].scores().tolist() == [2.5, 1.5] and out[3].field("nbr_counts").tolist() == [7, 8]
    assert out[1].ids().tolist() == ["a"] and out[1].field("nbr_counts").tolist() == [9]
    for b in (0, 2):
        assert out[b].scores().dtype == np.float32 and out[b].numbers(vocabulary=VOCAB).dtype == np.int32


def test_rank_size():
    n_max = int(_lib.lib().lk_topn_max())
    assert batch.rank_size(10, 5) == 5
    assert batch.rank_size(3, 5) == 3
    assert batch.rank_size(0, 5) == 0 and batch.rank_size(-2, 5) == 0 and batch.rank_size(4, 0) == 0
    assert batch.rank_size(n_max + 10, n_max) == n_max
    with pytest.raises(ValueError, match="engine limit"):
        batch.rank_size(n_max + 1, n_max + 5)


def test_check_exclude():
    batch.check_exclude("query")
    batch.check_exclude(None)
    with pytest.raises(ValueError, match="exclude"):
        batch.check_exclude("all")


def test_sorted_exclusions():
    indptr = torch.tensor([0, 5, 5, 8])
    items = torch.tensor([4, -1, 2, 4, 9, 3, 0, 3], dtype=torch.int32)
    ptr, ex = engine._sorted_exclusions(indptr, items, 5, 3, "cpu")
    assert ptr.tolist() == [0, 3, 3, 6]
    assert ex.dtype == torch.int32 and ex.tolist() == [2, 4, 4, 0, 3, 3]
    ptr, ex = engine._sorted_exclusions(torch.tensor([0, 1]), torch.tensor([7]), 5, 1, "cpu")
    assert ptr.tolist() == [0, 0] and ex.numel() == 1  # a placeholder address the kernel never reads
    with pytest.raises(ValueError, match="excl_indptr"):
        engine._sorted_exclusions(torch.tensor([0, 1]), torch.tensor([1]), 5, 2, "cpu")
