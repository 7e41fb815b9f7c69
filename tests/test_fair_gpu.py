"""
FAIRReranker on the device (``lk_fair_rerank``), exactly against the host: ``rerank_batch`` against the sequence of
``__call__``s, and ``rank_scores`` against ``__call__`` on argtopn's top N of each row (``oracle.argtopn``, the C
restatement of the reference's heap), with the query's items excluded.
"""

import pickle

import numpy as np
import pytest
import torch

import oracle
from lkpy_b200 import _lib, engine
from lkpy_b200.components import Dataset, ItemList, RecQuery, Vocabulary
from lkpy_b200.reranking import FAIRReranker

pytestmark = pytest.mark.gpu


def trained(n: int, p: float, ids, flags) -> FAIRReranker:
    r = FAIRReranker(n=n, p=p, alpha=0.1)
    r.train(Dataset(None, users=Vocabulary(np.zeros(0, np.int64), "user"), items=Vocabulary(ids, "item"),
                    item_attributes={"protected": flags}))  # fmt: skip
    return r


def same(a: ItemList, b: ItemList) -> bool:
    sa, sb = a.scores(), b.scores()
    scores = (sa is None and sb is None) or np.array_equal(sa.view(np.int32), sb.view(np.int32))
    return np.array_equal(a.ids(), b.ids()) and scores and a.ordered and b.ordered


@pytest.mark.parametrize("cfg_n", [10, 200, 1024])
def test_rerank_batch_equals_calls(cuda_lib, cfg_n):
    """Ragged lists (empty, shorter and longer than n, unknown items, no or only protected items, protected items
    deep in the list), B of 2,500 lists over many CTAs, every kind of runtime n; each result keeps its fields."""
    rng = np.random.default_rng(cfg_n)
    ids = np.arange(5000) * 2 + 1
    flags = rng.random(5000) < 0.3
    r = trained(cfg_n, 0.6, ids, flags)
    lists = []
    for b in range(2500 if cfg_n < 1024 else 300):  # the host calls of the longest lists are slow
        L = int(rng.integers(0, 3 * cfg_n + 5)) if b % 7 else int(rng.integers(0, 4))
        it = rng.choice(ids, L, replace=False)
        if b % 11 == 1:
            it[::4] = 100_000 + b  # not in the vocabulary
        if b % 13 == 2:
            it = np.concatenate([rng.choice(ids[~flags], 2 * cfg_n, replace=False), rng.choice(ids[flags], 40, replace=False)])
        if b % 17 == 3:
            it = rng.choice(ids[flags], min(L, 1000), replace=False)
        lists.append(ItemList(item_ids=it, scores=rng.standard_normal(len(it)).astype(np.float32),
                              rating=np.arange(len(it)), ordered=True))  # fmt: skip
    for n in (None, cfg_n, cfg_n // 2 + 1, 0, 1):
        got = r.rerank_batch(lists, n)
        for g, it in zip(got, lists):
            want = r(it, n)
            assert same(g, want) and np.array_equal(g.field("rating"), want.field("rating"))


def host_topn_fair(r: FAIRReranker, S: np.ndarray, vocab, hists, N: int, n):
    """``TopNRanker(n=N)`` (argtopn over the row, the query's items as NaN) then ``r(list, n)``, per row."""
    out = []
    for b in range(S.shape[0]):
        row = S[b].copy()
        row[hists[b]] = np.nan
        top = oracle.argtopn(row, N)
        out.append(r(ItemList(item_nums=top, vocabulary=vocab, scores=row[top], ordered=True), n))
    return out


CASES = {
    # name: (n_items, B, N, n, ties, specials, strided)
    "ties_straddle": (3000, 64, 100, 10, True, False, False),
    "nan_inf": (2048, 48, 50, 20, False, True, False),
    "N_equals_n": (999, 40, 30, 30, True, False, True),
    "N_1024": (5003, 24, 1024, 100, True, True, True),
    "odd_items_strided": (4001, 70, 200, 50, False, False, True),
}


@pytest.mark.parametrize("name", list(CASES))
def test_rank_scores_equals_topn_then_call(cuda_lib, name):
    """Tied scores across the two classes, NaN, ±inf and all-NaN rows, excluded query items, N = n and N = 1024,
    n_items off a multiple of 32, and the transpose of an item-major matrix (no copy)."""
    n_items, B, N, n, ties, specials, strided = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    dev = _lib.require_device()
    S = rng.standard_normal((B, n_items)).astype(np.float32)
    if ties:
        S = np.round(S * 2).astype(np.float32)  # few distinct values: ties at the cut and inside the list
    if specials:
        bad = rng.random(S.shape)
        S[bad < 0.05] = np.nan
        S[(bad >= 0.05) & (bad < 0.06)] = np.inf
        S[(bad >= 0.06) & (bad < 0.07)] = -np.inf
        S[3] = np.nan
        S[4, : n_items - 5] = np.nan  # fewer valid items than N
    ids = np.arange(n_items) * 5 + 2
    vocab = Vocabulary(ids, "item")
    r = trained(max(n, 2 * n), 0.55, ids, rng.random(n_items) < 0.25)
    hists = [rng.choice(n_items, int(rng.integers(0, 60)), replace=False) for _ in range(B)]
    queries = [RecQuery(None, ItemList(item_ids=ids[h])) if len(h) else RecQuery(None, None) for h in hists]
    M = torch.from_numpy(S.T.copy()).to(dev).T if strided else torch.from_numpy(S).to(dev)
    assert M.is_contiguous() != strided
    got = r.rank_scores(M, queries, vocab, n, candidates=N)
    want = host_topn_fair(r, S, vocab, hists, N, n)
    for b, (g, w) in enumerate(zip(got, want)):
        assert same(g, w), (name, b)
    if specials:
        assert len(got[3]) == 0  # an all-NaN row
    none = r.rank_scores(M, queries, vocab, n, candidates=N, exclude=None)
    want = host_topn_fair(r, S, vocab, [np.zeros(0, np.int64)] * B, N, n)
    assert all(same(g, w) for g, w in zip(none, want))


def test_rank_scores_of_another_vocabulary(cuda_lib):
    """A score matrix over a vocabulary other than the trained one: its items' flags are looked up by id, unknown
    items unprotected."""
    rng = np.random.default_rng(3)
    ids = np.arange(800)
    r = trained(20, 0.7, ids, rng.random(800) < 0.2)
    vocab = Vocabulary(np.arange(400, 1300), "item")
    S = rng.standard_normal((16, 900)).astype(np.float32)
    got = r.rank_scores(torch.from_numpy(S).to(_lib.require_device()), [None] * 16, vocab, candidates=300)
    want = host_topn_fair(r, S, vocab, [np.zeros(0, np.int64)] * 16, 300, None)
    assert all(same(g, w) for g, w in zip(got, want))


def test_engine_list_mode_matches_the_merge(cuda_lib):
    """``engine.fair_rerank``'s list mode on raw flags: lists of up to 70,000 positions with the protected ones last,
    so that the merge scans far for them."""
    from lkpy_b200.reranking import fair_merge, minimum_protected

    rng = np.random.default_rng(9)
    m = minimum_protected(1024, 0.5, 0.1)
    flags = [np.concatenate([np.zeros(L - 30, bool), np.ones(30, bool)]) for L in (31, 1000, 70000)]
    flags.append(rng.random(5000) < 0.5)
    indptr = np.concatenate([[0], np.cumsum([len(f) for f in flags])])
    lens = np.array([min(len(f), 1024) for f in flags], np.int32)
    idx, _v, cnt = engine.fair_rerank(m, 1024, np.concatenate(flags), indptr=indptr, lengths=lens)
    idx, cnt = idx.cpu().numpy(), cnt.cpu().numpy()
    for b, f in enumerate(flags):
        assert cnt[b] == lens[b] and np.array_equal(idx[b, : lens[b]], fair_merge(f, m, lens[b]))
        assert (idx[b, lens[b] :] == -1).all()


def test_pickle_round_trip(cuda_lib):
    rng = np.random.default_rng(6)
    ids = np.arange(500) + 10
    r = trained(30, 0.5, ids, rng.random(500) < 0.4)
    r2 = pickle.loads(pickle.dumps(r))
    lists = [ItemList(item_ids=rng.permutation(ids)[: int(rng.integers(0, 100))], ordered=True) for _ in range(40)]
    assert all(same(a, b) for a, b in zip(r.rerank_batch(lists), r2.rerank_batch(lists)))
    S = torch.from_numpy(rng.standard_normal((8, 500)).astype(np.float32)).to(_lib.require_device())
    vocab = Vocabulary(ids, "item")
    a, b = r.rank_scores(S, [None] * 8, vocab, candidates=100), r2.rank_scores(S, [None] * 8, vocab, candidates=100)
    assert all(same(x, y) for x, y in zip(a, b))
