"""
StochasticTopNRanker on the device (``lk_stochastic_topn``) against the host restatements in
tests/stochastic_oracle.py: the PCG64 stream and the generator state left behind exactly, the selection exactly over
the device's own keys, and the keys within the tolerance the host's transcendentals allow (DESIGN.md §4.19).
"""

import pickle

import numpy as np
import pytest
import torch

import stochastic_oracle as so
from lkpy_b200 import _lib, engine
from lkpy_b200.components import ItemList, RecQuery, Vocabulary
from lkpy_b200.stochastic import StochasticTopNRanker, derivable_rng, generator_words

pytestmark = pytest.mark.gpu

#: relative key tolerance: 2 f64 ulps where only the f64 log may differ, 1e-6 where the f32 exp does too
TOL = {None: 4.5e-16, "linear": 4.5e-16, "softmax": 1e-6}


def ulps(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a.view(np.int64) - b.view(np.int64))


def packed(lists: list[np.ndarray]) -> torch.Tensor:
    L = max((len(s) for s in lists), default=0)
    m = np.full((len(lists), L), np.nan, np.float32)
    for b, s in enumerate(lists):
        m[b, : len(s)] = s
    return torch.from_numpy(m).to(_lib.require_device())


def all_keys(idx, key, cnt, L) -> np.ndarray:
    """Per-position keys from a key-mode result (NaN where not valid)."""
    out = np.full((len(cnt), L), np.nan)
    for b in range(len(cnt)):
        out[b, idx[b, : cnt[b]]] = key[b, : cnt[b]]
    return out


def random_list(rng, L: int, ties: bool = False) -> np.ndarray:
    s = rng.standard_normal(L).astype(np.float32)
    if ties:
        s = np.round(s * 4) / 4
    bad = rng.random(L)
    s[bad < 0.05] = np.nan
    s[(bad >= 0.05) & (bad < 0.07)] = np.inf
    s[(bad >= 0.07) & (bad < 0.08)] = -np.inf
    return s


def compare(got: ItemList, want_pos, want_keys, transform, ids) -> int:
    """Keys within tolerance of the oracle's, and the same list unless two oracle keys lie within that tolerance;
    returns 1 for such an exception."""
    gk = got.field("weight")
    if len(got) == len(want_pos) and np.array_equal(got.ids(), ids[want_pos]):
        if transform == "softmax":
            assert np.allclose(gk, want_keys, rtol=TOL[transform], atol=0)
        else:
            assert ulps(gk, want_keys).max(initial=0) <= 2
        return 0
    srt = np.sort(want_keys)[::-1]
    gaps = np.abs(np.diff(srt)) / np.maximum(np.abs(srt[1:]), 1e-300)
    assert len(got) == len(want_pos) and gaps.size and gaps.min() < 2 * TOL[transform], "lists differ without a near-tie"
    return 1


def test_stream_is_numpy_pcg64(cuda_lib, monkeypatch):
    """With transform=None and every score 1.0 the key is log(u): the k-th valid position takes the k-th uniform of
    its stream, within 1 ulp of np.log of NumPy's uniforms.  Per-query streams and one shared stream across split
    launches (a small split forces the stream offsets and the device-side position through several launches)."""
    rng = np.random.default_rng(3)
    lens = [1, 31, 32, 33, 100, 1000, 4097, 70000]
    lists = []
    for L in lens:
        s = np.ones(L, np.float32)
        s[rng.random(L) < 0.1] = np.nan
        lists.append(s)
    S = packed(lists)
    seeds = [11 + b for b in range(len(lens))]
    states = np.array([generator_words(np.random.default_rng(x)) for x in seeds], np.uint64)
    idx, _v, key, cnt, _d = (t.cpu().numpy() if t is not None else None for t in engine.stochastic_topn(
        S, None, transform=None, scale=1.0, states=states, shared=False, with_keys=True))  # fmt: skip
    K = all_keys(idx, key, cnt, S.shape[1])
    for b, (x, s) in enumerate(zip(seeds, lists)):
        ok = np.isfinite(s)
        want = np.log(np.random.default_rng(x).uniform(0, 1, int(ok.sum())))
        assert cnt[b] == ok.sum() and ulps(K[b, : len(s)][ok], want).max(initial=0) <= 1
        assert np.isnan(K[b, : len(s)][~ok]).all() and np.isnan(K[b, len(s) :]).all()
    monkeypatch.setattr(engine, "STOCHASTIC_SPLIT_BYTES", 3 * (8 * 70000 + 64))
    gen = np.random.default_rng(99)
    idx, _v, key, cnt, drawn = (t.cpu().numpy() if t is not None else None for t in engine.stochastic_topn(
        S, None, transform=None, scale=1.0, states=np.array([generator_words(gen)], np.uint64), shared=True,
        with_keys=True))  # fmt: skip
    K = all_keys(idx, key, cnt, S.shape[1])
    for b, s in enumerate(lists):
        ok = np.isfinite(s)
        assert ulps(K[b, : len(s)][ok], np.log(gen.uniform(0, 1, int(ok.sum())))).max(initial=0) <= 1
    assert int(drawn[0]) == sum(int(np.isfinite(s).sum()) for s in lists)


@pytest.mark.parametrize("transform", ["softmax", "linear", None])
@pytest.mark.parametrize("scale", [1.0, 0.1, 1e4])
def test_batch_equals_sequence(cuda_lib, transform, scale):
    """Under a fixed generator, rank_batch gives the sequence of oracle calls in order (NaN, ±inf, ties, empty and
    all-invalid lists among them), and leaves the generator's state equal to the one those calls leave."""
    rng = np.random.default_rng(int(scale * 10) + len(str(transform)))
    lists = [random_list(rng, int(L), ties=b % 2 == 1) for b, L in enumerate(rng.integers(1, 3000, 14))]
    lists += [np.zeros(0, np.float32), np.full(50, np.nan, np.float32), np.array([np.inf, -np.inf], np.float32)]
    lists += [random_list(rng, 40)]
    items = [ItemList(item_ids=np.arange(len(s)) + 1000, scores=s, rating=np.arange(len(s))) for s in lists]
    exceptions = 0
    for n in (10, None):
        r = StochasticTopNRanker(rng=42, transform=transform, scale=scale, n=n)
        gen = np.random.default_rng(42)
        got = r.rank_batch(items, include_weights=True)
        for g, s, it in zip(got, lists, items):
            pos, k = so.rank(s, n, transform, scale, gen)
            exceptions += compare(g, pos, k, transform, it.ids())
            assert np.array_equal(g.field("rating"), it.field("rating")[g.ids() - 1000])
            assert np.array_equal(g.scores(), s[g.ids() - 1000])
        assert r._rng_factory.rng.bit_generator.state == gen.bit_generator.state
    assert exceptions == 0, f"{exceptions} near-tie exceptions"


def test_derived_rng_per_user(cuda_lib):
    """(seed, "user"): int, str and missing user ids, in order; a query without one spawns from the base seed."""
    rng = np.random.default_rng(5)
    lists = [random_list(rng, int(L)) for L in rng.integers(1, 500, 7)]
    users = [17, "alice", None, 17, None, "bob", 3]
    r = StochasticTopNRanker(rng=(7, "user"), transform="linear", n=20)
    got = r.rank_batch([ItemList(item_ids=np.arange(len(s)), scores=s) for s in lists], users, include_weights=True)
    f = derivable_rng((7, "user"))
    for g, s, u in zip(got, lists, users):
        pos, k = so.rank(s, 20, "linear", 1.0, f(RecQuery(u)))
        assert compare(g, pos, k, "linear", np.arange(len(s))) == 0
    # the spawn counter moved as two calls with no user id move it
    assert r._rng_factory.seed.n_children_spawned == 2


@pytest.mark.parametrize("n", [1, 5, 100, 1024])
def test_selection_is_argtopn_over_the_device_keys(cuda_lib, n):
    """Rank mode selects and orders exactly as argtopn over the keys the device computes (read in key mode from the
    same states)."""
    rng = np.random.default_rng(n)
    lists = [random_list(rng, int(L), ties=True) for L in (3, 200, 5000, 20000)]
    S = packed(lists)
    states = np.array([generator_words(np.random.default_rng(x)) for x in range(len(lists))], np.uint64)
    run = lambda m: [t.cpu().numpy() for t in engine.stochastic_topn(  # noqa: E731
        S, m, transform="softmax", scale=3.0, states=states, shared=False, with_keys=True)[:4]]  # fmt: skip
    idx, _v, key, cnt = run(None)
    K = all_keys(idx, key, cnt, S.shape[1])
    idx, val, key, cnt = run(n)
    for b in range(len(lists)):
        want = so.argtopn(K[b], n)
        assert np.array_equal(idx[b, : cnt[b]], want)
        assert np.array_equal(key[b, : cnt[b]], K[b, want])
        assert np.array_equal(val[b, : cnt[b]], lists[b][want])
        assert (idx[b, cnt[b] :] == -1).all() and np.isnan(val[b, cnt[b] :]).all()


@pytest.mark.parametrize("L", [1, 7, 8, 9, 127, 128, 129, 136, 255, 256, 257, 1000, 65537, 70001])
def test_row_lengths_across_the_pairwise_tree(cuda_lib, L):
    """Row lengths across the 8 / 128 leaf sizes and the splits, and beyond 2^16: the exact linear transform's keys
    within 2 ulps, for n of 0, 1, 100, more than the valid count, lk_topn_max(), beyond it, and every item."""
    rng = np.random.default_rng(L)
    s = rng.standard_normal(L).astype(np.float32)
    s[rng.random(L) < 0.03] = np.nan
    it = ItemList(item_ids=np.arange(L), scores=s)
    n_max = int(cuda_lib.lk_topn_max())
    for n in (0, 1, 100, int(np.isfinite(s).sum()) + 3, n_max, n_max + 7, -1):
        r = StochasticTopNRanker(rng=L, transform="linear")
        gen = np.random.default_rng(L)
        got = r(it, None, n, include_weights=True)
        pos, k = so.rank(s, None if n < 0 else n, "linear", 1.0, gen)
        if n == 0:
            pos, k = pos[:0], k[:0]
        assert compare(got, pos, k, "linear", np.arange(L)) == 0
        assert r._rng_factory.rng.bit_generator.state == gen.bit_generator.state


@pytest.mark.parametrize("contiguous", [False, True])
def test_rank_scores_of_a_factor_score_matrix(cuda_lib, contiguous):
    """rank_scores on an item-major score matrix's transpose (no copy) and on a contiguous one: each query's list is
    every item minus its query items, against the oracle on those candidate lists; an unscorable query (a NaN
    column) gets an empty list and draws nothing."""
    rng = np.random.default_rng(8)
    n_items, B, k = 3000, 24, 16
    dev = _lib.require_device()
    q = torch.from_numpy((rng.standard_normal((n_items, k)) * 0.3).astype(np.float32)).to(dev)
    x = torch.from_numpy((rng.standard_normal((B, k)) * 0.3).astype(np.float32)).to(dev)
    S = engine.als_recommend(q, x)  # [n_items, B]
    S[:, 5] = float("nan")
    M = S.T.contiguous() if contiguous else S.T
    vocab = Vocabulary(np.arange(n_items) * 3 + 1, "item")
    hists = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(B)]
    queries = [RecQuery(None, ItemList(item_ids=vocab.ids(h))) if len(h) else RecQuery(None, None) for h in hists]
    host = S.T.cpu().numpy()
    exceptions = 0
    for transform in ("softmax", "linear"):
        r = StochasticTopNRanker(rng=9, transform=transform, scale=2.0)
        got = r.rank_scores(M, queries, vocab, 50, include_weights=True)
        gen = np.random.default_rng(9)
        for b, (g, h) in enumerate(zip(got, hists)):
            cand = np.setdiff1d(np.arange(n_items), h)
            pos, kk = so.rank(host[b, cand], 50, transform, 2.0, gen)
            exceptions += compare(g, cand[pos], kk, transform, vocab.ids())
            assert np.array_equal(g.scores(), host[b, g.numbers()])
        assert len(got[5]) == 0
        assert r._rng_factory.rng.bit_generator.state == gen.bit_generator.state
    assert exceptions == 0, f"{exceptions} near-tie exceptions"
    none = StochasticTopNRanker(rng=9).rank_scores(M, queries, vocab, 10, exclude=None)
    assert all(len(x) == (0 if b == 5 else 10) for b, x in enumerate(none))


def test_pickled_ranker_continues_the_stream(cuda_lib):
    rng = np.random.default_rng(2)
    it = ItemList(item_ids=np.arange(300), scores=rng.standard_normal(300).astype(np.float32))
    r = StochasticTopNRanker(rng=4, n=10)
    r(it)
    r2 = pickle.loads(pickle.dumps(r))
    a, b = r(it, include_weights=True), r2(it, include_weights=True)
    assert np.array_equal(a.ids(), b.ids()) and np.array_equal(a.field("weight"), b.field("weight"))
    assert r._rng_factory.rng.bit_generator.state == r2._rng_factory.rng.bit_generator.state
