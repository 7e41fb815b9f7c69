"""
Batched ALS scoring and recommendation on the device (``lk_als_recommend_batch``) against the oracle, bit for bit:

    score mode   S = als_scores(Q, X, item_offset, query_offset)      (tests/als_oracle.py)
    rank mode    for each query: argtopn over S[:, b] with the excluded items set to NaN (oracle.argtopn)

and the ALS components' ``recommend_batch`` against the host composition: candidates = all items minus the
query's items, scores from the ``score_matrix`` column, ``oracle.argtopn``.
"""

import pickle

import numpy as np
import pytest
import torch
from als_oracle import als_scores

import oracle
from lkpy_b200 import _lib, engine
from lkpy_b200.components import Dataset, ItemList, RecQuery, TrainingOptions

pytestmark = pytest.mark.gpu

IT = 128  # items per tile (als_recommend.cu)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_lib.require_device())


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _factors(rng, n_items, B, k, integer=False):
    if integer:  # small integers: many scores tie exactly
        return (rng.integers(-2, 3, (n_items, k)).astype(np.float32), rng.integers(-2, 3, (B, k)).astype(np.float32))
    return rng.standard_normal((n_items, k)).astype(np.float32), rng.standard_normal((B, k)).astype(np.float32)


def _excl_lists(rng, n_items, B):
    lists = []
    for b in range(B):
        kind = b % 5
        if kind == 0:
            e = np.zeros(0, np.int64)  # empty
        elif kind == 1:
            e = rng.integers(0, n_items, int(rng.integers(1, 40)))  # unsorted, repeats
        elif kind == 2:
            e = np.concatenate([[-1, -1], rng.integers(0, n_items, 10), [-1]])  # negative entries
        elif kind == 3:
            e = rng.permutation(n_items)  # every item: count 0
        else:
            e = np.concatenate([rng.integers(0, n_items, 5), [n_items + 3]])  # an unknown number
        lists.append(np.asarray(e, dtype=np.int32))
    ptr = np.zeros(B + 1, np.int64)
    ptr[1:] = np.cumsum([len(e) for e in lists])
    return lists, ptr, np.concatenate(lists) if lists else np.zeros(0, np.int32)


def _check_rank(idx, val, cnt, S, n, lists=None):
    for b in range(S.shape[1]):
        col = S[:, b].copy()
        if lists is not None:
            e = lists[b]
            col[e[(e >= 0) & (e < len(col))]] = np.nan
        want = oracle.argtopn(col, n)
        c = int(cnt[b])
        assert c == len(want), b
        assert np.array_equal(idx[b, :c], want), b
        assert np.array_equal(_bits(val[b, :c]), _bits(col[want])), b
        assert (idx[b, c:] == -1).all() and np.isnan(val[b, c:]).all(), b


@pytest.mark.parametrize("k", [1, 8, 33, 64, 100, 128])
@pytest.mark.parametrize("B", [1, 7, 65, 1000])
def test_score_mode_bit_exact(cuda_lib, k, B):
    rng = np.random.default_rng(k * 1000 + B)
    n_items = 3 * IT + 37  # not a multiple of the item tile
    Q, X = _factors(rng, n_items, B, k)
    io = rng.standard_normal(n_items).astype(np.float32)
    qo = rng.standard_normal(B).astype(np.float32)
    for item_off, query_off in ((None, None), (io, None), (None, qo), (io, qo)):
        S = engine.als_recommend(
            _t(Q), _t(X), None, None if item_off is None else _t(item_off), None if query_off is None else _t(query_off)
        ).cpu().numpy()
        want = als_scores(Q, X, item_off, query_off)
        assert S.shape == (n_items, B)
        assert np.array_equal(_bits(S), _bits(want)), (item_off is not None, query_off is not None)


@pytest.mark.parametrize("n", [1, 10, 100, 1024])
@pytest.mark.parametrize("integer", [False, True])
def test_rank_mode_bit_exact(cuda_lib, n, integer):
    rng = np.random.default_rng(n + 7 * integer)
    n_items, B, k = 9 * IT + 5, 130, 24
    Q, X = _factors(rng, n_items, B, k, integer)
    io = rng.integers(-1, 2, n_items).astype(np.float32) if integer else rng.standard_normal(n_items).astype(np.float32)
    S = als_scores(Q, X, io)
    lists, ptr, items = _excl_lists(rng, n_items, B)
    idx, val, cnt = (t.cpu().numpy() for t in engine.als_recommend(_t(Q), _t(X), n, _t(io), None, _t(ptr), _t(items)))
    _check_rank(idx, val, cnt, S, n, lists)
    assert cnt[3] == 0  # query 3 excludes every item
    idx, val, cnt = (t.cpu().numpy() for t in engine.als_recommend(_t(Q), _t(X), n, _t(io)))
    _check_rank(idx, val, cnt, S, n)


def test_rank_mode_more_than_candidates(cuda_lib):
    rng = np.random.default_rng(3)
    n_items, B, k = 50, 20, 8
    Q, X = _factors(rng, n_items, B, k, integer=True)
    qo = rng.standard_normal(B).astype(np.float32)
    S = als_scores(Q, X, None, qo)
    lists, ptr, items = _excl_lists(rng, n_items, B)
    for n in (50, 200, 1024):
        idx, val, cnt = (t.cpu().numpy() for t in engine.als_recommend(_t(Q), _t(X), n, None, _t(qo), _t(ptr), _t(items)))
        _check_rank(idx, val, cnt, S, n, lists)
    with pytest.raises(ValueError):
        engine.als_recommend(_t(Q), _t(X), 1025)


def test_batch_independence(cuda_lib):
    rng = np.random.default_rng(17)
    n_items, B, k = 20 * IT + 3, 4096, 64
    Q, X = _factors(rng, n_items, B, k)
    io = rng.standard_normal(n_items).astype(np.float32)
    qo = rng.standard_normal(B).astype(np.float32)
    dQ, dX, dio, dqo = _t(Q), _t(X), _t(io), _t(qo)
    S_all = engine.als_recommend(dQ, dX, None, dio, dqo).cpu().numpy()
    r_all = [t.cpu().numpy() for t in engine.als_recommend(dQ, dX, 100, dio, dqo)]
    for size in (1, 33):
        for b0 in (0, 1000, 4096 - size):
            sl = slice(b0, b0 + size)
            S = engine.als_recommend(dQ, dX[sl], None, dio, dqo[sl]).cpu().numpy()
            assert np.array_equal(_bits(S), _bits(S_all[:, sl])), (size, b0)
            idx, val, cnt = (t.cpu().numpy() for t in engine.als_recommend(dQ, dX[sl], 100, dio, dqo[sl]))
            assert np.array_equal(idx, r_all[0][sl]) and np.array_equal(cnt, r_all[2][sl]), (size, b0)
            assert np.array_equal(_bits(val), _bits(r_all[1][sl])), (size, b0)
    # argtopn of a score-mode column is the rank-mode list
    for b in range(0, B, 97):
        want = oracle.argtopn(S_all[:, b], 100)
        assert np.array_equal(r_all[0][b], want), b


def test_many_tiles(cuda_lib):
    rng = np.random.default_rng(59047)
    n_items, B, k = 59047, 4096, 64
    Q = (rng.standard_normal((n_items, k)) * 0.1).astype(np.float32)
    X = (rng.standard_normal((B, k)) * 0.1).astype(np.float32)
    sample = np.sort(rng.choice(B, 64, replace=False))
    lists, ptr, items = _excl_lists(rng, n_items, B)
    S_dev = engine.als_recommend(_t(Q), _t(X), None)
    S_sample = S_dev[:, torch.from_numpy(sample).to(S_dev.device)].cpu().numpy()
    del S_dev
    want = als_scores(Q, X[sample])
    assert np.array_equal(_bits(S_sample), _bits(want))
    idx, val, cnt = (t.cpu().numpy() for t in engine.als_recommend(_t(Q), _t(X), 100, None, None, _t(ptr), _t(items)))
    _check_rank(idx[sample], val[sample], cnt[sample], want, 100, [lists[b] for b in sample])


# ---------------------------------------------------------------------------------------------
# components
# ---------------------------------------------------------------------------------------------


def _models(ml_small):
    from lkpy_b200.als import BiasedMFScorer, ImplicitMFScorer

    ds = Dataset(ml_small)
    out = []
    for m in (ImplicitMFScorer(features=32, epochs=3), ImplicitMFScorer(features=24, epochs=3, use_ratings=True),
              BiasedMFScorer(features=16, epochs=3)):  # fmt: skip
        m.train(ds, TrainingOptions(rng=7))
        out.append(m)
    return ds, out


def _queries(ml_small, ds):
    empty = ItemList(item_ids=ds.user_history(5).ids()[:0])
    return [
        RecQuery(user_id=ml_small.user_ids[3]),  # known user, no history given
        RecQuery(user_id=ml_small.user_ids[50], query_items=ds.user_history(50)),  # fold-in, own history
        RecQuery(user_id=None, query_items=ds.user_history(77)),  # fold-in, anonymous
        RecQuery(user_id=-12345),  # unknown user, no history
        RecQuery(user_id=-12345, query_items=empty),  # empty history
        RecQuery(user_id=ml_small.user_ids[400], query_items=empty),  # known user, empty history
    ]


def _host_expected(model, q, S_col, n, exclude):
    n_items = len(S_col)
    cands = np.arange(n_items, dtype=np.int32)
    if exclude == "query" and q.query_items is not None and len(q.query_items) > 0:
        nums = q.query_items.numbers(vocabulary=model.items, missing="negative")
        cands = np.setdiff1d(cands, nums[nums >= 0]).astype(np.int32)
    sc = S_col[cands]
    top = oracle.argtopn(sc, n)
    return cands[top], sc[top]


@pytest.mark.parametrize("exclude", ["query", None])
def test_components_match_host_composition(cuda_lib, ml_small, exclude):
    ds, models = _models(ml_small)
    queries = _queries(ml_small, ds)
    for m in models:
        S = m.score_matrix(queries).cpu().numpy()
        for n in (1, 10, 100, 1024):
            recs = m.recommend_batch(queries, n, exclude=exclude)
            assert len(recs) == len(queries)
            for b, q in enumerate(queries):
                if np.isnan(S[:, b]).all():
                    assert len(recs[b]) == 0, b
                    continue
                items, scores = _host_expected(m, q, S[:, b], n, exclude)
                assert np.array_equal(recs[b].numbers(vocabulary=m.items), items), (type(m).__name__, n, b)
                assert np.array_equal(recs[b].ids(), ml_small.item_ids[items])
                assert np.array_equal(_bits(recs[b].scores()), _bits(scores)), (type(m).__name__, n, b)
        assert all(len(r) == 0 for r in m.recommend_batch(queries, 0, exclude=exclude))
        assert all(len(r) == 0 for r in m.recommend_batch(queries, -3, exclude=exclude))
        with pytest.raises(ValueError):
            m.recommend_batch(queries, 1025, exclude=exclude)
    # the unknown user without history is unscorable
    assert len(models[0].recommend_batch(queries, 10)[3]) == 0


def test_components_pickle_round_trip(cuda_lib, ml_small):
    ds, models = _models(ml_small)
    queries = _queries(ml_small, ds)
    for m in models:
        before = m.recommend_batch(queries, 50, exclude="query")
        m2 = pickle.loads(pickle.dumps(m))
        # the device item table stays out of the pickle: it loads without a GPU
        state = [x for v in m2.__dict__.values() for x in (v if isinstance(v, tuple) else (v,))]
        assert not any(isinstance(x, torch.Tensor) for x in state)
        after = m2.recommend_batch(queries, 50, exclude="query")
        for r0, r1 in zip(before, after):
            assert np.array_equal(r0.numbers(vocabulary=m.items), r1.numbers(vocabulary=m2.items))
            assert np.array_equal(_bits(r0.scores()), _bits(r1.scores()))
