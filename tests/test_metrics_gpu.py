"""
The ranking metrics on the device (``lk_rank_metrics``, ``lk_item_exposure``) against the host restatements of
lkpy_b200/metrics.py, bit for bit with NaN in the same places: on the recorded reference cases, on randomised
batches, from a top-n kernel's output (``measure_topn``), and at the benchmark's shape (ML-25M-shaped synthetic,
every user with a rating, top-100 from the bias scorer, about 20 % of each user's items held out).
"""

import os
import warnings

import numpy as np
import pytest
import torch

import metrics_ref_sandbox as mrs
from lkpy_b200 import data, engine
from lkpy_b200 import metrics as lm
from lkpy_b200.basic import BiasScorer
from lkpy_b200.components import Dataset, ItemList, Vocabulary
from lkpy_b200.data import Interactions
from test_metrics import cases, metric, reference_golden, same_bits

pytestmark = pytest.mark.gpu

LIST_CONFIGS = [k for k, (c, _kw) in mrs.CONFIGS.items() if c not in mrs.GINI]
GINI_CONFIGS = [k for k, (c, _kw) in mrs.CONFIGS.items() if c in mrs.GINI]


def host(metrics, outputs, tests):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return lm.measure_lists_host(metrics, outputs, tests)


def check_run(got: lm.RunMetrics, want: lm.RunMetrics):
    """Per-list values bit for bit, and the summaries equal (NaN matching NaN)."""
    assert list(got.list_metrics.columns) == list(want.list_metrics.columns)
    for c in want.list_metrics.columns:
        assert same_bits(got.list_metrics[c].to_numpy(), want.list_metrics[c].to_numpy()), c
    assert got.summary_metrics.keys() == want.summary_metrics.keys()
    for k, v in want.summary_metrics.items():
        assert same_bits([got.summary_metrics[k]], [v]), k


@pytest.mark.parametrize("name", LIST_CONFIGS)
def test_recorded_cases(cuda_lib, name):
    """The device on every recorded list the reference measures, bit for bit with the recording; a batch holding a
    list where the reference divides by zero raises ``ZeroDivisionError`` as the reference does."""
    g = reference_golden("metrics_values")
    recs, tests, vocab, stats = cases()
    m = metric(name, vocab, stats)
    ok = ~g[f"raised_{name}"]
    sel = np.flatnonzero(ok)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = lm.measure_batch([m], [recs[b] for b in sel], [tests[b] for b in sel])
    assert same_bits(got.list_metrics[m.label].to_numpy(), g[name][ok]), name
    if not ok.all():
        with pytest.raises(ZeroDivisionError):
            lm.measure_batch([m], recs, tests)


def test_recorded_cases_together(cuda_lib):
    """A metric of every kind and option in one batch, against the host path; and the Gini metrics against the
    recording: per-item totals bit for bit, coefficients equal."""
    g = reference_golden("metrics_values")
    all_recs, all_tests, vocab, stats = cases()
    known = mrs.known([r.ids() for r in all_recs])
    keep = known & ~np.any([g[f"raised_{n}"] for n in LIST_CONFIGS], axis=0)
    recs = [r for r, k in zip(all_recs, keep) if k]
    tests = [t for t, k in zip(all_tests, keep) if k]
    ms, labels = [], set()
    for n in mrs.CONFIGS:  # one metric per label, as a collector requires
        m = metric(n, vocab, stats)
        if m.label not in labels:
            ms.append(m)
            labels.add(m.label)
    check_run(lm.measure_batch(ms, recs, tests), host(ms, recs, tests))
    recs_k = [r for r, k in zip(all_recs, known) if k]
    tests_k = [t for t, k in zip(all_tests, known) if k]
    lens = np.array([len(r) for r in recs_k])
    ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)])).cuda()
    items = torch.from_numpy(np.concatenate([vocab.numbers(r.ids()) for r in recs_k]).astype(np.int32)).cuda()
    for n in GINI_CONFIGS:
        m = metric(n, vocab, stats)
        assert lm.measure_batch([m], recs_k, tests_k).summary_metrics[m.label] == float(g[f"gini_{n}"]), n
        assert same_bits(lm._gini_totals(m, vocab, ptr, items, lens).totals, g[f"totals_{n}"]), n


def random_batch(rng, B: int, n_items: int, max_len: int, ordered=True):
    ids = np.arange(n_items, dtype=np.int64) * 3 + 1
    vocab = Vocabulary(ids, "item")
    recs, tests = [], []
    for _ in range(B):
        L = int(rng.choice([0, 1, 5, 8, 20, 100, 127, 129, max_len])) if rng.random() < 0.3 else int(rng.integers(0, max_len + 1))
        nums = rng.choice(n_items, L, replace=False).astype(np.int32)
        recs.append(ItemList(item_ids=ids[nums], item_nums=nums, vocabulary=vocab, ordered=ordered))
        T = int(rng.integers(0, 3 * L + 5)) if rng.random() < 0.9 else 0
        t = rng.choice(ids, min(T, n_items), replace=False)
        if rng.random() < 0.2 and len(t):
            t = np.concatenate([t, t[:2], [-7]])
        tests.append(ItemList(item_ids=rng.permutation(t)))
    return vocab, recs, tests


def test_randomised_batches(cuda_lib):
    """Random lists (up to 1024 items, a shared vocabulary) with every metric and option, against the host path."""
    rng = np.random.default_rng(17)
    for _ in range(3):
        vocab, recs, tests = random_batch(rng, 400, 3000, 1024)
        n_users = 50
        inter = Interactions(np.repeat(np.arange(n_users, dtype=np.int32), 60),
                             np.concatenate([np.sort(rng.choice(3000, 60, replace=False)) for _ in range(n_users)]).astype(np.int32),
                             np.ones(n_users * 60, np.float32), n_users, 3000, item_ids=vocab.ids())  # fmt: skip
        ds = Dataset(inter)
        ms = [lm.Hit(10), lm.Precision(), lm.Recall(20), lm.RecipRank(), lm.DCG(), lm.NDCG(), lm.NDCG(100),
              lm.RBP(patience=0.6),
              lm.MeanPopRank(ds, n=30), lm.MeanPopRank(ds), lm.ListGini(items=vocab), lm.ExposureGini(20, items=ds)]
        # AveragePrecision raises on an empty test set, and RBP normalised by list sums on an empty list
        ok = [len(t) > 0 and len(r) > 0 for r, t in zip(recs, tests)]
        ms_ap = [lm.AveragePrecision(), lm.AveragePrecision(10), lm.RBP(normalize=True),
                 lm.RBP(50, weight=lm.LogRankWeight(base=3, offset=2))]
        check_run(lm.measure_batch(ms, recs, tests), host(ms, recs, tests))
        r2 = [r for r, k in zip(recs, ok) if k]
        t2 = [t for t, k in zip(tests, ok) if k]
        check_run(lm.measure_batch(ms_ap, r2, t2), host(ms_ap, r2, t2))
    # more metrics than one launch takes (32): two groups
    many = [lm.Precision(n) for n in range(1, 41)] + [lm.NDCG(n) for n in (1, 2, 1000)]
    check_run(lm.measure_batch(many, recs, tests), host(many, recs, tests))


def test_lists_without_a_vocabulary_and_unordered_lists(cuda_lib):
    rng = np.random.default_rng(8)
    vocab, recs, tests = random_batch(rng, 60, 500, 40)
    bare = [ItemList(item_ids=r.ids(), ordered=True) for r in recs]
    ms = [lm.NDCG(10), lm.Hit(), lm.MeanPopRank(lm.item_counts(Interactions(
        np.zeros(3, np.int32), np.arange(3, dtype=np.int32), np.ones(3, np.float32), 1, 500, item_ids=vocab.ids())))]
    check_run(lm.measure_batch(ms, bare, tests), host(ms, bare, tests))
    unordered = [ItemList(item_ids=r.ids()) for r in recs]
    with pytest.raises(ValueError, match="ordered"):
        lm.measure_batch([lm.Hit(5)], unordered, tests)
    with pytest.raises(TypeError, match="not ordered"):
        lm.measure_batch([lm.DCG()], unordered, tests)
    check_run(lm.measure_batch([lm.Hit(), lm.Recall()], unordered, tests), host([lm.Hit(), lm.Recall()], unordered, tests))
    with pytest.raises(ValueError, match="1024"):
        lm.measure_batch([lm.Hit()], [ItemList(item_ids=np.arange(1025), ordered=True)], [ItemList(item_ids=[1])])


def test_measure_topn_is_measure_batch(cuda_lib, ml_small):
    """``measure_topn`` on ``BiasScorer.recommend_batch``'s output gives what ``measure_batch`` gives on its lists."""
    scorer = BiasScorer()
    ds = Dataset(ml_small)
    scorer.train(ds)
    users = ds.users.ids()[:300]
    lists = [ItemList(r, ordered=True) for r in scorer.recommend_batch(list(users), 60)]
    rng = np.random.default_rng(4)
    tests = [ItemList(item_ids=np.concatenate([rng.choice(r.ids(), 5), rng.choice(ds.items.ids(), 20)])) for r in lists]
    n = max(len(r) for r in lists)
    idx = np.full((len(lists), n), -1, np.int32)
    for b, r in enumerate(lists):
        idx[b, : len(r)] = r.numbers()
    cnt = torch.tensor([len(r) for r in lists], dtype=torch.int32, device="cuda")
    ms = [lm.NDCG(), lm.NDCG(10), lm.RBP(), lm.Recall(20), lm.AveragePrecision(), lm.MeanPopRank(ds, n=10),
          lm.ListGini(items=ds.items), lm.ExposureGini(10, items=ds.items)]  # fmt: skip
    got = lm.measure_topn(ms, ds.items, torch.from_numpy(idx).cuda(), cnt, tests)
    check_run(got, lm.measure_batch(ms, lists, tests))
    check_run(got, host(ms, lists, tests))


# ---------------------------------------------------------------------------------------------------------------
# the benchmark's shape
# ---------------------------------------------------------------------------------------------------------------


def ml25m_topn(seed: int = 31, n: int = 100):
    """The ML-25M shape split into train and about 20 % test per user, the bias scorer trained on train, and each
    user's top ``n`` over the items not in their train set: ``(vocab, idx, cnt, tests)``."""
    it = data.synth_interactions_cached(os.environ.get("LK_BENCH_DATA_CACHE"), **data.ML25M_SHAPE)
    test = np.random.default_rng(seed).random(it.nnz) < 0.2
    # every user keeps at least one test item (AveragePrecision divides by the test length)
    rated = np.bincount(it.users, minlength=it.n_users) > 0
    none = np.flatnonzero(rated & (np.bincount(it.users[test], minlength=it.n_users) == 0))
    test[np.searchsorted(it.users, none)] = True
    users = np.flatnonzero(rated)  # the users with a test set: a user without ratings has none to measure
    tr = Interactions(it.users[~test], it.items[~test], it.ratings[~test], it.n_users, it.n_items)
    scorer = BiasScorer()
    ds = Dataset(tr)
    scorer.train(ds)
    dev = torch.device("cuda")
    # each user's training items, excluded from their list (users without ratings have empty rows: dropped)
    excl_indptr = torch.from_numpy(np.searchsorted(tr.users, np.append(users, it.n_users)).astype(np.int64)).to(dev)
    excl_items = torch.from_numpy(tr.items.astype(np.int32)).to(dev)
    idx, _val, cnt = engine.offset_scores(scorer._device_base(), len(users), None, n, excl_indptr, excl_items)
    tptr = np.searchsorted(it.users[test], np.arange(it.n_users + 1))
    titems = ds.items.ids(it.items[test])
    tests = [ItemList(item_ids=titems[tptr[u] : tptr[u + 1]]) for u in users]
    return ds, idx, cnt, tests


TEN = lambda ds: [lm.NDCG(), lm.NDCG(10), lm.DCG(), lm.RBP(), lm.RecipRank(), lm.Hit(10), lm.Precision(10),  # noqa: E731
                  lm.Recall(10), lm.AveragePrecision(), lm.MeanPopRank(ds)]  # fmt: skip


def test_ml25m_shape(cuda_lib):
    ds, idx, cnt, tests = ml25m_topn()
    B = idx.shape[0]
    assert B > 150_000 and int(cnt.min()) == 100 and min(len(t) for t in tests) >= 1
    ms = TEN(ds) + [lm.ListGini(items=ds.items), lm.ExposureGini(items=ds.items)]
    got = lm.measure_topn(ms, ds.items, idx, cnt, tests)
    # sampled lists and the longest test sets against the host path
    nrel = np.array([len(t) for t in tests])
    rng = np.random.default_rng(6)
    sample = np.unique(np.concatenate([rng.choice(B, 1500, replace=False), np.argsort(nrel)[-50:]]))
    assert nrel[sample].max() == nrel.max() and nrel.max() > 1000
    idx_h = idx[torch.from_numpy(sample).cuda()].cpu().numpy()
    lists = [ItemList(item_nums=idx_h[j], vocabulary=ds.items, ordered=True) for j in range(len(sample))]
    want = host(TEN(ds), lists, [tests[b] for b in sample])
    for c in want.list_metrics.columns:
        assert same_bits(got.list_metrics[c].to_numpy()[sample], want.list_metrics[c].to_numpy()), c
    # the summaries: the reference's statements over the device's values
    for c in want.list_metrics.columns:
        v = got.list_metrics[c].to_numpy()
        v = v[~np.isnan(v)]
        assert got.summary_metrics[f"{c}.n"] == len(v) and got.summary_metrics[f"{c}.mean"] == np.mean(v)
        assert got.summary_metrics[f"{c}.median"] == np.median(v) and got.summary_metrics[f"{c}.std"] == np.std(v)
    # Gini totals: the host accumulator over every list
    all_idx = idx.cpu().numpy()
    for m in ms[-2:]:
        acc = m.create_accumulator()
        for b in range(B):
            acc.add(m.measure_list(ItemList(item_nums=all_idx[b], vocabulary=ds.items, ordered=True), tests[b]))
        lens = np.full(B, 100)
        dev = idx.device
        ptr = torch.arange(B + 1, dtype=torch.int64, device=dev) * 100
        totals = lm._gini_totals(m, ds.items, ptr, idx.reshape(-1).contiguous(), lens).totals
        assert same_bits(totals, acc.totals), m.label
        assert got.summary_metrics[m.label] == acc.accumulate()
