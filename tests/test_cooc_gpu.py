"""
Co-occurrence counting and association scoring on the GPU, bit for bit against ``tests/cooc_oracle.py``.
"""

import numpy as np
import pyarrow as pa
import pytest
import torch

import cooc_oracle as co
import oracle
from lkpy_b200 import _lib, accel, data, engine
from lkpy_b200.association import AssociationScorer
from lkpy_b200.components import Dataset, ItemList

pytestmark = pytest.mark.gpu


def _dup_data(seed=3, n_groups=300, n_items=700, nnz=20_000):
    """Groups ascending, items in any order within a group, repeats inside groups, empty groups and items."""
    rng = np.random.default_rng(seed)
    g = np.sort(rng.integers(0, n_groups, nnz)).astype(np.int32)
    i = (rng.zipf(1.3, nnz) % (n_items - 5)).astype(np.int32)  # the last five items never occur
    g[g == 7] = 8  # group 7 is empty
    return n_groups, n_items, np.sort(g, kind="stable"), i


def _run(task):
    return accel.run_accel_task(task)


@pytest.mark.parametrize("diagonal", [True, False])
@pytest.mark.parametrize("which", ["ml_small", "dups"])
def test_count_and_dense_cooc(cuda_lib, ml_small, which, diagonal):
    if which == "ml_small":
        ng, ni, g, i = ml_small.n_users, ml_small.n_items, ml_small.users, ml_small.items
    else:
        ng, ni, g, i = _dup_data()
    got = _run(accel.data.count_cooc(ng, ni, pa.array(g), pa.array(i), diagonal=diagonal))
    want = co.count_cooc(ng, ni, g, i, diagonal=diagonal)
    assert len(got) == len(want)
    for b, w in zip(got, want):
        assert b.schema.names == ["row", "col", "count"]
        assert all(not f.nullable and f.type == pa.int32() for f in b.schema)
        for k, col in enumerate(("row", "col", "count")):
            assert np.array_equal(b.column(col).to_numpy(), w[k]), col
    dense = _run(accel.data.dense_cooc(ng, ni, pa.array(g), pa.array(i), diagonal=diagonal))
    assert dense.dtype == np.float32 and np.array_equal(dense, co.dense_cooc(ng, ni, g, i, diagonal=diagonal))


def test_count_rows_at_ml25m_shape(cuda_lib):
    """Sampled rows, the most expensive ones included, at the ML-25M shape, against XᵀX rows."""
    it = data.synth_interactions(**data.ML25M_SHAPE)
    dev = _lib.require_device()
    plan = engine.CoocPlan.create(it.n_users, it.n_items, torch.from_numpy(it.users).to(dev),
                                  torch.from_numpy(it.items).to(dev))  # fmt: skip
    indptr, cols, cnt = (t.cpu().numpy() for t in plan.count(full_rows=False))
    cost = plan.row_cost(False).cpu().numpy()
    X = co.count_matrix(it.n_users, it.n_items, it.users, it.items).tocsc()
    rng = np.random.default_rng(0)
    rows = np.unique(np.concatenate([np.argsort(-cost, kind="stable")[:4], rng.integers(0, it.n_items, 12)]))
    for r in rows:
        full = (X[:, [int(r)]].T @ X).toarray()[0]
        full[: r + 1] = 0
        nz = np.flatnonzero(full)
        lo, hi = indptr[r], indptr[r + 1]
        assert np.array_equal(cols[lo:hi], nz) and np.array_equal(cnt[lo:hi], full[nz]), r
    print(f"ML-25M shape: {int(indptr[-1])} upper-triangle entries")


def test_count_cancel_stops_the_kernel(cuda_lib):
    ng, ni, g, i = _dup_data()
    dev = _lib.require_device()
    plan = engine.CoocPlan.create(ng, ni, torch.from_numpy(g).to(dev), torch.from_numpy(i).to(dev))
    raised = torch.ones(1, dtype=torch.int32, device=dev)
    indptr, _c, _v = plan.count(attach=lambda counter, units: raised)
    assert int(indptr[-1]) == 0 and int(plan.work_counter.item()) == 0  # no unit was handed out
    task = accel.data.count_cooc(ng, ni, pa.array(g), pa.array(i))
    orig = task._attach

    def attach(counter, units):
        task._cancelled.set()  # cancelled once the kernel's flag exists: the flag is raised before the launch
        return orig(counter, units)

    task._attach = attach
    with pytest.raises(RuntimeError, match="cancelled"):
        task.invoke()


def _dataset(which, ml_small):
    if which == "ml_small":
        return Dataset(ml_small)
    it = data.synth_interactions(900, 400, 30_000, seed=5)
    return Dataset(it)


CONFIGS = [dict(method="probability"), dict(method="lift"), dict(method="lift", damping=0.1)]


@pytest.mark.parametrize("cfg", CONFIGS)
def test_assoc_matrix(cuda_lib, ml_small, cfg):
    it = ml_small
    m = AssociationScorer(**cfg)
    m.train(Dataset(it))
    want = co.assoc_matrix(it.n_users, it.n_items, it.users, it.items, cfg["method"], cfg.get("damping", 0.0))
    got = m.assoc_scores
    assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data.view(np.int32), want.data.astype(np.float32).view(np.int32))
    assert np.array_equal(m.item_freqs, np.bincount(it.items, minlength=it.n_items))


def _queries(ds, rng, n=40):
    it = ds.interactions
    qs = []
    for u in rng.choice(it.n_users, n, replace=False):
        h = ds.user_history(int(u))
        nums = h.numbers()
        if len(nums) and u % 3 == 0:  # repeated reference items
            nums = np.concatenate([nums, nums[: max(1, len(nums) // 3)]])
        qs.append(nums)
    qs.append(np.zeros(0, np.int32))  # empty query
    qs.append(np.array([0, 0, 0], np.int32))
    return qs


@pytest.mark.parametrize("max_nbrs", [None, 1])
@pytest.mark.parametrize("cfg", CONFIGS)
def test_score_batch(cuda_lib, ml_small, cfg, max_nbrs):
    ds = Dataset(ml_small)
    m = AssociationScorer(**cfg, max_nbrs=max_nbrs)
    m.train(ds)
    A = m.assoc_scores
    rng = np.random.default_rng(1)
    qs = _queries(ds, rng)
    ids = ds.items.ids()
    hist = [ItemList(item_ids=np.concatenate([ids[q], [ids.max() + 1]]) if len(q) else ids[q]) for q in qs]
    tgt_nums = rng.integers(0, len(ids), 300)
    tgt = ItemList(item_ids=np.concatenate([ids[tgt_nums], [ids.max() + 1]]))
    got = m.score_batch(hist, [tgt] * len(hist))
    for q, g in zip(qs, got):
        full = co.score(A, q, max_nbrs)
        want = np.concatenate([full[tgt_nums], [np.nan]]).astype(np.float32)
        s = g.scores()
        assert np.array_equal(np.isnan(s), np.isnan(want))
        ok = ~np.isnan(want)
        assert np.array_equal(s[ok].view(np.int32), want[ok].view(np.int32))
    one = m(hist[0], tgt)
    assert np.array_equal(one.scores(), got[0].scores(), equal_nan=True)


@pytest.mark.parametrize("exclude", ["query", None])
@pytest.mark.parametrize("max_nbrs", [None, 1])
@pytest.mark.parametrize("which", ["ml_small", "synth"])
def test_recommend_batch(cuda_lib, ml_small, which, max_nbrs, exclude):
    ds = _dataset(which, ml_small)
    m = AssociationScorer(method="lift", damping=0.1 if which == "synth" else 0.0, max_nbrs=max_nbrs)
    m.train(ds)
    A = m.assoc_scores
    rng = np.random.default_rng(2)
    qs = _queries(ds, rng, 30)
    qs.append(np.array([int(np.argmin(np.diff(A.indptr)))], np.int32))  # few non-zero scores: lists fill with 0 ties
    hist = [ItemList(item_nums=q, vocabulary=ds.items) for q in qs]
    n_items = ds.item_count
    for n in (1, 10, 1024):
        got = m.recommend_batch(hist, n, exclude=exclude)
        for q, g in zip(qs, got):
            s = co.score(A, q, max_nbrs).copy()
            if exclude == "query":
                s[q] = np.nan
            want = oracle.argtopn(s, min(n, n_items))
            assert np.array_equal(g.numbers(), want)
            assert np.array_equal(g.scores().view(np.int32), s[want].view(np.int32))
    m.config = m.config.model_copy(update={"max_nbrs": 3})
    with pytest.raises(NotImplementedError):
        m.recommend_batch(hist, 5)


def test_pickle_round_trip(cuda_lib, ml_small):
    import pickle

    ds = Dataset(ml_small)
    m = AssociationScorer(method="lift")
    m.train(ds)
    hist = [ds.user_history(3), ds.user_history(11)]
    a = m.recommend_batch(hist, 20)
    m2 = pickle.loads(pickle.dumps(m))
    b = m2.recommend_batch(hist, 20)
    for x, y in zip(a, b):
        assert np.array_equal(x.numbers(), y.numbers()) and np.array_equal(x.scores(), y.scores())
