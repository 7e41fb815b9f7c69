"""
GPU parity: item-kNN build (bit-exact vs the oracle) and scoring (exact vs the
oracle's ScoreAccumulator emulation, and against the reference's golden CSV).
"""

import os
from pathlib import Path

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sps
import torch

import oracle
from lkpy_b200 import _lib, data, engine

from helpers import small_synth

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


def _build(ui, iu, min_sim, save_nbrs, order=None, world=1):
    dev = _lib.require_device()
    d_ui = engine.DeviceCSR.from_host(ui, dev)
    d_iu = engine.DeviceCSR.from_host(iu, dev)
    plan = engine.KnnBuildPlan.create(d_ui, d_iu, world=world)
    if save_nbrs:
        cols, vals, cnt = plan.build_topk(min_sim, save_nbrs, order)
        indptr, c, v = engine.topk_rows_to_csr(cols, vals, cnt)
    else:
        indptr, c, v = plan.build_unbounded(min_sim, order)
    torch.cuda.synchronize()
    n = iu.shape[0]
    return sps.csr_array((v.cpu().numpy(), c.cpu().numpy(), indptr.cpu().numpy()), shape=(n, n)), plan


def _assert_same(got: sps.csr_array, ref: sps.csr_array):
    assert np.array_equal(got.indptr, ref.indptr)
    assert np.array_equal(got.indices, ref.indices)  # bit-exact top-k indices (north_star)
    assert np.array_equal(got.data.view(np.int32), ref.data.view(np.int32))  # and values


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("save_nbrs", [None, 20, 100])
def test_build_ml_small_bit_exact(cuda_lib, ml_small, explicit, save_nbrs):
    ui, iu, _ = data.knn_item_matrices(ml_small, explicit)
    ref = oracle.knn_build(ui, iu, 1e-6, save_nbrs)
    got, _ = _build(ui, iu, 1e-6, save_nbrs)
    _assert_same(got, ref)
    if save_nbrs is None and explicit:
        assert got.nnz == 8_780_790


def test_build_toy(cuda_lib):
    z = np.load(GOLD / "knn_prep.npz")
    toy = data.Interactions(z["toy_users"], z["toy_items"], z["toy_ratings"], 6, 4)
    for explicit in (True, False):
        ui, iu, _ = data.knn_item_matrices(toy, explicit)
        for K in (None, 500, 1, 2):
            _assert_same(_build(ui, iu, 1e-6, K)[0], oracle.knn_build(ui, iu, 1e-6, K))


@pytest.mark.parametrize("ctas,warps", [("8", "8"), ("4", "16"), ("1", "32")])
def test_build_multi_half_geometry(cuda_lib, ml_small, ctas, warps, lk_options):
    """Small shared-memory budgets force several column halves and the merge path."""
    lk_options("LK_KNN_CTAS", int(ctas))
    lk_options("LK_KNN_WARPS", int(warps))
    ui, iu, _ = data.knn_item_matrices(ml_small, False)  # implicit: 76% of rows tie at K=20
    ref = oracle.knn_build(ui, iu, 1e-6, 20)
    got, plan = _build(ui, iu, 1e-6, 20)
    if ctas == "8":
        assert plan.geom.n_halves > 1
    _assert_same(got, ref)
    ref = oracle.knn_build(ui, iu, 1e-6, None)
    got, _ = _build(ui, iu, 1e-6, None)
    _assert_same(got, ref)


@pytest.mark.parametrize("explicit", [True, False])
def test_build_hot_items_cut_into_column_pieces(cuda_lib, lk_options, explicit):
    """A plan made for many GPUs cuts the (item, half) units of expensive items into 2 / 4 / 8 column
    pieces handled by different CTAs (knn_build.cu): same bits as the unsplit build and the oracle —
    every dots[j] still sums its users in ascending order."""
    lk_options("LK_KNN_CTAS", 4)  # several column halves as well
    inter = small_synth(3000, 2500, 150000, seed=9)
    ui, iu, _ = data.knn_item_matrices(inter, explicit)
    ref = oracle.knn_build(ui, iu, 1e-6, 20)
    got, plan = _build(ui, iu, 1e-6, 20, world=64)
    pieces = plan.units(split_hot=True)["units"][:, 3]
    assert int(pieces.max()) == 8 and len(torch.unique(pieces)) >= 2  # hot items cut finer than the tail
    _assert_same(got, ref)
    got1, _ = _build(ui, iu, 1e-6, 20, world=1)
    _assert_same(got1, ref)
    # the unbounded build never splits (pool segments must stay in column order)
    refu = oracle.knn_build(ui, iu, 1e-6, None)
    gotu, planu = _build(ui, iu, 1e-6, None, world=64)
    assert int(planu.units(split_hot=False)["units"][:, 3].max()) == 1
    _assert_same(gotu, refu)


def test_build_synthetic_and_min_sim_edges(cuda_lib):
    inter = small_synth(3000, 2500, 150000, seed=9)
    for explicit in (True, False):
        ui, iu, _ = data.knn_item_matrices(inter, explicit)
        for min_sim, K in ((1e-6, 20), (0.05, 7), (np.finfo(np.float64).smallest_normal, 20), (1e-6, None)):
            ref = oracle.knn_build(ui, iu, min_sim, K)
            got, _ = _build(ui, iu, min_sim, K)
            _assert_same(got, ref)


def test_build_row_subset(cuda_lib, ml_small):
    """Item-sharded build (multi-GPU partitioning): only the rows in `order` are produced."""
    ui, iu, _ = data.knn_item_matrices(ml_small, True)
    dev = _lib.require_device()
    rows = torch.arange(1000, 3000, dtype=torch.int32, device=dev)
    got, _ = _build(ui, iu, 1e-6, 20, order=rows)
    ref = oracle.knn_build(ui, iu, 1e-6, 20, rows=(1000, 3000))
    sub = got[1000:3000]
    assert np.array_equal(sub.indptr, ref.indptr)
    assert np.array_equal(sub.indices, ref.indices)
    assert np.array_equal(sub.data.view(np.int32), ref.data.view(np.int32))
    assert got[:1000].nnz == 0 and got[3000:].nnz == 0


def test_build_unbounded_pool_overflow_is_reported(cuda_lib, ml_small):
    """A similarity pool too small for the kept pairs raises instead of returning a truncated matrix, and the
    plan builds the whole matrix afterwards."""
    ui, iu, _ = data.knn_item_matrices(ml_small, True)
    dev = _lib.require_device()
    plan = engine.KnnBuildPlan.create(engine.DeviceCSR.from_host(ui, dev), engine.DeviceCSR.from_host(iu, dev))
    with pytest.raises(_lib.EngineError, match="overflow"):
        plan.build_unbounded(1e-6, capacity=3)
    indptr, _c, _v = plan.build_unbounded(1e-6)
    assert int(indptr[-1]) == 8_780_790


def _score_gpu(S, queries, max_nbrs, min_nbrs, explicit=True):
    dev = _lib.require_device()
    st = engine.KnnScorerState.create(S.shape[0], S.indptr, S.indices, S.data, dev)
    ref_ptr = np.cumsum([0] + [len(q[0]) for q in queries])
    tgt_ptr = np.cumsum([0] + [len(q[2]) for q in queries])
    ri = np.concatenate([q[0] for q in queries]).astype(np.int32)
    rv = np.concatenate([q[1] for q in queries]).astype(np.float32)
    ti = np.concatenate([q[2] for q in queries]).astype(np.int32)
    sc, ct = st.score(
        torch.from_numpy(ref_ptr).to(dev), torch.from_numpy(ri).to(dev),
        torch.from_numpy(rv).to(dev) if explicit else None,
        torch.from_numpy(tgt_ptr).to(dev), torch.from_numpy(ti).to(dev), max_nbrs, min_nbrs,
    )  # fmt: skip
    return sc.cpu().numpy(), ct.cpu().numpy(), tgt_ptr


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("max_nbrs,save_nbrs", [(20, None), (5, None), (20, 20), (3, 50)])
def test_score_matches_oracle_exactly(cuda_lib, ml_small, explicit, max_nbrs, save_nbrs):
    """Batched scoring equals the ScoreAccumulator emulation bit for bit (incl. heap ties)."""
    ui, iu, means = data.knn_item_matrices(ml_small, explicit)
    S = oracle.knn_build(ui, iu, 1e-6, save_nbrs)
    R = ml_small.coo().tocsr()
    rng = np.random.default_rng(17)
    queries = []
    for u in rng.choice(ml_small.n_users, 40, replace=False):
        s, e = R.indptr[u], R.indptr[u + 1]
        ri = R.indices[s:e].astype(np.int32)
        perm = rng.permutation(len(ri))  # history order matters, exercise it
        ri = ri[perm]
        rv = R.data[s:e][perm].astype(np.float32)
        if explicit:
            rv = rv - means[ri]
        ti = rng.choice(ml_small.n_items, 300).astype(np.int32)  # with duplicates
        ti[::37] = -1  # null targets
        if len(ri) > 3:
            ri = ri.copy()
            ri[2] = -1  # a null reference item is skipped
        queries.append((ri, rv, ti))
    queries.append((np.zeros(0, np.int32), np.zeros(0, np.float32), np.arange(50, dtype=np.int32)))
    sc, ct, tptr = _score_gpu(S, queries, max_nbrs, 1, explicit)
    for qi, (ri, rv, ti) in enumerate(queries):
        osc, oct_ = oracle.knn_score(S, ri, rv if explicit else None, ti, max_nbrs, 1)
        g = sc[tptr[qi] : tptr[qi + 1]]
        assert np.array_equal(ct[tptr[qi] : tptr[qi + 1]], oct_)
        assert np.array_equal(np.isnan(g), np.isnan(osc))
        ok = ~np.isnan(osc)
        assert np.array_equal(g[ok].view(np.int32), osc[ok].view(np.int32))


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("max_nbrs,save_nbrs", [(20, 20), (5, None)])
def test_score_all_items_dense_kernel(cuda_lib, ml_small, explicit, max_nbrs, save_nbrs, monkeypatch):
    """Every query against all items (knn_score_dense_kernel): the same bits as the oracle's ScoreAccumulator,
    heap ties included; with the unbounded model the heaviest users overflow the CTA's shared target list and
    come back through the list kernel."""
    ui, iu, means = data.knn_item_matrices(ml_small, explicit)
    S = oracle.knn_build(ui, iu, 1e-6, save_nbrs)
    R = ml_small.coo().tocsr()
    rng = np.random.default_rng(23)
    users = np.concatenate([[int(np.argmax(np.diff(R.indptr)))], rng.choice(ml_small.n_users, 30, replace=False)])
    dev = _lib.require_device()
    st = engine.KnnScorerState.create(S.shape[0], S.indptr, S.indices, S.data, dev)
    hists = []
    for u in users:
        s, e = R.indptr[u], R.indptr[u + 1]
        ri = R.indices[s:e].astype(np.int32)
        perm = rng.permutation(len(ri))
        ri = ri[perm].copy()
        rv = R.data[s:e][perm].astype(np.float32)
        if explicit:
            rv = rv - means[ri]
        if len(ri) > 4:
            ri[1] = -1  # a null reference item
        hists.append((ri, rv))
    hists.append((np.zeros(0, np.int32), np.zeros(0, np.float32)))  # an empty history
    ptr_ = np.cumsum([0] + [len(h[0]) for h in hists])
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    sc, ct = st.score_all_items(
        t(ptr_), t(np.concatenate([h[0] for h in hists])),
        t(np.concatenate([h[1] for h in hists])) if explicit else None, max_nbrs, 1,
    )  # fmt: skip
    sc, ct = sc.cpu().numpy(), ct.cpu().numpy()
    all_items = np.arange(ml_small.n_items, dtype=np.int32)
    for qi, (ri, rv) in enumerate(hists):
        osc, oct_ = oracle.knn_score(S, ri, rv if explicit else None, all_items, max_nbrs, 1)
        assert np.array_equal(ct[qi], oct_)
        assert np.array_equal(np.isnan(sc[qi]), np.isnan(osc))
        ok = ~np.isnan(osc)
        assert np.array_equal(sc[qi][ok].view(np.int32), osc[ok].view(np.int32))


def test_score_empty_histories_and_no_targets(cuda_lib, ml_small):
    """Zero-length inputs give the oracle's answer, in item and user mode: a batch whose histories (neighbour
    lists) are all empty scores every target as having no neighbours, and a call with no targets (or, for all
    items, no queries) returns empty results."""
    ui, iu, _ = data.knn_item_matrices(ml_small, True)
    S = oracle.knn_build(ui, iu, 1e-6, 20)
    R = ml_small.coo().tocsr().astype(np.float32)
    dev = _lib.require_device()
    t = lambda a: torch.from_numpy(np.asarray(a)).to(dev)  # noqa: E731
    none_i, none_f = np.zeros(0, np.int32), np.zeros(0, np.float32)
    hist_i, hist_f = np.array([1, 5, 30], np.int32), np.array([0.5, -1.0, 0.25], np.float32)
    ti = np.array([3, -1, 7, 31, 5, 3], np.int32)

    def check(got, ref):
        sc, ct = (x.cpu().numpy() for x in got)
        osc, oct_ = ref
        assert sc.shape == osc.shape and np.array_equal(ct, oct_)
        assert np.array_equal(np.isnan(sc), np.isnan(osc))
        ok = ~np.isnan(osc)
        assert np.array_equal(sc[ok].view(np.int32), osc[ok].view(np.int32))

    item = engine.KnnScorerState.create(S.shape[0], S.indptr, S.indices, S.data, dev)
    for explicit in (True, False):
        rv = none_f if explicit else None
        got = item.score(t([0, 0, 0]), t(none_i), None if rv is None else t(rv), t([0, 4, 6]), t(ti), 20, 1)
        check(got, oracle.knn_score(S, none_i, rv, ti, 20, 1))
        hv = hist_f if explicit else None
        got = item.score(t([0, 3]), t(hist_i), None if hv is None else t(hv), t([0, 0]), t(none_i), 20, 1)
        check(got, oracle.knn_score(S, hist_i, hv, none_i, 20, 1))
        sc, ct = item.score_all_items(t([0, 0, 0]), t(none_i), None if rv is None else t(rv), 20, 1)
        all_items = np.arange(S.shape[0], dtype=np.int32)
        for q in range(2):
            check((sc[q], ct[q]), oracle.knn_score(S, none_i, rv, all_items, 20, 1))
        sc, ct = item.score_all_items(t([0]), t(none_i), None if rv is None else t(rv), 20, 1)
        assert sc.shape == ct.shape == (0, S.shape[0])

    for explicit in (True, False):
        user = engine.KnnScorerState.create(R.shape[1], R.indptr, R.indices, R.data if explicit else None, dev,
                                            user_mode=True)  # fmt: skip
        got = user.score(t([0, 0]), t(none_i), t(none_f), t([0, 6]), t(ti), 20, 1)
        check(got, oracle.user_score(R, none_i, none_f, ti, 20, 1, explicit))
        got = user.score(t([0, 3]), t(hist_i), t(np.abs(hist_f)), t([0, 0]), t(none_i), 20, 1)
        check(got, oracle.user_score(R, hist_i, np.abs(hist_f), none_i, 20, 1, explicit))


def test_golden_predictions_end_to_end(cuda_lib, ml_small):
    """tests/models/item-item-preds.csv through GPU build + GPU scoring."""
    ui, iu, means = data.knn_item_matrices(ml_small, True)
    S, _ = _build(ui, iu, 1e-6, None)
    known = pd.read_csv(GOLD / "item-item-preds.csv")
    uidx = {u: i for i, u in enumerate(ml_small.user_ids)}
    iidx = {it: i for i, it in enumerate(ml_small.item_ids)}
    R = ml_small.coo().tocsr()
    queries, expected = [], []
    for uid, grp in known.groupby("user_id"):
        u = uidx[uid]
        s, e = R.indptr[u], R.indptr[u + 1]
        ri = R.indices[s:e].astype(np.int32)
        rv = R.data[s:e].astype(np.float32) - means[ri]
        ti = np.array([iidx.get(i, -1) for i in grp.item_id], dtype=np.int32)
        queries.append((ri, rv, ti))
        expected.append(grp.prediction.values)
    sc, ct, tptr = _score_gpu(S, queries, 20, 1, True)
    ti_all = np.concatenate([q[2] for q in queries])
    pred = sc + means[np.maximum(ti_all, 0)]
    err = np.abs(pred - np.concatenate(expected))
    assert len(err) == 1288 and not np.isnan(err).any()
    assert (err > 1e-5).sum() <= 3  # the three boundary-tie rows of SURVEY.md §8c


def _arrow_rows(csr, large=False):
    """The reference's storage of a sparse row array (data/matrix.py:388-424): List (or LargeList) of
    Struct{index: int32, value: float32}."""
    import pyarrow as pa

    elems = pa.StructArray.from_arrays(
        [pa.array(csr.indices, type=pa.int32()), pa.array(csr.values, type=pa.float32())], names=["index", "value"]
    )
    if large:
        return pa.LargeListArray.from_arrays(pa.array(np.asarray(csr.indptr, dtype=np.int64)), elems)
    return pa.ListArray.from_arrays(pa.array(np.asarray(csr.indptr, dtype=np.int32)), elems)


def test_accel_api_mirror(cuda_lib, ml_small):
    """lenskit._accel.knn with the reference's own argument types: Arrow List<Struct{index,value}> matrices in
    (csr.rs:160-209), LargeList chunks out (consumer.rs:96-142) that combine the way knn/item.py:173-177
    combines them, Arrow arrays with nulls for the scoring calls."""
    import pyarrow as pa

    from lkpy_b200 import accel

    ui, iu, means = data.knn_item_matrices(ml_small, True)
    a_ui, a_iu = _arrow_rows(ui), _arrow_rows(iu)
    shape = (ml_small.n_users, ml_small.n_items)
    chunks = accel.run_accel_task(accel.knn.compute_similarities(a_ui, a_iu, shape, 1e-6, 20))
    assert isinstance(chunks, list) and all(pa.types.is_large_list(c.type) for c in chunks)
    elem = chunks[0].type.value_type  # Struct{index: lenskit.sparse_index(n_items) over int32, value: float32}
    assert [elem.field(i).name for i in range(elem.num_fields)] == ["index", "value"]
    assert elem.field("index").type.extension_name == "lenskit.sparse_index"  # consumer.rs:109
    assert elem.field("index").type.storage_type == pa.int32() and elem.field("index").type.dimension == ml_small.n_items
    assert elem.field("value").type == pa.float32()
    smat = pa.chunked_array(chunks).combine_chunks()  # knn/item.py:173-177
    assert len(smat) == ml_small.n_items
    ref = oracle.knn_build(ui, iu, 1e-6, 20)
    got = accel.as_host_csr(smat, ml_small.n_items)
    assert np.array_equal(got.indptr, ref.indptr) and got.indptr.dtype == np.int64
    assert np.array_equal(got.indices, ref.indices)
    assert np.array_equal(got.values.view(np.int32), ref.data.view(np.int32))
    # several chunks: row order is the only contract (consumer.rs:137-142)
    old = accel.RESULT_CHUNK_ROWS
    try:
        accel.RESULT_CHUNK_ROWS = 1000
        many = accel.run_accel_task(accel.knn.compute_similarities(ui, iu, shape, 1e-6, 20))
    finally:
        accel.RESULT_CHUNK_ROWS = old
    assert len(many) == -(-ml_small.n_items // 1000)
    assert pa.chunked_array(many).combine_chunks().equals(smat)
    # the unbounded build through the same door
    full = accel.run_accel_task(accel.knn.compute_similarities(a_ui, a_iu, shape, 1e-6, None))
    assert sum(len(c.values) for c in full) == 8_780_790

    ri = pa.array([1, 5, 30, None, 100], type=pa.int32())
    rv = pa.array([0.5, -1.0, 0.25, None, 1.5], type=pa.float32())
    ti = pa.array([3, None, 7, 31, 5], type=pa.int32())
    scores, counts = accel.knn.score_explicit(smat, ri, rv, ti, 20, 1)
    assert isinstance(scores, pa.Array) and isinstance(counts, pa.Array)
    assert counts.null_count == 1 and scores[1].as_py() is None
    osc, oct_ = oracle.knn_score(
        ref, np.array([1, 5, 30, -1, 100], np.int32), np.array([0.5, -1.0, 0.25, 0, 1.5], np.float32),
        np.array([3, -1, 7, 31, 5], np.int32), 20, 1,
    )  # fmt: skip
    got = scores.to_numpy(zero_copy_only=False)
    assert np.array_equal(np.isnan(got), np.isnan(osc))
    assert np.allclose(got[~np.isnan(osc)], osc[~np.isnan(osc)], rtol=0, atol=0)
    s2, c2 = accel.knn.score_implicit(smat, ri, ti, 20, 1)
    assert len(s2) == 5
    with pytest.raises(TypeError):
        accel.as_host_csr(pa.array([1.0, 2.0]))  # not a list array (csr.rs:160-195)
    bad = pa.ListArray.from_arrays(pa.array([0, 1], type=pa.int32()), pa.array([0.5], type=pa.float64()))
    with pytest.raises(TypeError):
        accel.as_host_csr(bad)


def test_build_cancel_flag_and_task(cuda_lib, ml_small):
    """The build stops handing out work when the device cancel flag is up (tasks/mod.rs:84-90 through
    item_train.rs's CancelAdapter): a flag raised before the launch leaves every row empty, a task cancelled
    before `invoke` raises, and a finished task reports (n_items, n_items)."""
    from lkpy_b200 import accel

    ui, iu, _ = data.knn_item_matrices(ml_small, True)
    dev = _lib.require_device()
    plan = engine.KnnBuildPlan.create(engine.DeviceCSR.from_host(ui, dev), engine.DeviceCSR.from_host(iu, dev))
    plan.cancel = torch.ones(1, dtype=torch.int32, device=dev)
    _cols, _vals, cnt = plan.build_topk(1e-6, 20)
    torch.cuda.synchronize()
    assert int(cnt.sum().item()) == 0
    plan.cancel.zero_()
    _cols, _vals, cnt = plan.build_topk(1e-6, 20)
    torch.cuda.synchronize()
    assert int(cnt.sum().item()) == oracle.knn_build(ui, iu, 1e-6, 20).nnz

    shape = (ml_small.n_users, ml_small.n_items)
    task = accel.knn.compute_similarities(ui, iu, shape, 1e-6, 20)
    assert task.current_progress() == (0, ml_small.n_items)
    task.cancel()
    with pytest.raises(RuntimeError, match="cancelled"):
        task.invoke()
    task = accel.knn.compute_similarities(ui, iu, shape, 1e-6, 20)
    task.invoke()
    assert task.current_progress() == (ml_small.n_items, ml_small.n_items)
