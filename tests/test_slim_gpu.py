"""
SLIM on the device: ``accel.slim.train_slim`` / ``engine.SlimPlan`` bit for bit against the C restatement
(``tests/slim_oracle.c``), and ``SLIMScorer.score_batch`` / ``recommend_batch`` bit for bit against the host
composition of ``x @ weights``, the candidate selector and ``argtopn``.
"""

import pickle

import numpy as np
import pyarrow as pa
import pytest
import torch

import oracle
import slim_oracle as so
from lkpy_b200 import _lib, accel, data, engine
from lkpy_b200.components import Dataset, ItemList
from lkpy_b200.slim import SLIMScorer

pytestmark = pytest.mark.gpu


def _structures(it):
    return so.structure(it.n_users, it.users, it.items), so.structure(it.n_items, it.items, it.users)


def _arrow(ip, cols, dim):
    """A sparse-row array with the column count in its index type, as ``SparseRowArray`` carries it."""
    csr = data.InteractionCSR(ip, cols, np.ones(len(cols), np.float32), (len(ip) - 1, dim))
    return pa.chunked_array(accel.csr_to_arrow_chunks(csr)).combine_chunks()


def _chunks_to_csr(chunks, n):
    arr = pa.chunked_array(chunks).combine_chunks()
    off = arr.offsets.to_numpy()
    st = arr.values
    idx = st.field("index")
    idx = idx.storage if isinstance(idx, pa.ExtensionArray) else idx
    return off, idx.to_numpy(), st.field("value").to_numpy()


def _assert_same(got, want):
    ip, c, v = got
    assert np.array_equal(ip, want.indptr)
    assert np.array_equal(c, want.indices)
    assert np.array_equal(np.asarray(v, np.float32).view(np.int32), want.data.view(np.int32))


CONFIGS = [
    (1.0, 1.0, 100, None),  # SLIMConfig defaults
    (1.0, 1.0, 10, None),
    (1.0, 1.0, 100, 1),
    (1.0, 1.0, 100, 20),
    (1.0, 1.0, 100, 100),
    (0.1, 0.3, 100, 20),  # neither is exact in f32
]


@pytest.mark.parametrize("l1,l2,iters,nbrs", CONFIGS)
def test_train_slim_matches_restatement_on_ml_small(cuda_lib, ml_small, l1, l2, iters, nbrs):
    it = ml_small
    ui, iu = _structures(it)
    task = accel.slim.train_slim(_arrow(*ui, it.n_items), _arrow(*iu, it.n_users), l1, l2, iters, nbrs)
    got = _chunks_to_csr(task.invoke(), it.n_items)
    assert task.current_progress() == (it.n_items, it.n_items)
    want = so.train(it.n_users, it.n_items, ui, iu, l1, l2, iters, nbrs)
    assert want.nnz > 0
    _assert_same(got, want)


def test_unsorted_rows_keep_stored_order(cuda_lib):
    """UI rows in a shuffled order change the active-set order and so fsSLIM's ties and the CD order."""
    it = data.synth_interactions(500, 300, 12_000, seed=3)
    rng = np.random.default_rng(1)
    perm = rng.permutation(it.nnz)
    ui = so.structure(it.n_users, it.users[perm], it.items[perm])
    iu = so.structure(it.n_items, it.items[perm], it.users[perm])
    for nbrs in (None, 5):
        got = _chunks_to_csr(accel.slim.train_slim(_arrow(*ui, 300), _arrow(*iu, 500), 0.5, 1.0, 50, nbrs).invoke(),
                             300)  # fmt: skip
        _assert_same(got, so.train(it.n_users, it.n_items, ui, iu, 0.5, 1.0, 50, nbrs))


def _ml25m():
    return data.synth_interactions(**data.ML25M_SHAPE, ratings=False)


@pytest.mark.parametrize("nbrs", [100, None])
def test_ml25m_shape_sample_matches_restatement(cuda_lib, nbrs):
    it = _ml25m()
    ui, iu = _structures(it)
    row_len = np.diff(ui[0])
    cost = np.bincount(it.items, weights=row_len[it.users], minlength=it.n_items)
    order = np.argsort(-cost, kind="stable")
    cols = order[[0, 1, 10, 100, 1000, 5000, 20000, 40000]]  # cost-stratified, the most expensive first
    dev = _lib.require_device()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    plan = engine.SlimPlan.create(it.n_users, it.n_items, t(ui[0]), t(ui[1]), t(iu[0]), t(iu[1]), 1.0, 1.0, 100, nbrs,
                                  columns=t(cols))  # fmt: skip
    assert int(plan.sched[0].item()) == int(cols[0])
    got = tuple(x.cpu().numpy() for x in plan.train())
    want = so.train(it.n_users, it.n_items, ui, iu, 1.0, 1.0, 100, nbrs, columns=cols)
    _assert_same(got, want)
    print(f"ML-25M shape, max_nbrs={nbrs}: {want.nnz} weights in {len(cols)} sampled columns")


def test_cancel_stops_the_kernel_and_overflow_retries(cuda_lib, ml_small):
    it = ml_small
    ui, iu = _structures(it)
    dev = _lib.require_device()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    plan = engine.SlimPlan.create(it.n_users, it.n_items, t(ui[0]), t(ui[1]), t(iu[0]), t(iu[1]), 1.0, 1.0, 100, 20)
    raised = torch.ones(1, dtype=torch.int32, device=dev)
    indptr, _c, _v = plan.train(attach=lambda counter, units: raised)
    assert int(indptr[-1]) == 0 and int(plan.work_counter.item()) == 0  # no column was handed out
    plan.cancel = None
    small = tuple(x.cpu().numpy() for x in plan.train(capacity=3))  # overflows, then retries with larger pools
    _assert_same(small, so.train(it.n_users, it.n_items, ui, iu, 1.0, 1.0, 100, 20))

    task = accel.slim.train_slim(_arrow(*ui, it.n_items), _arrow(*iu, it.n_users), 1.0, 1.0, 100, 20)
    orig = task._attach

    def attach(counter, units):
        task._cancelled.set()  # cancelled once the kernel's flag exists: the flag is raised before the launch
        return orig(counter, units)

    task._attach = attach
    with pytest.raises(RuntimeError, match="cancelled"):
        task.invoke()


@pytest.fixture(scope="module")
def scorer():
    it = data.load_ml_small()
    m = SLIMScorer(max_nbrs=50)
    m.train(Dataset(it))
    return it, m


def _histories(it):
    rng = np.random.default_rng(7)
    out = []
    for u in (0, 3, 100, 414, 670):
        nums = it.items[it.users == u]
        h = rng.permutation(nums)  # unsorted
        out.append(np.concatenate([h, h[:3]]))  # repeats
    out.append(np.array([], np.int64))
    return out


def _queries(it, hists):
    qs = [ItemList(item_ids=it.item_ids[h]) for h in hists]
    qs.append(ItemList(item_ids=np.array([-5, -6])))  # history of unknown items only: zeros everywhere
    qs.append(None)
    return qs


def test_scorer_weights_and_scores(cuda_lib, scorer):
    it, m = scorer
    ui, iu = _structures(it)
    want = so.train(it.n_users, it.n_items, ui, iu, 1.0, 1.0, 100, 50)
    W = m.weights
    Wt = want.T.tocsr()
    assert np.array_equal(W.indptr, Wt.indptr) and np.array_equal(W.indices, Wt.indices)
    assert np.array_equal(W.data.view(np.int32), Wt.data.view(np.int32))
    hists = _histories(it)
    qs = _queries(it, hists)
    tgt = ItemList(item_ids=np.concatenate([it.item_ids[::7], [-1]]))
    outs = m.score_batch(qs, [tgt] * len(qs))
    for k, out in enumerate(outs):
        s = out.scores()
        if k < len(hists) and len(hists[k]):
            full = so.score(Wt, hists[k])
            assert np.array_equal(s[:-1].view(np.int32), full[::7].view(np.int32)) and np.isnan(s[-1])
        elif k == len(hists):  # unknown items only
            assert np.all(s[:-1] == 0) and np.isnan(s[-1])
        else:  # empty or missing history
            assert np.all(np.isnan(s))
    one = m(qs[1], tgt)
    assert np.array_equal(one.scores().view(np.int32), outs[1].scores().view(np.int32))


@pytest.mark.parametrize("n", [1, 10, 1024])
@pytest.mark.parametrize("exclude", ["query", None])
def test_recommend_batch_matches_host_composition(cuda_lib, scorer, n, exclude):
    it, m = scorer
    Wt = m.weights
    hists = _histories(it)
    qs = _queries(it, hists)
    recs = m.recommend_batch(qs, n, exclude=exclude)
    for k, rec in enumerate(recs):
        if k < len(hists) and len(hists[k]):
            s = so.score(Wt, hists[k])
            if exclude == "query":
                s[hists[k]] = np.nan
        elif k == len(hists):
            s = np.zeros(it.n_items, np.float32)
        else:
            assert len(rec) == 0
            continue
        want = oracle.argtopn(s, n)
        assert np.array_equal(rec.numbers(), want), (k, n)
        assert np.array_equal(rec.scores().view(np.int32), s[want].view(np.int32))


def test_pickle_round_trip(cuda_lib, scorer):
    it, m = scorer
    hists = _histories(it)
    qs = _queries(it, hists)
    m2 = pickle.loads(pickle.dumps(m))
    a, b = m.recommend_batch(qs, 20), m2.recommend_batch(qs, 20)
    for x, y in zip(a, b):
        assert np.array_equal(x.numbers(), y.numbers()) and np.array_equal(x.scores(), y.scores())
    tgt = ItemList(item_ids=it.item_ids)
    for x, y in zip(m.score_batch(qs, [tgt] * len(qs)), m2.score_batch(qs, [tgt] * len(qs))):
        assert np.array_equal(x.scores().view(np.int32), y.scores().view(np.int32))
