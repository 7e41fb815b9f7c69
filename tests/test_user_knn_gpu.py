"""
User-kNN scoring (SURVEY.md §8f N3): the accumulator kernel in user mode against the oracle's
restatement of src/accel/knn/user_score.rs:21-98 (bit-exact, ScoreAccumulator element movement
included), the _accel-level mirror, and the UserKNNScorer component against the reference's
algorithm restated with NumPy (user.py:157-255).
"""

import numpy as np
import pyarrow as pa
import pytest
import torch

import oracle
from lkpy_b200 import _lib, accel, data, engine
from lkpy_b200.components import Dataset, ItemList, RecQuery
from lkpy_b200.knn_user import UserKNNScorer

from helpers import small_synth

pytestmark = pytest.mark.gpu


def _bits_equal(got_s, got_c, ref_s, ref_c):
    assert np.array_equal(got_c, ref_c)
    assert np.array_equal(np.isnan(got_s), np.isnan(ref_s))
    ok = ~np.isnan(ref_s)
    assert np.array_equal(got_s[ok].view(np.int32), ref_s[ok].view(np.int32))


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("max_nbrs", [20, 3, 1, 128])  # 1 and 128: the smallest and largest accumulator
def test_user_score_matches_oracle_exactly(cuda_lib, ml_small, explicit, max_nbrs):
    m = UserKNNScorer(feedback="explicit" if explicit else "implicit", max_nbrs=max_nbrs)
    m.train(Dataset(ml_small))
    R = m.user_ratings
    dev = _lib.require_device()
    st = engine.KnnScorerState.create(R.shape[1], R.indptr, R.indices, R.values if explicit else None, dev, user_mode=True)
    rng = np.random.default_rng(5)
    queries = []
    for _ in range(24):
        n_nb = int(rng.integers(1, 200))
        nb = rng.choice(ml_small.n_users, n_nb, replace=False).astype(np.int32)
        sims = np.round(rng.random(n_nb).astype(np.float32), 2)  # coarse: ties at the heap boundary
        ti = rng.choice(ml_small.n_items, 400).astype(np.int32)
        ti[::41] = -1
        queries.append((nb, sims, ti))
    ref_ptr = np.cumsum([0] + [len(q[0]) for q in queries])
    tgt_ptr = np.cumsum([0] + [len(q[2]) for q in queries])
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    sc, ct = st.score(
        t(ref_ptr), t(np.concatenate([q[0] for q in queries])), t(np.concatenate([q[1] for q in queries])),
        t(tgt_ptr), t(np.concatenate([q[2] for q in queries])), max_nbrs, 2,
    )  # fmt: skip
    sc, ct = sc.cpu().numpy(), ct.cpu().numpy()
    for qi, (nb, sims, ti) in enumerate(queries):
        osc, oct_ = oracle.user_score(R, nb, sims, ti, max_nbrs, 2, explicit)
        _bits_equal(sc[tgt_ptr[qi] : tgt_ptr[qi + 1]], ct[tgt_ptr[qi] : tgt_ptr[qi + 1]], osc, oct_)


def test_accel_user_score_mirror(cuda_lib, ml_small):
    """_accel.knn.user_score_items_* with Arrow inputs: null neighbours / similarities are dropped
    pairwise (user_score.rs:41-44), null targets give nulls."""
    m = UserKNNScorer()
    m.train(Dataset(ml_small))
    R = m.user_ratings
    rng = np.random.default_rng(2)
    nb = rng.choice(ml_small.n_users, 60, replace=False).astype(np.int32)
    sims = rng.random(60).astype(np.float32)
    ti = rng.choice(ml_small.n_items, 300, replace=False).astype(np.int32)
    nb_mask = np.zeros(60, bool)
    nb_mask[[3, 17]] = True
    sim_mask = np.zeros(60, bool)
    sim_mask[[5]] = True
    ti_mask = np.zeros(300, bool)
    ti_mask[[0, 9]] = True
    for explicit, fn in ((True, accel.knn.user_score_items_explicit), (False, accel.knn.user_score_items_implicit)):
        out = fn(pa.array(ti, mask=ti_mask), pa.array(nb, mask=nb_mask), pa.array(sims, mask=sim_mask), R, 20, 1)
        keep = ~(nb_mask | sim_mask)
        tin = np.where(ti_mask, -1, ti).astype(np.int32)
        osc, _ = oracle.user_score(R, nb[keep], sims[keep], tin, 20, 1, explicit)
        got = out.to_numpy(zero_copy_only=False)
        assert out.null_count == int(np.isnan(osc).sum())
        ok = ~np.isnan(osc)
        assert np.array_equal(got[ok].astype(np.float32).view(np.int32), osc[ok].view(np.int32))


@pytest.mark.parametrize("explicit", [True, False])
def test_user_knn_component_matches_numpy_restatement(cuda_lib, ml_small, explicit):
    """The component against user.py:157-255 restated with NumPy: top-max_nbrs neighbours per item by
    similarity, weighted average of centred ratings (explicit) or sum of similarities (implicit)."""
    m = UserKNNScorer(feedback="explicit" if explicit else "implicit", max_nbrs=15, min_nbrs=2)
    ds = Dataset(ml_small)
    m.train(ds)
    R = m.user_ratings.to_scipy().tocsc()
    rng = np.random.default_rng(3)
    users = rng.choice(ml_small.n_users, 6, replace=False)
    items = ItemList(item_nums=rng.choice(ml_small.n_items, 500, replace=False).astype(np.int32), vocabulary=ds.items)
    outs = m.score_batch([RecQuery(user_id=ds.users.id(int(u))) for u in users], [items] * len(users))
    for u, out in zip(users, outs):
        vec = m.user_vectors[[int(u)], :].toarray()[0]
        sims = m.user_vectors @ vec
        sims[u] = 0
        got = out.scores()
        for pos, inum in enumerate(items.numbers(vocabulary=ds.items)):
            col = R[:, [inum]]
            raters = col.indices
            s = sims[raters]
            keep = s >= m.config.min_sim
            raters, s, vals = raters[keep], s[keep], np.asarray(col.data)[keep]
            if len(s) < 2:
                assert np.isnan(got[pos])
                continue
            if len(s) > 15 and np.sum(s == np.sort(s)[-15]) > 1:
                continue  # tie at the cut: decided by heap order, covered by the exact test above
            top = np.argsort(-s, kind="stable")[:15]
            if explicit:
                want = float(np.sum(s[top] * vals[top]) / np.sum(s[top])) + float(m.user_means[u])
            else:
                want = float(np.sum(s[top]))
            assert got[pos] == pytest.approx(want, rel=2e-5, abs=2e-5)
    # a query with an explicit history and no known user id
    hist = ds.user_history(int(users[0]))
    a = m(RecQuery(user_id=None, query_items=hist), items)
    assert np.isfinite(a.scores()).any()
    assert np.isnan(m(RecQuery(user_id="nobody"), items).scores()).all()
