"""
FlexMF implicit on the device: the sampler against its NumPy restatement (bit for bit), ``lk_flexmf_step`` against the
plain-torch restatement of the reference's step (``flexmf_oracle``), determinism, and the scorer's batched interface.
"""

import pickle

import numpy as np
import pytest
import torch

import flexmf_oracle as fo
import oracle
from lkpy_b200 import engine, flexmf, prep
from lkpy_b200.components import Dataset, ItemList, RecQuery, TrainingOptions
from lkpy_b200.flexmf import FlexMFImplicitScorer

pytestmark = pytest.mark.gpu
LR, REG, PW = 0.01, 0.05, 1.5


def _params(n_users, n_items, k, ub, ib, seed=3):
    return flexmf.initial_parameters(n_users, n_items, k, ub, ib, torch.Generator().manual_seed(seed))


def _state(params, users, items, loss, reg_method, n, B, **kw):
    return engine.FlexMFState(params, users, items, loss=loss, reg_method=reg_method, negative_count=n, batch_size=B,
                              learning_rate=LR, regularization=REG, positive_weight=PW, **kw)  # fmt: skip


def _update_error(new, want, old) -> float:
    """‖new − want‖ / ‖want − old‖: the error of the update, not of the parameter."""
    new, want, old = (np.asarray(x, dtype=np.float64) for x in (new, want, old))
    return float(np.linalg.norm(new - want) / max(np.linalg.norm(want - old), 1e-300))


def _check_steps(st, params, batches, loss, reg_method, tol=1e-5, residue=(), residue_step=1e-3 * LR):
    """Run the batches on the device and in the f32 and f64 restatements; compare after every step.  Tensors named
    in ``residue`` have a loss gradient that is zero but for rounding: they are compared absolutely instead."""
    kw = dict(loss=loss, reg_method=reg_method, regularization=REG, positive_weight=PW)
    m32, m64 = fo.Model(params, reg_method != "AdamW"), fo.Model(params, reg_method != "AdamW", torch.float64)
    o32, o64 = fo.make_optimizer(m32, reg_method, LR, REG), fo.make_optimizer(m64, reg_method, LR, REG)
    for users, pos, neg in batches:
        old = {n: t.clone() for n, t in m32.state_dict().items()}
        old_mom = fo.moments(m32, o32)
        got = float(st.step(torch.from_numpy(users), torch.from_numpy(pos), torch.from_numpy(neg)).item())
        fo.train_step(m32, o32, users, pos, neg, **kw)
        want64 = fo.train_step(m64, o64, users, pos, neg, **kw)
        assert abs(got - want64) <= 1e-6 * abs(want64)
        mom = fo.moments(m32, o32)
        for name, want in m32.state_dict().items():
            if name in residue:
                assert float((st.params[name].cpu() - want).abs().max()) < residue_step, name
                assert float((st.moments[name][0].cpu() - mom[name][0]).abs().max()) < 1e-8, name
                continue
            assert _update_error(st.params[name].cpu(), want, old[name]) < tol, name
            for which in (0, 1):
                err = _update_error(st.moments[name][which].cpu(), mom[name][which], old_mom[name][which])
                assert err < tol, (name, which)
        # the next step starts from the restatement's f32 state, so that errors do not accumulate into the tolerance
        for name, t in m32.state_dict().items():
            st.params[name].copy_(t)
            for which in (0, 1):
                st.moments[name][which].copy_(mom[name][which])


def _batches(ml_small, B, n, count, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        at = rng.integers(0, ml_small.nnz, B)
        out.append((ml_small.users[at].astype(np.int32), ml_small.items[at].astype(np.int32),
                    rng.integers(0, ml_small.n_items, (B, n)).astype(np.int32)))  # fmt: skip
    return out


@pytest.mark.parametrize("popular", [False, True])
@pytest.mark.parametrize("n", [1, 4])
def test_sampler_equals_restatement(ml_small, popular, n):
    st = _state(_params(ml_small.n_users, ml_small.n_items, 8, True, True), ml_small.users, ml_small.items,
                "logistic", None, n, 1000, popular=popular, seed=2**63 + 12345)  # fmt: skip
    rows = np.random.default_rng(1).integers(0, ml_small.n_users, 5000).astype(np.int32)
    got = st.sample(torch.from_numpy(rows), step0=7).cpu().numpy()
    indptr = np.concatenate([[0], np.cumsum(np.bincount(ml_small.users, minlength=ml_small.n_users))])
    want = fo.sample_negatives(indptr, ml_small.items, rows, ml_small.n_items, n, seed=2**63 + 12345, step0=7,
                               batch_size=1000, popular=popular)  # fmt: skip
    assert np.array_equal(got, want)


@pytest.mark.parametrize("loss", ["logistic", "pairwise"])
@pytest.mark.parametrize("reg_method", ["AdamW", "L2", None])
@pytest.mark.parametrize("biases", [True, False])
@pytest.mark.parametrize("n, k", [(1, 64), (4, 32), (1, 50), (4, 50)])
def test_steps_match_restatement(ml_small, loss, reg_method, biases, n, k):
    """One step and five consecutive steps."""
    B = 512
    params = _params(ml_small.n_users, ml_small.n_items, k, biases, biases)
    st = _state(params, ml_small.users, ml_small.items, loss, reg_method, n, B)
    # a user bias cancels out of the pairwise loss.  The kernel makes its loss gradient an exact zero and adds only the
    # L2 term; autograd adds the L2 term's pieces (1e-6) to the two cancelling loss terms (1e-3) first, which costs
    # it about 6e-11 absolute (measured: 3e-5 of a small gradient).  So that tensor is compared absolutely: a wrong
    # L2 or decay factor would show as 1e-6 in the first moment and several 1e-3 lr in the parameter
    residue = ("u_bias.weight",) if loss == "pairwise" and biases else ()
    _check_steps(st, params, _batches(ml_small, B, n, 5), loss, reg_method, residue=residue)
    assert st.steps_done == 5


@pytest.mark.parametrize("loss, reg_method", [("logistic", "AdamW"), ("logistic", "L2"), ("pairwise", None)])
def test_one_user_and_one_item_fill_half_the_batch(ml_small, loss, reg_method):
    B, n = 1024, 2
    (users, pos, neg), = _batches(ml_small, B, n, 1, seed=5)
    users[::2], pos[::2], neg[1::2, 0] = 17, 23, 23  # item 23 also as a negative of the other half
    params = _params(ml_small.n_users, ml_small.n_items, 64, True, True)
    params["i_embed.weight"][40] = 0  # an all-zero row under the L2 term: its norm's gradient is 0
    neg[5, 1] = 40
    st = _state(params, ml_small.users, ml_small.items, loss, reg_method, n, B)
    # 512-term sums of coefficients of both signs, added in units of 64 here and in one chain by torch: the
    # cancellation leaves up to 1.5e-5 of the update in the second moment of the hot user's bias (measured)
    residue = ("u_bias.weight",) if loss == "pairwise" else ()
    # the hot user's residue adds up over 512 samples: a few 1e-9, which SparseAdam turns into about lr / 50
    _check_steps(st, params, [(users, pos, neg)] * 2, loss, reg_method, tol=1e-4, residue=residue, residue_step=0.1 * LR)


@pytest.mark.parametrize("reg_method", ["L2", None])
def test_sparse_adam_leaves_other_rows_alone(ml_small, reg_method):
    B, n = 256, 1
    params = _params(ml_small.n_users, ml_small.n_items, 32, True, True)
    st = _state(params, ml_small.users, ml_small.items, "logistic", reg_method, n, B)
    for name in st.params:  # non-zero moments, so that an unwanted decay would show
        st.moments[name][0].fill_(0.25)
        st.moments[name][1].fill_(0.5)
    before = {n_: (t.clone(), st.moments[n_][0].clone(), st.moments[n_][1].clone()) for n_, t in st.params.items()}
    (users, pos, neg), = _batches(ml_small, B, n, 1)
    st.step(torch.from_numpy(users), torch.from_numpy(pos), torch.from_numpy(neg))
    touched = {"u": np.unique(users), "i": np.unique(np.concatenate([pos, neg.flatten()]))}
    for name, t in st.params.items():
        rest = torch.from_numpy(np.setdiff1d(np.arange(t.shape[0]), touched[name[0]])).to(t.device)
        hit = torch.from_numpy(touched[name[0]]).to(t.device).long()
        for got, old in zip((t, *st.moments[name]), before[name]):
            assert torch.equal(got[rest], old[rest]), name
            assert not torch.equal(got[hit], old[hit]), name


def _train(ml_small, seed, **kw):
    m = FlexMFImplicitScorer(embedding_size=32, epochs=2, batch_size=4096, **kw)
    m.train(Dataset(ml_small), TrainingOptions(rng=seed))
    return m


@pytest.mark.parametrize("kw", [{}, {"preset": "bpr", "reg_method": "L2", "negative_count": 3, "negative_strategy": "popular"}])
def test_training_is_deterministic(ml_small, kw):
    a, b, c = _train(ml_small, 11, **kw), _train(ml_small, 11, **kw), _train(ml_small, 12, **kw)
    for name in ("user_embeddings", "item_embeddings", "user_bias", "item_bias"):
        x, y, z = getattr(a, name), getattr(b, name), getattr(c, name)
        if x is None:
            assert y is None and "bpr" in kw.values()
            continue
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), name
        assert not np.array_equal(x, z), name
    assert a.training_log == b.training_log


def test_trainer_initial_state_order_and_losses(ml_small):
    """The trainer starts from the reference's initial parameters and first permutation; its per-batch losses over
    two epochs follow the restatement fed the same negatives, and the epoch loss falls over five epochs."""
    m = FlexMFImplicitScorer(embedding_size=16, batch_size=8192, epochs=5)
    tr = m.create_trainer(Dataset(ml_small), TrainingOptions(rng=5))
    ucnt, icnt = np.bincount(ml_small.users, minlength=ml_small.n_users), np.bincount(ml_small.items, minlength=ml_small.n_items)
    want = flexmf.initial_parameters(ml_small.n_users, ml_small.n_items, 16, True, True, torch.Generator().manual_seed(5), ucnt, icnt)
    for name, t in want.items():
        assert torch.equal(tr.state.params[name].cpu(), t), name
    assert not m.is_trained()  # nothing is handed to the scorer before the first epoch
    assert np.array_equal(tr.epoch_permutation(), np.random.default_rng(5).permutation(ml_small.nnz).astype(np.int32))

    model = fo.Model(want, sparse=False)
    opt = fo.make_optimizer(model, "AdamW", 0.01, 0.01)
    st, rng = tr.state, np.random.default_rng(77)
    st.seed = 99
    for _epoch in range(2):
        perm = rng.permutation(ml_small.nnz)
        users, pos = ml_small.users[perm].astype(np.int32), ml_small.items[perm].astype(np.int32)
        neg = st.sample(torch.from_numpy(users))
        got = st.train_batches(torch.from_numpy(users), torch.from_numpy(pos), neg).cpu().numpy()
        neg = neg.cpu().numpy()
        for s, g in enumerate(got):
            sl = slice(s * 8192, (s + 1) * 8192)
            w = fo.train_step(model, opt, users[sl], pos[sl], neg[sl], loss="logistic", reg_method="AdamW",
                              regularization=0.01, positive_weight=1.0)  # fmt: skip
            assert abs(g - w) <= 1e-3 * abs(w)
    m2 = FlexMFImplicitScorer(embedding_size=16, batch_size=8192, epochs=5)
    m2.train(Dataset(ml_small), TrainingOptions(rng=5))
    log = [e["loss"] for e in m2.training_log]
    assert len(log) == 5 and log[4] < log[0]


def test_parameters_round_trip(ml_small):
    m = FlexMFImplicitScorer(embedding_size=16, batch_size=8192, epochs=1)
    tr = m.create_trainer(Dataset(ml_small), TrainingOptions(rng=5))
    tr.train_epoch()
    saved = {n: t.clone() for n, t in tr.get_parameters().items()}
    assert set(saved) == {"u_bias.weight", "i_bias.weight", "u_embed.weight", "i_embed.weight"}
    tr.train_epoch()
    assert not np.array_equal(m.item_embeddings, saved["i_embed.weight"].numpy())
    tr.load_parameters(saved)
    assert np.array_equal(m.item_embeddings, saved["i_embed.weight"].numpy())
    tr.finalize()
    assert m.is_trained()


@pytest.mark.parametrize("kw", [{}, {"preset": "bpr"}])
def test_scorer_batched_interface(ml_small, kw):
    ds = Dataset(ml_small)
    m = _train(ml_small, 3, **kw)
    uids = [ds.users.id(u) for u in (0, 5, 77, 300)]
    queries = [RecQuery(uid, ds.user_history(u)) for uid, u in zip(uids, (0, 5, 77, 300))] + [RecQuery(-999, None)]
    S = m.score_matrix(queries).cpu().numpy()
    assert np.isnan(S[:, -1]).all() and not np.isnan(S[:, :-1]).any()
    for exclude in (None, "query"):
        recs = m.recommend_batch(queries, 25, exclude=exclude)
        assert len(recs[-1]) == 0
        for b, rec in enumerate(recs[:-1]):
            col = S[:, b].copy()
            if exclude == "query":
                col[queries[b].query_items.numbers(vocabulary=m.items)] = np.nan
            want = oracle.argtopn(col, 25)
            assert np.array_equal(rec.numbers(), want)
            assert np.array_equal(rec.scores().view(np.int32), col[want].view(np.int32))
    targets = [ItemList(item_ids=np.concatenate([ds.items.ids()[b::7], [-5]])) for b in range(len(queries))]
    scored = m.score_batch(queries, targets)
    for b, (tgt, out) in enumerate(zip(targets, scored)):
        s = out.scores()
        assert np.isnan(s[-1])
        nums = tgt.numbers(vocabulary=m.items, missing="negative")[:-1]
        assert np.array_equal(s[:-1].view(np.int32), S[nums, b].view(np.int32))
        one = m(queries[b], tgt).scores()
        assert np.array_equal(np.isnan(one), np.isnan(s)) and np.allclose(one[:-1], s[:-1], rtol=1e-6, atol=1e-6, equal_nan=True)
    # ub + ib + u·i in f64
    u = 77
    want = m.item_embeddings.astype(np.float64) @ m.user_embeddings[u].astype(np.float64)
    want += (m.item_bias if m.item_bias is not None else 0.0) + (m.user_bias[u] if m.user_bias is not None else 0.0)
    assert np.allclose(S[:, 2], want, rtol=1e-5, atol=1e-6)
    m2 = pickle.loads(pickle.dumps(m))
    assert np.array_equal(m2.score_matrix(queries[:2]).cpu().numpy().view(np.int32), S[:, :2].view(np.int32))


@pytest.mark.parametrize("reg_method", ["AdamW", None])
def test_more_rows_than_a_batch_touches(reg_method):
    """20,000 x 8,000 with 1 M interactions and batches of 4,096: most rows are untouched by a step, and the popular
    items make long groups."""
    users, items, _ = prep.synth_interactions_device(20_000, 8_000, 1_000_000, seed=4)
    params = _params(20_000, 8_000, 64, True, True)
    st = _state(params, users, items, "logistic", reg_method, 1, 4096, popular=True, seed=8)
    at = torch.from_numpy(np.random.default_rng(2).integers(0, 1_000_000, 3 * 4096)).to(users.device)
    u, p = users[at], items[at]
    neg = st.sample(u)
    got = st.train_batches(u, p, neg).cpu().numpy()
    model = fo.Model(params, sparse=reg_method != "AdamW")
    opt = fo.make_optimizer(model, reg_method, LR, REG)
    u, p, neg = u.cpu().numpy(), p.cpu().numpy(), neg.cpu().numpy()
    for s in range(3):
        sl = slice(s * 4096, (s + 1) * 4096)
        w = fo.train_step(model, opt, u[sl], p[sl], neg[sl], loss="logistic", reg_method=reg_method, regularization=REG,
                          positive_weight=PW)  # fmt: skip
        assert abs(got[s] - w) <= 1e-5 * abs(w)
    for name, want in model.state_dict().items():
        assert _update_error(st.params[name].cpu(), want, params[name]) < 1e-4, name  # three steps' rounding
