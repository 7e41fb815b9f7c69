"""
FlexMF explicit on the device: ``lk_flexmf_step`` with the MSE loss against the plain-torch restatement
(``flexmf_explicit_oracle``), ``FlexMFExplicitScorer`` trained on ml-latest-small against the reference's own trainer (the
golden files of ``test_flexmf_explicit``), determinism, held-out accuracy, and the scorer's batched interface.
"""

import pickle

import numpy as np
import pytest
import torch

import flexmf_explicit_oracle as feo
import flexmf_oracle as fo
import oracle
import test_flexmf_explicit as host
from lkpy_b200 import engine, flexmf
from lkpy_b200.components import Dataset, ItemList, RecQuery, TrainingOptions
from lkpy_b200.data import Interactions
from lkpy_b200.flexmf import FlexMFExplicitScorer

pytestmark = pytest.mark.gpu
LR, REG = 0.01, 0.1
# The device and the reference differ by rounding in every step (the dot product and the norms are summed in another
# order), and Adam turns such a difference into one relative to the update.  Measured on an H100 against the three
# recordings, after two epochs (26 steps): sampled tables within 1.3e-7 (relative Frobenius), epoch losses within
# 1e-7 (relative), scores within 1.4e-8.  The bounds leave a factor of about 70.
GOLD_TABLE_TOL, GOLD_LOSS_TOL, GOLD_SCORE_TOL = 1e-5, 1e-6, 1e-6


def _update_error(new, want, old) -> float:
    """‖new − want‖ / ‖want − old‖: the error of the update, not of the parameter."""
    new, want, old = (np.asarray(x, dtype=np.float64) for x in (new, want, old))
    return float(np.linalg.norm(new - want) / max(np.linalg.norm(want - old), 1e-300))


def _state(params, ml_small, reg_method, B):
    targets = np.zeros(ml_small.nnz, np.float32)  # per-interaction targets: only epoch() reads them
    return engine.FlexMFState(params, ml_small.users, ml_small.items, loss="mse", reg_method=reg_method,
                              negative_count=0, batch_size=B, learning_rate=LR, regularization=REG, ratings=targets)  # fmt: skip


def _check_steps(st, params, batches, reg_method, tol=1e-5):
    """Run the batches on the device and in the f32 and f64 restatements; compare after every step."""
    kw = dict(reg_method=reg_method, regularization=REG)
    m32, m64 = fo.Model(params, reg_method != "AdamW"), fo.Model(params, reg_method != "AdamW", torch.float64)
    o32, o64 = fo.make_optimizer(m32, reg_method, LR, REG), fo.make_optimizer(m64, reg_method, LR, REG)
    for users, items, t in batches:
        old = {n: x.clone() for n, x in m32.state_dict().items()}
        old_mom = fo.moments(m32, o32)
        got = float(st.step(torch.from_numpy(users), torch.from_numpy(items), ratings=torch.from_numpy(t)).item())
        feo.train_step(m32, o32, users, items, torch.from_numpy(t), **kw)
        want64 = feo.train_step(m64, o64, users, items, torch.from_numpy(t).double(), **kw)
        assert abs(got - want64) <= 1e-6 * abs(want64)
        mom = fo.moments(m32, o32)
        for name, want in m32.state_dict().items():
            assert _update_error(st.params[name].cpu(), want, old[name]) < tol, name
            for which in (0, 1):
                assert _update_error(st.moments[name][which].cpu(), mom[name][which], old_mom[name][which]) < tol, (name, which)
        # the next step starts from the restatement's f32 state, so that errors do not accumulate into the tolerance
        for name, x in m32.state_dict().items():
            st.params[name].copy_(x)
            for which in (0, 1):
                st.moments[name][which].copy_(mom[name][which])


def _batches(ml_small, B, count, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        at = rng.integers(0, ml_small.nnz, B)
        t = (ml_small.ratings[at] - np.float32(3.5)).astype(np.float32)
        out.append((ml_small.users[at].astype(np.int32), ml_small.items[at].astype(np.int32), t))
    return out


@pytest.mark.parametrize("reg_method", ["L2", "AdamW", None])
@pytest.mark.parametrize("biases", [False, True])
@pytest.mark.parametrize("k", [64, 50])
def test_steps_match_restatement(ml_small, reg_method, biases, k):
    """One step and four more.  ``biases=False`` is the reference's model; with biases the kernel's MSE bias terms
    (the user and item L2 weights of the header) are checked too.  k = 50 is the scalar-row path."""
    B = 512
    params = flexmf.initial_parameters(ml_small.n_users, ml_small.n_items, k, biases, biases, torch.Generator().manual_seed(3))
    st = _state(params, ml_small, reg_method, B)
    _check_steps(st, params, _batches(ml_small, B, 5), reg_method)
    assert st.steps_done == 5


@pytest.mark.parametrize("reg_method", ["L2", "AdamW", None])
def test_one_user_and_one_item_fill_half_the_batch(ml_small, reg_method):
    B = 1024
    (users, items, t), = _batches(ml_small, B, 1, seed=5)
    users[::2], items[::2] = 17, 23
    params = flexmf.initial_parameters(ml_small.n_users, ml_small.n_items, 64, True, True, torch.Generator().manual_seed(3))
    params["i_embed.weight"][40] = 0  # an all-zero row under the L2 term: its norm's gradient is 0
    items[5] = 40
    st = _state(params, ml_small, reg_method, B)
    # 512-term sums of coefficients of both signs, added in units of 64 here and in one chain by torch
    _check_steps(st, params, [(users, items, t)] * 2, reg_method, tol=1e-4)


def _train(data, seed, **kw):
    m = FlexMFExplicitScorer(**({"embedding_size": 16, "epochs": 2} | kw))
    m.train(Dataset(data), TrainingOptions(rng=seed))
    return m


@pytest.mark.parametrize("reg_method", ["L2", "AdamW", None])
def test_training_follows_the_reference_trainer(ml_small, reg_method):
    """``FlexMFExplicitScorer(embedding_size=16, epochs=2)`` with seed 42 against the reference's own trainer:
    the same mean, the same initial tables, and its losses, tables and scores after two epochs within rounding."""
    theirs = host.reference_golden(ml_small, reg_method)
    m = FlexMFExplicitScorer(embedding_size=16, epochs=2, reg_method=reg_method)
    tr = m.create_trainer(Dataset(ml_small), TrainingOptions(rng=42))
    assert m.global_bias == float(theirs["mu"])
    assert set(tr.get_parameters()) == set(host.TABLES)
    for name in host.TABLES:
        got = host.sampled(name, tr.state.params[name].cpu())
        assert np.array_equal(got.view(np.int32), theirs[f"init/{name}"].view(np.int32)), name
    losses = []
    for e in range(2):
        losses.append(tr.train_epoch()["loss"])
        for name in host.TABLES:
            err = host.rel_err(host.sampled(name, tr.state.params[name].cpu()), theirs[f"epoch{e + 1}/{name}"])
            print(f"{reg_method} epoch {e + 1} {name}: {err:.2e}")
            assert err < GOLD_TABLE_TOL, (e, name)
    tr.finalize()
    print(f"{reg_method} losses {losses} against {theirs['losses']}")
    assert np.allclose(losses, theirs["losses"], rtol=GOLD_LOSS_TOL, atol=0)
    ds = Dataset(ml_small)
    got = np.stack([m(ds.users.id(u), ItemList(item_ids=ds.items.ids()[host.SCORE_ITEMS])).scores() for u in host.SCORE_USERS])
    err = host.rel_err(got, theirs["scores"])
    print(f"{reg_method} scores: {err:.2e}")
    assert err < GOLD_SCORE_TOL


def test_training_is_deterministic(ml_small):
    a, b, c = _train(ml_small, 11), _train(ml_small, 11), _train(ml_small, 12)
    for name in ("user_embeddings", "item_embeddings"):
        x, y, z = getattr(a, name), getattr(b, name), getattr(c, name)
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), name
        assert not np.array_equal(x, z), name
    assert a.user_bias is None and a.item_bias is None and a.global_bias == b.global_bias
    assert a.training_log == b.training_log


def test_held_out_rmse_matches_the_restatement(ml_small):
    """An 80/20 split of ml-latest-small: five epochs on the device and in the CPU restatement with the same seed
    predict the held-out ratings with RMSEs within 0.01 of each other."""
    rng = np.random.default_rng(9)
    test = rng.random(ml_small.nnz) < 0.2
    train = Interactions(ml_small.users[~test], ml_small.items[~test], ml_small.ratings[~test], ml_small.n_users,
                         ml_small.n_items, ml_small.user_ids, ml_small.item_ids)  # fmt: skip
    epochs, k = 5, 16
    m = _train(train, 4, embedding_size=k, epochs=epochs)
    tu, ti, tr_ = ml_small.users[test], ml_small.items[test], ml_small.ratings[test].astype(np.float64)
    pred = (m.user_embeddings[tu].astype(np.float64) * m.item_embeddings[ti]).sum(1) + m.global_bias
    rmse_dev = float(np.sqrt(np.mean((pred - tr_) ** 2)))

    ucnt = np.bincount(train.users, minlength=train.n_users)
    icnt = np.bincount(train.items, minlength=train.n_items)
    params = flexmf.initial_parameters(train.n_users, train.n_items, k, False, False, flexmf._torch_generator(4), ucnt, icnt)
    values = torch.from_numpy(train.ratings)
    mu = values.mean()
    model = fo.Model(params, sparse=True)
    opt = fo.make_optimizer(model, "L2", LR, REG)
    prng = np.random.default_rng(4)
    for _ in range(epochs):
        feo.explicit_epoch(model, opt, train.users, train.items, (values - mu).numpy(), prng.permutation(train.nnz), 8192,
                           reg_method="L2", regularization=REG)  # fmt: skip
    t = {n: x.numpy().astype(np.float64) for n, x in model.state_dict().items()}
    pred = (t["u_embed.weight"][tu] * t["i_embed.weight"][ti]).sum(1) + mu.item()
    rmse_cpu = float(np.sqrt(np.mean((pred - tr_) ** 2)))
    print(f"held-out RMSE: device {rmse_dev:.5f}, restatement {rmse_cpu:.5f}")
    assert abs(rmse_dev - rmse_cpu) < 0.01 and rmse_dev < 1.5


def test_parameters_round_trip(ml_small):
    m = FlexMFExplicitScorer(embedding_size=16, epochs=1)
    tr = m.create_trainer(Dataset(ml_small), TrainingOptions(rng=5))
    tr.train_epoch()
    saved = {n: t.clone() for n, t in tr.get_parameters().items()}
    assert set(saved) == {"u_embed.weight", "i_embed.weight"}
    tr.train_epoch()
    assert not np.array_equal(m.item_embeddings, saved["i_embed.weight"].numpy())
    tr.load_parameters(saved)
    assert np.array_equal(m.item_embeddings, saved["i_embed.weight"].numpy())
    tr.finalize()
    assert m.is_trained()


def test_scorer_batched_interface(ml_small):
    ds = Dataset(ml_small)
    m = _train(ml_small, 3)
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
    assert np.array_equal(m.recommend_batch(queries[:2], 10)[0].numbers(), oracle.argtopn(S[:, 0].copy(), 10))  # default: every item
    targets = [ItemList(item_ids=np.concatenate([ds.items.ids()[b::7], [-5]])) for b in range(len(queries))]
    scored = m.score_batch(queries, targets)
    for b, (tgt, out) in enumerate(zip(targets, scored)):
        s = out.scores()
        assert np.isnan(s[-1])  # unknown item
        nums = tgt.numbers(vocabulary=m.items, missing="negative")[:-1]
        assert np.array_equal(s[:-1].view(np.int32), S[nums, b].view(np.int32))
        one = m(queries[b], tgt).scores()
        assert np.array_equal(one.view(np.int32), s.view(np.int32))
    assert np.isnan(scored[-1].scores()).all()  # unknown user
    # u·i + mu in f64
    u = 77
    want = m.item_embeddings.astype(np.float64) @ m.user_embeddings[u].astype(np.float64) + m.global_bias
    assert np.allclose(S[:, 2], want, rtol=1e-5, atol=1e-5)
    m2 = pickle.loads(pickle.dumps(m))
    assert m2.global_bias == m.global_bias
    assert np.array_equal(m2.score_matrix(queries[:2]).cpu().numpy().view(np.int32), S[:, :2].view(np.int32))
