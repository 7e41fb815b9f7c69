"""
FlexMF explicit, host side: the configuration surface, the torch restatement's MSE step against hand-written update
formulas, the step's host validation of the MSE arguments, and the reference's own trainer (``flexmf/_explicit.py``
over ``_training.py``, ``_model.py``, loaded by tests/flexmf_ref_sandbox.py) against the restatement.  CPU only.

The reference's side comes from a lenskit/lkpy checkout when there is one, else from
``tests/golden/reference_classes/flexmf_explicit_*.npz``, which ``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites from the
checkout (on the CPU, without ``torch.compile``).
"""

import ctypes as C
import os
import warnings
from pathlib import Path

import numpy as np
import pytest
import torch

import flexmf_explicit_oracle as feo
import flexmf_oracle as fo
import flexmf_ref_sandbox
import ref_sandbox
from lkpy_b200 import _lib, flexmf
from lkpy_b200.flexmf import FlexMFExplicitConfig, FlexMFExplicitScorer, FlexMFImplicitConfig

GOLD = Path(__file__).resolve().parent / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"
ROWS_U = np.random.default_rng(0).choice(671, 120, replace=False)
ROWS_I = np.random.default_rng(1).choice(9066, 300, replace=False)
SCORE_USERS = (0, 5, 77, 300)
SCORE_ITEMS = np.arange(0, 9066, 37)
K, EPOCHS, SEED = 16, 2, 42
REG_METHODS = ["L2", "AdamW", None]
TABLES = ("u_embed.weight", "i_embed.weight")  # the reference's model scores without its bias tables
# On the CPU the restatement's tables after two epochs are the reference's bit for bit (measured, all three
# reg_methods).  The epoch loss differs in how the batch losses are averaged (an f32 running sum divided in Python,
# against an f64 mean): 3e-8 relative, measured.  The scores differ by the reference's f32 evaluation against this
# test's f64 one: 2e-8 relative, measured.
LOSS_TOL, SCORE_TOL = 1e-6, 1e-6


def gold_name(reg_method) -> str:
    return f"flexmf_explicit_{reg_method or 'none'}"


def sampled(name: str, t) -> np.ndarray:
    """The golden files' rows of a table: ``ROWS_U`` of the user tables, ``ROWS_I`` of the item tables."""
    t = np.asarray(t, dtype=np.float32)
    return t[ROWS_U if name.startswith("u_") else ROWS_I]


def _record(ml_small, reg_method) -> dict:
    """The reference's trainer on ml-latest-small: mu, the epoch losses, the sampled tables at the start and after
    every epoch, and its ``__call__`` scores."""
    with flexmf_ref_sandbox.flexmf_modules() as ref, warnings.catch_warnings():
        warnings.simplefilter("ignore")
        exp, training, items_mod = ref["lenskit.flexmf._explicit"], ref["lenskit.training"], ref["lenskit.data._items"]
        m = exp.FlexMFExplicitScorer(embedding_size=K, epochs=EPOCHS, reg_method=reg_method)
        opts = training.TrainingOptions(rng=SEED, device="cpu", environment={"LK_TORCH_COMPILE": "0"})
        tr = m.create_trainer(flexmf_ref_sandbox.FlexMFDataset(ml_small), opts)
        assert isinstance(tr, exp.FlexMFExplicitTrainer) and tr._compiled_model is None
        # the class attributes u_bias = i_bias = None shadow the registered bias modules: they are never used
        out = {"mu": np.float64(m.global_bias), "biases_inactive": np.array(m.model.u_bias is None and m.model.i_bias is None)}
        for name in TABLES:
            out[f"init/{name}"] = sampled(name, m.model.state_dict()[name])
        losses = []
        for e in range(EPOCHS):
            losses.append(tr.train_epoch()["loss"])
            for name in TABLES:
                out[f"epoch{e + 1}/{name}"] = sampled(name, m.model.state_dict()[name])
        tr.finalize()
        out["losses"] = np.array(losses)
        ItemList = items_mod.ItemList
        out["scores"] = np.stack([
            np.asarray(m(ml_small.user_ids[u], ItemList(item_ids=ml_small.item_ids[SCORE_ITEMS])).scores("numpy"),
                       dtype=np.float32)
            for u in SCORE_USERS
        ])  # fmt: skip
        return out


def reference_golden(ml_small, reg_method) -> dict:
    """The reference's values: recorded live when asked to, else read from the golden file."""
    path = GOLD / f"{gold_name(reg_method)}.npz"
    if RECORD:
        assert ref_sandbox.available(), "recording needs the reference checkout"
        np.savez_compressed(path, **_record(ml_small, reg_method))
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def restated_training(ml_small, reg_method, params, epochs=EPOCHS, dtype=torch.float32):
    """The plain-torch restatement of the explicit trainer with the reference's data, seed and sample order:
    ``(model, mu, epoch losses, tables after every epoch)``."""
    values = torch.from_numpy(ml_small.ratings).to(torch.float32)
    mu = values.mean()
    targets = (values - mu).numpy()
    c = FlexMFExplicitConfig(embedding_size=K, reg_method=reg_method)
    model = fo.Model(params, sparse=reg_method != "AdamW", dtype=dtype)
    opt = fo.make_optimizer(model, reg_method, c.learning_rate, c.regularization)
    rng = np.random.default_rng(SEED)
    losses, tables = [], []
    for _ in range(epochs):
        perm = rng.permutation(ml_small.nnz)
        bl = feo.explicit_epoch(model, opt, ml_small.users, ml_small.items, targets, perm, c.batch_size,
                                reg_method=reg_method, regularization=c.regularization)  # fmt: skip
        losses.append(float(np.mean(bl)))
        tables.append({n: t.clone() for n, t in model.state_dict().items()})
    return model, mu.item(), losses, tables


def initial(ml_small):
    ucnt = np.bincount(ml_small.users, minlength=ml_small.n_users)
    icnt = np.bincount(ml_small.items, minlength=ml_small.n_items)
    return flexmf.initial_parameters(ml_small.n_users, ml_small.n_items, K, False, False,
                                     flexmf._torch_generator(SEED), ucnt, icnt)  # fmt: skip


def rel_err(got, want) -> float:
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.linalg.norm(got - want) / np.linalg.norm(want))


# ------------------------------------------------------------------------------------------------------------
# configuration
# ------------------------------------------------------------------------------------------------------------


def test_config_defaults_and_alias():
    c = FlexMFExplicitConfig()
    assert (c.embedding_size, c.batch_size, c.learning_rate, c.epochs) == (64, 8192, 0.01, 10)
    assert (c.regularization, c.reg_method) == (0.1, "L2")
    assert FlexMFExplicitConfig(embedding_size_exp=4).embedding_size == 16
    assert FlexMFExplicitConfig(reg_method=None).reg_method is None
    assert FlexMFExplicitConfig(reg_method="AdamW").reg_method == "AdamW"
    assert FlexMFExplicitScorer(embedding_size=8).config.embedding_size == 8
    # the implicit model keeps its own defaults
    assert (FlexMFImplicitConfig().regularization, FlexMFImplicitConfig().reg_method) == (0.01, "AdamW")


@pytest.mark.parametrize("kw, named", [({"embedding_size": 129}, "embedding_size"), ({"reg_method": "adam"}, "reg_method"),
                                       ({"embedding_size_exp": 8}, "embedding_size")])  # fmt: skip
def test_rejected_options_are_named(kw, named):
    with pytest.raises(ValueError, match=named):
        FlexMFExplicitConfig(**kw)


def test_no_ratings_is_a_clear_error(ml_small):
    from lkpy_b200.components import Dataset, TrainingOptions
    from lkpy_b200.data import Interactions

    bare = Interactions(ml_small.users, ml_small.items, None, ml_small.n_users, ml_small.n_items)
    m = FlexMFExplicitScorer(embedding_size=8, epochs=1)
    # the device is asked for first; without one the engine's own error comes before the data is read
    with pytest.raises((ValueError, _lib.EngineError), match="ratings|no CPU fallback"):
        m.train(Dataset(bare), TrainingOptions(rng=1))


# ------------------------------------------------------------------------------------------------------------
# the MSE step of the restatement against the update formulas written out by hand in f64
# ------------------------------------------------------------------------------------------------------------


def _toy(rng, n_users=7, n_items=9, k=5):
    p = {"u_embed.weight": rng.normal(0, 0.1, (n_users, k)), "i_embed.weight": rng.normal(0, 0.1, (n_items, k)),
         "u_bias.weight": rng.normal(0, 0.1, (n_users, 1)), "i_bias.weight": rng.normal(0, 0.1, (n_items, 1))}  # fmt: skip
    return {n: v.astype(np.float64) for n, v in p.items()}


@pytest.mark.parametrize("reg_method", REG_METHODS)
def test_oracle_mse_step_is_the_documented_update(reg_method):
    """The gradient by finite differences of ``mse(s, t) + [L2] reg * mean(norm)``, pushed through the optimiser
    formulas of ``include/lkpy_b200.h``, gives the restatement's step (f64); the loss it reports is the squared
    error alone."""
    rng = np.random.default_rng(0)
    p0 = _toy(rng)
    users, items = np.array([0, 3, 3, 6, 1]), np.array([1, 2, 8, 1, 1])
    t = torch.tensor([0.5, -1.0, 1.5, 0.0, -0.5], dtype=torch.float64)
    lr, reg = 0.01, 0.1
    model = fo.Model(p0, sparse=reg_method != "AdamW", dtype=torch.float64)
    opt = fo.make_optimizer(model, reg_method, lr, reg)
    got_loss = feo.train_step(model, opt, users, items, t, reg_method=reg_method, regularization=reg)

    def f(params, with_norm=True):
        with torch.no_grad():
            m = fo.Model(params, sparse=False, dtype=torch.float64)
            u, i = torch.as_tensor(users), torch.as_tensor(items)
            s = (m.tables["u_embed.weight"][u] * m.tables["i_embed.weight"][i]).sum(1)
            s = s + m.tables["u_bias.weight"][u, 0] + m.tables["i_bias.weight"][i, 0]
            out = ((s - t) ** 2).mean()
            if with_norm and reg_method == "L2":
                nrm = (m.tables["u_bias.weight"][u, 0] ** 2 + m.tables["i_bias.weight"][i, 0] ** 2
                       + m.tables["u_embed.weight"][u].norm(dim=1) + m.tables["i_embed.weight"][i].norm(dim=1))  # fmt: skip
                out = out + reg * nrm.mean()
            return float(out)

    assert got_loss == pytest.approx(f(p0, with_norm=False), rel=1e-12)
    touched = {"u": set(users.tolist()), "i": set(items.tolist())}
    b1, b2, eps = 0.9, 0.999, 1e-8
    for name, w in p0.items():
        g = np.zeros_like(w)
        for idx in np.ndindex(*w.shape):
            hi, lo = {n: v.copy() for n, v in p0.items()}, {n: v.copy() for n, v in p0.items()}
            hi[name][idx] += 1e-6
            lo[name][idx] -= 1e-6
            g[idx] = (f(hi) - f(lo)) / 2e-6
        m, v = (1 - b1) * g, (1 - b2) * g * g
        if reg_method == "AdamW":
            want = w * (1 - lr * reg) - lr / (1 - b1) * m / (np.sqrt(v) / np.sqrt(1 - b2) + eps)
        else:
            want = w - lr * np.sqrt(1 - b2) / (1 - b1) * m / (np.sqrt(v) + eps)
            rows = [r for r in range(len(w)) if r not in touched[name[0]]]
            want[rows] = w[rows]
        got = dict(model.state_dict())[name].numpy()
        assert np.allclose(got, want, rtol=0, atol=2e-4 * lr), name


def test_item_l2_weight_is_twice_the_implicit_positive():
    """The header's per-occurrence L2 weights, from autograd: an item row gets ``reg/B`` under MSE and
    ``0.5 reg/B`` as an implicit positive; a user row gets ``reg/B`` under both."""
    p0 = _toy(np.random.default_rng(3))
    users, items, reg = np.array([0, 1, 2, 3]), np.array([4, 5, 6, 7]), 0.2
    grads = {}
    for loss in ("mse", "logistic"):
        g = {}
        for reg_method in ("L2", None):
            model = fo.Model(p0, sparse=False, dtype=torch.float64)
            if loss == "mse":
                out, _ = feo.mse_terms(model, users, items, torch.zeros(4, dtype=torch.float64), reg_method=reg_method,
                                       regularization=reg)  # fmt: skip
            else:
                out = fo.batch_loss(model, users, items, [[8]] * 4, loss=loss, reg_method=reg_method,
                                    regularization=reg, positive_weight=1.0)  # fmt: skip
            out.backward()
            g[reg_method] = {n: t.grad.clone() for n, t in model.named_parameters()}
        grads[loss] = {n: g["L2"][n] - g[None][n] for n in g["L2"]}  # the L2 term's share
    ib = torch.as_tensor(p0["i_bias.weight"])
    assert torch.allclose(grads["mse"]["i_bias.weight"][4], reg / 4 * 2 * ib[4])
    assert torch.allclose(grads["logistic"]["i_bias.weight"][4], 0.5 * reg / 4 * 2 * ib[4])
    ub = torch.as_tensor(p0["u_bias.weight"])
    for loss in ("mse", "logistic"):
        assert torch.allclose(grads[loss]["u_bias.weight"][0], reg / 4 * 2 * ub[0])


# ------------------------------------------------------------------------------------------------------------
# the step's host validation of the MSE arguments (the built library, no device)
# ------------------------------------------------------------------------------------------------------------


def test_step_validates_mse_arguments_on_the_host(cuda_lib):
    need = C.c_int64()
    assert cuda_lib.lk_flexmf_workspace_bytes(8192, 0, 64, C.byref(need)) == 0 and need.value > 0
    assert cuda_lib.lk_flexmf_workspace_bytes(8192, -1, 64, C.byref(need)) == -1
    ratings = (C.c_float * 4)()
    cases = [
        (_lib.LK_FLEXMF_MSE, 1, C.cast(ratings, C.c_void_p).value, b"negatives"),
        (_lib.LK_FLEXMF_LOGISTIC, 0, None, b"negatives"),
        (_lib.LK_FLEXMF_PAIRWISE, 0, None, b"negatives"),
        (_lib.LK_FLEXMF_MSE, 0, None, b"d_ratings"),
    ]
    for loss, n_neg, d_ratings, msg in cases:
        a = _lib.LkFlexmfStepArgs()
        a.batch, a.n_neg, a.k, a.loss = 4, n_neg, 64, loss
        assert cuda_lib.lk_flexmf_workspace_bytes(4, n_neg, 64, C.byref(need)) == 0
        a.d_workspace, a.workspace_bytes = 1, need.value  # never dereferenced: the checks are on the host
        a.d_ratings = d_ratings
        assert cuda_lib.lk_flexmf_step(C.byref(a), None) == -1, (loss, n_neg)  # LK_ERR_INVALID
        assert msg in cuda_lib.lk_last_error(), cuda_lib.lk_last_error()


# ------------------------------------------------------------------------------------------------------------
# the reference's own trainer against the restatement
# ------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("reg_method", REG_METHODS)
def test_reference_trainer_equals_the_restatement(ml_small, reg_method):
    """``FlexMFExplicitScorer(embedding_size=16, epochs=2)`` trained by the reference with seed 42: its mean and
    initial tables are this package's bit for bit; its tables after each epoch are the restatement's, fed the same
    permutations, bit for bit, and its epoch losses within ``LOSS_TOL``; its scores are ``u·i + mu`` of its own
    tables: its bias tables take no part."""
    theirs = reference_golden(ml_small, reg_method)
    assert bool(theirs["biases_inactive"])
    params = initial(ml_small)
    for name in TABLES:
        assert np.array_equal(sampled(name, params[name]).view(np.int32), theirs[f"init/{name}"].view(np.int32)), name
    _model, mu, losses, tables = restated_training(ml_small, reg_method, params)
    assert mu == float(theirs["mu"])
    assert np.allclose(losses, theirs["losses"], rtol=LOSS_TOL, atol=0)
    for e in range(EPOCHS):
        for name in TABLES:
            got = sampled(name, tables[e][name])
            assert np.array_equal(got.view(np.int32), theirs[f"epoch{e + 1}/{name}"].view(np.int32)), (e, name)
    assert theirs["scores"].shape == (len(SCORE_USERS), len(SCORE_ITEMS)) and np.isfinite(theirs["scores"]).all()
    assert rel_err(restated_scores(tables[-1], mu), theirs["scores"]) < SCORE_TOL


def restated_scores(tables, mu) -> np.ndarray:
    """``u·i + mu`` of ``SCORE_USERS`` x ``SCORE_ITEMS`` in f64."""
    t = {n: np.asarray(v, dtype=np.float64) for n, v in tables.items()}
    return t["u_embed.weight"][np.array(SCORE_USERS)] @ t["i_embed.weight"][SCORE_ITEMS].T + mu
