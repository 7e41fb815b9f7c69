"""
FlexMF implicit, host side: the configuration surface (defaults, aliases, presets, and every option the engine
rejects), the sampler's NumPy restatement, the torch restatement of the step against hand-written update formulas,
the initial parameters, the ABI structs' layout and the absence of a fallback.  CPU only.
"""

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import flexmf_oracle as fo
from lkpy_b200 import _lib, flexmf
from lkpy_b200.components import Dataset, TrainingOptions
from lkpy_b200.flexmf import FlexMFImplicitConfig, FlexMFImplicitScorer

ROOT = Path(__file__).resolve().parent.parent


def test_config_defaults_and_aliases():
    c = FlexMFImplicitConfig()
    assert (c.embedding_size, c.batch_size, c.learning_rate, c.epochs, c.regularization) == (64, 8192, 0.01, 10, 0.01)
    assert (c.reg_method, c.loss, c.negative_strategy, c.negative_count, c.positive_weight) == ("AdamW", "logistic", None, 1, 1.0)
    assert (c.user_bias, c.item_bias, c.preset, c.convolution_layers) == (None, True, None, 0)
    assert c.selected_negative_strategy() == "uniform" and c.selected_user_bias() is True
    assert FlexMFImplicitConfig(loss="pairwise").selected_user_bias() is False
    assert FlexMFImplicitConfig(loss="pairwise", user_bias=True).selected_user_bias() is True
    assert FlexMFImplicitConfig(embedding_size_exp=5).embedding_size == 32
    assert FlexMFImplicitConfig(reg_method=None).reg_method is None
    assert FlexMFImplicitScorer(embedding_size=16, negative_strategy="popular").config.selected_negative_strategy() == "popular"


def test_preset_bpr_yields_to_explicit_options():
    c = FlexMFImplicitConfig(preset="bpr")
    assert (c.loss, c.user_bias, c.item_bias) == ("pairwise", False, False)
    assert FlexMFImplicitConfig(preset="bpr", item_bias=True).item_bias is True


@pytest.mark.parametrize(
    "kw, named",
    [
        ({"loss": "warp"}, "loss"),
        ({"negative_strategy": "misranked"}, "negative_strategy"),
        ({"preset": "warp"}, "preset"),
        ({"preset": "lightgcn"}, "preset"),
        ({"convolution_layers": 2}, "convolution_layers"),
        ({"embedding_size": 129}, "embedding_size"),
        ({"negative_count": 0}, "negative_count"),
        ({"reg_method": "adam"}, "reg_method"),
    ],
)
def test_uncovered_options_are_rejected_by_name(kw, named):
    with pytest.raises(ValueError, match=named):
        FlexMFImplicitConfig(**kw)


# ------------------------------------------------------------------------------------------------------------
# sampler restatement
# ------------------------------------------------------------------------------------------------------------


def _csr(ml_small):
    indptr = np.concatenate([[0], np.cumsum(np.bincount(ml_small.users, minlength=ml_small.n_users))])
    return indptr, ml_small.items


def test_draw_is_the_header_definition():
    """One draw worked with Python integers, the header's formulas taken literally."""
    M = (1 << 64) - 1

    def mix(x):
        x ^= x >> 30
        x = (x * 0xBF58476D1CE4E5B9) & M
        x ^= x >> 27
        x = (x * 0x94D049BB133111EB) & M
        return x ^ (x >> 31)

    G = 0x9E3779B97F4A7C15
    for seed, step, pos, rep, att, m in [(0, 0, 0, 0, 0, 9724), (2**63 + 5, 3051, 8191, 3, 10, 25_000_095), (7, 1, 2, 1, 4, 1)]:
        h = mix((seed + G * (step + 1)) & M)
        h = mix((h + G * (pos + 1)) & M)
        h = mix((h + G * ((rep << 32) + att + 1)) & M)
        assert int(fo.draw(seed, step, pos, rep, att, m)) == ((h >> 32) * m) >> 32


def test_sampler_avoids_training_items_and_always_answers(ml_small):
    indptr, cols = _csr(ml_small)
    rows = np.random.default_rng(3).integers(0, ml_small.n_users, 4000)
    for popular in (False, True):
        neg = fo.sample_negatives(indptr, cols, rows, ml_small.n_items, 2, seed=11, popular=popular, max_attempts=200)
        seen = set(zip(ml_small.users.tolist(), ml_small.items.tolist()))
        assert not any((int(u), int(i)) in seen for u, row in zip(rows, neg) for i in row)
    # a user who has every item still gets an answer, after max_attempts rejections
    full_ptr, full_cols = np.array([0, 5]), np.arange(5, dtype=np.int32)
    neg = fo.sample_negatives(full_ptr, full_cols, np.zeros(50, np.int64), 5, 3, seed=1)
    assert neg.shape == (50, 3) and neg.min() >= 0 and neg.max() < 5


def test_sampler_distributions(ml_small):
    """Fixed-seed chi-square bounds: uniform draws are flat over the items; popular draws follow the item counts."""
    n_items, S = 40, 200_000
    counts = np.arange(1, n_items + 1)
    table = np.repeat(np.arange(n_items, dtype=np.int32), counts)  # the item of every interaction
    indptr, cols = np.array([0, 0]), np.zeros(0, np.int32)  # the sampled user owns nothing: every draw is kept
    rows = np.zeros(S, np.int64)
    for popular, p in ((False, np.full(n_items, 1 / n_items)), (True, counts / counts.sum())):
        neg = fo.sample_negatives(indptr, cols, rows, n_items, 1, seed=5, popular=popular, batch_size=8192,
                                  coo_items=table)
        obs = np.bincount(neg[:, 0], minlength=n_items)
        chi2 = float(((obs - S * p) ** 2 / (S * p)).sum())
        assert chi2 < 80.0  # 39 degrees of freedom: the 0.9999 quantile is 77
    assert not np.array_equal(
        fo.sample_negatives(indptr, cols, rows[:100], n_items, 1, seed=5),
        fo.sample_negatives(indptr, cols, rows[:100], n_items, 1, seed=6),
    )


# ------------------------------------------------------------------------------------------------------------
# step restatement: torch autograd + torch.optim against the update formulas written out by hand in f64
# ------------------------------------------------------------------------------------------------------------


def _toy(rng, n_users=7, n_items=9, k=5, ub=True, ib=True):
    p = {"u_embed.weight": rng.normal(0, 0.1, (n_users, k)), "i_embed.weight": rng.normal(0, 0.1, (n_items, k))}
    if ub:
        p["u_bias.weight"] = rng.normal(0, 0.1, (n_users, 1))
    if ib:
        p["i_bias.weight"] = rng.normal(0, 0.1, (n_items, 1))
    return {n: v.astype(np.float64) for n, v in p.items()}


@pytest.mark.parametrize("loss", ["logistic", "pairwise"])
@pytest.mark.parametrize("reg_method", ["AdamW", "L2", None])
def test_oracle_step_is_the_documented_update(loss, reg_method):
    """The gradient by finite differences of the oracle's own loss, pushed through the optimiser formulas of
    ``include/lkpy_b200.h``, gives the oracle's step (f64)."""
    rng = np.random.default_rng(0)
    p0 = _toy(rng)
    users, pos = np.array([0, 3, 3, 6]), np.array([1, 2, 8, 1])
    neg = np.array([[4, 5], [5, 5], [0, 7], [3, 2]])
    kw = dict(loss=loss, reg_method=reg_method, regularization=0.05, positive_weight=1.5)
    lr = 0.01
    model = fo.Model(p0, sparse=reg_method != "AdamW", dtype=torch.float64)
    opt = fo.make_optimizer(model, reg_method, lr, 0.05)
    got_loss = fo.train_step(model, opt, users, pos, neg, **kw)

    def f(params):
        with torch.no_grad():
            return float(fo.batch_loss(fo.Model(params, sparse=False, dtype=torch.float64), users, pos, neg, **kw))

    assert got_loss == pytest.approx(f(p0), rel=1e-12)
    touched = {"u": set(users.tolist()), "i": set(pos.tolist()) | set(neg.flatten().tolist())}
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
            want = w * (1 - lr * 0.05) - lr / (1 - b1) * m / (np.sqrt(v) / np.sqrt(1 - b2) + eps)
        else:
            want = w - lr * np.sqrt(1 - b2) / (1 - b1) * m / (np.sqrt(v) + eps)
            rows = [r for r in range(len(w)) if r not in touched[name[0]]]
            want[rows] = w[rows]  # SparseAdam leaves rows outside the batch alone
        got = dict(model.state_dict())[name].numpy()
        assert np.allclose(got, want, rtol=0, atol=2e-4 * lr), name  # finite-difference accuracy through m / sqrt(v)


def test_l2_norm_gradient_at_zero_is_zero():
    """An all-zero embedding row gets nothing from the L2 term: its gradient is that of the loss without the term,
    while a non-zero row's gradient moves."""
    p0 = _toy(np.random.default_rng(1))
    p0["i_embed.weight"][4] = 0.0
    grads = {}
    for reg_method in ("L2", None):
        model = fo.Model(p0, sparse=False, dtype=torch.float64)
        fo.batch_loss(model, [0, 1], [4, 2], [[4], [3]], loss="logistic", reg_method=reg_method, regularization=1.0,
                      positive_weight=1.0).backward()  # fmt: skip
        grads[reg_method] = model.tables["i_embed.weight"].grad
    assert torch.equal(grads["L2"][4], grads[None][4]) and grads[None][4].abs().sum() > 0
    assert not torch.allclose(grads["L2"][2], grads[None][2])


# ------------------------------------------------------------------------------------------------------------
# initial parameters, ABI layout, no fallback
# ------------------------------------------------------------------------------------------------------------


def test_initial_parameters_follow_the_normal_sequence():
    gen = flexmf._torch_generator(1234)
    ucnt, icnt = np.array([3, 0, 2, 1]), np.array([0, 1, 1, 4, 0])
    p = flexmf.initial_parameters(4, 5, 8, True, True, gen, ucnt, icnt)
    ref = torch.Generator().manual_seed(1234)
    for name, shape, cnt in (("u_bias.weight", (4, 1), ucnt), ("i_bias.weight", (5, 1), icnt),
                             ("u_embed.weight", (4, 8), ucnt), ("i_embed.weight", (5, 8), icnt)):  # fmt: skip
        want = torch.nn.init.normal_(torch.empty(shape), std=0.1, generator=ref)
        want[torch.as_tensor(cnt == 0)] = 0
        assert torch.equal(p[name], want), name
    # without the user bias the stream moves on: the item bias takes the first draws
    q = flexmf.initial_parameters(4, 5, 8, False, True, flexmf._torch_generator(1234))
    assert "u_bias.weight" not in q
    assert torch.equal(q["i_bias.weight"], torch.nn.init.normal_(torch.empty(5, 1), std=0.1, generator=torch.Generator().manual_seed(1234)))
    # a NumPy generator seeds torch with one int32 draw, as the reference's random_generator(type="torch") does
    i32 = np.iinfo(np.int32)
    want_seed = int(np.random.default_rng(9).integers(i32.min, i32.max))
    assert flexmf._torch_generator(np.random.default_rng(9)).initial_seed() == torch.Generator().manual_seed(want_seed).initial_seed()


STRUCTS = {
    "lk_flexmf_sample_args": _lib.LkFlexmfSampleArgs,
    "lk_flexmf_groups": _lib.LkFlexmfGroups,
    "lk_flexmf_step_args": _lib.LkFlexmfStepArgs,
}


def test_ctypes_structs_match_header(tmp_path):
    expected, lines = [], []
    for cname, cls in STRUCTS.items():
        for field in cls._fields_:
            name = field[0]
            expected.append((f"{cname}.{name}", getattr(cls, name).offset))
            lines.append(f'    printf("{cname}.{name} %zu\\n", offsetof({cname}, {name}));')
        expected.append((f"sizeof {cname}", C.sizeof(cls)))
        lines.append(f'    printf("sizeof {cname} %zu\\n", sizeof({cname}));')
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "lkpy_b200.h"\n\nint main(void)\n{\n'
                   + "\n".join(lines) + "\n    return 0;\n}\n")  # fmt: skip
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert [(line.rsplit(" ", 1)[0], int(line.rsplit(" ", 1)[1])) for line in out] == expected


def test_step_validates_its_workspace_on_the_host(cuda_lib):
    need = C.c_int64()
    assert cuda_lib.lk_flexmf_workspace_bytes(8192, 1, 64, C.byref(need)) == 0 and need.value > 0
    assert cuda_lib.lk_flexmf_workspace_bytes(8192, 1, 129, C.byref(need)) == -3  # LK_ERR_UNSUPPORTED
    a = _lib.LkFlexmfStepArgs()
    a.batch, a.n_neg, a.k = 8192, 1, 64
    a.d_workspace, a.workspace_bytes = 1, need.value - 1  # never dereferenced: the size check comes first
    assert cuda_lib.lk_flexmf_step(C.byref(a), None) == -1  # LK_ERR_INVALID
    assert b"workspace" in cuda_lib.lk_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a device")
def test_no_fallback_without_a_device(ml_small):
    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        FlexMFImplicitScorer(embedding_size=8, epochs=1).train(Dataset(ml_small), TrainingOptions(rng=1))
