"""
StochasticTopNRanker without a GPU: the PCG64 restatement and the jump constants against NumPy, the derivable-RNG
restatement, the key statements of tests/stochastic_oracle.py against recordings of the reference's own class
(``tests/golden/reference_classes/stochastic_*.npz``, which ``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites from a
reference checkout through tests/stochastic_ref_sandbox.py), the configuration, and the ABI.
"""

import ctypes as C
import os
from pathlib import Path

import numpy as np
import pydantic
import pytest

import stochastic_oracle as so
import stochastic_ref_sandbox as srs
from lkpy_b200 import _lib, engine
from lkpy_b200.components import RecQuery
from lkpy_b200.stochastic import (
    DerivingRNG, FixedRNG, StochasticTopNConfig, StochasticTopNRanker, advance, derivable_rng, generator_words, make_seed,
)  # fmt: skip
from test_flexmf import test_ctypes_structs_match_header as _layout_check

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"


@pytest.mark.parametrize("seed", [0, 42, 2**40 + 17])
def test_pcg64_restatement_is_numpy(seed):
    """Step then XSL-RR of the new state is ``random_raw``; ``uniform(0, 1, N)`` is N raw draws as
    ``(raw >> 11) * 2^-53``."""
    bg = np.random.default_rng(seed).bit_generator
    st = bg.state["state"]
    out, end = so.raw(st["state"], st["inc"], 100)
    assert out == [int(x) for x in bg.random_raw(100)]
    assert end == bg.state["state"]["state"]
    g = np.random.default_rng(seed)
    u = g.uniform(0, 1, 100)
    assert np.array_equal(u, np.array([(x >> 11) * 2.0**-53 for x in out]))
    assert g.bit_generator.state == bg.state


def test_jump_constants_are_numpy_advance():
    """``engine.pcg64_jump`` (square and multiply) is the closed form of tests/stochastic_oracle.py, its table is the
    one the kernel takes, and a jump of j lands where ``bit_generator.advance(j)`` does."""
    assert np.array_equal(engine.stochastic_jump_table(), so.jump_table_words())
    assert engine.stochastic_jump_table().size == _lib.LK_STOCH_JUMP_WORDS
    for j in (0, 1, 2, 31, 32, 33, 1000, 123_456_789, 2**63 + 5):
        assert engine.pcg64_jump(j) == so.jump(j)
        bg = np.random.default_rng(j).bit_generator
        st = bg.state["state"]
        m, g = engine.pcg64_jump(j)
        bg.advance(j)
        assert (m * st["state"] + g * st["inc"]) % 2**128 == bg.state["state"]["state"]
    # raw steps: a jump of j equals j single steps
    s, inc = 12345, 0xDA3E39CB94B95BDB
    for j in range(40):
        m, g = engine.pcg64_jump(j)
        assert (m * s + g * inc) % 2**128 == so.raw(s, inc, j)[1]


def test_advance_leaves_the_state_of_the_draws():
    """``advance(gen, k)`` leaves the whole state dict that k uniforms leave, a buffered 32-bit half included."""
    for pre in (False, True):
        a, b = np.random.default_rng(3), np.random.default_rng(3)
        if pre:
            a.integers(0, 10, dtype=np.uint32), b.integers(0, 10, dtype=np.uint32)
        a.uniform(0, 1, 777)
        advance(b, 777)
        assert a.bit_generator.state == b.bit_generator.state


def test_derived_rng_restatement():
    """Per-query generators: (seed, "user") hashes string ids with md5 and appends int ids to the base entropy; a
    query without a user id spawns from the base sequence, in call order; a seed gives one shared generator."""
    f = derivable_rng((7, "user"))
    assert isinstance(f, DerivingRNG) and f.seed.entropy == [7]
    g = f(RecQuery(12))
    assert g.bit_generator.state == np.random.default_rng(np.random.SeedSequence([7, 12])).bit_generator.state
    digest = np.frombuffer(__import__("hashlib").md5(b"alice").digest(), np.int32)
    h = abs(int(digest[0] ^ digest[1] ^ digest[2] ^ digest[3]))
    assert make_seed(f.seed, "alice").entropy == [7, h]
    s1, s2 = f(RecQuery(None)), f(None)
    base = np.random.SeedSequence([7])
    assert s1.bit_generator.state == np.random.default_rng(base.spawn(1)[0]).bit_generator.state
    assert s2.bit_generator.state == np.random.default_rng(base.spawn(1)[0]).bit_generator.state
    fx = derivable_rng(5)
    assert isinstance(fx, FixedRNG) and fx(None) is fx(RecQuery(3))
    assert isinstance(derivable_rng("user"), DerivingRNG) and isinstance(derivable_rng(None), FixedRNG)
    with pytest.raises(ValueError):
        derivable_rng((1, "item"))
    w = generator_words(np.random.default_rng(1))
    st = np.random.default_rng(1).bit_generator.state["state"]
    assert w == [st["state"] >> 64, st["state"] % 2**64, st["inc"] >> 64, st["inc"] % 2**64]
    with pytest.raises(TypeError, match="PCG64"):
        generator_words(np.random.Generator(np.random.MT19937(1)))


def test_config_defaults_and_validation():
    c = StochasticTopNConfig()
    assert (c.n, c.rng, c.transform, c.scale) == (None, None, "softmax", 1.0)
    assert StochasticTopNConfig(rng=(3, "user")).rng == (3, "user")
    assert StochasticTopNConfig(rng="user").rng == "user" and StochasticTopNConfig(rng=[1, 2]).rng == [1, 2]
    assert StochasticTopNConfig(transform=None).transform is None
    for bad in ({"transform": "exp"}, {"rng": (3, "item")}, {"rng": "item"}, {"count": 3}, {"scale": "big"}):
        with pytest.raises(pydantic.ValidationError):
            StochasticTopNConfig(**bad)
    r = StochasticTopNRanker(n=5, rng=1, transform="linear", scale=2.0)
    assert r.config.n == 5 and isinstance(r._rng_factory, FixedRNG)
    assert r._n(None) == 5 and r._n(-3) == 5 and r._n(0) == 0 and r._n(7) == 7
    assert StochasticTopNRanker(n=0)._n(None) is None and StochasticTopNRanker()._n(-1) is None


def test_oracle_argtopn_is_the_heap():
    """The f64 heap replay against ``oracle.argtopn`` (the C restatement of argtopn) on f32-exact values with ties,
    NaN and every cut."""
    import oracle

    rng = np.random.default_rng(0)
    v = (np.round(rng.standard_normal(500) * 3) / 3).astype(np.float32)
    v[rng.random(500) < 0.1] = np.nan
    for n in (0, 1, 2, 7, 100, 449, 500, 600):
        assert np.array_equal(so.argtopn(v.astype(np.float64), n), oracle.argtopn(v, n))


def test_ctypes_structs_match_header(tmp_path, monkeypatch):
    import test_flexmf

    monkeypatch.setattr(test_flexmf, "STRUCTS", {"lk_stochastic_args": _lib.LkStochasticArgs})
    _layout_check(tmp_path)


def test_entry_point_checks_arguments_on_the_host(cuda_lib):
    a = _lib.LkStochasticArgs()
    a.n_queries, a.n_items, a.n = 2, 10, 1025
    assert cuda_lib.lk_stochastic_topn(C.byref(a), None) == -3  # n beyond lk_topn_max(): LK_ERR_UNSUPPORTED
    a.n = -1
    assert cuda_lib.lk_stochastic_topn(C.byref(a), None) == -1
    a.n, a.transform = 5, 7
    assert cuda_lib.lk_stochastic_topn(C.byref(a), None) == -1 and b"transform" in cuda_lib.lk_last_error()
    a.transform = _lib.LK_STOCH_SOFTMAX
    assert cuda_lib.lk_stochastic_topn(C.byref(a), None) == -1 and b"null" in cuda_lib.lk_last_error()
    a.n_items = 2**31 - 1
    assert cuda_lib.lk_stochastic_topn(C.byref(a), None) == -3  # positions must fit in int32
    # never dereferenced: every check comes before a launch
    a.n_items, a.d_scores, a.d_state, a.d_jump, a.d_workspace, a.d_out_cnt = 10, 8, 8, 8, 8, 8
    a.d_out_idx, a.d_out_val, a.shared_stream = 8, 8, 1
    assert cuda_lib.lk_stochastic_topn(C.byref(a), None) == -1 and b"d_position" in cuda_lib.lk_last_error()
    a.d_position, a.workspace_bytes = 8, 10
    assert cuda_lib.lk_stochastic_topn(C.byref(a), None) == -1 and b"workspace" in cuda_lib.lk_last_error()
    assert cuda_lib.lk_stochastic_workspace_bytes(3, 10, _lib.LK_STOCH_SOFTMAX) == 20 * 4 + 4 * 3 * 10
    assert cuda_lib.lk_stochastic_workspace_bytes(3, 10, _lib.LK_STOCH_NONE) == 20 * 4
    z = _lib.LkStochasticArgs()
    assert cuda_lib.lk_stochastic_topn(C.byref(z), None) == 0  # an empty batch does nothing


def test_ranker_checks_before_the_device():
    from lkpy_b200.components import ItemList

    r = StochasticTopNRanker(rng=1)
    with pytest.raises(ValueError, match="scores"):
        r.rank_batch([ItemList(item_ids=[1, 2])])
    with pytest.raises(ValueError, match="exclude"):
        r.rank_scores(None, [], None, exclude="history")


# ---------------------------------------------------------------------------
# the host statements against the reference class
# ---------------------------------------------------------------------------


_recorded: list[bool] = []


def reference_golden(name: str) -> dict:
    """The reference's recording ``name`` (stochastic_ref_sandbox.record): recorded live when asked to, else read."""
    if RECORD and not _recorded:
        import ref_sandbox

        assert ref_sandbox.available(), "recording needs the reference checkout"
        for n, d in srs.record().items():
            np.savez_compressed(GOLD / f"{n}.npz", **d)
        _recorded.append(True)
    with np.load(GOLD / f"{name}.npz") as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", list(srs.CASES))
def test_host_statements_are_the_reference(name):
    """The key statements of tests/stochastic_oracle.py, with this package's derivable RNG, reproduce the reference
    class's calls: the same items in the same order, keys within 2 ulps (1e-6 relative where NumPy's f32 exp, which
    depends on the CPU's SIMD level, is involved), and a fixed generator's final state exactly."""
    g = reference_golden(name)
    cfg = srs.CASES[name]
    f = derivable_rng(cfg["rng"])
    cfg_n = cfg.get("n")
    for c in range(len(g["lens"])):
        s = g["scores"][c, : g["lens"][c]]
        kind, uid = int(g["user_kind"][c]), str(g["users"][c])
        user = None if kind == 0 else (int(uid) if kind == 1 else uid)
        n = None if g["n"][c] == srs.NONE_N else int(g["n"][c])
        if n is None or n < 0:
            n = cfg_n or -1
        pos, keys = so.rank(s, None if n < 0 else n, cfg["transform"], cfg.get("scale", 1.0), f(RecQuery(user)))
        lo, hi = g["ptr"][c], g["ptr"][c + 1]
        assert np.array_equal(pos, g["pos"][lo:hi]), (name, c)
        if g["weights"][c]:
            if cfg["transform"] == "softmax":
                assert np.allclose(keys, g["keys"][lo:hi], rtol=1e-6, atol=0)
            else:
                assert (np.abs(keys.view(np.int64) - g["keys"][lo:hi].view(np.int64)) <= 2).all()
    if "state" in g:
        st = f(None).bit_generator.state["state"]
        assert engine.pcg64_words(st["state"], st["inc"]) == [int(x) for x in g["state"]]
