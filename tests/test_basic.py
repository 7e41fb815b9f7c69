"""
BiasScorer and PopScorer without a GPU: configurations, the pairwise-mean restatement of ``lk_bias_learn`` against
NumPy, the ctypes layouts, host-side argument checks, and the host statements against the recordings of the
reference's own classes on ml-latest-small (``tests/golden/reference_classes/basic_*.npz``, which
``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites from a reference checkout through tests/basic_ref_sandbox.py).
"""

import ctypes as C
import os
from pathlib import Path

import numpy as np
import pandas as pd
import pydantic
import pytest
import torch

import basic_oracle as bo
import basic_ref_sandbox as brs
import ref_sandbox
from lkpy_b200 import _lib
from lkpy_b200.basic import BiasConfig, BiasModel, BiasScorer, PopConfig, PopScorer, damping_pair
from lkpy_b200.components import Dataset, ItemList, RecQuery
from test_flexmf import test_ctypes_structs_match_header as _layout_check

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"


_recorded: list[bool] = []


def reference_golden(name: str, ml_small) -> dict:
    """The reference's recording ``name`` (basic_ref_sandbox.record): recorded live when asked to, else read."""
    if RECORD and not _recorded:
        assert ref_sandbox.available(), "recording needs the reference checkout"
        for n, d in brs.record(ml_small).items():
            np.savez_compressed(GOLD / f"{n}.npz", **d)
        _recorded.append(True)
    with np.load(GOLD / f"{name}.npz") as z:
        return {k: z[k] for k in z.files}


def test_config_defaults_and_validation():
    c = BiasConfig()
    assert c.entities == {"user", "item"} and c.damping == 0.0
    assert c.model_dump() == {"entities": ["item", "user"], "damping": 0.0}
    assert BiasConfig(damping={"user": 2.0}).entity_damping("item") == 0.0
    assert BiasConfig(damping=5).entity_damping("user") == 5.0
    for bad in ({"damping": -1.0}, {"damping": {"user": -1.0}}, {"entities": {"group"}}, {"dampening": 1.0}):
        with pytest.raises(pydantic.ValidationError):
            BiasConfig(**bad)
    assert PopConfig().score == "quantile"
    with pytest.raises(pydantic.ValidationError):
        PopConfig(score="mean")
    assert BiasScorer(damping=2.5).config.damping == 2.5 and PopScorer(score="rank").config.score == "rank"
    assert not BiasScorer().is_trained() and not PopScorer().is_trained()


def test_damping_forms():
    assert damping_pair(0.5) == (0.5, 0.5)
    assert damping_pair((1.0, 2.0)) == (1.0, 2.0)
    assert damping_pair({"item": 3.0}) == (0.0, 3.0)
    with pytest.raises(ValueError):
        damping_pair((-1.0, 0.0))


@pytest.mark.parametrize("n", [1, 8, 9, 128, 129, 1000, 2**20 + 3])
def test_pairwise_mean_restatement_is_numpy(n):
    """``lk_bias_learn``'s evaluation of the mean — the pairwise tree cut into subtrees and recombined — against
    ``np.mean`` of the same f32 array, bit for bit."""
    rng = np.random.default_rng(n)
    a = (rng.integers(1, 11, n) * 0.5).astype(np.float32) + rng.standard_normal(n).astype(np.float32)
    assert bo.kernel_mean(a).view(np.int32) == np.mean(a).view(np.int32)
    assert bo.kernel_mean(a).view(np.int32) == np.float32(np.float64(bo.pairwise(a)) / n).view(np.int32)


def test_ctypes_structs_match_header(tmp_path, monkeypatch):
    import test_flexmf

    monkeypatch.setattr(test_flexmf, "STRUCTS", {
        "lk_bias_learn_args": _lib.LkBiasLearnArgs, "lk_offset_score_args": _lib.LkOffsetScoreArgs,
    })  # fmt: skip
    _layout_check(tmp_path)


def test_entry_points_check_arguments_on_the_host(cuda_lib):
    a = _lib.LkBiasLearnArgs()
    assert cuda_lib.lk_bias_learn(C.byref(a), None) == -3  # nnz = 0: LK_ERR_UNSUPPORTED
    a.nnz, a.n_users, a.n_items = 10, 2, 2
    assert cuda_lib.lk_bias_learn(C.byref(a), None) == -1  # null ratings
    a.d_ratings, a.d_workspace, a.d_mean, a.damping_item = 8, 8, 8, -1.0  # never dereferenced: checks come first
    assert cuda_lib.lk_bias_learn(C.byref(a), None) == -1 and b"damping" in cuda_lib.lk_last_error()
    a.damping_item, a.d_item_bias = 0.0, 8
    assert cuda_lib.lk_bias_learn(C.byref(a), None) == -1 and b"item pass" in cuda_lib.lk_last_error()
    assert cuda_lib.lk_bias_learn_workspace_bytes() > 0
    o = _lib.LkOffsetScoreArgs()
    o.n_items, o.n_queries, o.n = 5, 1, 1025
    assert cuda_lib.lk_offset_score_batch(C.byref(o), None) == -3
    o.n, o.d_base = 3, 8
    assert cuda_lib.lk_offset_score_batch(C.byref(o), None) == -1  # no outputs
    o.n_items = 0
    assert cuda_lib.lk_offset_score_batch(C.byref(o), None) == -1


def test_scorers_check_arguments_before_the_device(ml_small):
    from lkpy_b200 import basic

    with pytest.raises(ValueError, match="entities"):
        basic.learn(Dataset(ml_small), 0.0, entities={"group"})
    with pytest.raises(ValueError, match="centered_dtype"):
        basic.learn(Dataset(ml_small), 0.0, centered_dtype=np.float16)
    with pytest.raises(ValueError, match="exclude"):
        BiasScorer().recommend_batch([1], 10, exclude="history")


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a device")
def test_no_fallback_without_a_device(ml_small):
    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        BiasScorer().train(Dataset(ml_small))
    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        PopScorer().train(Dataset(ml_small))


# ---------------------------------------------------------------------------
# the host statements against the reference classes
# ---------------------------------------------------------------------------


def our_queries(ml_small, vocab_items):
    out = []
    for uid, hist, ratings in brs.queries(ml_small):
        h = None
        if hist is not None:
            h = ItemList(item_ids=hist, **({} if ratings is None else {"rating": ratings}))
        out.append(RecQuery(uid, h))
    return out


@pytest.mark.parametrize("name", list(brs.BIAS_CONFIGS))
def test_host_bias_statements_are_the_reference(ml_small, name):
    """``basic.BiasModel.learn`` (the oracle of ``lk_bias_learn``) on the f32 ratings and ``compute_for_items``'
    statements reproduce the reference BiasScorer's model and scores bit for bit."""
    g = reference_golden(f"basic_bias_{name}", ml_small)
    cfg = BiasConfig(**brs.BIAS_CONFIGS[name])
    m = BiasModel.learn(ml_small, damping_pair(cfg.damping), np.float32, cfg.entities)
    assert m.global_bias == float(g["global_bias"])
    for ours, key, has in ((m.item_biases, "item_biases", "has_items"), (m.user_biases, "user_biases", "has_users")):
        assert (ours is not None) == bool(g[has])
        if ours is not None:
            assert np.array_equal(ours.view(np.int32), g[key].view(np.int32))
    ds = Dataset(ml_small)
    targets = ItemList(item_ids=brs.score_item_ids(ml_small))
    for q, want in zip(our_queries(ml_small, ds.items), g["scores"]):
        got = bo.bias_scores(m, ds.users, ds.items, q, targets)
        assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_user_bias_for_items_is_compute_for_items(ml_small):
    """``BiasModel.user_bias_for_items`` against ``compute_for_items``' statements, in the ratings' dtype: unknown
    items, NaN ratings, an all-NaN query, infinite ratings (an infinite bias stays infinite, as in the reference), and a
    model without item biases."""
    ds = Dataset(ml_small)
    ids = ds.items.ids()
    cases = [([ids[0], ids[5], -7], [4.0, 3.5, 2.0]), ([ids[1], ids[2], ids[3]], [np.nan, 5.0, 1.0]),
             ([ids[1], ids[2]], [np.nan, np.nan]), ([ids[4], ids[9]], [np.inf, 3.0]),
             ([ids[4], ids[9]], [-np.inf, 3.0]), ([ids[4], ids[9]], [np.inf, -np.inf])]  # fmt: skip
    for entities in (("user", "item"), ("user",)):
        m = BiasModel.learn(ml_small, (2.5, 1.0), np.float32, entities)
        for item_ids, ratings in cases:
            for dtype in (np.float32, np.float64):
                q = ItemList(item_ids=item_ids, rating=np.array(ratings, dtype=dtype))
                got = m.user_bias_for_items(q.numbers(vocabulary=ds.items, missing="negative"), q.field("rating"))
                want = bo.rated_user_bias(m, ds.items, q)
                assert np.float64(got).view(np.int64) == np.float64(want).view(np.int64), (entities, ratings, dtype)
        q = ItemList(item_ids=[ids[4], ids[9]], rating=[np.inf, 3.0])
        assert m.user_bias_for_items(q.numbers(vocabulary=ds.items), q.field("rating")) == np.inf
        q = ItemList(item_ids=[ids[1], ids[2]], rating=[np.nan, np.nan])
        assert m.user_bias_for_items(q.numbers(vocabulary=ds.items), q.field("rating")) == 0.0


@pytest.mark.parametrize("mode", brs.POP_SCORES)
def test_host_pop_statements_are_the_reference(ml_small, mode):
    """PopScorer's pandas statements on the item counts, and its ``__call__``, against the reference class.
    Quantiles of tied counts depend on the order an unstable sort leaves the ties in, which may differ between
    CPUs: they are compared as sorted groups of equal counts."""
    g = reference_golden(f"basic_pop_{mode}", ml_small)
    ds = Dataset(ml_small)
    counts = np.bincount(ml_small.items, minlength=ml_small.n_items).astype(np.int64)
    m = PopScorer(score=mode)
    ours = np.require(m._train_internal(pd.Series(counts, index=ds.items.ids())).values, np.float32)
    want = g["item_scores"]
    if mode == "quantile":
        for c in np.unique(counts):
            at = counts == c
            assert np.array_equal(np.sort(ours[at]), np.sort(want[at]))
    else:
        assert np.array_equal(ours.view(np.int32), want.view(np.int32))
    m.items, m.item_scores = ds.items, want
    got = m(ItemList(item_ids=brs.score_item_ids(ml_small))).scores()
    assert np.array_equal(got, g["scores"], equal_nan=True) and np.isnan(got[-1])
