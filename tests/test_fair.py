"""
FAIRReranker without a GPU: the training and merge restatements of lkpy_b200/reranking.py against recordings of the
reference's own class (``tests/golden/reference_classes/fair_*.npz``, which ``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites
from a reference checkout through tests/fair_ref_sandbox.py), the configuration and its ``n`` rules, the ABI, and the
argument checks made before the device.
"""

import ctypes as C
import logging
import os
import pickle
from pathlib import Path

import numpy as np
import pydantic
import pytest
import torch

import fair_ref_sandbox as frs
from lkpy_b200 import _lib
from lkpy_b200.components import Dataset, ItemList, Vocabulary
from lkpy_b200.reranking import (
    FAIRReranker, FAIRRerankerConfig, adjusted_significance, fair_merge, minimum_protected,
)  # fmt: skip
from test_flexmf import test_ctypes_structs_match_header as _layout_check

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"

_recorded: list[bool] = []


def reference_golden(name: str) -> dict:
    """The reference's recording ``name`` (fair_ref_sandbox.record): recorded live when asked to, else read."""
    if RECORD and not _recorded:
        import ref_sandbox

        assert ref_sandbox.available(), "recording needs the reference checkout"
        for n, d in frs.record().items():
            np.savez_compressed(GOLD / f"{n}.npz", **d)
        _recorded.append(True)
    with np.load(GOLD / f"{name}.npz") as z:
        return {k: z[k] for k in z.files}


def dataset(ids, flags, name: str = "protected") -> Dataset:
    """This package's ``Dataset`` over the items ``ids`` with the per-item attribute ``name``."""
    return Dataset(None, users=Vocabulary(np.zeros(0, np.int64), "user"), items=Vocabulary(ids, "item"),
                   item_attributes={name: np.asarray(flags)})  # fmt: skip


def trained(cfg: dict, ids, flags) -> FAIRReranker:
    r = FAIRReranker(**cfg)
    r.train(dataset(ids, flags, cfg.get("protected_attribute", "protected")))
    return r


def test_thresholds_are_the_reference():
    """``alpha_c`` to the bit and ``m_list`` exactly for every recorded ``(n, p, alpha)``, including n = 1, n = 1000
    and configurations whose m_list is all zero."""
    g = reference_golden("fair_thresholds")
    assert any(g["m_list"][g["m_ptr"][k] : g["m_ptr"][k + 1]].max() == 0 for k in range(len(g["n"])))
    for k in range(len(g["n"])):
        n, p, alpha = int(g["n"][k]), float(g["p"][k]), float(g["alpha"][k])
        ac = adjusted_significance(n, p, alpha)
        assert ac == g["alpha_c"][k], (n, p, alpha)
        assert np.array_equal(minimum_protected(n, p, ac), g["m_list"][g["m_ptr"][k] : g["m_ptr"][k + 1]])


@pytest.mark.parametrize("name", list(frs.CASES))
def test_calls_are_the_reference(name):
    """Training on this package's ``Dataset`` and every recorded call: the same ``alpha_c`` and ``m_list`` and the same
    ids in the same order, with unknown items, lists with no or only protected items, short lists, runtime ``n`` of
    None, 0, 1, below and equal to the config's, and protected items deep in the list."""
    g = reference_golden(name)
    cfg = frs.CASES[name]
    assert np.array_equal(g["vocab"], frs.vocabulary(name)[0])
    r = trained(cfg, g["vocab"], g["protected"])
    assert r.alpha_c == float(g["alpha_c"]) and np.array_equal(r.m_list, g["m_list"])
    for c in range(len(g["n"])):
        items = g["lists"][g["list_ptr"][c] : g["list_ptr"][c + 1]]
        n = None if g["n"][c] == frs.NONE_N else int(g["n"][c])
        got = r(ItemList(item_ids=items, ordered=True), n)
        assert np.array_equal(got.ids(), g["out"][g["out_ptr"][c] : g["out_ptr"][c + 1]]), (name, c)
        assert got.ordered


def test_published_thresholds_and_expected_output():
    """Table 2 of Zehlike et al. (2017) at (10, 0.5, 0.1), and the reference test's exact output for a list whose last
    item has no attribute."""
    m = minimum_protected(10, 0.5, 0.1)
    assert (m[3], m[6], m[8], len(m)) == (1, 2, 3, 10)
    items = np.array([1, 2, 3, 4, 5, 31, 32, 33, 34, 35])
    prot = [False, False, False, False, False, False, True, False, True]
    r = trained({"n": 10}, items[:-1], prot)
    got = r(ItemList(item_ids=items, ordered=True))
    assert np.array_equal(got.ids(), [1, 2, 3, 32, 4, 5, 34, 31, 33, 35])


def test_merge_meets_the_thresholds():
    """Every prefix of a merged list holds at least m_list protected items whenever the list has them."""
    rng = np.random.default_rng(4)
    m = minimum_protected(60, 0.6, adjusted_significance(60, 0.6, 0.1))
    for _ in range(50):
        flags = rng.random(int(rng.integers(60, 200))) < rng.uniform(0.2, 0.9)
        pos = fair_merge(flags, m, 60)
        assert len(np.unique(pos)) == 60
        counts = np.cumsum(flags[pos])
        assert np.all((counts >= m) | (counts == flags.sum()))


def test_fields_and_n_rules(caplog):
    rng = np.random.default_rng(1)
    ids = np.arange(30) + 7
    r = trained({"n": 8, "p": 0.6}, ids, rng.random(30) < 0.3)
    it = ItemList(item_ids=ids[::-1], scores=np.linspace(1, 0, 30, dtype=np.float32), rating=np.arange(30))
    got = r(it)
    pos = fair_merge(r._flags(it), r.m_list, 8)
    assert np.array_equal(got.ids(), it.ids()[pos]) and np.array_equal(got.field("rating"), pos)
    assert np.array_equal(got.scores(), it.scores()[pos])
    with pytest.raises(ValueError, match="exceeds configured n=8"):
        r(it, 9)
    with caplog.at_level(logging.WARNING, logger="lkpy_b200.reranking"):
        assert len(r(it, 5)) == 5
    assert "trained for n=8 used on n=5" in caplog.text
    caplog.clear()
    with caplog.at_level(logging.WARNING, logger="lkpy_b200.reranking"):
        assert np.array_equal(r(it, 0).ids(), got.ids()) and np.array_equal(r(it, 8).ids(), got.ids())
    assert len(r(ItemList(item_ids=ids[:3]))) == 3 and len(r(ItemList(item_ids=ids[:0]))) == 0


def test_train_inputs():
    """The flags are ``attribute == True``; a missing attribute raises, as does one of the wrong length; a LensKit
    ``Dataset`` is read through ``entities("item")``."""
    ids = np.arange(5)
    r = trained({"n": 3}, ids, np.array([True, None, 1, "yes", False], dtype=object))
    assert r.protected_attributes.tolist() == [True, False, True, False, False]
    with pytest.raises(ValueError, match="missing required 'flag'"):
        FAIRReranker(n=3, protected_attribute="flag").train(dataset(ids, [True] * 5))
    with pytest.raises(ValueError, match="values for"):
        FAIRReranker(n=3).train(dataset(ids, [True] * 4))

    class Ent:
        attributes = ["protected"]
        vocabulary = Vocabulary(ids, "item")

        def attribute(self, name):
            return type("A", (), {"numpy": lambda _s: np.array([0, 1, 1, 0, 1], bool)})()

    r = FAIRReranker(n=3)
    r.train(type("DS", (), {"entities": lambda _s, kind: Ent()})())
    assert r.protected_attributes.tolist() == [False, True, True, False, True] and r.is_trained()


def test_config_defaults_and_validation():
    c = FAIRRerankerConfig(n=5)
    assert (c.n, c.p, c.alpha, c.protected_attribute) == (5, 0.5, 0.1, "protected")
    for bad in ({}, {"n": 0}, {"n": -2}, {"n": 5, "p": 0.0}, {"n": 5, "p": 1.0}, {"n": 5, "alpha": 0.0},
                {"n": 5, "alpha": 1.5}, {"n": 5, "count": 3}):  # fmt: skip
        with pytest.raises(pydantic.ValidationError):
            FAIRRerankerConfig(**bad)
    assert FAIRReranker(n=4, alpha=0.2).config.alpha == 0.2 and not FAIRReranker(n=4).is_trained()


def test_pickle_keeps_the_model():
    ids = np.arange(20) * 2
    r = trained({"n": 6, "p": 0.4}, ids, np.arange(20) % 3 == 0)
    r2 = pickle.loads(pickle.dumps(r))
    assert r2.alpha_c == r.alpha_c and np.array_equal(r2.m_list, r.m_list) and r2.vocab == r.vocab
    assert np.array_equal(r2.protected_attributes, r.protected_attributes)
    it = ItemList(item_ids=ids[::-1])
    assert np.array_equal(r2(it).ids(), r(it).ids())


def test_item_list_ordered_flag():
    """The shim's ``ordered``: False by default, kept by a copy unless given."""
    a = ItemList(item_ids=[1, 2])
    assert a.ordered is False and ItemList(item_ids=[1], ordered=True).ordered is True
    b = ItemList(ItemList(item_ids=[1], ordered=True))
    assert b.ordered is True and ItemList(b, ordered=False).ordered is False


def test_ctypes_structs_match_header(tmp_path, monkeypatch):
    import test_flexmf

    monkeypatch.setattr(test_flexmf, "STRUCTS", {"lk_fair_args": _lib.LkFairArgs})
    _layout_check(tmp_path)


def test_entry_point_checks_arguments_on_the_host(cuda_lib):
    a = _lib.LkFairArgs()
    a.mode, a.n_queries, a.n = 7, 2, 5
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -1 and b"mode" in cuda_lib.lk_last_error()
    a.mode, a.n = _lib.LK_FAIR_LISTS, 1025
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -3  # beyond lk_topn_max(): LK_ERR_UNSUPPORTED
    a.n = 0
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -1
    a.n = 5
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -1 and b"null" in cuda_lib.lk_last_error()
    # never dereferenced: every check comes before a launch
    a.d_m, a.d_out_idx, a.d_out_cnt = 8, 8, 8
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -1 and b"list" in cuda_lib.lk_last_error()
    a.mode, a.n_candidates = _lib.LK_FAIR_SCORES, 0
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -1 and b"n_candidates" in cuda_lib.lk_last_error()
    a.n_candidates = 1025
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -3
    a.n_candidates, a.n_items = 100, 2**31 - 1
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -3  # item numbers must fit in int32
    a.n_items, a.d_scores, a.d_item_protected, a.d_excl_indptr = 10, 8, 8, 8
    assert cuda_lib.lk_fair_rerank(C.byref(a), None) == -1 and b"d_excl_items" in cuda_lib.lk_last_error()
    z = _lib.LkFairArgs()
    z.n = 1
    assert cuda_lib.lk_fair_rerank(C.byref(z), None) == 0  # an empty batch does nothing


def test_reranker_checks_before_the_device(cuda_lib):
    ids = np.arange(3000)
    r = trained({"n": 2000}, ids, ids % 2 == 0)
    with pytest.raises(ValueError, match="engine limit"):
        r.rerank_batch([ItemList(item_ids=ids[:1500])])
    with pytest.raises(ValueError, match="exceeds configured"):
        r.rerank_batch([ItemList(item_ids=ids[:10])], 2001)
    vocab, S = Vocabulary(ids, "item"), torch.zeros((2, 3000))
    with pytest.raises(ValueError, match="exclude"):
        r.rank_scores(S, [None, None], vocab, candidates=10, exclude="history")
    for bad in (0, 1025):
        with pytest.raises(ValueError, match="candidates"):
            r.rank_scores(S, [None, None], vocab, candidates=bad)
    with pytest.raises(ValueError, match="scores must be"):
        r.rank_scores(S, [None], vocab, candidates=10)
    with pytest.raises(ValueError, match="exceeds configured"):
        r.rank_scores(S, [None, None], vocab, 2001, candidates=10)
    # nothing to merge: no launch
    assert [len(x) for x in r.rerank_batch([ItemList(item_ids=ids[:0])] * 2)] == [0, 0]
