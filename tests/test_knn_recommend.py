"""
CPU tests of batched kNN recommendation (``lk_knn_recommend_batch``): the ctypes mirror of its argument
struct, and the facts about ``argtopn`` the ranking mode of the dense scoring kernel relies on, pinned with the
oracle's restatement of the reference heap (``oracle.argtopn``).
"""

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle
from lkpy_b200 import _lib
from lkpy_b200.components import ItemList
from lkpy_b200.data import InteractionCSR
from lkpy_b200.knn import ItemKNNScorer
from lkpy_b200.knn_user import UserKNNScorer

ROOT = Path(__file__).resolve().parent.parent


def test_rank_args_layout_matches_header(tmp_path):
    cls, cname = _lib.LkKnnRankArgs, "lk_knn_rank_args"
    expected = [(f"{cname}.{f[0]}", getattr(cls, f[0]).offset) for f in cls._fields_] + [(f"sizeof {cname}", C.sizeof(cls))]
    lines = [f'    printf("{cname}.{f[0]} %zu\\n", offsetof({cname}, {f[0]}));' for f in cls._fields_]
    lines.append(f'    printf("sizeof {cname} %zu\\n", sizeof({cname}));')
    src = tmp_path / "rank_layout.c"
    src.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "lkpy_b200.h"\n\nint main(void)\n{\n'
        + "\n".join(lines)
        + "\n    return 0;\n}\n"
    )
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "rank_layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert [(ln.rsplit(" ", 1)[0], int(ln.rsplit(" ", 1)[1])) for ln in out] == expected


def test_exclusion_is_a_nan_offer():
    """Fact 1: argtopn over the candidate list (excluded items taken out, positions mapped back to items) equals
    argtopn over every item with the excluded items' scores set to NaN — the heap returns on a NaN offer before
    it touches anything, and the candidates keep their relative order."""
    rng = np.random.default_rng(5)
    for trial in range(300):
        n_items = int(rng.integers(1, 400))
        scores = rng.integers(0, 6, n_items).astype(np.float32)  # few values: large tie groups
        scores[rng.random(n_items) < 0.2] = np.nan  # untouched / below min_nbrs
        excl = rng.choice(n_items, int(rng.integers(0, n_items + 1)), replace=True)  # repeats allowed
        n = int(rng.integers(1, n_items + 5))
        cands = np.setdiff1d(np.arange(n_items), excl)
        want = cands[oracle.argtopn(scores[cands], n)]
        masked = scores.copy()
        masked[excl] = np.nan
        got = oracle.argtopn(masked, n)
        assert np.array_equal(got, want), trial


def test_offer_order_is_item_order():
    """Fact 2: the order of the offers decides the order of equal scores, so the kernel cannot offer in the
    touched list's (atomic arrival) order."""
    scores = np.float32([5, 5, 5, 4])
    assert oracle.argtopn(scores, 3).tolist() == [1, 2, 0]
    arrival = np.array([2, 0, 3, 1])  # the same items offered in another order
    assert arrival[oracle.argtopn(scores[arrival], 3)].tolist() == [0, 2, 1]


def test_no_threshold_prefilter():
    """Fact 3: dropping candidates below the n-th score before the heap sees them changes the tie order; only
    the full heap's own root is an exact filter."""
    scores = np.float32([1, 5, 5, 5])
    assert oracle.argtopn(scores, 2).tolist() == [1, 2]
    fives = np.flatnonzero(scores == 5)
    assert fives[oracle.argtopn(scores[fives], 2)].tolist() == [2, 1]


def test_root_filter_is_exact():
    """Fact 3, the allowed filter: once the heap is full, offering only the candidates strictly above the root
    the heap had at the start of a chunk (what the kernel's chunked walk does) gives argtopn's result."""
    rng = np.random.default_rng(9)
    for trial in range(200):
        n_items = int(rng.integers(1, 3000))
        scores = rng.integers(0, 8, n_items).astype(np.float32)
        scores[rng.random(n_items) < 0.3] = np.nan
        n = int(rng.integers(1, 64))
        chunk = int(rng.choice([1, 7, 64, 2048]))
        heap_vals: list[float] = []  # only the multiset matters for the root: the n largest offered so far
        kept = []
        for c0 in range(0, n_items, chunk):
            root = min(heap_vals) if len(heap_vals) == n else None
            for i in range(c0, min(c0 + chunk, n_items)):
                s = scores[i]
                if s != s or (root is not None and not s > root):
                    continue
                kept.append(i)
            heap_vals = sorted(heap_vals + [float(scores[i]) for i in kept if i >= c0], reverse=True)[:n]
        masked = np.full(n_items, np.nan, np.float32)
        masked[kept] = scores[kept]
        assert np.array_equal(oracle.argtopn(masked, n), oracle.argtopn(scores, n)), trial


def test_no_fallback_without_device():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    from lkpy_b200.components import Vocabulary

    items = Vocabulary(np.arange(4), "item")
    m = ItemKNNScorer()
    m.sim_matrix = InteractionCSR(np.zeros(5, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32), (4, 4))
    m.items, m.item_means = items, np.zeros(4, np.float32)
    q = ItemList(item_nums=np.int32([1]), vocabulary=items, rating=np.float32([4.0]))
    with pytest.raises(_lib.EngineError):  # nothing is computed on the host
        m.recommend_batch([q], 2)
    u = UserKNNScorer()
    u.user_ratings = InteractionCSR(np.zeros(3, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32), (2, 4))
    u.items = items
    with pytest.raises(_lib.EngineError):
        u.recommend_batch([q], 2)
