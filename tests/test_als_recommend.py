"""
CPU tests of batched ALS scoring and recommendation (``lk_als_recommend_batch``): the ctypes mirror of its
argument struct, the host restatement of the kernel's FMA chain (``als_oracle.als_scores``, checked against the
C library's ``fmaf``), the exclusion fact the rank mode relies on, and the component's argument checks.
"""

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
from als_oracle import als_scores, fmaf

import oracle
from lkpy_b200 import _lib
from lkpy_b200.als import ImplicitMFScorer
from lkpy_b200.components import ItemList, Vocabulary

ROOT = Path(__file__).resolve().parent.parent


def test_rec_args_layout_matches_header(tmp_path):
    cls, cname = _lib.LkAlsRecArgs, "lk_als_rec_args"
    expected = [(f"{cname}.{f[0]}", getattr(cls, f[0]).offset) for f in cls._fields_] + [(f"sizeof {cname}", C.sizeof(cls))]
    lines = [f'    printf("{cname}.{f[0]} %zu\\n", offsetof({cname}, {f[0]}));' for f in cls._fields_]
    lines.append(f'    printf("sizeof {cname} %zu\\n", sizeof({cname}));')
    src = tmp_path / "rec_layout.c"
    src.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "lkpy_b200.h"\n\nint main(void)\n{\n'
        + "\n".join(lines)
        + "\n    return 0;\n}\n"
    )
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "rec_layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert [(ln.rsplit(" ", 1)[0], int(ln.rsplit(" ", 1)[1])) for ln in out] == expected


@pytest.mark.parametrize("k", [1, 8, 33, 64, 128])
def test_oracle_scores_match_f64_product(k):
    rng = np.random.default_rng(k)
    Q = rng.standard_normal((300, k)).astype(np.float32)
    X = rng.standard_normal((17, k)).astype(np.float32)
    io = rng.standard_normal(300).astype(np.float32)
    qo = rng.standard_normal(17).astype(np.float32)
    exact = Q.astype(np.float64) @ X.T.astype(np.float64)
    # each FMA rounds once: |error| <= k * eps * sum |q_d x_d|, plus one rounding per offset add
    mag = np.abs(Q.astype(np.float64)) @ np.abs(X.T.astype(np.float64))
    eps = np.finfo(np.float32).eps
    S = als_scores(Q, X)
    assert S.dtype == np.float32 and S.shape == (300, 17)
    assert (np.abs(S - exact) <= k * eps * mag + 1e-30).all()
    So = als_scores(Q, X, io, qo)
    want = exact + io[:, None] + qo[None, :]
    tol = k * eps * mag + 2 * eps * (np.abs(exact) + np.abs(io)[:, None] + np.abs(qo)[None, :])
    assert (np.abs(So - want) <= tol).all()
    # the offsets are separate f32 adds after the chain, item offset first
    assert np.array_equal(So.view(np.int32), ((S + io[:, None]) + qo[None, :]).view(np.int32))


def _c_fmaf(tmp_path):
    src = tmp_path / "fmaf.c"
    src.write_text(
        "#include <math.h>\n#include <stdint.h>\n"
        "void run(const float *a, const float *b, const float *c, float *out, int64_t n)\n"
        "{ for (int64_t i = 0; i < n; i++) out[i] = fmaf(a[i], b[i], c[i]); }\n"
    )
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed for the fmaf reference"
    so = tmp_path / "libfmaf.so"
    subprocess.run([cc, "-O0", "-shared", "-fPIC", str(src), "-o", str(so), "-lm"], check=True)
    fn = C.CDLL(str(so)).run
    f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    fn.argtypes, fn.restype = [f32p, f32p, f32p, f32p, C.c_int64], None

    def run(a, b, c):
        out = np.empty_like(a)
        fn(a, b, c, out, len(a))
        return out

    return run


def test_host_fmaf_matches_c_fmaf(tmp_path):
    """The NumPy fmaf of ``als_oracle`` rounds exactly like the C library's, on random triples over a wide exponent
    range and on built cases where the f64 sum lands on an f32 midpoint with a nonzero TwoSum error."""
    c_fmaf = _c_fmaf(tmp_path)
    rng = np.random.default_rng(23)
    m = 200_000

    def rand(lo, hi):
        return (rng.standard_normal(m) * np.exp2(rng.integers(lo, hi, m))).astype(np.float32)

    a, b, c = rand(-40, 40), rand(-40, 40), rand(-80, 80)
    c[::7] = -(a[::7] * b[::7])  # near-cancellation
    c[::11] = 0.0
    # midpoint cases: c with an odd last bit, p = h (1 - 2^-46) with h half an ulp of c (the exact sum lies just
    # below the midpoint c + h, which is the f64 sum); ties-to-even on the f64 sum would round the wrong way
    e = rng.integers(-20, 20, m)
    mant = (rng.integers(2**23, 2**24, m) | 1).astype(np.float64)
    sign = rng.choice([-1.0, 1.0], m)
    c2 = (sign * mant * np.exp2(e - 23)).astype(np.float32)
    h = np.exp2(e - 24)
    a2 = (np.float64(1 + 2**-23) * np.exp2(e - 12)).astype(np.float32)
    b2 = (sign * np.float64(1 - 2**-23) * (h / np.exp2(e - 12))).astype(np.float32)
    a, b, c = np.concatenate([a, a2]), np.concatenate([b, b2]), np.concatenate([c, c2])
    got, want = fmaf(a, b, c), c_fmaf(a, b, c)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    # and the built cases do exercise the midpoint correction
    naive = (a2.astype(np.float64) * b2.astype(np.float64) + c2.astype(np.float64)).astype(np.float32)
    assert (naive.view(np.int32) != want[m:].view(np.int32)).all()


def test_oracle_scores_are_one_fma_chain():
    """A sum whose value depends on fusing: fmaf(a, a, s) keeps the low bits of a*a that a separate f32 product
    rounds away."""
    a = np.float32(1 + 2**-12)  # a*a = 1 + 2^-11 + 2^-24 exactly; its f32 rounding drops the 2^-24
    c = np.float32(1 + 2**-11)
    # d = 0: s = fmaf(-1, c, +0) = -c;  d = 1: s = fmaf(a, a, -c) = 2^-24 exactly (0 without the fusion)
    assert als_scores(np.float32([[-1.0, a]]), np.float32([[c, a]]))[0, 0] == np.float32(2**-24)


def test_exclusion_is_a_nan_offer_with_ties():
    """argtopn over the candidate list with the excluded items taken out (the reference's ``items.remove``)
    equals argtopn over every item with the excluded items' scores set to NaN, on tie-heavy score vectors."""
    rng = np.random.default_rng(11)
    for trial in range(300):
        n_items = int(rng.integers(1, 500))
        scores = rng.integers(-3, 4, n_items).astype(np.float32)  # few values: large tie groups
        excl = rng.integers(-1, n_items, int(rng.integers(0, n_items + 2)))  # repeats and -1 allowed
        n = int(rng.integers(1, n_items + 5))
        drop = excl[excl >= 0]
        cands = np.setdiff1d(np.arange(n_items), drop)
        want = cands[oracle.argtopn(scores[cands], n)]
        masked = scores.copy()
        masked[drop] = np.nan
        assert np.array_equal(oracle.argtopn(masked, n), want), trial


def _tiny_model():
    m = ImplicitMFScorer(features=4)
    m.items = Vocabulary(np.arange(5), "item")
    m.users = Vocabulary(np.arange(3), "user")
    m.item_embeddings = np.ones((5, 4), np.float32)
    m.user_embeddings = np.ones((3, 4), np.float32)
    return m


def test_recommend_batch_needs_a_device():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    m = _tiny_model()
    with pytest.raises(_lib.EngineError):  # nothing is computed on the host
        m.recommend_batch([1], 2)
    with pytest.raises(_lib.EngineError):
        m.recommend_batch([ItemList(item_nums=np.int32([1]), vocabulary=m.items)], 2, exclude="query")


@pytest.mark.parametrize("bad", ["all", "items", 1, True])
def test_recommend_batch_rejects_bad_exclude(bad):
    m = _tiny_model()
    with pytest.raises(ValueError):
        m.recommend_batch([1], 2, exclude=bad)
