"""
NMF without a GPU: the restatements of tests/nmf_oracle.py against scikit-learn's compiled sweep, NumPy's sequential
f32 sum and ``non_negative_factorization``, the configuration surface, and the C struct layouts.  CPU only.
"""

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import scipy.sparse as sps
import torch

import nmf_oracle as no
from lkpy_b200 import _lib
from lkpy_b200.components import Dataset
from lkpy_b200.nmf import NMFConfig, NMFScorer

ROOT = Path(__file__).resolve().parent.parent
SWEEP_K = (1, 16, 64, 128)


def sweep_case(k: int, n: int = 257, seed: int = 0):
    """Random sweep operands with exact zeros in W, a zero Gram diagonal entry, and l1 and l2 terms applied."""
    rng = np.random.default_rng(seed + k)
    W = np.abs(rng.standard_normal((n, k))).astype(np.float32)
    W[rng.random((n, k)) < 0.25] = 0
    HHt = no.gram(np.abs(rng.standard_normal((40, k))).astype(np.float32))
    HHt.flat[:: k + 1] += 0.75  # l2
    if k > 1:
        HHt[:, k // 2] = 0
        HHt[k // 2, :] = 0  # a component with a zero Hessian: left as it is
    XHt = (rng.random((n, k)) * 4).astype(np.float32)
    XHt -= 0.5  # l1
    return W, HHt, XHt


def adversarial_sums() -> dict[str, np.ndarray]:
    """Inputs for the sequential sum: ties at every binade, jumps over several binades, subnormals, zeros, inf, NaN."""
    rng = np.random.default_rng(7)
    ties = []
    for e in range(-140, 120, 3):  # 2^e, then half an ulp (a tie to even), three halves, one ulp
        ties += [2.0**e, 2.0 ** (e - 24), 3 * 2.0 ** (e - 24), 2.0 ** (e - 23), 2.0 ** (e - 24)]
    f32 = lambda a: np.asarray(a, dtype=np.float32)  # noqa: E731
    return {
        "empty": f32([]),
        "zeros": np.zeros(1000, np.float32),
        "ties": f32(ties),
        "ulp_steps": f32(np.float32(1 + 2**-23) * np.ones(5000)),
        "half_ulps": f32(np.where(rng.random(20000) < 0.5, 0, rng.integers(1, 8, 20000) * 2.0**-24)),
        "jumps_up": f32([2.0**e for e in range(-149, 127, 5)]),
        "jumps_down": f32([2.0**e for e in range(126, -150, -5)]),
        "subnormals": f32([1e-45] * 3000 + [3e-42] * 100 + [1.2e-38] * 7 + [1.0] + [1e-8] * 1000),
        "inf": f32([0, 1, np.inf, 3, 2]),
        "inf_then_nan": f32([1, np.inf, 3, np.nan, 4]),
        "nan_then_inf": f32([1, np.nan, np.inf]),
        "overflow": f32([3e38, 3e38, 1]),
        "wide_range": f32(np.abs(rng.standard_normal(20000) * np.exp(rng.uniform(-40, 40, 20000)))),
    }


def violation_like(n: int = 10_000_000, seed: int = 11) -> np.ndarray:
    """n |pg|-like values: half-normal magnitudes spread over several binades, a third of them exact zeros."""
    rng = np.random.default_rng(seed)
    x = (np.abs(rng.standard_normal(n)) * np.exp(rng.uniform(-6, 2, n))).astype(np.float32)
    x[rng.random(n) < 0.3] = 0
    return x


def same_bits(a, b) -> bool:
    a, b = np.float32(a), np.float32(b)
    return bool(a.view(np.uint32) == b.view(np.uint32) or (np.isnan(a) and np.isnan(b)))


def cumsum_f32(x: np.ndarray) -> np.float32:
    return np.cumsum(x, dtype=np.float32)[-1] if len(x) else np.float32(0)


@pytest.mark.parametrize("k", SWEEP_K)
def test_sweep_restatement_is_sklearn(k):
    cdnmf = pytest.importorskip("sklearn.decomposition._cdnmf_fast")
    W, HHt, XHt = sweep_case(k)
    theirs = W.copy()
    v = cdnmf._update_cdnmf_fast(theirs, HHt, XHt, np.arange(k, dtype=np.intp))
    ours = W.copy()
    pg = no.cd_sweep(ours, HHt, XHt)
    assert np.array_equal(ours.view(np.uint32), theirs.view(np.uint32))
    assert same_bits(no.seq_sum(pg.ravel()), v)


@pytest.mark.parametrize("name", sorted(adversarial_sums()))
def test_seq_sum_restatement_is_cumsum(name):
    x = adversarial_sums()[name]
    with np.errstate(over="ignore", invalid="ignore"):
        assert same_bits(no.seq_sum(x), cumsum_f32(x))


def test_seq_sum_restatement_on_ten_million_values():
    x = violation_like()
    assert same_bits(no.seq_sum(x), cumsum_f32(x))


def test_host_loop_is_non_negative_factorization(ml_small):
    """The restated loop with the f64 Gram, from scikit-learn's own initialisation, against
    ``non_negative_factorization`` at k = 16.  Measured on ml-latest-small: the same 120 iterations, W and H within
    3e-5 relative Frobenius, W H within 3.1e-6; the bounds leave a factor of about three."""
    skd = pytest.importorskip("sklearn.decomposition")
    from sklearn.decomposition._nmf import _initialize_nmf

    X = sps.csr_matrix((np.ones(ml_small.nnz, np.float32), (ml_small.users, ml_small.items)),
                       shape=(ml_small.n_users, ml_small.n_items))  # fmt: skip
    np.random.seed(3)
    W0, H0 = _initialize_nmf(X, 16)
    np.random.seed(3)
    W, H, n_iter = skd.non_negative_factorization(X, n_components=16, max_iter=200)
    oW, oH, o_iter = no.fit(X, W0, H0, max_iter=200)
    assert o_iter == n_iter
    rel = lambda a, b: np.linalg.norm(a.astype(np.float64) - b) / np.linalg.norm(b.astype(np.float64))  # noqa: E731
    assert rel(oW, W) < 1e-4 and rel(oH, H) < 1e-4
    assert rel(oW.astype(np.float64) @ oH, W.astype(np.float64) @ H) < 1e-5


def test_config():
    c = NMFConfig()
    assert (c.beta_loss, c.max_iter, c.embedding_size, c.alpha_W, c.alpha_H, c.l1_ratio, c.method) == (
        "frobenius", 200, 64, 0.0, "same", 0.0, "full")  # fmt: skip
    assert NMFConfig(epochs=7).max_iter == 7
    assert NMFConfig(n_components=12).embedding_size == 12
    assert NMFConfig(embedding_size_exp=5).embedding_size == 32
    assert NMFScorer(n_components=8).config.embedding_size == 8
    assert NMFConfig(alpha_W=0.5, l1_ratio=0.25).regularization(10, 20) == (2.5, 1.25, 7.5, 3.75)
    assert NMFConfig(alpha_W=0.5, alpha_H=1.0).regularization(10, 20) == (0.0, 0.0, 10.0, 10.0)
    with pytest.raises(ValueError, match="minibatch"):
        NMFConfig(method="minibatch")
    with pytest.raises(ValueError, match="beta_loss"):
        NMFConfig(beta_loss="kullback-leibler")
    with pytest.raises(ValueError, match="embedding_size=None"):
        NMFConfig(embedding_size=None)
    with pytest.raises(ValueError, match="engine limit"):
        NMFConfig(embedding_size=129)
    with pytest.raises(ValueError):
        NMFConfig(max_iter=0)


@pytest.mark.parametrize("struct", ["lk_nmf_cd_sweep_args", "lk_f32_seq_sum_args"])
def test_structs_match_header(tmp_path, struct):
    cls = {"lk_nmf_cd_sweep_args": _lib.LkNmfCdSweepArgs, "lk_f32_seq_sum_args": _lib.LkF32SeqSumArgs}[struct]
    lines = [f'    printf("{struct}.{f[0]} %zu\\n", offsetof({struct}, {f[0]}));' for f in cls._fields_]
    lines.append(f'    printf("sizeof %zu\\n", sizeof({struct}));')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"lkpy_b200.h\"\n\nint main(void)\n{\n"
                   + "\n".join(lines) + "\n    return 0;\n}\n")  # fmt: skip
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    expected = []
    for f in cls._fields_:
        expected += [f"{struct}.{f[0]}", str(getattr(cls, f[0]).offset)]
    assert out == expected + ["sizeof", str(C.sizeof(cls))]


def test_host_validation(cuda_lib):
    a = _lib.LkNmfCdSweepArgs()
    a.n, a.k = 4, 129
    assert cuda_lib.lk_nmf_cd_sweep(C.byref(a), None) == -3  # LK_ERR_UNSUPPORTED
    a.k = 0
    assert cuda_lib.lk_nmf_cd_sweep(C.byref(a), None) == -3
    a.k = 8
    assert cuda_lib.lk_nmf_cd_sweep(C.byref(a), None) == -1  # null pointers, caught before any launch
    sums = (_lib.LkF32SeqSumArgs * 9)()
    assert cuda_lib.lk_f32_seq_sum(sums, 9, None) == -1  # at most 8 sums
    sums[0].n = 5
    assert cuda_lib.lk_f32_seq_sum(sums, 1, None) == -1


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a device")
def test_no_fallback_without_a_device(ml_small):
    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        NMFScorer(embedding_size=8).train(Dataset(ml_small))
