"""
BiasedSVD without a GPU: the restatements of tests/svd_oracle.py against SciPy's products and scikit-learn's
``TruncatedSVD``, the restatement against the reference's recordings, the configuration surface, ``lk_spmm``'s host
validation and C struct layout, and the absence of a fallback without a device.  CPU only.

The reference's side comes from a lenskit/lkpy checkout when there is one, else from
``tests/golden/reference_classes/biased_svd_k*.npz``, which ``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites from the
checkout (tests/svd_ref_sandbox.py).
"""

import ctypes as C
import os
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import scipy.sparse as sps
import torch

import ref_sandbox
import svd_oracle as so
import svd_ref_sandbox as srs
from lkpy_b200 import _lib
from lkpy_b200.basic import BiasModel
from lkpy_b200.components import Dataset
from lkpy_b200.svd import BiasedSVDConfig, BiasedSVDScorer

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"
GOLDEN_K = (16, 64)


def reference_golden(ml_small, k: int) -> dict:
    """The reference's values for ``embedding_size=k``: recorded live when asked to, else read from the golden file."""
    path = GOLD / f"biased_svd_k{k}.npz"
    if RECORD:
        assert ref_sandbox.available(), "recording needs the reference checkout"
        np.savez_compressed(path, **srs.record(ml_small, k))
    with np.load(path) as z:
        return {name: z[name] for name in z.files}


def ml_residuals(ml_small, damping=5.0):
    bias = BiasModel.learn(ml_small, damping, np.float32)
    X = so.residuals(ml_small.users, ml_small.items, ml_small.ratings, ml_small.n_users, ml_small.n_items,
                     bias.global_bias, bias.item_biases, bias.user_biases)  # fmt: skip
    return bias, X


# ------------------------------------------------------------------------------------------------------------
# restatements
# ------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("W", [1, 17, 74])
def test_product_restatement_is_scipy(ml_small, W):
    _bias, X = ml_residuals(ml_small)
    XT = sps.csr_array(X.T)
    XT.sort_indices()
    rng = np.random.default_rng(W)
    d_items = rng.standard_normal((X.shape[1], W)).astype(np.float32)
    d_users = rng.standard_normal((X.shape[0], W)).astype(np.float32)
    ours = so.spmm(X.indptr, X.indices, X.data, d_items)
    assert np.array_equal(ours.view(np.uint32), (X @ d_items).view(np.uint32))
    ours_t = so.spmm(XT.indptr, XT.indices, XT.data, d_users)
    assert np.array_equal(ours_t.view(np.uint32), (X.T @ d_users).view(np.uint32))
    assert np.array_equal(ours_t.T.view(np.uint32), np.ascontiguousarray(d_users.T @ X).view(np.uint32))


@pytest.mark.parametrize("n_iter", [2, 5])
@pytest.mark.parametrize("transposed", [True, False])
def test_restatement_is_truncated_svd(ml_small, n_iter, transposed):
    TruncatedSVD = pytest.importorskip("sklearn.decomposition").TruncatedSVD
    _bias, X = ml_residuals(ml_small)
    if not transposed:  # a tall matrix: the items as rows
        X = sps.csr_array(X.T)
        X.sort_indices()
    assert (X.shape[0] < X.shape[1]) == transposed
    k = 16
    theirs = TruncatedSVD(k, algorithm="randomized", n_iter=n_iter, random_state=np.random.RandomState(3))
    xt = theirs.fit_transform(X)
    vt, s, ours_xt = so.truncated_svd(X, k, n_iter, so.start_matrix(X.shape, k, np.random.RandomState(3)))
    for a, b in ((vt, theirs.components_), (s, theirs.singular_values_), (ours_xt, xt)):
        assert a.dtype == b.dtype == np.float32
        assert np.array_equal(a, b)


@pytest.mark.parametrize("k", GOLDEN_K)
def test_restatement_is_the_reference(ml_small, k):
    """The restatement, with the bias model of ``lkpy_b200.basic`` and the start matrix drawn after
    ``np.random.seed``, reproduces the reference's recording (the biases bit for bit) and leaves the global state
    where it did."""
    g = reference_golden(ml_small, k)
    bias, X = ml_residuals(ml_small)
    assert bias.global_bias == g["global_bias"]
    assert np.array_equal(bias.item_biases, g["item_biases"]) and np.array_equal(bias.user_biases, g["user_biases"])
    np.random.seed(srs.SEED)
    vt, s, xt = so.truncated_svd(X, k, 5, so.start_matrix(X.shape, k, np.random.mtrand._rand))
    state = np.random.get_state()
    assert np.array_equal(state[1], g["state_keys"]) and state[2] == g["state_pos"]
    assert np.array_equal([state[3], state[4]], g["state_gauss"])
    # the LU, QR and SVD are LAPACK's, whose blocked routines round differently under another BLAS thread count
    # than the recording had (measured: singular values 5e-7 apart, user components 7e-5 at k = 64), so the dense
    # results are compared to rounding, with the bounds the device run is held to
    assert np.abs(s / g["singular_values"] - 1).max() < 1e-5
    assert np.abs(vt[:, srs.ROWS_I] - g["components"]).max() < 1e-3
    want = g["user_components"].astype(np.float64)
    assert np.linalg.norm(xt[srs.ROWS_U] - want) / np.linalg.norm(want) < 1e-3


# ------------------------------------------------------------------------------------------------------------
# configuration, ABI, no fallback
# ------------------------------------------------------------------------------------------------------------


def test_config():
    c = BiasedSVDConfig()
    assert (c.embedding_size, c.damping, c.algorithm, c.n_iter) == (64, 5, "randomized", 5)
    assert BiasedSVDConfig(features=2).embedding_size == 2
    assert BiasedSVDConfig(embedding_size=25, damping=10).embedding_size == 25
    assert BiasedSVDConfig(embedding_size_exp=5).embedding_size == 32
    assert BiasedSVDScorer(features=8).config.embedding_size == 8
    assert BiasedSVDConfig(damping={"user": 3}).damping == {"user": 3.0}
    with pytest.raises(ValueError, match="algorithm='arpack'"):
        BiasedSVDConfig(algorithm="arpack")
    with pytest.raises(ValueError, match="engine limit"):
        BiasedSVDConfig(embedding_size=129)
    with pytest.raises(ValueError):
        BiasedSVDConfig(n_iter=-1)


def test_dict_damping(ml_small):
    both = BiasModel.learn(ml_small, (3.0, 0.0))
    d = BiasModel.learn(ml_small, {"user": 3.0})
    assert d.damping == (3.0, 0.0)
    assert np.array_equal(d.item_biases, both.item_biases) and np.array_equal(d.user_biases, both.user_biases)


def test_spmm_struct_matches_header(tmp_path):
    cls = _lib.LkSpmmArgs
    lines = [f'    printf("lk_spmm_args.{f[0]} %zu\\n", offsetof(lk_spmm_args, {f[0]}));' for f in cls._fields_]
    lines.append('    printf("sizeof %zu\\n", sizeof(lk_spmm_args));')
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
        expected += [f"lk_spmm_args.{f[0]}", str(getattr(cls, f[0]).offset)]
    assert out == expected + ["sizeof", str(C.sizeof(cls))]


def test_spmm_host_validation(cuda_lib):
    a = _lib.LkSpmmArgs()
    a.n_rows, a.n_src, a.width = 4, 4, 0
    assert cuda_lib.lk_spmm(C.byref(a), None) == -1  # LK_ERR_INVALID
    a.width, a.nnz = 8, 2**31
    assert cuda_lib.lk_spmm(C.byref(a), None) == -3  # LK_ERR_UNSUPPORTED: int32 offsets
    assert b"2^31" in cuda_lib.lk_last_error()
    a.nnz = 10
    assert cuda_lib.lk_spmm(C.byref(a), None) == -1  # null pointers, caught before any launch


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a device")
def test_no_fallback_without_a_device(ml_small):
    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        BiasedSVDScorer(embedding_size=8).train(Dataset(ml_small))
