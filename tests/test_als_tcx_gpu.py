"""
GPU parity of the tf32 gather path of als_tc.cu at k = 64 and k = 128 — the tensor-core ALS kernel for fp32
gathered rows and non-uniform confidence weights (tf32 hi/lo split Gram, three MMAs per accumulator tile and
8 rows) — against the f64 oracle with
UNROUNDED inputs (fp32 rows: the reference's own arithmetic, north-star tolerance 1e-4) and against
the SIMT kernel on the same inputs.
"""

import numpy as np
import pytest
import torch

import oracle
from lkpy_b200 import _lib, data, engine

from helpers import rel_fro, small_synth

pytestmark = pytest.mark.gpu


def _run(mode, csr, this, other, reg, bf16=False, chunk_nnz=engine.DEFAULT_CHUNK_NNZ):
    dev = _lib.require_device()
    dm = engine.DeviceCSR.from_host(csr, dev)
    k = this.shape[1]
    plan = engine.ALSHalfPlan.create(dm, k, chunk_nnz)
    d_this = torch.from_numpy(this.copy()).to(dev)
    d_other = torch.from_numpy(other).to(dev)
    obf = torch.empty_like(d_other, dtype=torch.bfloat16) if bf16 else None
    ws = engine.OtorWorkspace.create(k, dev)
    otor = engine.als_otor(d_other, reg, ws, obf)
    engine.als_half_epoch(
        plan, _lib.LK_ALS_IMPLICIT if mode == "implicit" else _lib.LK_ALS_EXPLICIT, d_this,
        obf if bf16 else d_other, otor=otor if mode == "implicit" else None, reg=reg,
    )  # fmt: skip
    torch.cuda.synchronize()
    assert int(plan.status.item()) == 0
    return d_this.cpu().numpy(), float(np.sqrt(plan.sqdelta.item())), plan


def _oracle(mode, csr, this, other, reg, bf16=False):
    _o32, o64 = oracle.otor(oracle.bf16_round(other) if bf16 else other, reg)
    return oracle.als_half_f64(mode, csr, this, other, otor_mat=o64, reg=reg, bf16_other=bf16)


def _matrices(inter, kind, rng):
    if kind == "implicit":
        return data.als_implicit_matrices(inter, 40.0)
    if kind == "weighted":
        return data.als_implicit_matrices(inter, 40.0, use_ratings=True)
    coo = inter.coo(rng.standard_normal(inter.nnz).astype(np.float32))
    return data.InteractionCSR.from_scipy(coo), data.InteractionCSR.from_scipy(coo.T)


@pytest.mark.parametrize("k", [64, 128])
@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("kind", ["implicit", "weighted", "explicit"])
def test_tcx_parity(cuda_lib, lk_options, kind, bf16, k):
    if kind == "implicit" and bf16:
        pytest.skip("bf16 rows with uniform weights take the bf16 MMAs (test_als_tc_gpu.py, test_als_tc128_gpu.py)")
    inter = small_synth(900, 500, 40000, seed=21)
    rng = np.random.default_rng(21)
    p = (rng.standard_normal((inter.n_users, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((inter.n_items, k)) * 0.1).astype(np.float32)
    ui, iu = _matrices(inter, kind, rng)
    mode = "explicit" if kind == "explicit" else "implicit"
    for csr, this, other in ((ui, p, q), (iu, q, p)):
        lk_options("LK_ALS_TC", 1)
        got, delta, plan = _run(mode, csr, this, other, 0.1, bf16)
        assert plan.vals_uniform == (kind == "implicit")
        ref, dref = _oracle(mode, csr, this, other, 0.1, bf16)
        assert rel_fro(got, ref) < 1e-4, rel_fro(got, ref)  # north-star tolerance vs the f64 oracle
        assert delta == pytest.approx(dref, rel=1e-3)
        assert np.all(got[np.diff(csr.indptr) == 0] == 0.0)
        lk_options("LK_ALS_TC", 0)  # the SIMT kernel on the same inputs
        simt, _, _ = _run(mode, csr, this, other, 0.1, bf16)
        # the tf32 x3 Gram drops the lo.lo term and truncates lo: it sits a few 1e-5 from true f32
        # arithmetic, inside the 1e-4 north-star tolerance
        assert rel_fro(got, simt) < 6e-5, rel_fro(got, simt)


@pytest.mark.parametrize("k", [64, 128])
def test_tcx_switch_off(cuda_lib, lk_options, k):
    """LK_ALS_TF32=0 sends fp32 rows back to the SIMT kernel (same bits as LK_ALS_TC=0)."""
    inter = small_synth(300, 200, 9000, seed=6)
    ui, _ = data.als_implicit_matrices(inter, 40.0)
    rng = np.random.default_rng(6)
    p = (rng.standard_normal((300, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((200, k)) * 0.1).astype(np.float32)
    lk_options("LK_ALS_TF32", 0)
    a, _, _ = _run("implicit", ui, p, q, 0.1)
    lk_options("LK_ALS_TF32", 1)
    lk_options("LK_ALS_TC", 0)
    b, _, _ = _run("implicit", ui, p, q, 0.1)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))


@pytest.mark.parametrize("k", [64, 128])
@pytest.mark.parametrize("kind", ["implicit", "weighted", "explicit"])
def test_tcx_split_rows_deterministic(cuda_lib, lk_options, kind, k):
    inter = small_synth(300, 200, 20000, seed=5)
    rng = np.random.default_rng(5)
    _ui, iu = _matrices(inter, kind, rng)
    mode = "explicit" if kind == "explicit" else "implicit"
    p = (rng.standard_normal((300, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((200, k)) * 0.1).astype(np.float32)
    a, _, plan = _run(mode, iu, q, p, 0.1, chunk_nnz=32)
    assert plan.n_split_rows > 0
    b, _, _ = _run(mode, iu, q, p, 0.1, chunk_nnz=32)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))  # bit-reproducible
    ref, _ = _oracle(mode, iu, q, p, 0.1)
    assert rel_fro(a, ref) < 1e-4
    c, _, _ = _run(mode, iu, q, p, 0.1, chunk_nnz=1 << 20)
    # split (32-nonzero parts added with round-to-nearest) vs unsplit (one tensor-core accumulation chain per
    # row): the accumulation orders differ, and the 128x128 solve amplifies that more than the 64x64 one; both
    # sit inside the 1e-4 tolerance against the oracle above
    assert rel_fro(a, c) < (1e-5 if k == 64 else 1e-4)


def test_tcx_badly_conditioned(cuda_lib, lk_options):
    """cond ~1e4 systems: the tf32-split Gram + tensor-core solve stays within a small factor of what the
    f32 oracle itself delivers."""
    inter = small_synth(400, 300, 60000, seed=9)
    ui, _ = data.als_implicit_matrices(inter, 40.0)
    rng = np.random.default_rng(9)
    p = (rng.standard_normal((400, 64)) * 0.1).astype(np.float32)
    q = rng.standard_normal((300, 64)).astype(np.float32)
    reg = 0.01
    got, _, _ = _run("implicit", ui, p, q, reg)
    ref, _ = _oracle("implicit", ui, p, q, reg)
    o32, _ = oracle.otor(q, reg)
    cpu32, _ = oracle.als_half("implicit", ui, p, q, otor_mat=o32)
    e_gpu, e_cpu = rel_fro(got, ref), rel_fro(cpu32, ref)
    assert e_gpu < max(1e-4, 3.0 * e_cpu), (e_gpu, e_cpu)


def test_tcx_ml_small_epochs(cuda_lib, ml_small):
    """Config 1 (ml-latest-small, reference init): three fp32 epochs on the tensor-core path track the
    f64 oracle as closely as the f32 oracle does (the init makes the first systems ill-conditioned)."""
    from helpers import implicit_init

    ui, iu = data.als_implicit_matrices(ml_small, 40.0)
    p, q = implicit_init(np.random.default_rng(42), ml_small.n_items, ml_small.n_users, 64)
    for csr, this, other in ((ui, p, q), (iu, q, p)):
        got, _, _ = _run("implicit", csr, this, other, 0.1)
        ref, _ = _oracle("implicit", csr, this, other, 0.1)
        o32, _ = oracle.otor(other, 0.1)
        cpu32, _ = oracle.als_half("implicit", csr, this, other, otor_mat=o32)
        assert rel_fro(got, ref) < max(1e-4, 1.5 * rel_fro(cpu32, ref)), (rel_fro(got, ref), rel_fro(cpu32, ref))


def test_tcx_not_positive_definite_is_reported(cuda_lib, lk_options):
    inter = small_synth(60, 40, 600, seed=2)
    ui, _ = data.als_implicit_matrices(inter, 40.0)
    dev = _lib.require_device()
    k = 64
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(ui, dev), k)
    this = torch.full((60, k), 0.5, device=dev)
    other = torch.zeros((40, k), device=dev)
    otor = -torch.eye(k, device=dev)
    engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, this, other, otor=otor)
    torch.cuda.synchronize()
    assert int(plan.status.item()) > 0
    nonempty = torch.from_numpy(np.diff(ui.indptr) > 0).to(dev)
    assert torch.all(this[nonempty] == 0.5)  # failed solves do not write
