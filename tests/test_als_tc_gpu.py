"""
GPU parity of the tensor-core ALS kernel (als_tc.cu: k = 64, bf16 gather,
unweighted / uniformly weighted Gram on bf16 MMAs) against the oracle that rounds the
gathered rows to bf16 the same way, and against the SIMT kernel.
"""

import numpy as np
import pytest
import torch

import oracle
from lkpy_b200 import _lib, data, engine

from helpers import rel_fro, small_synth

pytestmark = pytest.mark.gpu

def _run(mode, csr, this, other, reg, chunk_nnz=engine.DEFAULT_CHUNK_NNZ):
    dev = _lib.require_device()
    dm = engine.DeviceCSR.from_host(csr, dev)
    k = this.shape[1]
    plan = engine.ALSHalfPlan.create(dm, k, chunk_nnz)
    d_this = torch.from_numpy(this.copy()).to(dev)
    d_other = torch.from_numpy(other).to(dev)
    obf = torch.empty_like(d_other, dtype=torch.bfloat16)
    ws = engine.OtorWorkspace.create(k, dev)
    otor = engine.als_otor(d_other, reg, ws, obf)  # also fills the bf16 copy
    engine.als_half_epoch(
        plan, _lib.LK_ALS_IMPLICIT if mode == "implicit" else _lib.LK_ALS_EXPLICIT, d_this, obf,
        otor=otor if mode == "implicit" else None, reg=reg,
    )  # fmt: skip
    torch.cuda.synchronize()
    assert int(plan.status.item()) == 0
    return d_this.cpu().numpy(), float(np.sqrt(plan.sqdelta.item())), plan


def _oracle(mode, csr, this, other, reg):
    _o32, o64 = oracle.otor(oracle.bf16_round(other), reg)
    return oracle.als_half_f64(mode, csr, this, other, otor_mat=o64, reg=reg, bf16_other=True)


@pytest.mark.parametrize("mode", ["implicit", "explicit"])
@pytest.mark.parametrize("chunk_nnz", [engine.DEFAULT_CHUNK_NNZ, 256, 64, 32])
def test_tc_kernel_parity(cuda_lib, lk_options, chunk_nnz, mode):
    """Parity with the f64 oracle and with the SIMT kernel, for row parts from whole rows down to 32 nonzeros
    (split rows are summed from their partial systems in slot order)."""
    lk_options("LK_ALS_TC", 1)
    inter = small_synth(900, 500, 40000, seed=21)
    rng = np.random.default_rng(21)
    k = 64
    p = (rng.standard_normal((inter.n_users, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((inter.n_items, k)) * 0.1).astype(np.float32)
    if mode == "implicit":
        ui, iu = data.als_implicit_matrices(inter, 40.0)
    else:
        coo = inter.coo(rng.standard_normal(inter.nnz).astype(np.float32))
        ui, iu = data.InteractionCSR.from_scipy(coo), data.InteractionCSR.from_scipy(coo.T)
    for csr, this, other in ((ui, p, q), (iu, q, p)):
        got, delta, plan = _run(mode, csr, this, other, 0.1, chunk_nnz)
        assert plan.vals_uniform == (mode == "implicit")
        if chunk_nnz < 64:
            assert plan.n_split_rows > 0
        ref, dref = _oracle(mode, csr, this, other, 0.1)
        assert rel_fro(got, ref) < 1e-4, rel_fro(got, ref)  # north_star tolerance
        assert delta == pytest.approx(dref, rel=1e-3)
        empty = np.diff(csr.indptr) == 0
        assert np.all(got[empty] == 0.0)
        # the SIMT kernel on the same inputs agrees to rounding
        lk_options("LK_ALS_TC", 0)
        simt, _, _ = _run(mode, csr, this, other, 0.1, chunk_nnz)
        lk_options("LK_ALS_TC", 1)
        assert rel_fro(got, simt) < 2e-5


@pytest.mark.parametrize("mode", ["implicit", "explicit"])
@pytest.mark.parametrize("chunk_nnz", [32, 64, 96])
def test_tc_split_rows_deterministic(cuda_lib, lk_options, chunk_nnz, mode):
    lk_options("LK_ALS_TC", 1)
    inter = small_synth(300, 200, 20000, seed=5)
    rng = np.random.default_rng(5)
    if mode == "implicit":
        _ui, iu = data.als_implicit_matrices(inter, 40.0)
    else:
        coo = inter.coo(rng.standard_normal(inter.nnz).astype(np.float32))
        iu = data.InteractionCSR.from_scipy(coo.T)
    p = (rng.standard_normal((300, 64)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((200, 64)) * 0.1).astype(np.float32)
    a, _, plan = _run(mode, iu, q, p, 0.1, chunk_nnz=chunk_nnz)
    assert plan.n_split_rows > 0
    b, _, _ = _run(mode, iu, q, p, 0.1, chunk_nnz=chunk_nnz)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))  # bit-reproducible
    ref, _ = _oracle(mode, iu, q, p, 0.1)
    assert rel_fro(a, ref) < 1e-4
    c, _, _ = _run(mode, iu, q, p, 0.1, chunk_nnz=1 << 20)
    assert rel_fro(a, c) < 1e-5


@pytest.mark.parametrize("reg", [1e-2, 1e-3])
def test_tc_solve_badly_conditioned(cuda_lib, lk_options, reg):
    """Large Gram, small ridge (cond ~1e4 and ~1e5): the tensor-core kernel stays within a small factor of
    what f32 arithmetic can deliver (the f32 oracle's own distance to the f64 oracle)."""
    lk_options("LK_ALS_TC", 1)
    inter = small_synth(400, 300, 60000, seed=9)
    ui, _ = data.als_implicit_matrices(inter, 40.0)
    rng = np.random.default_rng(9)
    p = (rng.standard_normal((400, 64)) * 0.1).astype(np.float32)
    q = rng.standard_normal((300, 64)).astype(np.float32)  # trained-scale-and-beyond item factors
    got, _, _ = _run("implicit", ui, p, q, reg)
    ref, _ = _oracle("implicit", ui, p, q, reg)
    o32, _ = oracle.otor(oracle.bf16_round(q), reg)
    cpu32, _ = oracle.als_half("implicit", ui, p, q, otor_mat=o32, bf16_other=True)
    e_gpu, e_cpu = rel_fro(got, ref), rel_fro(cpu32, ref)
    assert e_gpu < max(1e-4, 3.0 * e_cpu), (e_gpu, e_cpu)


def test_tc_zero_weight_falls_back(cuda_lib, lk_options):
    """weight = 0 makes every confidence 0: A = OtOr, the Gram scaled by zero."""
    lk_options("LK_ALS_TC", 1)
    inter = small_synth(200, 150, 5000, seed=3)
    ui, _ = data.als_implicit_matrices(inter, 0.0)
    rng = np.random.default_rng(3)
    p = (rng.standard_normal((200, 64)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((150, 64)) * 0.1).astype(np.float32)
    got, _, _ = _run("implicit", ui, p, q, 0.1)
    ref, _ = _oracle("implicit", ui, p, q, 0.1)
    assert np.isfinite(got).all()
    assert rel_fro(got, ref) < 1e-4


def test_tc_non_uniform_weights_leave_the_bf16_fast_path(cuda_lib, lk_options):
    """use_ratings=True confidences are not uniform: the kernel leaves the bf16 MMAs for the tf32 x3 Gram of
    sqrt(v)-scaled rows."""
    lk_options("LK_ALS_TC", 1)
    inter = small_synth(400, 300, 15000, seed=8)
    ui, _ = data.als_implicit_matrices(inter, 40.0, use_ratings=True)
    rng = np.random.default_rng(8)
    p = (rng.standard_normal((400, 64)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((300, 64)) * 0.1).astype(np.float32)
    got, _, plan = _run("implicit", ui, p, q, 0.1)
    assert not plan.vals_uniform
    ref, _ = _oracle("implicit", ui, p, q, 0.1)
    assert rel_fro(got, ref) < 1e-4


@pytest.mark.parametrize("gram", ["bf16", "fp32", "weighted"])
def test_tc_not_positive_definite_is_reported(cuda_lib, lk_options, gram):
    """A system that is not positive definite (the reference's `ALS solve error`, implicit.rs:79) sets the
    status word and leaves the row untouched — on each Gram path of the tensor-core kernel: bf16 MMAs,
    tf32 x3 on fp32 rows, tf32 x3 on sqrt(v)-scaled rows (per-nonzero confidences)."""
    lk_options("LK_ALS_TC", 1)
    inter = small_synth(60, 40, 600, seed=2)
    ui, _ = data.als_implicit_matrices(inter, 40.0, use_ratings=gram == "weighted")
    dev = _lib.require_device()
    k = 64
    dm = engine.DeviceCSR.from_host(ui, dev)
    plan = engine.ALSHalfPlan.create(dm, k)
    assert plan.vals_uniform == (gram != "weighted")
    this = torch.full((60, k), 0.5, device=dev)
    other = torch.zeros((40, k), device=dev, dtype=torch.bfloat16 if gram == "bf16" else torch.float32)
    otor = -torch.eye(k, device=dev)
    engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, this, other, otor=otor)
    torch.cuda.synchronize()
    assert int(plan.status.item()) > 0
    nonempty = torch.from_numpy(np.diff(ui.indptr) > 0).to(dev)
    assert torch.all(this[nonempty] == 0.5)  # failed solves do not write
