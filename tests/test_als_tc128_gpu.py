"""
GPU parity of als_tc.cu at k = 128 (four warps, one 64x64 Gram quadrant each, the 128x128 system solved
in shared memory; BASELINE configs[3]) — against the f64 oracle that
rounds the gathered rows to bf16 the same way, and against the SIMT kernel on the same inputs.
"""

import numpy as np
import pytest
import torch

import oracle
from lkpy_b200 import _lib, data, engine

from helpers import rel_fro, small_synth

pytestmark = pytest.mark.gpu
K = 128


def _run(mode, csr, this, other, reg, chunk_nnz=engine.DEFAULT_CHUNK_NNZ):
    dev = _lib.require_device()
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), K, chunk_nnz)
    d_this = torch.from_numpy(this.copy()).to(dev)
    d_other = torch.from_numpy(other).to(dev)
    obf = torch.empty_like(d_other, dtype=torch.bfloat16)
    ws = engine.OtorWorkspace.create(K, dev)
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
def test_tc128_parity(cuda_lib, lk_options, mode):
    inter = small_synth(900, 500, 40000, seed=31)
    rng = np.random.default_rng(31)
    p = (rng.standard_normal((inter.n_users, K)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((inter.n_items, K)) * 0.1).astype(np.float32)
    if mode == "implicit":
        ui, iu = data.als_implicit_matrices(inter, 40.0)
    else:
        coo = inter.coo(rng.standard_normal(inter.nnz).astype(np.float32))
        ui, iu = data.InteractionCSR.from_scipy(coo), data.InteractionCSR.from_scipy(coo.T)
    for csr, this, other in ((ui, p, q), (iu, q, p)):
        lk_options("LK_ALS_TC", 1)
        got, delta, _ = _run(mode, csr, this, other, 0.1)
        ref, dref = _oracle(mode, csr, this, other, 0.1)
        assert rel_fro(got, ref) < 1e-4, rel_fro(got, ref)  # north-star tolerance
        assert delta == pytest.approx(dref, rel=1e-3)
        assert np.all(got[np.diff(csr.indptr) == 0] == 0.0)
        lk_options("LK_ALS_TC", 0)  # the SIMT kernel on the same inputs agrees to rounding
        simt, _, _ = _run(mode, csr, this, other, 0.1)
        assert rel_fro(got, simt) < 3e-5, rel_fro(got, simt)


@pytest.mark.parametrize("mode", ["implicit", "explicit"])
def test_tc128_split_rows_deterministic(cuda_lib, lk_options, mode):
    inter = small_synth(300, 200, 20000, seed=5)
    rng = np.random.default_rng(5)
    if mode == "implicit":
        _ui, iu = data.als_implicit_matrices(inter, 40.0)
    else:
        iu = data.InteractionCSR.from_scipy(inter.coo(rng.standard_normal(inter.nnz).astype(np.float32)).T)
    p = (rng.standard_normal((300, K)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((200, K)) * 0.1).astype(np.float32)
    a, _, plan = _run(mode, iu, q, p, 0.1, chunk_nnz=32)
    assert plan.n_split_rows > 0
    b, _, _ = _run(mode, iu, q, p, 0.1, chunk_nnz=32)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))  # bit-reproducible
    ref, _ = _oracle(mode, iu, q, p, 0.1)
    assert rel_fro(a, ref) < 1e-4
    c, _, _ = _run(mode, iu, q, p, 0.1, chunk_nnz=1 << 20)
    assert rel_fro(a, c) < 1e-5


def test_tc128_badly_conditioned(cuda_lib, lk_options):
    inter = small_synth(400, 300, 60000, seed=9)
    ui, _ = data.als_implicit_matrices(inter, 40.0)
    rng = np.random.default_rng(9)
    p = (rng.standard_normal((400, K)) * 0.1).astype(np.float32)
    q = rng.standard_normal((300, K)).astype(np.float32)
    reg = 0.01
    got, _, _ = _run("implicit", ui, p, q, reg)
    ref, _ = _oracle("implicit", ui, p, q, reg)
    o32, _ = oracle.otor(oracle.bf16_round(q), reg)
    cpu32, _ = oracle.als_half("implicit", ui, p, q, otor_mat=o32, bf16_other=True)
    e_gpu, e_cpu = rel_fro(got, ref), rel_fro(cpu32, ref)
    assert e_gpu < max(1e-4, 3.0 * e_cpu), (e_gpu, e_cpu)


def test_tc128_short_and_odd_rows(cuda_lib, lk_options):
    """Rows of 1..40 nonzeros (not multiples of the 16-row stage), an odd number of chunks, empty rows."""
    rng = np.random.default_rng(3)
    n_rows, n_other = 77, 150
    lens = rng.integers(0, 41, n_rows)
    lens[[0, 5]] = 0
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = np.concatenate([np.sort(rng.choice(n_other, n, replace=False)) for n in lens]).astype(np.int32)
    csr = data.InteractionCSR(indptr, cols, np.full(len(cols), 40.0, np.float32), (n_rows, n_other))
    p = (rng.standard_normal((n_rows, K)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((n_other, K)) * 0.1).astype(np.float32)
    got, _, _ = _run("implicit", csr, p, q, 0.1)
    ref, _ = _oracle("implicit", csr, p, q, 0.1)
    assert rel_fro(got, ref) < 1e-4
    assert np.all(got[lens == 0] == 0.0)


def test_tc128_not_positive_definite_is_reported(cuda_lib, lk_options):
    inter = small_synth(60, 40, 600, seed=2)
    ui, _ = data.als_implicit_matrices(inter, 40.0)
    dev = _lib.require_device()
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(ui, dev), K)
    this = torch.full((60, K), 0.5, device=dev)
    other = torch.zeros((40, K), device=dev, dtype=torch.bfloat16)
    otor = -torch.eye(K, device=dev)
    engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, this, other, otor=otor)
    torch.cuda.synchronize()
    assert int(plan.status.item()) > 0
    nonempty = torch.from_numpy(np.diff(ui.indptr) > 0).to(dev)
    assert torch.all(this[nonempty] == 0.5)  # failed solves do not write
