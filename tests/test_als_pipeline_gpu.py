"""
The k = 64 tensor-core ALS kernel's gather pipeline and work hand-out (als_tc.cu): the three-stage ring of
bulk copies wraps across many chunks, rows of every length class relative to a 32-row stage, split rows whose
last parts finish in varying order, a work index claimed one chunk ahead, and the lower-triangle Gram — on the
bf16, fp32 and weighted (sqrt(v)-scaled tf32) Grams, implicit and explicit.
"""

import time

import numpy as np
import pytest
import torch

import oracle
from lkpy_b200 import _lib, data, engine

from helpers import rel_fro

pytestmark = pytest.mark.gpu

K = 64
# empty, shorter than a stage, exactly 32 m nonzeros, one past a stage boundary, long rows that split at 32 / 64
LENGTHS = [0, 1, 5, 31, 32, 0, 33, 64, 96, 97, 0, 150, 255, 256, 300, 3, 2]


def _csr(lengths, n_cols, kind, rng):
    indptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    cols = np.concatenate([np.sort(rng.choice(n_cols, n, replace=False)) for n in lengths]).astype(np.int32)
    nnz = int(indptr[-1])
    if kind == "explicit":
        vals = rng.standard_normal(nnz)
    elif kind == "weighted":
        vals = 1.0 + 40.0 * rng.integers(1, 11, nnz) / 2.0  # per-nonzero confidences
    else:
        vals = np.full(nnz, 40.0)
    return data.InteractionCSR(indptr, cols, vals.astype(np.float32), (len(lengths), n_cols))


def _run(mode, csr, this, other, gram, reg=0.1, chunk_nnz=engine.DEFAULT_CHUNK_NNZ, otor=None, cancel=None):
    dev = _lib.require_device()
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), K, chunk_nnz)
    d_this = torch.from_numpy(this.copy()).to(dev)
    d_other = torch.from_numpy(other).to(dev)
    obf = torch.empty_like(d_other, dtype=torch.bfloat16) if gram == "bf16" else None
    ws = engine.OtorWorkspace.create(K, dev)
    o = engine.als_otor(d_other, reg, ws, obf)
    if otor is not None:
        o = torch.from_numpy(otor).to(dev)
    engine.als_half_epoch(
        plan, _lib.LK_ALS_IMPLICIT if mode == "implicit" else _lib.LK_ALS_EXPLICIT, d_this,
        obf if gram == "bf16" else d_other, otor=o if mode == "implicit" else None, reg=reg, cancel=cancel,
    )  # fmt: skip
    torch.cuda.synchronize()
    return d_this.cpu().numpy(), plan


def _oracle(mode, csr, this, other, gram, reg=0.1, otor=None):
    bf16 = gram == "bf16"
    if otor is None:
        _o32, otor = oracle.otor(oracle.bf16_round(other) if bf16 else other, reg)
    return oracle.als_half_f64(mode, csr, this, other, otor_mat=otor, reg=reg, bf16_other=bf16)[0]


def _factors(rng, n_rows, n_cols):
    this = (rng.standard_normal((n_rows, K)) * 0.1).astype(np.float32)
    other = (rng.standard_normal((n_cols, K)) * 0.1).astype(np.float32)
    return this, other


@pytest.mark.parametrize("chunk_nnz", [32, 64, engine.DEFAULT_CHUNK_NNZ])
@pytest.mark.parametrize("mode", ["implicit", "explicit"])
@pytest.mark.parametrize("gram", ["bf16", "fp32", "weighted"])
def test_ring_wraps_over_mixed_rows(cuda_lib, gram, mode, chunk_nnz):
    """Hundreds of chunks of every length class: reproducible to the bit, and within 1e-4 of the f64 oracle."""
    if gram == "weighted" and mode == "explicit":
        pytest.skip("the explicit Gram is unweighted")
    rng = np.random.default_rng(chunk_nnz + len(gram))
    lengths = np.array(LENGTHS * 24)
    rng.shuffle(lengths)
    csr = _csr(lengths, 400, "weighted" if gram == "weighted" else mode, rng)
    this, other = _factors(rng, len(lengths), 400)
    a, plan = _run(mode, csr, this, other, gram, chunk_nnz=chunk_nnz)
    assert int(plan.status.item()) == 0
    assert plan.vals_uniform == (gram != "weighted" and mode == "implicit")
    assert plan.n_chunks > 8 * len(LENGTHS)
    if chunk_nnz < 256:
        assert plan.n_split_rows > 0
    b, _ = _run(mode, csr, this, other, gram, chunk_nnz=chunk_nnz)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    assert np.all(a[lengths == 0] == 0.0)
    ref = _oracle(mode, csr, this, other, gram)
    assert rel_fro(a, ref) < 1e-4, rel_fro(a, ref)


@pytest.mark.parametrize("gram", ["bf16", "fp32"])
def test_many_tiny_rows(cuda_lib, gram):
    """Tens of thousands of one- to three-nonzero rows: the work hand-out, not the Gram, sets the pace."""
    rng = np.random.default_rng(4)
    lengths = rng.integers(0, 4, 30000)
    csr = _csr(lengths, 300, "implicit", rng)
    this, other = _factors(rng, len(lengths), 300)
    a, plan = _run("implicit", csr, this, other, gram)
    assert int(plan.status.item()) == 0
    b, _ = _run("implicit", csr, this, other, gram)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    assert rel_fro(a, _oracle("implicit", csr, this, other, gram)) < 1e-4


@pytest.mark.parametrize("gram", ["bf16", "fp32", "weighted"])
def test_non_positive_definite_row_leaves_the_others_solved(cuda_lib, gram):
    """With OtOr = -I, rows of fewer than k nonzeros are indefinite and long rows stay positive definite: the
    status word names a short row, the short rows keep their old values, and every long row is solved."""
    rng = np.random.default_rng(6)
    lengths = np.array([0, 3, 300, 20, 400, 63, 250, 1, 500] * 8)
    csr = _csr(lengths, 600, "weighted" if gram == "weighted" else "implicit", rng)
    this = (rng.standard_normal((len(lengths), K)) * 0.1).astype(np.float32)
    other = rng.standard_normal((600, K)).astype(np.float32)
    otor = -np.eye(K, dtype=np.float32)
    got, plan = _run("implicit", csr, this, other, gram, otor=otor)
    short = (lengths > 0) & (lengths < K)
    status = int(plan.status.item())
    assert status > 0 and short[status - 1]
    assert np.array_equal(got[short], this[short])
    long_ = lengths >= 200
    sub = csr.to_scipy()[np.flatnonzero(long_)]
    ref = _oracle("implicit", data.InteractionCSR.from_scipy(sub), this[long_], other, gram, otor=otor.astype(np.float64))
    assert rel_fro(got[long_], ref) < 1e-4


def test_raised_cancel_flag_ends_the_launch(cuda_lib):
    """A cancel flag raised before the launch: no chunk is handed out and nothing is written."""
    dev = _lib.require_device()
    rng = np.random.default_rng(8)
    lengths = np.array(LENGTHS * 40)
    csr = _csr(lengths, 400, "implicit", rng)
    this, other = _factors(rng, len(lengths), 400)
    got, plan = _run("implicit", csr, this, other, "bf16", cancel=torch.ones(1, dtype=torch.int32, device=dev))
    assert np.array_equal(got.view(np.int32), this.view(np.int32))
    assert float(plan.sqdelta.item()) == 0.0 and int(plan.status.item()) == 0


@pytest.mark.parametrize("gram", ["bf16", "fp32"])
def test_cancel_mid_launch_finishes_exactly_the_claimed_chunks(cuda_lib, gram):
    """The flag raised by a copy engine while the launch runs: every chunk the work counter handed out, the
    one each CTA claimed ahead included, is finished and bit-equal to an uncancelled run, and no other row
    is touched."""
    dev = _lib.require_device()
    rng = np.random.default_rng(9)
    lengths = rng.integers(0, 120, 200_000)
    indptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    cols = rng.integers(0, 4000, int(indptr[-1])).astype(np.int32)
    csr = data.InteractionCSR(indptr, cols, np.full(len(cols), 40.0, np.float32), (len(lengths), 4000))
    this, other = _factors(rng, len(lengths), 4000)
    dm = engine.DeviceCSR.from_host(csr, dev)
    plan = engine.ALSHalfPlan.create(dm, K, 1 << 20)  # whole rows: a row is written by the chunk that holds it
    assert plan.n_split_rows == 0
    d_other = torch.from_numpy(other).to(dev)
    obf = torch.empty_like(d_other, dtype=torch.bfloat16)
    otor = engine.als_otor(d_other, 0.1, engine.OtorWorkspace.create(K, dev), obf)
    gather = obf if gram == "bf16" else d_other
    full = torch.from_numpy(this).to(dev)
    engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, full, gather, otor=otor)
    full = full.cpu().numpy()
    rows = plan.chunks[: plan.n_chunks, 0].cpu().numpy()
    one = torch.ones(1, dtype=torch.int32).pin_memory()
    side = torch.cuda.Stream(device=dev)
    partial = False
    for delay in (1e-3, 5e-4, 2e-3):
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        d_this = torch.from_numpy(this).to(dev)
        torch.cuda.synchronize()
        engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, d_this, gather, otor=otor, cancel=flag)
        time.sleep(delay)
        with torch.cuda.stream(side):
            flag.copy_(one, non_blocking=True)
        torch.cuda.synchronize()
        handed = min(int(plan.work_counter.item()), plan.n_chunks)
        got = d_this.cpu().numpy()
        done, rest = rows[:handed], rows[handed:]
        assert np.array_equal(got[done].view(np.int32), full[done].view(np.int32))
        assert np.array_equal(got[rest].view(np.int32), this[rest].view(np.int32))
        assert int(plan.status.item()) == 0
        if 0 < handed < plan.n_chunks:
            partial = True
            break
    assert partial, "the flag never landed while the launch ran"
