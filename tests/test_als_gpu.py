"""
GPU parity: ALS half-epoch kernels (through the C ABI) vs the oracle.

Tolerances (SURVEY.md §7, north_star "within 1e-4 relative on ALS factors"):
one half-step from identical inputs, matrix-level relative Frobenius error
against the f64 oracle <= 1e-4, and no worse than 3x the f32 oracle's own
distance to f64 (+1e-6).  bf16-gather runs are compared with an oracle that
rounds the gathered rows to bf16 the same way.
"""

import numpy as np
import pytest
import torch

from pathlib import Path

import oracle
from lkpy_b200 import _lib, data, engine

from helpers import explicit_init, implicit_init, rel_fro, small_synth

pytestmark = pytest.mark.gpu

TOL = 1e-4
GOLD = Path(__file__).resolve().parent / "golden"


@pytest.fixture(autouse=True)
def _simt_for_fp32_rows(lk_options):
    """This file pins the general SIMT kernel (als_kernels.cu) to "as good as f32 arithmetic": fp32 rows at
    k = 64 are kept off the tf32 tensor-core path, which has its own tests and tolerance
    (tests/test_als_rows_gpu.py); bf16 rows at k = 64 still take als_tc.cu."""
    lk_options("LK_ALS_TF32", 0)


def _half(mode, csr, this, other, *, reg, bf16=False, chunk_nnz=engine.DEFAULT_CHUNK_NNZ):
    dev = _lib.require_device()
    dm = engine.DeviceCSR.from_host(csr, dev)
    k = this.shape[1]
    plan = engine.ALSHalfPlan.create(dm, k, chunk_nnz)
    d_this = torch.from_numpy(this.copy()).to(dev)
    d_other = torch.from_numpy(other).to(dev)
    otor = None
    d_gather = d_other
    if mode == "implicit":
        ws = engine.OtorWorkspace.create(k, dev)
        obf = torch.empty_like(d_other, dtype=torch.bfloat16) if bf16 else None
        otor = engine.als_otor(d_other, reg, ws, obf)
        if bf16:
            d_gather = obf
    elif bf16:
        d_gather = d_other.to(torch.bfloat16)
    engine.als_half_epoch(
        plan, _lib.LK_ALS_IMPLICIT if mode == "implicit" else _lib.LK_ALS_EXPLICIT,
        d_this, d_gather, otor=otor, reg=reg,
    )  # fmt: skip
    torch.cuda.synchronize()
    return (
        d_this.cpu().numpy(),
        float(np.sqrt(plan.sqdelta.item())),
        int(plan.status.item()),
        None if otor is None else otor.cpu().numpy(),
        plan,
    )


def _check(mode, csr, this, other, reg, bf16=False, chunk_nnz=engine.DEFAULT_CHUNK_NNZ, tol=TOL, ill_conditioned_ok=False):
    got, delta, status, otor_gpu, plan = _half(mode, csr, this, other, reg=reg, bf16=bf16, chunk_nnz=chunk_nnz)
    assert status == 0
    other_eff = oracle.bf16_round(other) if bf16 else other
    o32, o64 = oracle.otor(other_eff, reg)
    if mode == "implicit":
        assert rel_fro(otor_gpu, o64) < 2e-6
    ref64, d64 = oracle.als_half_f64(mode, csr, this, other, otor_mat=o64, reg=reg, bf16_other=bf16)
    ref32, d32 = oracle.als_half(mode, csr, this, other, otor_mat=o32, reg=reg, bf16_other=bf16)
    e_gpu = rel_fro(got, ref64)
    e_cpu = rel_fro(ref32, ref64)
    # Bar: 1e-4 relative (north_star) wherever f32 arithmetic can deliver it.  With the
    # reference's (0.01 N(0,1))^2 init the early ml-latest-small systems are so
    # ill-conditioned that the f32 *reference arithmetic itself* sits ~1e-3 from f64
    # (SURVEY.md §7); there the bar is "no worse than the f32 oracle".
    if e_cpu <= tol / 3:
        assert e_gpu <= tol, (e_gpu, e_cpu)
    else:
        assert ill_conditioned_ok, (e_gpu, e_cpu)
    assert e_gpu <= 1.5 * e_cpu + 2e-6, (e_gpu, e_cpu)
    assert delta == pytest.approx(d64, rel=1e-3)
    empty = np.diff(csr.indptr) == 0
    assert np.all(got[empty] == 0.0)
    return got, plan


@pytest.mark.parametrize("k", [32, 64])
def test_implicit_half_steps_ml_small(cuda_lib, ml_small, k):
    """Config 1 shape: ml-latest-small, reference init, user step then item step."""
    ui, iu = data.als_implicit_matrices(ml_small, 40.0)
    p, q = implicit_init(np.random.default_rng(42), ml_small.n_items, ml_small.n_users, k)
    # the very first user step sees a tiny Q (1e-4 entries): the systems are reg-dominated
    p1, _ = _check("implicit", ui, p, q, 0.1)
    q1, _ = _check("implicit", iu, q, p1, 0.1, ill_conditioned_ok=True)
    p2, _ = _check("implicit", ui, p1, q1, 0.1, ill_conditioned_ok=True)
    _check("implicit", iu, q1, p2, 0.1, ill_conditioned_ok=True)


def test_explicit_half_steps_ml_small(cuda_lib, ml_small):
    k = 64
    r = ml_small.ratings - ml_small.ratings.mean()
    coo = ml_small.coo(r.astype(np.float32))
    ui = data.InteractionCSR.from_scipy(coo)
    iu = data.InteractionCSR.from_scipy(coo.T)
    p, q = explicit_init(np.random.default_rng(42), ml_small.n_items, ml_small.n_users, k)
    p1, _ = _check("explicit", ui, p, q, 0.1)
    _check("explicit", iu, q, p1, 0.1)


@pytest.mark.parametrize("k", [8, 20, 50, 64, 96, 128])
def test_feature_sizes_and_padding(cuda_lib, k):
    """k not a multiple of 4 takes the non-bulk gather; k < KP is zero-padded."""
    inter = small_synth(500, 300, 12000, seed=k)
    ui, iu = data.als_implicit_matrices(inter, 40.0)
    rng = np.random.default_rng(k)
    p = (rng.standard_normal((500, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((300, k)) * 0.1).astype(np.float32)
    _check("implicit", ui, p, q, 0.1)
    vals = rng.standard_normal(inter.nnz).astype(np.float32)
    ue = data.InteractionCSR.from_scipy(inter.coo(vals))
    _check("explicit", ue, p, q, 0.05)


@pytest.mark.parametrize("mode", ["implicit", "explicit"])
def test_split_rows_are_deterministic(cuda_lib, mode):
    """Rows longer than chunk_nnz go through the partial-Gram path; same bits every run."""
    inter = small_synth(300, 200, 20000, seed=5)
    ui, iu = data.als_implicit_matrices(inter, 40.0)
    rng = np.random.default_rng(5)
    k = 64
    p = (rng.standard_normal((300, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((200, k)) * 0.1).astype(np.float32)
    csr = iu if mode == "implicit" else data.InteractionCSR.from_scipy(
        inter.coo(rng.standard_normal(inter.nnz).astype(np.float32)).T
    )
    a, plan = _check(mode, csr, q, p, 0.1, chunk_nnz=32)
    assert plan.n_split_rows > 0
    b, _ = _check(mode, csr, q, p, 0.1, chunk_nnz=32)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    c, plan2 = _check(mode, csr, q, p, 0.1, chunk_nnz=1 << 20)
    assert plan2.n_split_rows == 0
    assert rel_fro(a, c) < 1e-5


def test_bf16_gather(cuda_lib, ml_small):
    """bf16-gather mode vs an oracle that rounds the gathered rows identically."""
    k = 64
    ui, iu = data.als_implicit_matrices(ml_small, 40.0)
    rng = np.random.default_rng(3)
    p = (rng.standard_normal((ml_small.n_users, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((ml_small.n_items, k)) * 0.1).astype(np.float32)
    _check("implicit", ui, p, q, 0.1, bf16=True)
    _check("implicit", iu, q, p, 0.1, bf16=True)


def test_not_positive_definite_is_reported(cuda_lib):
    inter = small_synth(40, 30, 300, seed=1)
    ui, _ = data.als_implicit_matrices(inter, 40.0)
    dev = _lib.require_device()
    k = 32
    dm = engine.DeviceCSR.from_host(ui, dev)
    plan = engine.ALSHalfPlan.create(dm, k)
    this = torch.zeros((40, k), device=dev)
    other = torch.zeros((30, k), device=dev)
    otor = -torch.eye(k, device=dev)
    engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, this, other, otor=otor)
    torch.cuda.synchronize()
    assert int(plan.status.item()) > 0


def test_accel_api_mirror(cuda_lib, ml_small):
    """lenskit._accel.als signatures: host arrays, `this` mutated in place, float result."""
    from lkpy_b200 import accel

    k = 32
    ui, iu = data.als_implicit_matrices(ml_small, 40.0)
    p, q = implicit_init(np.random.default_rng(42), ml_small.n_items, ml_small.n_users, k)
    o32, o64 = oracle.otor(q, 0.1)
    ref, dref = oracle.als_half_f64("implicit", ui, p, q, otor_mat=o64)
    p_in = p.copy()
    delta = accel.run_accel_task(accel.als.train_implicit_matrix(ui, p_in, q, o32))
    assert isinstance(delta, float)
    assert rel_fro(p_in, ref) < TOL
    assert delta == pytest.approx(dref, rel=1e-3)
    task = accel.als.train_explicit_matrix(ui, p_in, q, 0.1)
    task.invoke()
    with pytest.raises(RuntimeError):
        task.invoke()
    with pytest.raises(TypeError):
        accel.als.train_implicit_matrix(ui, p_in.astype(np.float64), q, o32)
    with pytest.raises(RuntimeError, match="accelerator task failed"):
        accel.run_accel_task(accel.als.train_implicit_matrix(ui, p_in, q, -np.eye(k, dtype=np.float32)))


def test_accel_arrow_matrix_and_live_cancel(cuda_lib, ml_small, lk_options):
    """The matrix argument as the reference passes it — an Arrow List<Struct{index:int32, value:float32}>
    (csr.rs:160-209) — and the task protocol's cancel / progress while the kernel runs (tasks/mod.rs:62-106)."""
    import threading

    import pyarrow as pa

    from lkpy_b200 import accel

    lk_options("LK_ALS_TF32", 1)  # the mirror's default path at k = 64: the tensor-core kernel
    k = 64
    ui, iu = data.als_implicit_matrices(ml_small, 40.0)
    p, q = implicit_init(np.random.default_rng(42), ml_small.n_items, ml_small.n_users, k)
    o32, o64 = oracle.otor(q, 0.1)
    ref, dref = oracle.als_half_f64("implicit", ui, p, q, otor_mat=o64)
    elems = pa.StructArray.from_arrays(
        [pa.array(ui.indices, type=pa.int32()), pa.array(ui.values, type=pa.float32())], names=["index", "value"]
    )
    arrow_ui = pa.ListArray.from_arrays(pa.array(ui.indptr.astype(np.int32)), elems)
    p_in = p.copy()
    task = accel.als.train_implicit_matrix(arrow_ui, p_in, q, o32)
    assert task.current_progress() == (0, ml_small.n_users)
    delta = accel.run_accel_task(task)
    assert rel_fro(p_in, ref) < 2 * TOL and delta == pytest.approx(dref, rel=1e-3)
    assert task.current_progress() == (ml_small.n_users, ml_small.n_users)

    # cancelled before it starts: nothing runs, `this` is untouched
    p_in = p.copy()
    task = accel.als.train_implicit_matrix(arrow_ui, p_in, q, o32)
    task.cancel()
    with pytest.raises(RuntimeError, match="cancelled"):
        task.invoke()
    assert np.array_equal(p_in, p)

    # cancelled while running (a large synthetic half-step; the flag is raised from another thread)
    inter = data.synth_interactions(60000, 20000, 6_000_000, seed=2)
    bui, _ = data.als_implicit_matrices(inter, 40.0)
    rng = np.random.default_rng(0)
    bp = (rng.standard_normal((inter.n_users, k)) * 0.1).astype(np.float32)
    bq = (rng.standard_normal((inter.n_items, k)) * 0.1).astype(np.float32)
    bo = (bq.T @ bq + 0.1 * np.eye(k, dtype=np.float32)).astype(np.float32)
    accel.run_accel_task(accel.als.train_implicit_matrix(bui, bp.copy(), bq, bo))  # upload + plan cached
    task = accel.als.train_implicit_matrix(bui, bp.copy(), bq, bo)
    seen = []

    def killer():
        while not task._invoked or task._counter is None:
            pass
        seen.append(task.current_progress())
        task.cancel()

    th = threading.Thread(target=killer)
    th.start()
    try:
        task.invoke()
        outcome = "finished"  # the kernel can beat the flag on a fast GPU: both outcomes are legal
    except RuntimeError as e:
        assert "cancelled" in str(e)
        outcome = "cancelled"
    th.join()
    assert outcome in ("finished", "cancelled") and isinstance(seen[0], tuple) and seen[0][1] == inter.n_users


@pytest.mark.parametrize("tf32", [0, 1])
def test_row_solves_match_reference_fold_in_vectors(cuda_lib, lk_options, tf32):
    """tests/golden/als_ref_rows.npz holds outputs of the REFERENCE's own fold-in code
    (_train_new_row als/_implicit.py:91-130, _train_bias_row_cholesky als/_explicit.py:121-147, run from the
    reference source by make_golden.py): the device row solve reproduces them for k = 8 .. 128, on the SIMT
    kernel and (k = 64) on the tensor-core kernel."""
    lk_options("LK_ALS_TF32", tf32)
    z = np.load(GOLD / "als_ref_rows.npz")
    dev = _lib.require_device()
    for c in range(int(z["n_cases"])):
        g = lambda name: z[f"c{c}_{name}"]  # noqa: E731
        k, other, items = int(g("k")), g("other"), g("items").astype(np.int32)
        order = np.argsort(items, kind="stable")
        for mode, vals, want in (("implicit", g("conf"), g("x_implicit")), ("explicit", g("rates"), g("x_explicit"))):
            csr = data.InteractionCSR(
                np.array([0, len(items)], dtype=np.int32), items[order], vals[order].astype(np.float32), (1, other.shape[0])
            )
            plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), k)
            x = torch.zeros((1, k), device=dev)
            d_other = torch.from_numpy(other).to(dev)
            otor = torch.from_numpy(g("otor")).to(dev) if mode == "implicit" else None
            engine.als_half_epoch(
                plan, _lib.LK_ALS_IMPLICIT if mode == "implicit" else _lib.LK_ALS_EXPLICIT, x, d_other,
                otor=otor, reg=float(g("reg")),
            )  # fmt: skip
            torch.cuda.synchronize()
            assert int(plan.status.item()) == 0
            got = x.cpu().numpy()[0]
            assert rel_fro(got, want) < 1e-4, (c, mode, k, rel_fro(got, want))
