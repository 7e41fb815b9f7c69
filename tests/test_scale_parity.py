"""
Parity at the benchmark's own shape (ML-25M-shaped synthetic, SURVEY.md §8d): the rows the small
fixtures cannot exercise — 80 k-nonzero item rows split into 20 parts, empty users, rows shorter than k,
the three-half kNN geometry, the hottest item — compared with the oracle on a row sample
(oracle/parity.py; the same checks bench.py emits in its `parity` object).
"""

import numpy as np
import pytest
import torch

from lkpy_b200 import _lib, data, engine
from oracle import parity

pytestmark = pytest.mark.gpu

K, WEIGHT, REG = 64, 40.0, 0.1


@pytest.fixture(scope="module")
def ml25m():
    import os

    return data.synth_interactions_cached(os.environ.get("LK_BENCH_DATA_CACHE"), **data.ML25M_SHAPE)


@pytest.mark.parametrize("gather", ["bf16", "fp32"])
def test_als_half_steps_at_ml25m_shape(cuda_lib, ml25m, gather):
    dev = _lib.require_device()
    ui, iu = data.als_implicit_matrices(ml25m, WEIGHT)
    rng = np.random.default_rng(1234)
    p0 = (rng.standard_normal((ml25m.n_users, K)) * 0.1).astype(np.float32)
    q0 = (rng.standard_normal((ml25m.n_items, K)) * 0.1).astype(np.float32)
    ws = engine.OtorWorkspace.create(K, dev)
    for which, csr, this0, other0 in (("user", ui, p0, q0), ("item", iu, q0, p0)):
        plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), K)
        if which == "item":
            assert plan.n_split_rows > 0  # the hot items are split (20 parts for the hottest)
        d_this = torch.from_numpy(this0).to(dev)
        d_other = torch.from_numpy(other0).to(dev)
        obf = torch.empty_like(d_other, dtype=torch.bfloat16) if gather == "bf16" else None
        otor = engine.als_otor(d_other, REG, ws, obf)
        engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, d_this, obf if obf is not None else d_other, otor=otor)
        torch.cuda.synchronize()
        assert int(plan.status.item()) == 0
        rows = parity.sample_als_rows(csr.indptr, K, engine.DEFAULT_CHUNK_NNZ, seed=7)
        got = d_this[torch.from_numpy(rows).to(dev)].cpu().numpy()
        r = parity.check_als_half("implicit", csr, rows, this0[rows], other0, got, REG, gather == "bf16")
        assert r["ok"], r
        assert r["rel_fro_vs_f64_oracle"] < 1e-4  # north-star tolerance, against the f64 oracle
        if which == "user":
            assert r["empty_rows"] > 0 and r["rows_shorter_than_k"] > 0
        del plan, d_this, d_other
        torch.cuda.empty_cache()


@pytest.mark.parametrize("gather", ["bf16", "fp32"])
def test_als_item_half_step_k128_at_ml25m_shape(cuda_lib, ml25m, gather):
    """features = 128 (BASELINE configs[3]'s width) on the long item rows of the ML-25M shape: the
    tensor-core Gram of als_tc.cu (bf16 MMAs for bf16 rows, tf32 x3 for fp32 rows), parts as long as the trainers plan them (ALSTrainerBase._chunk_nnz)."""
    dev = _lib.require_device()
    k = 128
    _ui, iu = data.als_implicit_matrices(ml25m, WEIGHT)
    rng = np.random.default_rng(99)
    p0 = (rng.standard_normal((ml25m.n_users, k)) * 0.1).astype(np.float32)
    q0 = (rng.standard_normal((ml25m.n_items, k)) * 0.1).astype(np.float32)
    chunk = engine.TF32_CHUNK_NNZ if gather == "bf16" else engine.TF32_CHUNK_NNZ_K128
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(iu, dev), k, chunk)
    assert plan.n_split_rows > 0
    d_this, d_other = torch.from_numpy(q0).to(dev), torch.from_numpy(p0).to(dev)
    obf = torch.empty_like(d_other, dtype=torch.bfloat16) if gather == "bf16" else None
    otor = engine.als_otor(d_other, REG, engine.OtorWorkspace.create(k, dev), obf)
    engine.als_half_epoch(plan, _lib.LK_ALS_IMPLICIT, d_this, obf if obf is not None else d_other, otor=otor)
    torch.cuda.synchronize()
    assert int(plan.status.item()) == 0
    rows = parity.sample_als_rows(iu.indptr, k, chunk, n_random=300, seed=11, max_nnz=20_000, n_split=24)
    got = d_this[torch.from_numpy(rows).to(dev)].cpu().numpy()
    r = parity.check_als_half("implicit", iu, rows, q0[rows], p0, got, REG, gather == "bf16")
    assert r["ok"] and r["rel_fro_vs_f64_oracle"] < 1e-4, r


def test_knn_build_rows_at_ml25m_shape(cuda_lib, ml25m):
    dev = _lib.require_device()
    kui, kiu, _ = data.knn_item_matrices(ml25m, True)
    plan = engine.KnnBuildPlan.create(engine.DeviceCSR.from_host(kui, dev), engine.DeviceCSR.from_host(kiu, dev))
    assert plan.geom.n_halves >= 2  # 59,047 f32 accumulators do not fit one CTA's shared memory
    cols, vals, cnt = plan.build_topk(1e-6, 20)
    indptr, c, v = engine.topk_rows_to_csr(cols, vals, cnt)
    cost = plan.cost.cpu().numpy()
    rows = parity.sample_knn_rows(cost, np.diff(kiu.indptr), seed=3)
    r = parity.check_knn_rows(kui, kiu, rows, indptr.cpu().numpy(), c.cpu().numpy(), v.cpu().numpy(), 1e-6, 20)
    assert r["ok"], r
    assert int(np.argmax(cost)) in rows  # the hottest item is part of the sample
