"""A row solve whose pivot is exactly zero (not NaN) must be reported and leave its row untouched.

Explicit mode with reg = 0 makes the system the bare Gram.  Gathered rows of `other` that are zero from
feature `f0` on give a Gram whose rows and columns from f0 on are exactly zero, so the factorisation meets
a zero pivot at column f0 (columns 0, the middle of a panel, and the last column are tried).  Every other
row gathers enough random rows to be well conditioned and must still be solved.
"""

from __future__ import annotations

import numpy as np
import pytest
import torch

from lkpy_b200 import _lib, data, engine

ROUTES = [
    pytest.param(32, False, {"LK_ALS_TC": 0}, id="simt-k32"),
    pytest.param(64, False, {"LK_ALS_TC": 0}, id="simt-k64"),
    pytest.param(64, True, {"LK_ALS_TC": 1, "LK_ALS_TF32": 1}, id="bf16mma-k64"),
    pytest.param(64, False, {"LK_ALS_TC": 1, "LK_ALS_TF32": 1}, id="tf32-k64"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("k,bf16,opts", ROUTES)
@pytest.mark.parametrize("where", ["first", "mid", "last"])
def test_zero_pivot_row_is_reported_and_untouched(cuda_lib, lk_options, k, bf16, opts, where):
    for name, v in opts.items():
        lk_options(name, v)
    f0 = {"first": 0, "mid": k // 2 + 3, "last": k - 1}[where]
    rng = np.random.default_rng([k, f0, 11])
    n_good, n_other, per_row = 40, 400, 3 * k
    other = (rng.standard_normal((n_other + 8, k)) * 0.5).astype(np.float32)
    other[n_other:, f0:] = 0.0  # the last 8 rows of `other` span only features 0 .. f0-1
    bad_row = 17
    cols, vals, indptr = [], [], [0]
    for r in range(n_good + 1):
        if r == bad_row:
            c = np.arange(n_other, n_other + 8)
        else:
            c = np.sort(rng.choice(n_other, per_row, replace=False))
        cols.append(c)
        vals.append(rng.uniform(1.0, 5.0, len(c)).astype(np.float32))
        indptr.append(indptr[-1] + len(c))
    csr = data.InteractionCSR(np.array(indptr, np.int32), np.concatenate(cols).astype(np.int32),
                              np.concatenate(vals), (n_good + 1, n_other + 8))  # fmt: skip
    this = (rng.standard_normal((n_good + 1, k)) * 0.1).astype(np.float32)

    dev = _lib.require_device()
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), k, 1024)
    d_this = torch.from_numpy(this.copy()).to(dev)
    src = torch.from_numpy(other).to(dev)
    if bf16:
        src = src.to(torch.bfloat16)
    engine.als_half_epoch(plan, _lib.LK_ALS_EXPLICIT, d_this, src, reg=0.0)
    torch.cuda.synchronize()
    got = d_this.cpu().numpy()

    assert int(plan.status.item()) == bad_row + 1
    assert np.array_equal(got[bad_row].view(np.int32), this[bad_row].view(np.int32))
    # the other rows: A x = O^T v with the (bf16-rounded) gathered rows, in f64
    o = src.float().cpu().numpy().astype(np.float64)
    for r in range(n_good + 1):
        if r == bad_row:
            continue
        c, v = csr.indices[csr.indptr[r] : csr.indptr[r + 1]], csr.values[csr.indptr[r] : csr.indptr[r + 1]]
        x = np.linalg.solve(o[c].T @ o[c], o[c].T @ v.astype(np.float64))
        assert np.linalg.norm(got[r] - x) <= 1e-3 * np.linalg.norm(x), r
