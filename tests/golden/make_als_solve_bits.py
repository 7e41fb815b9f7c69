#!/usr/bin/env python
"""
Record ``als_solve_bits.npz``: the exact f32 bits of factor rows, and the status word, that one ALS half-step
leaves on every route whose systems the one-warp Cholesky (``chol_solve_warp``) factors:

* ``als_tc_kernel`` at k = 64 with bf16 and fp32 rows, implicit with a uniform confidence, implicit with
  per-nonzero confidences, and explicit;
* the SIMT kernel (``LK_ALS_TC=0``) at k = 32 and 64 (KP = 32 and 64), in the same three modes.

Each problem is generated from a seed (``problem``) and holds empty rows, rows shorter than k, rows split over
several parts and rows whose system is nearly singular.  ``tests/test_als_solve_bits_gpu.py`` regenerates the
problems and requires the same bits, so a change to the solve that reorders one floating-point operation is
caught.  The bits depend on the CUDA toolchain (recorded with CUDA 12.9 for sm_90a); re-record them when the
toolchain changes, from a commit whose solve is trusted.

Run on a GPU from the repository root: ``python tests/golden/make_als_solve_bits.py``.
"""

from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
OUT = Path(__file__).resolve().parent / "als_solve_bits.npz"

N_OTHER = 1000
N_COLLINEAR = 100  #: the last rows of `other`, whose last two features nearly coincide
CHUNK = 64
REG_IMPLICIT = 0.1
REG_EXPLICIT = 1e-3
UNIFORM_CONF = 40.0
#: rows shorter than k, at the kernels' 8-, 16- and 32-row steps, and rows of 2 to 5 parts of CHUNK
LENGTHS = (1, 2, 3, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 40, 63, 64, 65, 100, 128, 129, 200, 300)
N_EMPTY = 4
N_NEAR_SINGULAR = 3
N_RANDOM = 120

ROUTES = {
    "tc64_bf16": dict(k=64, bf16=True, opts={"LK_ALS_TC": 1, "LK_ALS_TF32": 1}),
    "tc64_f32": dict(k=64, bf16=False, opts={"LK_ALS_TC": 1, "LK_ALS_TF32": 1}),
    "simt32": dict(k=32, bf16=False, opts={"LK_ALS_TC": 0}),
    "simt64": dict(k=64, bf16=False, opts={"LK_ALS_TC": 0}),
}
KINDS = ("uniform", "weighted", "explicit")


def cases():
    for route in ROUTES:
        for kind in KINDS:
            yield f"{route}_{kind}", route, kind


def problem(k: int, kind: str, seed: int = 0):
    """(csr, this, other, reg): the seeded problem for feature count k and mode kind."""
    from lkpy_b200 import data

    rng = np.random.default_rng([seed, k, KINDS.index(kind), 2026])
    other = (rng.standard_normal((N_OTHER, k)) * 0.5).astype(np.float32)
    c = other[N_OTHER - N_COLLINEAR :]
    c[:, k - 1] = c[:, k - 2] + (rng.standard_normal(N_COLLINEAR) * 1e-3).astype(np.float32)

    lens = list(LENGTHS) + [0] * N_EMPTY
    lens += np.minimum(np.round(rng.lognormal(2.5, 1.25, N_RANDOM)), 400).astype(int).tolist()
    cols = []
    for n in lens:
        cols.append(np.sort(rng.choice(N_OTHER - N_COLLINEAR, n, replace=False)))
    for _ in range(N_NEAR_SINGULAR):  # explicit: nearly singular Gram; implicit: OtOr keeps it well posed
        n = int(rng.integers(2 * k, 3 * k))
        cols.append(np.sort(rng.choice(np.arange(N_OTHER - N_COLLINEAR, N_OTHER), min(n, N_COLLINEAR), replace=False)))
        lens.append(len(cols[-1]))
    order = rng.permutation(len(lens))
    lens = [lens[i] for i in order]
    cols = [cols[i] for i in order]
    indices = np.concatenate(cols).astype(np.int32)
    nnz = len(indices)
    if kind == "uniform":
        vals = np.full(nnz, UNIFORM_CONF, dtype=np.float32)
    elif kind == "weighted":
        vals = rng.uniform(0.5, 40.0, nnz).astype(np.float32)
    else:
        vals = rng.standard_normal(nnz).astype(np.float32)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    csr = data.InteractionCSR(indptr, indices, vals, (len(lens), N_OTHER))
    this = (rng.standard_normal((len(lens), k)) * 0.1).astype(np.float32)
    reg = REG_EXPLICIT if kind == "explicit" else REG_IMPLICIT
    return csr, this, other, reg


def run(route: str, kind: str, set_option) -> tuple[np.ndarray, int]:
    """One half-step of `route` on its problem: (factor rows as int32 bits, status word)."""
    import torch

    import oracle
    from lkpy_b200 import _lib, engine

    r = ROUTES[route]
    k, bf16 = r["k"], r["bf16"]
    for name, value in r["opts"].items():
        set_option(name, value)
    csr, this, other, reg = problem(k, kind)
    dev = _lib.require_device()
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), k, CHUNK)
    assert plan.n_split_rows > 0
    d_this = torch.from_numpy(this.copy()).to(dev)
    src = torch.from_numpy(other).to(dev)
    if bf16:
        src = src.to(torch.bfloat16)
    otor = None
    if kind != "explicit":
        o32, _ = oracle.otor(oracle.bf16_round(other) if bf16 else other, reg)
        otor = torch.from_numpy(o32).to(dev)
    mode = _lib.LK_ALS_EXPLICIT if kind == "explicit" else _lib.LK_ALS_IMPLICIT
    engine.als_half_epoch(plan, mode, d_this, src, otor=otor, reg=reg)
    torch.cuda.synchronize()
    return d_this.cpu().numpy().view(np.int32).copy(), int(plan.status.item())


def main() -> None:
    sys.path.insert(0, str(ROOT))
    from lkpy_b200 import _build, _lib

    _build.build()
    _lib.lib()
    saved = {}

    def set_option(name, value):
        saved.setdefault(name, _lib.get_option(name))
        _lib.set_option(name, value)

    out = {}
    for name, route, kind in cases():
        bits, status = run(route, kind, set_option)
        for n, v in saved.items():
            _lib.set_option(n, v)
        out[f"{name}_x"] = bits
        out[f"{name}_status"] = np.array(status, dtype=np.int64)
        print(name, bits.shape, "status", status)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
