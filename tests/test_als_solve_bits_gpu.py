"""
The one-warp ALS row solve (``chol_solve_warp``) keeps its results bit for bit.

ALS carries small differences from epoch to epoch, so a solve that reorders one floating-point operation moves
the benchmark's factors measurably after a few dozen epochs.  The other ALS tests check a tolerance against the
oracle and reproducibility within one build; this one pins the exact bits across changes to the solve.
``tests/golden/make_als_solve_bits.py`` generated the seeded problems and recorded ``als_solve_bits.npz``: the
factor rows and status word one half-step leaves on the k = 64 tensor-core kernel (bf16 and fp32 rows) and on
the SIMT kernel at KP = 32 and 64, in implicit uniform, implicit weighted and explicit mode.  The problems hold
empty rows, rows shorter than k, split rows and nearly singular systems.

The recorded bits are those of nvcc from CUDA 12.9 for sm_90a; a different toolchain may contract or schedule
the same source differently, and the fixture is then re-recorded from a commit whose solve is trusted.
"""

from __future__ import annotations

import importlib.util
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

_GOLDEN = Path(__file__).resolve().parent / "golden"
_spec = importlib.util.spec_from_file_location("make_als_solve_bits", _GOLDEN / "make_als_solve_bits.py")
bits = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(bits)


@pytest.fixture(scope="module")
def golden():
    with np.load(bits.OUT) as z:
        return {name: z[name] for name in z.files}


@pytest.mark.parametrize("name,route,kind", [pytest.param(*c, id=c[0]) for c in bits.cases()])
def test_solve_bits_match_recording(cuda_lib, lk_options, golden, name, route, kind):
    got, status = bits.run(route, kind, lk_options)
    want = golden[f"{name}_x"]
    assert status == int(golden[f"{name}_status"])
    diff = np.flatnonzero(np.any(got != want, axis=1))
    assert diff.size == 0, f"{name}: {diff.size} of {len(want)} rows differ in their bits, first rows {diff[:8].tolist()}"
