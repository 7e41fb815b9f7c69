"""
Registers and spills of the k = 64 tensor-core ALS kernels, from ptxas (no device needed).

The benchmark's route (bf16 rows, implicit feedback, uniform confidence) runs 16 one-warp CTAs per SM, so it
must fit 65,536 / (16 x 32) = 128 registers per thread; it may keep the single 4-byte spill it has outside the
Gram and solve loops.  The other k = 64 routes do not spill.
"""

import os
import re
import subprocess

from lkpy_b200 import _build

# als_tc_kernel<64, ET, MODE, WEIGHTED> (LK_ALS_IMPLICIT = 0, LK_ALS_EXPLICIT = 1)
BENCH_ROUTE = "_ZN2lk13als_tc_kernelILi64E13__nv_bfloat16Li0ELb0EEEv11lk_als_args"
OTHER_K64_ROUTES = {
    "_ZN2lk13als_tc_kernelILi64E13__nv_bfloat16Li0ELb1EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64E13__nv_bfloat16Li1ELb0EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64EfLi0ELb0EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64EfLi0ELb1EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64EfLi1ELb0EEEv11lk_als_args",
}
BENCH_CTAS_PER_SM = 16


def ptxas_usage(tmp_path) -> dict:
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    cmd = [_build._nvcc(), *_build.NVCC_FLAGS, "-Xptxas", "-v", "-ccbin", "/usr/bin/g++",
           "-c", str(_build.CSRC / "als_tc.cu"), "-o", str(tmp_path / "als_tc.o")]  # fmt: skip
    out = subprocess.run(cmd, capture_output=True, text=True, env=env, check=True).stderr
    usage, name = {}, None
    for line in out.splitlines():
        if m := re.search(r"Compiling entry function '(\w+)'", line):
            name = m.group(1)
            usage[name] = {}
        elif name and (m := re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)):
            usage[name]["spill"] = (int(m.group(1)), int(m.group(2)))
        elif name and (m := re.search(r"Used (\d+) registers", line)):
            usage[name]["regs"] = int(m.group(1))
    return usage


def test_k64_register_budget_and_spills(tmp_path):
    usage = ptxas_usage(tmp_path)
    assert {BENCH_ROUTE} | OTHER_K64_ROUTES <= set(usage)
    bench = usage[BENCH_ROUTE]
    assert bench["regs"] <= 65536 // (32 * BENCH_CTAS_PER_SM), bench
    assert bench["spill"][0] <= 4 and bench["spill"][1] <= 4, bench
    for name in OTHER_K64_ROUTES:
        assert usage[name]["spill"] == (0, 0), (name, usage[name])
