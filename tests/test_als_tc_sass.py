"""
Instructions of the k = 64 tensor-core ALS kernels, from the compiled object's SASS (no device needed).

The k = 64 routes gather their staged rows with per-lane 16-byte cp.async copies (LDGSTS), not with
cp.async.bulk (UBLKCP), whose uniform-register operands turn per-lane calls into a loop that sends one row per
pass.  On the bf16-MMA routes the one warp's B fragments are its A fragments in another order, so a Gram
k-step loads four ldmatrix.x4 (LDSM), not eight.
"""

import os
import re
import subprocess

from lkpy_b200 import _build

# als_tc_kernel<64, ET, MODE, WEIGHTED> (LK_ALS_IMPLICIT = 0, LK_ALS_EXPLICIT = 1)
BF16MMA_K64_ROUTES = {
    "_ZN2lk13als_tc_kernelILi64E13__nv_bfloat16Li0ELb0EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64E13__nv_bfloat16Li1ELb0EEEv11lk_als_args",
}
K64_ROUTES = BF16MMA_K64_ROUTES | {
    "_ZN2lk13als_tc_kernelILi64E13__nv_bfloat16Li0ELb1EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64EfLi0ELb0EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64EfLi0ELb1EEEv11lk_als_args",
    "_ZN2lk13als_tc_kernelILi64EfLi1ELb0EEEv11lk_als_args",
}


def sass_by_function(tmp_path) -> dict:
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    obj = tmp_path / "als_tc.o"
    cmd = [_build._nvcc(), *_build.NVCC_FLAGS, "-ccbin", "/usr/bin/g++",
           "-c", str(_build.CSRC / "als_tc.cu"), "-o", str(obj)]  # fmt: skip
    subprocess.run(cmd, capture_output=True, text=True, env=env, check=True)
    cuobjdump = os.path.join(os.path.dirname(_build._nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r"^\s*Function : ", sass, flags=re.M)[1:]:
        name, body = part.split("\n", 1)
        funcs[name.strip()] = body
    return funcs


def opcodes(body: str, op: str) -> int:
    return len(re.findall(rf"\b{op}\b", body))


def test_k64_gather_and_fragment_loads(tmp_path):
    funcs = sass_by_function(tmp_path)
    assert K64_ROUTES <= set(funcs)
    for name in K64_ROUTES:
        assert opcodes(funcs[name], "UBLKCP") == 0, name
        assert opcodes(funcs[name], "LDGSTS") > 0, name
    # the Gram's k-step loop is compiled once (not unrolled), so its LDSMs are all the function has
    for name in BF16MMA_K64_ROUTES:
        assert opcodes(funcs[name], "LDSM") == 4, name
