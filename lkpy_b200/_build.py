"""
In-tree build of the CUDA library ``lkpy_b200/csrc/liblkpy_b200.so`` for sm_90a (H100).

``nvcc`` cross-compiles without a GPU, so this runs in the CPU build container;
the resulting ``.so`` is git-ignored but travels to the GPU box with the tree.
"""

from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
LIB = CSRC / "liblkpy_b200.so"
SOURCES = ["capi.cu", "als_kernels.cu", "als_tc.cu", "knn_build.cu", "knn_score.cu", "knn_user.cu", "topn.cu", "prep.cu",
           "als_recommend.cu", "cooc.cu", "ease.cu", "slim.cu", "flexmf.cu",
           "spmm.cu", "nmf.cu", "basic.cu", "stochastic.cu", "fair.cu", "metrics.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17", "--extended-lambda",
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
]  # fmt: skip


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def _stale() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = [CSRC / s for s in SOURCES] + [
        CSRC / "common.cuh", CSRC / "als_common.cuh", CSRC / "topn_heap.cuh", CSRC / "tiles.cuh", CSRC / "pairwise.cuh",
    ]  # fmt: skip
    deps.append(CSRC.parent.parent / "include" / "lkpy_b200.h")
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not _stale():
        return LIB
    # one builder at a time: the ranks of a torchrun launch all import this module, and a stale library
    # must not be rebuilt by eight processes into the same object files
    import fcntl

    CSRC.joinpath("build").mkdir(exist_ok=True)
    with open(CSRC / "build" / ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not _stale():  # another process built it while this one waited
                return LIB
            return _build_locked(verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose: bool) -> Path:
    nvcc = _nvcc()
    objdir = CSRC / "build"
    objdir.mkdir(exist_ok=True)
    env = dict(os.environ)
    # the image's CC/CXX point at a wrapper without OpenMP specs; nvcc wants the system g++
    env.pop("CC", None)
    env.pop("CXX", None)

    def one(src: str) -> Path:
        obj = objdir / (src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-ccbin", "/usr/bin/g++", "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        subprocess.run(cmd, check=True, env=env)
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(one, SOURCES))
    tmp = LIB.with_suffix(".so.tmp")
    cmd = [nvcc, "-shared", "-Wno-deprecated-gpu-targets", "-ccbin", "/usr/bin/g++", "-o", str(tmp), *map(str, objs)]
    subprocess.run(cmd, check=True, env=env)
    os.replace(tmp, LIB)  # readers never see a half-written library
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
