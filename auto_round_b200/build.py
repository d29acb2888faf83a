"""Build libar_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

    python -m auto_round_b200.build [--force]

nvcc cross-compiles for sm_90a (H100) without a GPU.  The objects and the .so are build products (git-ignored);
they are rebuilt when a source, a header or this file (the flags) is newer.  `-fmad=false`: the fake-quant numerics must not be contracted into FMAs (bit-exact parity
with the reference's separate mul/add/div ops, see csrc/ar_qdq_math.cuh).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB = os.path.join(CSRC, "libar_b200.so")
SOURCES = ["ar_capi.cu", "ar_qdq.cu", "ar_pack.cu", "ar_loop.cu", "ar_block.cu", "ar_search.cu", "ar_outlier.cu", "ar_moe.cu", "ar_gemm.cu"]
HEADERS = ["ar_common.cuh", "ar_qdq_math.cuh", os.path.join("..", "..", "include", "ar_b200.h")]
NVCC_FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false",
              "-Xcompiler", "-fPIC", "-diag-suppress", "177"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_library(force: bool = False, verbose: bool = False) -> str:
    # the flags live in this file: editing it rebuilds everything
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    objs, jobs = [], []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(CSRC, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            jobs.append([_nvcc(), *NVCC_FLAGS, "-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout + r.stderr)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(run, jobs))
    if jobs or force or _stale(LIB, objs):
        run([_nvcc(), "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"])
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
