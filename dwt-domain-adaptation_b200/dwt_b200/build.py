"""Build libdwt_b200.so in-tree with nvcc for sm_90a (no torch headers, no libtorch).

    python dwt-domain-adaptation_b200/dwt_b200/build.py [--force] [--verbose]

The library is a plain C-ABI shared object (include/dwt_b200.h) with a statically linked
CUDA runtime; it cross-compiles on a machine without a GPU.  The built file is git-ignored.
"""
from __future__ import annotations

import os
import shlex
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libdwt_b200.so")
SOURCES = ["api.cu", "norm_small.cu", "norm_tiled.cu", "norm_tc.cu", "norm_tc_apply.cu", "norm_dense.cu", "norm_cl.cu", "norm_ldbn.cu", "mec.cu", "augment.cu", "pool.cu"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]
NVCC_FLAGS += shlex.split(os.environ.get("DWT_NVCC_EXTRA", ""))     # development only, e.g. -DDWT_PROF_DENSE (phase clocks)


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "..", "include", "dwt_b200.h"))
    deps.append(os.path.abspath(__file__))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "lib", src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stdout.write(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {src}")
    link = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", *objs, "-o", LIB]
    subprocess.check_call(link)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
