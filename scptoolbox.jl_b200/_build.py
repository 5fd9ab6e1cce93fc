"""Build libscpb.so (sm_90a, H100) in-tree with nvcc.  Called by __graft_entry__.build()."""
from __future__ import annotations

import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libscpb.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def stale() -> bool:
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + \
        glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", SO] + sources()
    subprocess.check_call(cmd)
    return SO
