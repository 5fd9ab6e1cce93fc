"""Local memory inside the loops of the 1024-thread interior-point kernel, read from the built library's SASS (no GPU,
no rebuild).  At 1024 threads a CTA has 64 registers per thread, and a subroutine called inside the solver's loops gets
fewer.  A value spilled inside a level or pass loop costs a local-memory round trip per pass, and local memory mostly
misses the L1 that the kernel's shared memory leaves over.

The substitution sweeps hold no local memory inside their loops but one load; the bounds for the factorisation (four
inlined copies, one per group size) and for the solver body are the counts of sm_90a code from CUDA 12.9's ptxas.  They
catch a change that pushes the level programs or the body back into local memory: with by-value argument blocks and
per-thread profile counters the sweeps had 12 and 6 such instructions, the single factorisation 71, the body 1 496."""
import importlib.util
import os
import shutil

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scptoolbox.jl_b200", "libscpb.so")
FACTOR = "_Z17kkt_factor_levelsv"
FORWARD, BACKWARD = "_Z11solve_sweepILi1EEvv", "_Z11solve_sweepILin1EEvv"


def _report():
    spec = importlib.util.spec_from_file_location("spill_report", os.path.join(ROOT, "scripts", "spill_report.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    if not os.path.exists(LIB):
        pytest.skip("libscpb.so is not built")
    if not os.path.exists(os.path.join(m.CUDA, "bin", "cuobjdump")) and not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    return m.local_memory_by_subroutine(LIB), m.KERNEL


def test_level_programs_take_no_argument_block():
    res, _ = _report()
    assert {FACTOR, FORWARD, BACKWARD} <= set(res), sorted(res)


def test_in_loop_local_memory_of_the_1024_thread_kernel():
    res, kernel = _report()
    in_loops = {n: r[2] + r[3] for n, r in res.items()}
    assert in_loops[FORWARD] == 0, in_loops
    assert in_loops[BACKWARD] <= 1, in_loops
    assert in_loops[FACTOR] <= 125, in_loops
    assert in_loops[kernel] <= 1188, in_loops
