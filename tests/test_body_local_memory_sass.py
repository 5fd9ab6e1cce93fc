"""Local memory of the 1024-thread interior-point kernel's body and of its sparse products, read from the built library's
SASS (no GPU, no rebuild).

The body reads its group's array bases from shared memory where it uses them (IpmGroup), instead of holding 39 64-bit
bases per thread in a stack frame, and the residual and KKT sparse products are separate subroutines with several loads
in flight.  Before that the body held 98 STL / 1 090 LDL inside loops and the factorisation 30 / 95.  The bounds are the
counts of sm_90a code from CUDA 12.9's ptxas.  The sparse products' gathers in flight must not be spilled: three of the
products hold no local memory inside their loops, the other two reload a few 64-bit values once per row, outside the
loops over a row's entries."""
import importlib.util
import os
import shutil

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scptoolbox.jl_b200", "libscpb.so")
FACTOR = "_Z17kkt_factor_levelsv"
SPMV = ("spmv_residuals", "spmv_kkt_rhs", "spmv_kkt_gdx<false>", "spmv_kkt_gdx<true>", "spmv_kkt_refine")


def _report():
    spec = importlib.util.spec_from_file_location("spill_report", os.path.join(ROOT, "scripts", "spill_report.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    if not os.path.exists(LIB):
        pytest.skip("libscpb.so is not built")
    if not os.path.exists(os.path.join(m.CUDA, "bin", "cuobjdump")) and not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    res = m.local_memory_by_subroutine(LIB)
    names = {n: m.demangle([n])[n].split("(")[0].replace("void ", "") for n in res}
    return res, names, m.KERNEL


BOUND = {"spmv_residuals": 3, "spmv_kkt_refine": 12}   # in-loop LDL; every other product: none


def test_sparse_products_are_subroutines_with_little_in_loop_local_memory():
    res, names, _ = _report()
    by_name = {names[n]: r for n, r in res.items()}
    assert set(SPMV) <= set(by_name), sorted(by_name)
    for f in SPMV:
        assert by_name[f][2] == 0 and by_name[f][3] <= BOUND.get(f, 0), (f, by_name[f])


def test_body_and_factorisation_in_loop_local_memory():
    res, _, kernel = _report()
    assert res[kernel][2] <= 96 and res[kernel][3] <= 377, res[kernel]
    assert res[FACTOR][2] + res[FACTOR][3] <= 37, res[FACTOR]
