"""Register and local-memory report of the cone solver, without a GPU.

1. Compiles csrc/conic_api.cu for sm_90a with `-Xptxas -v` (into a temporary directory) and prints registers, stack,
   spill stores and spill loads of every k_ipm_solve instantiation and of the device functions it calls.
2. Reads the SASS of k_ipm_solve<1024, 0> from a built library or object (default: the package's libscpb.so) and
   counts STL / LDL per subroutine: in total and inside loops.  Subroutines are found by CALL.REL target (their
   extents come from the ELF symbol table); a loop is the range a backward branch jumps over.

    python scripts/spill_report.py                      # both parts, for the tree's sources and library
    python scripts/spill_report.py --no-ptxas --lib X   # SASS part only, of another build
    python scripts/spill_report.py --csrc DIR           # ptxas part for other sources (e.g. a parent commit's)
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "scptoolbox.jl_b200")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
KERNEL = "_Z11k_ipm_solveILi1024ELi0EEv10IpmProgram7IpmData7IpmOpts"   # k_ipm_solve<1024, 0>
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def ptxas_table(csrc: str):
    """[(entry, function, regs or None, stack, spill stores, spill loads)] from `nvcc -Xptxas -v`."""
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([os.path.join(CUDA, "bin", "nvcc")] + NVCC_FLAGS + ["-c", "-Xptxas", "-v",
                           os.path.join(csrc, "conic_api.cu"), "-o", os.path.join(tmp, "conic_api.o")],
                           capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(r.stderr)
    rows, entry, cur = [], None, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            entry = m.group(1)
            continue
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            rows.append([entry, cur, None] + [int(x) for x in m.groups()])
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and rows and rows[-1][1] == entry:
            rows[-1][2] = int(m.group(1))
    return [r for r in rows if r[0] and "k_ipm_solve" in r[0]]


def subroutines(lib: str, kernel: str):
    """{name: (start, end)} of the subroutines of `kernel`, from the ELF symbol table."""
    out = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-elf", lib], capture_output=True, text=True,
                         check=True).stdout
    subs = {}
    pre = "$" + kernel + "$"
    for line in out.splitlines():
        f = line.split()
        if len(f) >= 7 and f[-1].startswith(pre) and f[1].startswith("0x") and f[2].startswith("0x"):
            start, size = int(f[1], 16), int(f[2], 16)
            subs[f[-1][len(pre):]] = (start, start + size)
    return subs


def sass(lib: str, kernel: str):
    """[(address, opcode, operand text)] of `kernel`."""
    out = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", "-fun", kernel, lib], capture_output=True,
                         text=True, check=True).stdout
    ins = []
    for line in out.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);", line)
        if m:
            ins.append((int(m.group(1), 16), m.group(3), m.group(4)))
    return ins


def local_memory_by_subroutine(lib: str, kernel: str = KERNEL):
    """{function: [STL, LDL, STL in loops, LDL in loops]}; the kernel body is listed under its own name."""
    ins = sass(lib, kernel)
    subs = subroutines(lib, kernel)
    called = {int(o.split()[0], 16) for _, op, o in ins if op.startswith("CALL.REL") and o.startswith("0x")}
    subs = {n: r for n, r in subs.items() if r[0] in called}
    loops = []
    for a, op, o in ins:
        if op.startswith("BRA") and o.split() and o.split()[-1].startswith("0x"):
            t = int(o.split()[-1], 16)
            if t <= a:
                loops.append((t, a))

    def owner(a):
        for n, (s, e) in subs.items():
            if s <= a < e:
                return n
        return kernel

    res = {n: [0, 0, 0, 0] for n in [kernel] + sorted(subs, key=lambda n: subs[n][0])}
    for a, op, _ in ins:
        k = 0 if op.startswith("STL") else 1 if op.startswith("LDL") else None
        if k is None:
            continue
        row = res[owner(a)]
        row[k] += 1
        if any(s <= a <= e for s, e in loops):
            row[k + 2] += 1
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--csrc", default=os.path.join(PKG, "csrc"), help="sources to compile for the ptxas table")
    ap.add_argument("--lib", default=os.path.join(PKG, "libscpb.so"), help="built library or object for the SASS table")
    ap.add_argument("--no-ptxas", action="store_true", help="skip the ptxas table (it compiles conic_api.cu)")
    ap.add_argument("--no-sass", action="store_true", help="skip the SASS table")
    a = ap.parse_args()
    if not a.no_ptxas:
        rows = ptxas_table(a.csrc)
        dm = demangle(sorted({r[0] for r in rows} | {r[1] for r in rows}))
        print("ptxas -v (sm_90a)")
        print(f"{'instantiation':<46} {'function':<44} {'regs':>4} {'stack':>6} {'st B':>6} {'ld B':>6}")
        for e, f, regs, st, ss, sl in rows:
            fn = "(body)" if f == e else dm[f].split("(")[0]
            print(f"{dm[e].split('(')[0][5:]:<46} {fn:<44} {regs if regs else '':>4} {st:>6} {ss:>6} {sl:>6}")
    if not a.no_sass:
        if not os.path.exists(a.lib):
            sys.exit(f"{a.lib} does not exist: build the library first")
        res = local_memory_by_subroutine(a.lib)
        dm = demangle(list(res))
        print(f"\nSASS of k_ipm_solve<1024, 0> in {os.path.relpath(a.lib, ROOT)}: local-memory instructions")
        print(f"{'function':<44} {'STL':>5} {'LDL':>5} {'STL in loops':>13} {'LDL in loops':>13}")
        for n, (s, l, sl, ll) in res.items():
            name = "(body)" if n == KERNEL else dm[n].split("(")[0]
            print(f"{name:<44} {s:>5} {l:>5} {sl:>13} {ll:>13}")


if __name__ == "__main__":
    main()
