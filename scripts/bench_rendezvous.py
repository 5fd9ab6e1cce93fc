"""Time the planar-rendezvous homotopy sweep (test/examples/rendezvous_planar/tests.jl:60-79: PTR, IMPULSE, N = 30,
Nsub = 10, ten kappa steps, each warm-started from the previous one) for a batch of seeded guesses on the GPU.

    python scripts/bench_rendezvous.py [--batch 256] [--repeats 3] [--chunks N]

The guesses are oracle/rendezvous.perturbed_guesses (seed --seed), the ones the GPU tests use.  Prints one JSON line: SCP
iterations per second (PTR iterations summed over seeds and steps, over the device time of the whole sweep, CUDA events
recorded on the library's stream), the per-step iteration counts, and the card name and power limit read in the same run.  Writes nothing in the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                      # noqa: BLE001
        pl = f"unavailable ({e})"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=3, help="timed sweeps (after one warm-up sweep)")
    ap.add_argument("--chunks", type=int, default=None, help="SCPB_PTR_CHUNKS for the run (default: the library's)")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if a.chunks is not None:
        os.environ["SCPB_PTR_CHUNKS"] = str(a.chunks)
    import torch
    import __graft_entry__ as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU path only")
    pkg = g.load_package()
    ex = pkg.examples.rendezvous_planar
    h = pkg.Handle(0)
    N = 30
    traj = pkg.problem.TrajectoryProblem(ex.PlanarRendezvousProblem())
    ex.define_problem(traj, "ptr")
    pbm = pkg.ptr.create(ex.ptr_parameters(N=N), traj, h)
    # the seeded perturbations of the straight-line guess that the GPU tests use (inputs only: nothing else of the
    # oracle runs here)
    from oracle.rendezvous import PlanarRendezvousProblem, perturbed_guesses
    X, U, P = perturbed_guesses(PlanarRendezvousProblem(N), a.batch, a.seed)
    stream = torch.cuda.ExternalStream(h.stream)
    runs = []
    for r in range(1 + a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        sols = ex.homotopy_sweep(pbm, (X, U, P))
        e1.record(stream)
        e1.synchronize()
        wall = time.perf_counter() - t0
        dev = e0.elapsed_time(e1) * 1e-3
        its = [int(s.iterations.sum()) for s in sols]
        runs.append(dict(device_s=dev, wall_s=wall, iterations=its,
                         solved_last_step=int(sum(st == "SCP_SOLVED" for st in sols[-1].status)),
                         max_iterations_per_step=[int(s.iterations.max()) for s in sols],
                         ipm_iterations=int(sum(s.timing["ipm_iterations"] for s in sols))))
    pbm.close()
    h.close()
    timed = runs[1:]
    rate = [sum(r["iterations"]) / r["device_s"] for r in timed]
    name, power = card()
    print(json.dumps({"metric": "SCP iterations/s (planar rendezvous homotopy sweep, 10 steps)", "value": float(np.median(rate)),
                      "unit": "SCP iterations/s", "all_runs": rate, "batch": a.batch, "N": N, "Nsub": 10,
                      "chunks": os.environ.get("SCPB_PTR_CHUNKS", "library default"),
                      "scp_iterations_per_step": timed[-1]["iterations"],
                      "max_iterations_per_step": timed[-1]["max_iterations_per_step"],
                      "solved_last_step": timed[-1]["solved_last_step"], "device_seconds": [r["device_s"] for r in timed],
                      "wall_seconds": [r["wall_s"] for r in timed], "ipm_iterations": timed[-1]["ipm_iterations"],
                      "gpu": name, "power_limit_and_max_sm_clock": power}))


if __name__ == "__main__":
    main()
