"""Time a sweep of the in-loop homotopy update threshold beta as ONE batch on the GPU: the planar rendezvous (PTR,
IMPULSE, N = 30, Nsub = 10, iter_max = 30) with kappa stepped through Homotopy(1e-3; delta_max = 5)(LinRange(0, 1, 10))
inside each solve by the schedule of examples/rendezvous_planar.homotopy_schedule, every seed from the straight-line
guess with its own beta = LinRange(0.1, 30, B) / 100 (the thresholds of the reference's test_homotopy_update,
test/examples/rendezvous_3d/tests.jl:189-231, at batch size B).

    python scripts/bench_rendezvous_schedule.py [--batch 256] [--repeats 3] [--chunks N]

Prints one JSON line: SCP iterations per second (PTR iterations summed over the seeds, over the device time of the solve,
CUDA events recorded on the library's stream), the iteration and grid-index spread, and the card name and power limit read
in the same run.  Writes nothing in the tree."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_rendezvous import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=3, help="timed solves (after one warm-up solve)")
    ap.add_argument("--chunks", type=int, default=None, help="SCPB_PTR_CHUNKS for the run (default: the library's)")
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
    ex.homotopy_schedule(traj, beta=0.1)
    pbm = pkg.ptr.create(ex.ptr_parameters(N=N), traj, h)
    betas = np.linspace(0.1, 30, a.batch) / 100
    x0, u0, p0 = traj.guess(N)
    G = (np.repeat(x0[None], a.batch, 0), np.repeat(u0[None], a.batch, 0), np.repeat(p0[None], a.batch, 0))
    stream = torch.cuda.ExternalStream(h.stream)
    runs = []
    for r in range(1 + a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        sol = pkg.ptr.solve(pbm, G, beta=betas)
        e1.record(stream)
        e1.synchronize()
        runs.append(dict(device_s=e0.elapsed_time(e1) * 1e-3, wall_s=time.perf_counter() - t0, sol=sol))
    pbm.close()
    h.close()
    timed = runs[1:]
    rate = [int(r["sol"].iterations.sum()) / r["device_s"] for r in timed]
    s = timed[-1]["sol"]
    name, power = card()
    print(json.dumps({"metric": "SCP iterations/s (planar rendezvous, in-loop homotopy, beta sweep in one batch)",
                      "value": float(np.median(rate)), "unit": "SCP iterations/s", "all_runs": rate, "batch": a.batch,
                      "N": N, "Nsub": 10, "chunks": os.environ.get("SCPB_PTR_CHUNKS", "library default"),
                      "scp_iterations": int(s.iterations.sum()), "iterations_min_median_max":
                      [int(s.iterations.min()), int(np.median(s.iterations)), int(s.iterations.max())],
                      "final_grid_index_histogram": np.bincount(s.hom_index, minlength=10).tolist(),
                      "solved": int(sum(st == "SCP_SOLVED" for st in s.status)),
                      "device_seconds": [r["device_s"] for r in timed], "wall_seconds": [r["wall_s"] for r in timed],
                      "gpu": name, "power_limit_and_max_sm_clock": power}))


if __name__ == "__main__":
    main()
