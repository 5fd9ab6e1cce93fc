"""Time the forced-oscillator deadband problem (test/examples/oscillator/tests.jl:22-80: PTR, FOH, N = 30, Nsub = 10,
iter_max = 10) on the GPU, two workloads in one run:
  * sweep:    the 10-step warm-started homotopy sweep of kappa = Homotopy(1e-8)(LinRange(0, 1, 10)) for a batch of
              seeded perturbed guesses (oracle/oscillator.perturbed_guesses, seed --seed), in the library's default
              lock-step loop;
  * schedule: the in-loop homotopy schedule over the same grid inside ONE solve, every seed from the reference guess with
              its own update threshold beta = LinRange(0.1, 30, B) / 100, in one batch.

    python scripts/bench_oscillator.py [--batch 256] [--repeats 3]

Prints one JSON line per workload: SCP iterations per second (PTR iterations summed over seeds and steps, over the device
time, CUDA events recorded on the library's stream), the iteration counts, and the card name, power limit and maximum SM
clock read in the same run.  Writes nothing in the tree."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_rendezvous import card  # noqa: E402


def timed(fn, stream, repeats):
    """one warm-up call, then `repeats` timed ones: [(device seconds, wall seconds, result)]"""
    import torch
    runs = []
    for _ in range(1 + repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        out = fn()
        e1.record(stream)
        e1.synchronize()
        runs.append((e0.elapsed_time(e1) * 1e-3, time.perf_counter() - t0, out))
    return runs[1:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=3, help="timed runs of each workload (after one warm-up run)")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU path only")
    pkg = g.load_package()
    ex = pkg.examples.oscillator
    h = pkg.Handle(0)
    N = 30
    stream = torch.cuda.ExternalStream(h.stream)
    name, power = card()
    common = dict(batch=a.batch, N=N, Nsub=10, iter_max=10, chunks=os.environ.get("SCPB_PTR_CHUNKS", "library default"),
                  gpu=name, power_limit_and_max_sm_clock=power)

    # the warm-started sweep; the guesses are the seeded perturbations the GPU tests use (inputs only: nothing else of
    # the oracle runs here)
    from oracle.oscillator import OscillatorProblem, perturbed_guesses
    X, U, P = perturbed_guesses(OscillatorProblem(N), a.batch, a.seed)
    traj = pkg.problem.TrajectoryProblem(ex.OscillatorProblem(N))
    ex.define_problem(traj, "ptr")
    pbm = pkg.ptr.create(ex.ptr_parameters(N=N), traj, h)
    runs = timed(lambda: ex.homotopy_sweep(pbm, (X, U, P)), stream, a.repeats)
    pbm.close()
    rate = [sum(int(s.iterations.sum()) for s in sols) / dev for dev, _, sols in runs]
    sols = runs[-1][2]
    print(json.dumps({"metric": "SCP iterations/s (oscillator homotopy sweep, 10 warm-started steps)",
                      "value": float(np.median(rate)), "unit": "SCP iterations/s", "all_runs": rate, **common,
                      "scp_iterations_per_step": [int(s.iterations.sum()) for s in sols],
                      "max_iterations_per_step": [int(s.iterations.max()) for s in sols],
                      "solved_last_step": int(sum(st == "SCP_SOLVED" for st in sols[-1].status)),
                      "device_seconds": [r[0] for r in runs], "wall_seconds": [r[1] for r in runs]}), flush=True)

    # the in-loop schedule, a beta sweep in one batch
    traj = pkg.problem.TrajectoryProblem(ex.OscillatorProblem(N))
    ex.define_problem(traj, "ptr")
    ex.homotopy_schedule(traj, beta=0.1)
    pbm = pkg.ptr.create(ex.ptr_parameters(N=N), traj, h)
    betas = np.linspace(0.1, 30, a.batch) / 100
    x0, u0, p0 = traj.guess(N)
    G = (np.repeat(x0[None], a.batch, 0), np.repeat(u0[None], a.batch, 0), np.repeat(p0[None], a.batch, 0))
    runs = timed(lambda: pkg.ptr.solve(pbm, G, beta=betas), stream, a.repeats)
    pbm.close()
    h.close()
    rate = [int(s.iterations.sum()) / dev for dev, _, s in runs]
    s = runs[-1][2]
    print(json.dumps({"metric": "SCP iterations/s (oscillator, in-loop homotopy, beta sweep in one batch)",
                      "value": float(np.median(rate)), "unit": "SCP iterations/s", "all_runs": rate, **common,
                      "scp_iterations": int(s.iterations.sum()), "iterations_min_median_max":
                      [int(s.iterations.min()), int(np.median(s.iterations)), int(s.iterations.max())],
                      "final_grid_index_histogram": np.bincount(s.hom_index, minlength=10).tolist(),
                      "solved": int(sum(st == "SCP_SOLVED" for st in s.status)),
                      "device_seconds": [r[0] for r in runs], "wall_seconds": [r[1] for r in runs]}), flush=True)


if __name__ == "__main__":
    main()
