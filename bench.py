#!/usr/bin/env python
"""bench.py -- SCP hot-path benchmark (contract in the task statement / DESIGN.md section 6).

  python bench.py --gpus N --steps K --warmup W            our arm  (CUDA path through the C ABI)
  python bench.py --impl reference --gpus N --steps K ...   reference arm (CPU oracle port, all host threads)

Workload (config.workload): BASELINE.json's north-star case -- starship_flip PTR, N=100 nodes, Nsub=100,
256 randomly perturbed initial guesses ("seeds"), fp64.  One "step" = one complete batched PTR solve
of those seeds (discretize! + formulate + conic solve + discretize! + stopping test, until every seed stops)
INCLUDING the final gather; the metric is SCP iterations per second = sum over seeds of PTR iterations / time.
The PTR loop runs as streamed chains (32 chunks of seed groups, each its own CUDA stream and PTR sequence, one hardware
queue per chunk: the two environment defaults set below, DESIGN.md section 4); SCPB_PTR_CHUNKS=0 gives the lock-step loop.
Seeds are independent: with N GPUs the 256 seeds are cut into blocks of ceil(256/N) per rank (SURVEY 8(e);
"scaling": "strong"), no collective on the data path, one NCCL all_gather of the per-seed results at the end, inside
the timed region (scptoolbox.jl_b200/sharded.py).  --weak keeps 256 seeds per GPU instead ("scaling": "weak").
--dump-outputs DIR writes the whole-batch solution of the last timed step as DIR/<name>.npy (float64); the seeds are
drawn from fixed random streams around a nominal guess computed on the CPU, so two builds run with the same arguments
solve the same inputs and can be compared array for array.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

# streamed PTR chains (scpb_ptr_solve): one hardware queue per chunk, or a 100 ms solver kernel at the head of a shared
# queue blocks the small kernels of another chunk behind it.  Must be in the environment before the CUDA context exists.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
os.environ.setdefault("SCPB_PTR_CHUNKS", "32")

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "SCP iterations/sec (batch)"
UNIT = "SCP iterations/s"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--batch", type=int, default=None, help="seeds in the batch (per GPU with --weak); default 256 "
                                                              "(ptr / scvx), 1024 (gusto)")
    ap.add_argument("--weak", action="store_true", help="weak scaling: --batch seeds on EVERY GPU (default: strong, "
                                                        "the batch is cut into ceil(batch/N) seeds per GPU)")
    ap.add_argument("--N", type=int, default=None, help="time nodes; default 100 (starship), 60 (quadrotor GuSTO)")
    ap.add_argument("--Nsub", type=int, default=None, help="RK4 sub-steps per interval; default 100 (starship), 15 (quadrotor)")
    ap.add_argument("--cpu-seeds", type=int, default=0, help="seeds in the CPU sample (0 = one per host thread)")
    ap.add_argument("--algo", default="ptr", choices=["ptr", "scvx", "gusto"],
                    help="ptr: the north-star workload (default); scvx: BASELINE configs[2], starship SCvx; "
                         "gusto: BASELINE configs[3], quadrotor obstacle avoidance with GuSTO")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the solution of the last timed step as DIR/<name>.npy (float64, at most 64 MiB)")
    a = ap.parse_args()
    dN, dNsub, dB = (60, 15, 1024) if a.algo == "gusto" else (100, 100, 256)
    a.N = a.N or dN; a.Nsub = a.Nsub or dNsub; a.batch = a.batch or dB
    return a


class ClockSampler:
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            parts = [x.strip() for x in r.split(",")]
            if len(parts) < 7:
                continue
            try:
                sm.append(float(parts[0])); mx.append(float(parts[1]))
            except ValueError:
                continue
            for n, v in zip(names, parts[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


def effective_cores():
    """Host cores this container may actually use: min(visible CPUs, cgroup cpu.max quota)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = max(1, min(n, int(round(int(q) / int(per)))))
    except Exception:
        pass
    return n


HBM_PEAK = (3350.0, "H100 SXM data sheet: 3.35 TB/s HBM3 at 700 W")


DUMP_BYTES = 64 * 1024 * 1024


def dump_outputs(sol, out_dir):
    """The arrays a caller of solve_sharded receives, as out_dir/<name>.npy in float64.  When they exceed DUMP_BYTES in
    all, a fixed seeded sample of the seeds is written instead, with the sampled seed numbers in seed_index.npy."""
    per_seed = {"xd": sol.xd, "ud": sol.ud, "p": sol.p, "cost": sol.cost, "deviation": sol.deviation,
                "iterations": sol.iterations, "feas": sol.feas, "status": sol.raw_status}
    per_seed = {k: np.asarray(v, dtype=np.float64) for k, v in per_seed.items()}
    B = per_seed["cost"].shape[0]
    td = np.asarray(sol.td, dtype=np.float64)
    row = sum(a.nbytes for a in per_seed.values()) // B + 8
    keep = (DUMP_BYTES - td.nbytes) // row
    os.makedirs(out_dir, exist_ok=True)
    if keep < B:
        idx = np.sort(np.random.default_rng(0).choice(B, keep, replace=False))
        per_seed = {k: v[idx] for k, v in per_seed.items()}
        np.save(os.path.join(out_dir, "seed_index.npy"), idx.astype(np.float64))
    for k, v in per_seed.items():
        np.save(os.path.join(out_dir, f"{k}.npy"), v)
    np.save(os.path.join(out_dir, "td.npy"), td)


# PTR constants of the reference test (starship_flip/tests.jl:33-47)
PTR = dict(iter_max=15, wvc=1e3, wtr=0.1, eps_abs=1e-5, eps_rel=0.01 / 100, feas_tol=5e-3)
# SCvx constants of the reference test (starship_flip/tests.jl:69-121)
SCVX = dict(iter_max=100, lam=5e2, rho_0=0.0, rho_1=0.1, rho_2=0.7, beta_sh=2.0, beta_gr=2.0, eta_init=1.0, eta_lb=1e-8,
            eta_ub=10.0, eps_abs=1e-5, eps_rel=0.01 / 100, feas_tol=5e-3)
# GuSTO constants of the reference test (quadrotor/tests.jl:81-145) with its commented-out stopping tolerances switched on
GUSTO = dict(iter_max=15, lam_init=1e4, lam_max=1e9, rho_0=0.1, rho_1=0.9, beta_sh=2.0, beta_gr=2.0, gamma_fail=5.0,
             eta_init=10.0, eta_lb=1e-3, eta_ub=10.0, mu=0.8, iter_mu=6, eps_abs=1e-5, eps_rel=0.01 / 100, feas_tol=1e-3)
ALGO = "ptr"


def workload_name(args):
    if args.algo == "gusto":
        return f"quadrotor GuSTO N={args.N} Nsub={args.Nsub}"
    return f"starship_flip {args.algo.upper()} N={args.N} Nsub={args.Nsub}"


def algo_constants(algo):
    return {"ptr": PTR, "scvx": SCVX, "gusto": GUSTO}[algo]


def workload_config(args, Btot, world):
    """The `config` object of the JSON line: what is solved -- identical in both arms (what happened in a run is `run`)."""
    return {"workload": workload_name(args), "batch_total": Btot, "batch_per_gpu": -(-Btot // world),
            "partition": "contiguous blocks of ceil(batch_total / n_gpus) seeds",
            "algorithm_constants": algo_constants(args.algo),
            "seeds": ("SURVEY 8(d): straight line + lateral half-sine of amplitude U[-1, 1] m, tdil ~ U[1, 2.5] s"
                      if args.algo == "gusto" else
                      "SURVEY 8(d): x += 0.05*Sx*N(0,1), u += 0.05*Su*N(0,1) clipped to the advised ranges, (t1, t2) x U[0.8, 1.2]"),
            "l2": "256 MiB buffer written between timed steps; solver working set (1.2 GB for 256 seeds) >> L2"}


def make_seeds_c4(base, nb, seed, r0, rf):
    """Synthetic seeds as SURVEY 8(d) specifies them for C4: the straight-line guess plus a lateral (horizontal, normal to
    the r0 -> rf line) half-sine of amplitude U[-1, 1] m -- which side of the obstacles the guess passes --, and the flight
    time tdil drawn from U[1, 2.5] s; seed 0 of stream 0 is the nominal guess."""
    rng = np.random.default_rng(0x5C94 + seed)
    x, u, p = base
    N = x.shape[0]
    d = np.asarray(rf, float) - np.asarray(r0, float)
    lat = np.array([-d[1], d[0], 0.0]); lat /= np.linalg.norm(lat)
    bump = np.sin(np.pi * np.arange(N) / (N - 1))
    X, U, P = [], [], []
    for b in range(nb):
        pert = bool(b or seed)
        xb = np.array(x, dtype=float)
        pb = np.array(p, dtype=float)
        if pert:
            xb[:, 0:3] += rng.uniform(-1.0, 1.0) * bump[:, None] * lat[None, :]
            pb[0] = rng.uniform(1.0, 2.5)
        X.append(xb); U.append(np.array(u, dtype=float)); P.append(pb)
    return np.array(X), np.array(U), np.array(P)


def make_seeds(base, Sx, Su, nb, seed, cx=None, cu=None):
    """Synthetic seeds as SURVEY 8(d) specifies them for C3: the nominal guess with x += 0.05*Sx*N(0,1),
    u += 0.05*Su*N(0,1) clipped to the advised ranges [c, c+S], and the two time-dilation parameters (t1, t2) drawn from
    U[0.8, 1.2] x nominal (the switch state xs stays nominal); seed 0 of stream 0 is the unperturbed nominal guess."""
    rng = np.random.default_rng(0x5C90 + seed)
    x, u, p = base
    X, U, P = [], [], []
    for b in range(nb):
        pert = bool(b or seed)
        xb = x + (0.05 * Sx * rng.standard_normal(x.shape) if pert else 0.0)
        ub = u + (0.05 * Su * rng.standard_normal(u.shape) if pert else 0.0)
        if pert and cx is not None:
            xb = np.clip(xb, cx, cx + Sx)
        if pert and cu is not None:
            ub = np.clip(ub, cu, cu + Su)
        pb = np.array(p, dtype=float)
        if pert:
            pb[:2] = pb[:2] * rng.uniform(0.8, 1.2, 2)
        X.append(xb); U.append(ub); P.append(pb)
    return np.array(X), np.array(U), np.array(P)


# ----------------------------------------------------------------------------------------------
def oracle_worker(args):
    """One seed through the oracle PTR (C discretize + HiGHS LP); returns (iterations, phase seconds)."""
    N, Nsub, hs, xd, ud, p = args[:6]
    algo = args[6] if len(args) > 6 else "ptr"
    from oracle import problems, ptr as optr, scvx as oscvx
    if algo == "gusto":
        from oracle import gusto as ogusto
        pb = problems.QuadrotorProblem(N)
        c = {k: v for k, v in GUSTO.items()}
        P = ogusto.GuSTO(pb, ogusto.Parameters(N=N, Nsub=Nsub, solver_tol=1e-9, **c))
        t0 = time.perf_counter()
        try:
            guess = optr.correct_convex(pb, P.scale, N, xd, ud, p, tol=1e-9)      # generate_initial_guess (gusto.jl:517-526)
        except RuntimeError as e:
            return 0, {"discretize": 0.0, "formulate": 0.0, "solve": time.perf_counter() - t0}, f"SCP_FAILED ({e})"
        out = P.solve(guess)
        tm = {"discretize": 0.0, "formulate": 0.0, "solve": 0.0}
        for s in out["history"]:
            for k in tm:
                tm[k] += s.timing.get(k, 0.0)
        return out["iterations"], tm, out["status"]
    pb = problems.StarshipProblem(N)
    pb.hs = hs
    if algo == "scvx":
        P = oscvx.SCvx(pb, oscvx.Parameters(N=N, Nsub=Nsub, solver_tol=1e-9, **SCVX))
    else:
        P = optr.PTR(pb, optr.Parameters(N=N, Nsub=Nsub, solver_tol=1e-9, **PTR))
    out = P.solve((xd, ud, p))
    tm = {"discretize": 0.0, "formulate": 0.0, "solve": 0.0}
    for s in out["history"]:
        for k in tm:
            tm[k] += s.timing.get(k, 0.0)
    return out["iterations"], tm, out["status"]


def cpu_run(N, Nsub, hs, X, U, P, nproc):
    import multiprocessing as mp
    # one seed per process, every process single-threaded (no BLAS / OpenMP / HiGHS thread pools fighting
    # over the cores): the reference is a single-threaded Julia process per trajectory
    for v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS", "HIGHS_NUM_THREADS"):
        os.environ[v] = "1"
    jobs = [(N, Nsub, hs, X[b], U[b], P[b], ALGO) for b in range(X.shape[0])]
    t0 = time.perf_counter()
    with mp.get_context("fork").Pool(nproc) as pool:
        res = pool.map(oracle_worker, jobs, chunksize=1)
    wall = time.perf_counter() - t0
    its = sum(r[0] for r in res)
    ph = {k: sum(r[1][k] for r in res) for k in ("discretize", "formulate", "solve")}
    return its, wall, ph, [r[2] for r in res]


def oracle_base_guess(N, algo="ptr"):
    from oracle import problems
    pb = problems.QuadrotorProblem(N) if algo == "gusto" else problems.StarshipProblem(N)
    g = pb.guess(N)
    return pb, g


def run_reference(args, rank):
    """Reference arm: the CPU restatement of the reference (Julia + ECOS are not installable here) on all host
    threads, one seed per process, on a bounded sample of the same workload."""
    if rank != 0:
        return
    cores = effective_cores()
    pb, g = oracle_base_guess(args.N)
    from oracle import ptr as optr
    sc = optr.Scaling(pb)
    nseeds = args.cpu_seeds or min(args.batch, 2 * cores)
    X, U, P = make_seeds(g, sc.Sx, sc.Su, nseeds, 0, sc.cx, sc.cu)      # the first seeds of the GPU arm's batch
    vals, walls = [], []
    cpu_run(args.N, args.Nsub, pb.hs, X[:min(8, nseeds)], U[:min(8, nseeds)], P[:min(8, nseeds)], min(cores, 8))  # warm-up
    for _ in range(args.steps):
        its, wall, ph, st = cpu_run(args.N, args.Nsub, pb.hs, X, U, P, min(cores, nseeds))
        vals.append(its); walls.append(wall)
    tot = sum(walls)
    val = sum(vals) / tot
    line = {"impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * tot / args.steps,
            "higher_is_better": True, "scaling": "weak" if args.weak else "strong", "vs_baseline": None, "dtype": "f64",
            "data": "synthetic",
            "config": workload_config(args, args.batch * (args.gpus if args.weak else 1), max(1, args.gpus)),
            "cpu_baseline": {"value": val, "unit": UNIT, "cores": cores, "kind": "port",
                             "sample": f"{nseeds} of {args.batch} seeds per step, one single-threaded process per core "
                                       f"(oracle: C discretize + Python formulate + "
                                       f"{'interior-point SOCP' if args.algo == 'gusto' else 'HiGHS LP'}); cores = "
                                       f"min(visible CPUs {os.cpu_count()}, cgroup cpu.max quota)",
                             "phase_cpu_seconds": ph, "seeds_solved": sum(x == "SCP_SOLVED" for x in st)},
            "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def k1_flops_per_seed(N, Nsub, nx, nu, np_):
    """SURVEY 8(d): algorithmic fp64 work of one discretize! call for one seed."""
    V = nx * (2 + 2 * nx + 2 * nu + np_)
    per = 2 * nx ** 3 + (8.0 / 3.0) * nx ** 3 + 2 * nx ** 2 * (2 * nu + np_ + 1 + nx) + 2 * nx * (nx + nu + np_) + 8 * V
    return (N - 1) * (Nsub - 1) * 4 * per


def run_ours(args, rank, local_rank, world):
    import torch
    import __graft_entry__ as g
    pkg = g.load_package()
    dist = None
    if world > 1:
        import torch.distributed as dist_
        dist = dist_
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    torch.cuda.set_device(local_rank)
    tc = torch.cuda
    dev = torch.device("cuda", local_rank)
    N, Nsub = args.N, args.Nsub
    Btot = args.batch * world if args.weak else args.batch      # seeds in the whole job
    h = pkg.Handle(local_rank)
    ex = pkg.examples.quadrotor if args.algo == "gusto" else pkg.examples.starship
    mdl = ex.QuadrotorProblem() if args.algo == "gusto" else ex.StarshipProblem()
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, args.algo if args.algo == "gusto" else "ptr", handle=h)
    algo = {"scvx": pkg.scvx, "ptr": pkg.ptr, "gusto": pkg.gusto}[args.algo]
    if args.algo == "gusto":
        c = GUSTO
        pars = pkg.gusto.Parameters(N, Nsub, c["iter_max"], pkg.ptr.FOH, c["lam_init"], c["lam_max"], c["rho_0"], c["rho_1"],
                                    c["beta_sh"], c["beta_gr"], c["gamma_fail"], c["eta_init"], c["eta_lb"], c["eta_ub"],
                                    c["mu"], c["iter_mu"], c["eps_abs"], c["eps_rel"], c["feas_tol"], "quad", 100.0, np.inf,
                                    np.inf, None, {"verbose": 0, "maxit": 100})
    elif args.algo == "scvx":
        pars = pkg.scvx.Parameters(N=N, Nsub=Nsub, disc_method=pkg.ptr.FOH, q_tr=np.inf, q_exit=np.inf,
                                   solver_opts={"verbose": 0, "maxit": 100}, **SCVX)
    else:
        pars = pkg.ptr.Parameters(N=N, Nsub=Nsub, disc_method=pkg.ptr.FOH, q_tr=np.inf, q_exit=np.inf,
                                  solver_opts={"verbose": 0, "maxit": 100}, **PTR)
    if args.algo == "gusto":
        base = traj.guess(N)                 # straight-line guess, computed on the host
    else:
        # nominal guess and seed scaling from the CPU restatement, as in the reference arm: the product's own generator
        # solves an SOCP batch with the library under test, so two builds would start from different seeds and could not
        # be compared output for output.  Outside the timed region.
        from oracle import ptr as optr
        pbo, base = oracle_base_guess(N)
        mdl.hs = pbo.hs
        sco = optr.Scaling(pbo, N)
    pbm = algo.create(pars, traj, h)
    if args.algo == "gusto":
        X, U, P = make_seeds_c4(base, Btot, 0, mdl.r0, mdl.rf)
        mdl.hs = 0.0
    else:
        X, U, P = make_seeds(base, sco.Sx, sco.Su, Btot, 0, sco.cx, sco.cu)      # the whole batch, identical on every rank
    lo, hi = pkg.sharded.shard_bounds(Btot, world, rank)
    Bloc = hi - lo
    info = pbm.cone.info()

    def barrier():
        if dist is not None:
            dist.barrier()
        tc.synchronize()

    l2_flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    W = max(args.warmup, 3)
    for _ in range(W):
        l2_flush.zero_()
        sol, loc = pkg.sharded.solve_sharded(algo, pbm, (X, U, P), dist=dist, device=dev)
    barrier()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    n0 = h.launches
    dev_t, wall_t, ipm, phases = 0.0, 0.0, 0, {"discretize": 0.0, "formulate": 0.0, "solve": 0.0, "overhead": 0.0}
    its, lock, k1_init = 0, 0, 0.0
    barrier()
    for _ in range(args.steps):
        l2_flush.zero_(); tc.synchronize()
        if dist is not None:
            dist.barrier()
        t0 = time.perf_counter()
        # the reference-facing call: host buffers in, host buffers out; shard -> device loop -> NCCL all_gather
        sol, loc = pkg.sharded.solve_sharded(algo, pbm, (X, U, P), dist=dist, device=dev)
        wall_t += time.perf_counter() - t0
        its += int(sol.iterations.sum())     # every rank holds the gathered whole-job result
        if loc is not None:
            dev_t += loc.timing["total"]     # CUDA events on the library's stream, H2D/D2H copies and the gather excluded
            ipm += loc.timing["ipm_iterations"]; lock += loc.timing["lockstep_iterations"]
            k1_init += loc.timing.get("initial_discretize", 0.0)
            for k in phases:
                phases[k] += loc.timing[k]
    barrier()
    launches = h.launches - n0
    clocks = sampler.stop() if rank == 0 else None
    t = torch.tensor([dev_t, wall_t], dtype=torch.float64, device="cuda")
    ln = torch.tensor([float(launches)], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(ln, op=dist.ReduceOp.SUM)
    dev_t, wall_t = float(t[0]), float(t[1])
    if rank == 0:
        if args.dump_outputs:
            dump_outputs(sol, args.dump_outputs)
        value = its / dev_t
        e2e = its / wall_t
        solved = sum(s_ == "SCP_SOLVED" for s_ in sol.status)
        itv = sol.iterations
        # ---- roofline of the dominant kernel (k_ipm_solve): algorithmic bytes per interior-point iteration ----
        nnzK = pbm.cp["nnzA"] + pbm.cp["nnzG"]
        n_, p_, m_ = pbm.cp["n"], pbm.cp["p"], pbm.cp["m"]
        nnzL, nk = info["nnzL"], info["nk"]
        # LDL' solve pairs per interior-point iteration (2 directions + the refinement steps the adaptive rule took):
        # counted by the kernel itself (CTA 0 of the last launch)
        cyc = pbm.cone.info()["cycles"]
        nsolve = cyc["ldl_count"] / max(cyc["factor_count"], 1)
        q_it = 8 * (nnzK + 3 * (nnzL + nk)                 # KKT assembly (read K, write Y) + factor (rw Y, write L)
                    + nsolve * (2 * nnzL + 4 * nk)         # forward+backward substitutions
                    + (2 + 2 * nsolve) * nnzK              # residual / refinement SpMVs (K and K')
                    + 12 * (n_ + p_ + 2 * m_))             # vector updates
        nch = int(loc.timing.get("chunks", 0))
        if nch > 1:
            # streamed chains: the step is n_chunks concurrent sequences of small k_ipm_solve launches (one CTA per seed
            # group), so a single launch says nothing about the device.  achieved = algorithmic bytes of ALL launches of the
            # step / the device time of the whole step (the other kernels of a chain overlap with the solves of the other
            # chains and cannot be subtracted); kernel_ms / kernel_share are those of chunk 0's own chain
            ng = -(-Bloc // pbm.cone.info()["group"]) if pbm.cone.info()["group"] else Bloc
            c0 = min(Bloc, -(-ng // nch) * max(pbm.cone.info()["group"], 1))
            k_ms = 1e3 * phases["solve"] / max(args.steps * int(loc.iterations[:c0].max()), 1)
            ach = q_it * ipm / max(dev_t, 1e-12) / 1e9
            chain = sum(phases.values())
            k_share = phases["solve"] / max(chain, 1e-12)
        else:
            k_ms = 1e3 * phases["solve"] / max(lock, 1)
            ach = q_it * ipm / max(phases["solve"], 1e-12) / 1e9
            k_share = phases["solve"] / max(dev_t, 1e-12)
        peak, peak_src = HBM_PEAK
        # ---- roofline of K1 (k_discretize_foh): fp64-FMA bound; W from SURVEY 8(d), peak measured here ----
        ncalls = lock + args.steps                           # one discretize! per lock-step iteration + the initial guess
        w_seed = k1_flops_per_seed(N, Nsub, traj.nx, traj.nu, traj.np)
        k1_s = phases["discretize"] / max(ncalls, 1)
        if nch > 1:                                          # K1 timed alone: the initial full-batch discretize! of each step
            k1_s = k1_init / max(args.steps, 1)
        try:
            fp64_peak = h.fp64_peak()
        except Exception:
            fp64_peak = None
        k1_ach = w_seed * Bloc / max(k1_s, 1e-12) / 1e12
        roof_k1 = {"bound": "fp64", "achieved": k1_ach, "peak": fp64_peak, "unit": "TFLOP/s",
                   "frac": (k1_ach / fp64_peak) if fp64_peak else None, "traffic": None, "kernel": "k_discretize_foh",
                   "kernel_ms": 1e3 * k1_s, "algorithmic_flops_per_seed_per_call": w_seed, "seeds_per_launch": Bloc,
                   "peak_source": "measured in this run (scpb_debug_fp64_peak: register-resident fp64 FMA microkernel)",
                   "kernel_share_of_step": phases["discretize"] / max(sum(phases.values()) if nch > 1 else dev_t, 1e-12)}
        # ---- CPU baseline on a bounded sample (rank 0, N=1 only) ----
        cpu = None
        if world == 1:
            cores = effective_cores()
            nseeds = args.cpu_seeds or min(Btot, 2 * cores)
            cits, cwall, cph, _ = cpu_run(N, Nsub, mdl.hs, X[:nseeds], U[:nseeds], P[:nseeds], min(cores, nseeds))
            cpu = {"value": cits / cwall, "unit": UNIT, "cores": cores, "kind": "port",
                   "sample": f"{nseeds} of {Btot} seeds, full {args.algo.upper()} solve each, one single-threaded process per core "
                             f"(oracle: C discretize + Python formulate + "
                             f"{'interior-point SOCP' if args.algo == 'gusto' else 'HiGHS LP'}); cores = min(visible CPUs "
                             f"{os.cpu_count()}, cgroup cpu.max quota)",
                   "phase_cpu_seconds": cph}
        nb_in = int(X.nbytes + U.nbytes + P.nbytes)
        line = {"metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": W,
                "ms_per_step": 1e3 * dev_t / args.steps, "higher_is_better": True,
                "scaling": "weak" if args.weak else "strong",
                "vs_baseline": None, "dtype": "f64", "data": "synthetic",
                "config": workload_config(args, Btot, world),
                "run": {"seeds_solved": int(solved), "seeds_total": Btot,
                        "scp_iterations_per_step": its / args.steps,
                        "scp_iterations_min_median_max": [int(itv.min()), float(np.median(itv)), int(itv.max())],
                        "longest_chain_iterations_per_step_rank0": lock / args.steps,
                        "chains_rank0": (f"{nch} chunks of seed groups, each its own stream and PTR sequence (no lock-step)"
                                         if nch > 1 else "one lock-step loop over the batch"),
                        "frozen_seed_fraction_rank0": (None if nch > 1 else
                                                       1.0 - (float(loc.iterations.sum()) / max(1, Bloc * (lock / args.steps))))},
                "gpu_launches": int(ln[0]),
                "e2e": {"value": e2e, "unit": UNIT, "h2d_bytes_per_step": nb_in,
                        "d2h_bytes_per_step": int(nb_in + Btot * (4 * 3 + 8 * 2)),
                        "includes": "H2D of the guesses, device loop, D2H of the results and the all_gather over NCCL"},
                "ms_per_socp_solve": k_ms,
                "phase_seconds_per_step": {k: v / args.steps for k, v in phases.items()},
                "roofline": {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                             "traffic": None, "peak_source": peak_src, "kernel": "k_ipm_solve",
                             "kernel_ms": k_ms, "algorithmic_bytes_per_ipm_iteration_per_seed": q_it,
                             "ipm_iterations_per_launch": ipm / max(lock, 1), "ldl_solves_per_ipm_iteration": nsolve,
                             "kernel_share_of_step": k_share,
                             "accounting": ("streamed chains: achieved = bytes of all launches of the step / device time of the "
                                            "step; kernel_ms, kernel_share_of_step and phase_seconds_per_step are those of "
                                            "chunk 0's chain") if nch > 1 else "lock-step: per launch",
                             "kernel_cycle_shares": {k: v / max(cyc["total"], 1) for k, v in cyc.items()
                                                     if k not in ("total", "ldl_count", "factor_count", "factor_retries")}},
                "roofline_k1": roof_k1,
                "cpu_baseline": cpu, "clocks": clocks}
        print(json.dumps(line))
    pbm.close()
    if dist is not None:
        dist.destroy_process_group()


def main():
    global ALGO
    args = parse()
    ALGO = args.algo
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        run_reference(args, rank)
    else:
        run_ours(args, rank, local_rank, world)


if __name__ == "__main__":
    main()
