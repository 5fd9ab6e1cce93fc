"""Generate tests/golden/oracle_ptr_oscillator.npz: the oracle's forced-oscillator deadband problem
(test/examples/oscillator/tests.jl:22-80: PTR, FOH, N = 30, Nsub = 10, iter_max = 10, ten kappa steps of
Homotopy(1e-8), each warm-started from the previous solution), with the oracle interior point at 1e-11 standing in for ECOS.
  * the full 10-step sweep from the problem's own guess: per step kappa, status, iterations, J_aug, xd, ud, p;
  * the first two steps from PERT_NB seeded perturbed guesses (oracle/oscillator.perturbed_guesses, seed PERT_SEED),
    keys pert_*;
  * the in-loop homotopy schedule (oracle/homotopy_update.py) over the same grid inside ONE solve from the problem's own
    guess, for each update threshold in BETAS (iter_max = 10): status, iterations, final grid index and iter_max, whether
    the loop stopped on the stopping rule, J_aug and the per-iteration history padded with NaN / -1 to HIST columns,
    keys sched_*.
    python scripts/make_golden_oscillator.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oscillator as osc, rendezvous as rz  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "oracle_ptr_oscillator.npz")
N, N_HOM, ITER_MAX = 30, 10, 10
PERT_NB, PERT_SEED, PERT_STEPS = 3, 2026, 2
BETAS = np.array([3e-3, 1e-2, 3e-2])
HIST = ITER_MAX + (N_HOM - 1) * (ITER_MAX - 1)


def _pack(res):
    return {"kappa": np.array([r["kappa"] for r in res]),
            "status": np.array([r["status"] for r in res]),
            "iterations": np.array([r["iterations"] for r in res]),
            "J_aug": np.array([r["sol"].J_aug for r in res]),
            "xd": np.array([r["sol"].xd for r in res]),
            "ud": np.array([r["sol"].ud for r in res]),
            "p": np.array([r["sol"].p for r in res])}


def main():
    pb = osc.OscillatorProblem(N)
    out = _pack(osc.homotopy_sweep(pb, pb.guess(N), n_hom=N_HOM, verbose=True))
    X, U, P = osc.perturbed_guesses(pb, PERT_NB, PERT_SEED)
    out.update(pert_xd0=X, pert_ud0=U, pert_p0=P)
    per = [_pack(osc.homotopy_sweep(pb, (X[b], U[b], P[b]), n_hom=N_HOM, steps=PERT_STEPS, verbose=True))
           for b in range(PERT_NB)]
    for k in per[0]:
        out["pert_" + k] = np.array([d[k] for d in per])
    # the in-loop schedule
    grid = np.array([osc.hom()(x) for x in rz.hom_grid(N_HOM)])
    out.update(sched_grid=grid, sched_beta=BETAS, sched_worsen_tol=np.array(-1e-3))
    rows = []
    for beta in BETAS:
        S = osc.OscillatorCallbackPTR(pb, osc.ptr_parameters(N=N, iter_max=ITER_MAX))
        rows.append(S.solve_with_schedule(pb.guess(N), grid, beta, verbose=True))
    out["sched_status"] = np.array([r["status"] for r in rows])
    for key in ("iterations", "index", "iter_max", "stopped_on_rule"):
        out["sched_" + key] = np.array([r[key] for r in rows])
    out["sched_J_aug"] = np.array([r["sol"].J_aug for r in rows])
    for key, fill, dt in (("improv_rel", np.nan, float), ("index", -1, np.int32), ("iter_max", -1, np.int32),
                          ("J_aug", np.nan, float)):
        h = np.full((len(rows), HIST), fill, dtype=dt)
        for b, r in enumerate(rows):
            v = r["history"][key]
            h[b, :v.size] = v
        out["sched_hist_" + key] = h
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    main()
