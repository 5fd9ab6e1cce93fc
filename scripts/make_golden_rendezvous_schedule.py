"""Generate tests/golden/oracle_ptr_rendezvous_schedule.npz: the oracle's planar rendezvous PTR loop (IMPULSE, N = 30,
Nsub = 10, iter_max = 30) with the in-loop homotopy callback of test/examples/rendezvous_3d/definition.jl:96-151
(oracle/homotopy_update.py): kappa steps through Homotopy(1e-3; delta_max = 5)(LinRange(0, 1, 10)) inside ONE solve from
the straight-line guess, for each update threshold in BETAS, with the oracle interior point at 1e-11 standing in for ECOS.
Per beta: status, iterations, final grid index, final iter_max, whether the loop stopped on the stopping rule, J_aug and
the per-iteration history (improv_rel, grid index, iter_max, J_aug; padded with NaN / -1 to HIST columns).
    python scripts/make_golden_rendezvous_schedule.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import homotopy_update as hu, rendezvous as rz  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "oracle_ptr_rendezvous_schedule.npz")
N, N_HOM, ITER_MAX = 30, 10, 30
BETAS = np.array([3e-3, 1e-2, 3e-2])
HIST = ITER_MAX + (N_HOM - 1) * (ITER_MAX - 1)


def main():
    pb = rz.PlanarRendezvousProblem(N)
    hom = rz.Homotopy(1e-3, delta_max=5.0)
    grid = np.array([hom(x) for x in rz.hom_grid(N_HOM)])
    out = dict(grid=grid, beta=BETAS, worsen_tol=np.array(-1e-3))
    rows = []
    for beta in BETAS:
        P = hu.CallbackPTR(pb, rz.ptr_parameters(N=N, iter_max=ITER_MAX))
        rows.append(P.solve_with_schedule(pb.guess(N), grid, beta, verbose=True))
    out["status"] = np.array([r["status"] for r in rows])
    for key in ("iterations", "index", "iter_max", "stopped_on_rule"):
        out[key] = np.array([r[key] for r in rows])
    out["J_aug"] = np.array([r["sol"].J_aug for r in rows])
    for key, fill, dt in (("improv_rel", np.nan, float), ("index", -1, np.int32), ("iter_max", -1, np.int32),
                          ("J_aug", np.nan, float)):
        h = np.full((len(rows), HIST), fill, dtype=dt)
        for b, r in enumerate(rows):
            v = r["history"][key]
            h[b, :v.size] = v
        out["hist_" + key] = h
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    main()
