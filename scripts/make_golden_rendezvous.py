"""Generate tests/golden/oracle_ptr_rendezvous.npz: the oracle's homotopy sweep of the planar rendezvous
(test/examples/rendezvous_planar/tests.jl:22-95: PTR, IMPULSE, N = 30, Nsub = 10, ten kappa steps, each warm-started from
the previous solution), with the oracle interior point at 1e-11 standing in for ECOS.
  * the full 10-step sweep from the problem's own straight-line guess: per step kappa, status, iterations, J_aug, xd, ud, p;
  * the first two steps from PERT_NB seeded perturbed guesses (oracle/rendezvous.perturbed_guesses, seed PERT_SEED).
    python scripts/make_golden_rendezvous.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import rendezvous as rz  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "oracle_ptr_rendezvous.npz")
N, PERT_NB, PERT_SEED, PERT_STEPS = 30, 3, 2026, 2


def _pack(res, prefix):
    return {f"{prefix}kappa": np.array([r["kappa"] for r in res]),
            f"{prefix}status": np.array([r["status"] for r in res]),
            f"{prefix}iterations": np.array([r["iterations"] for r in res]),
            f"{prefix}J_aug": np.array([r["sol"].J_aug for r in res]),
            f"{prefix}xd": np.array([r["sol"].xd for r in res]),
            f"{prefix}ud": np.array([r["sol"].ud for r in res]),
            f"{prefix}p": np.array([r["sol"].p for r in res])}


def main():
    pb = rz.PlanarRendezvousProblem(N)
    out = _pack(rz.homotopy_sweep(pb, pb.guess(N), verbose=True), "")
    X, U, P = rz.perturbed_guesses(pb, PERT_NB, PERT_SEED)
    out.update(pert_xd0=X, pert_ud0=U, pert_p0=P)
    per = [_pack(rz.homotopy_sweep(pb, (X[b], U[b], P[b]), steps=PERT_STEPS, verbose=True), "") for b in range(PERT_NB)]
    for k in per[0]:
        out["pert_" + k] = np.array([d[k] for d in per])
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    main()
