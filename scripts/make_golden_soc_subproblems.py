"""Generate tests/golden/oracle_soc_subproblems.npz: the oracle interior point's answers (status, objective) to the
starship PTR subproblems with L1 / SOC / GEOM trust regions of tests/test_conic_seeds_gpu.py.
    python scripts/make_golden_soc_subproblems.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import conic  # noqa: E402
from tests.test_conic_seeds_gpu import SUB_CASES, SUB_GOLDEN, SUB_NB, starship_soc_subproblems  # noqa: E402


def main():
    out = {}
    for q_tr, N in SUB_CASES:
        refs = [conic.solve_ipm(s["cp"], tol=1e-10) for s in starship_soc_subproblems(N, SUB_NB, q_tr, seed=N + q_tr)]
        out[f"obj_q{q_tr}_N{N}"] = np.array([r["obj"] for r in refs])
        out[f"status_q{q_tr}_N{N}"] = np.array([r["status"] for r in refs])
        print(q_tr, N, [r["status"] for r in refs], flush=True)
    np.savez(SUB_GOLDEN, **out)


if __name__ == "__main__":
    main()
