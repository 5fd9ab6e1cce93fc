"""GPU tests of features whose device path is not validated yet: on an H100 they do not pass.  They are marked xfail
(non-strict) and live in the file pytest collects last, so that whatever they do cannot disturb a validated test."""
import numpy as np
import pytest

from oracle import problems, ptr as optr
from tests.test_ptr_gpu import _setup

pytestmark = pytest.mark.gpu


@pytest.mark.xfail(reason="the PTR loop with a trust-region norm other than LINF ends 1e-4..1e-3 (ex(phys)) away from "
                          "the oracle loop after 5 iterations; the cone solves of the q_tr = 4 subproblems match the "
                          "oracle (test_conic_seeds_gpu.py::test_starship_soc_subproblems_match_the_oracle) and q_tr = 1, "
                          "which has no second-order cone, deviates the same way (test_ptr_with_soc_trust_regions_"
                          "matches_the_oracle_loop), so the cause is in the loop, not in the GEOM / SOC cone solve",
                   strict=False)
def test_ptr_with_the_squared_two_norm_trust_region(pkg, handle):
    """q_tr = 4 (ptr.jl:582, 604-630: SOC trust-region cones whose radius enters through the GEOM cone): the batched PTR
    against the oracle PTR on the starship problem, 5 forced iterations."""
    N, Nsub, K = 12, 60, 5
    mdl, traj, pars = _setup(pkg, handle, N, Nsub, iter_max=K)
    pars.q_tr = 4
    pars.eps_abs = 0.0
    pars.eps_rel = 0.0
    pbo = problems.StarshipProblem(N)
    g = pbo.guess(N)
    mdl.hs = pbo.hs
    P = optr.PTR(pbo, optr.Parameters(N=N, Nsub=Nsub, iter_max=K, wvc=1e3, wtr=0.1, eps_abs=0.0, eps_rel=0.0, feas_tol=5e-3,
                                      q_tr=4, solver_tol=1e-10))
    sc = P.scale
    X0, U0, P0 = np.array([g[0]]), np.array([g[1]]), np.array([g[2]])
    pbm = pkg.ptr.create(pars, traj, handle)
    sol = pkg.ptr.solve(pbm, (X0, U0, P0), feastol=1e-10, abstol=1e-10, reltol=1e-10)
    pbm.close()
    ref = P.solve((X0[0], U0[0], P0[0]), prefer="ipm")
    rs = ref["sol"]
    ex7 = np.abs((sol.xd[0][:, :7] - rs.xd[:, :7]) / sc.Sx[:7]).max()
    dJ = abs(sol.cost[0] - rs.J_aug) / max(1.0, abs(rs.J_aug))
    print("q_tr = 4 parity: iterations", sol.iterations[0], ref["iterations"], "ex(phys)", ex7, "dJ", dJ, sol.status[0], ref["status"])
    assert sol.status[0] == ref["status"] == "SCP_SOLVED" and int(sol.iterations[0]) == ref["iterations"] == K
    assert ex7 <= 1e-4 and dJ <= 1e-6
