"""GPU parity of the batched SCvx loop (scpb_scvx_solve through the host API) vs the oracle's SCvx loop
(oracle/scvx.py restating src/solvers/scvx.jl) on the same initial guesses -- the reference's own starship SCvx test
configuration (starship_flip/tests.jl:69-121: N = 31, Nsub = 100, lambda = 5e2, eta in [1e-8, 10], iter_max = 100).

SCvx with the reference's predicted-improvement rule does not stop at a minimiser but when the trust region has
collapsed (deviation <= eps_abs after ~40 accept / reject steps), and every LP subproblem has flat directions, so the
end point depends on the whole path: two solvers that agree to 1e-7 per subproblem end 1e-3 apart.  Asserted: identical
accept / reject sequence, identical iteration count and final radius; at the end the trajectories of the two loops are
only compared loosely (the end point of a collapsed trust region is not a minimiser).  Stated tolerance: both SCP_SOLVED, iteration counts and
final radius equal, final augmented cost within 2e-3 relative, physical trajectory within 2e-2 of its ranges; the
three-iteration test asserts 1e-7 / 1e-7."""
import numpy as np
import pytest

from oracle import problems, scvx as oscvx

pytestmark = pytest.mark.gpu

TOL = dict(feastol=1e-11, abstol=1e-11, reltol=1e-11)      # cone-solver tolerances of the parity runs

KW = dict(lam=5e2, rho_0=0.0, rho_1=0.1, rho_2=0.7, beta_sh=2.0, beta_gr=2.0, eta_init=1.0, eta_lb=1e-8, eta_ub=10.0,
          eps_abs=1e-5, eps_rel=0.01 / 100, feas_tol=5e-3)


def _setup(pkg, handle, N, Nsub, iter_max):
    ex = pkg.examples.starship
    mdl = ex.StarshipProblem()
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "scvx", handle=handle)
    pars = pkg.scvx.Parameters(N=N, Nsub=Nsub, iter_max=iter_max, disc_method=pkg.ptr.FOH, q_tr=np.inf, q_exit=np.inf,
                               solver_opts={"verbose": 0, "maxit": 1000}, **KW)
    return mdl, traj, pars


@pytest.mark.parametrize("N,Nsub,nb,iter_max", [(12, 60, 3, 100), (31, 100, 2, 100)])
def test_batched_scvx_matches_oracle_scvx(pkg, handle, N, Nsub, nb, iter_max):
    mdl, traj, pars = _setup(pkg, handle, N, Nsub, iter_max)
    pbo = problems.StarshipProblem(N)
    g = pbo.guess(N)
    mdl.hs = pbo.hs
    S = oscvx.SCvx(pbo, oscvx.Parameters(N=N, Nsub=Nsub, iter_max=iter_max, solver_tol=1e-11, **KW))
    sc = S.scale
    rng = np.random.default_rng(N)
    X0 = np.array([g[0] + (0.01 * sc.Sx * rng.standard_normal(g[0].shape) if b else 0.0) for b in range(nb)])
    U0 = np.array([g[1] + (0.01 * sc.Su * rng.standard_normal(g[1].shape) if b else 0.0) for b in range(nb)])
    P0 = np.array([g[2] * (1 + (0.02 * rng.uniform(-1, 1, g[2].shape) if b else 0.0)) for b in range(nb)])
    pbm = pkg.scvx.create(pars, traj, handle)
    sol = pkg.scvx.solve(pbm, (X0, U0, P0), **TOL)
    pbm.close()
    for b in range(nb):
        ref = S.solve((X0[b], U0[b], P0[b]), prefer="ipm")
        rs = ref["sol"]
        ex7 = np.abs((sol.xd[b][:, :7] - rs.xd[:, :7]) / sc.Sx[:7]).max()
        eu2 = np.abs((sol.ud[b][:, :2] - rs.ud[:, :2]) / sc.Su[:2]).max()
        ep = np.abs((sol.p[b] - rs.p) / sc.Sp).max()
        dJ = abs(sol.cost[b] - rs.J_aug) / max(1.0, abs(rs.J_aug))
        print("scvx parity seed", b, "iters", sol.iterations[b], ref["iterations"], "eta", sol.eta[b], ref["eta"],
              "ex(phys)", ex7, "eu", eu2, "ep", ep, "dJ", dJ, sol.status[b], ref["status"])
        assert sol.status[b] == ref["status"] == "SCP_SOLVED", (sol.status, sol.raw_status)
        assert int(sol.iterations[b]) == ref["iterations"] and sol.eta[b] == ref["eta"]     # same accept / reject path
        assert dJ <= 2e-3 and max(ex7, eu2, ep) <= 2e-2
        dn = np.abs(rs.defect * sc.iSx).max()             # feasibility flag: compare unless it sits on the tolerance
        if abs(dn - KW["feas_tol"]) > 0.05 * KW["feas_tol"]:
            assert bool(sol.feas[b]) == bool(rs.feas)


def test_scvx_first_iterations_are_identical(pkg, handle):
    """Three SCvx iterations (no stopping: eps = 0): before path effects accumulate the two loops must agree to solver
    accuracy -- radius history exactly, augmented cost and physical trajectory to 1e-5."""
    N, Nsub, K = 20, 60, 3
    mdl, traj, pars = _setup(pkg, handle, N, Nsub, K)
    pars.eps_abs = 0.0; pars.eps_rel = 0.0
    pbo = problems.StarshipProblem(N)
    g = pbo.guess(N)
    mdl.hs = pbo.hs
    kw = dict(KW); kw["eps_abs"] = 0.0; kw["eps_rel"] = 0.0
    S = oscvx.SCvx(pbo, oscvx.Parameters(N=N, Nsub=Nsub, iter_max=K, solver_tol=1e-11, **kw))
    sc = S.scale
    pbm = pkg.scvx.create(pars, traj, handle)
    sol = pkg.scvx.solve(pbm, (g[0][None], g[1][None], g[2][None]), **TOL)
    pbm.close()
    ref = S.solve(g, prefer="ipm")
    rs = ref["sol"]
    assert int(sol.iterations[0]) == ref["iterations"] == K
    assert sol.eta[0] == ref["eta"]
    ex7 = np.abs((sol.xd[0][:, :7] - rs.xd[:, :7]) / sc.Sx[:7]).max()
    dJ = abs(sol.cost[0] - rs.J_aug) / max(1.0, abs(rs.J_aug))
    print("scvx 3 iterations: ex(phys)", ex7, "dJ", dJ, "J", sol.cost[0], rs.J_aug)
    assert dJ <= 1e-7 and ex7 <= 1e-7


def test_scvx_refuses_a_constraint_pack_it_has_no_penalty_for(pkg, handle):
    """The nonlinear cost of SCvx has the nonconvex-constraint penalty of the starship's pack only: a problem with
    another pack (the quadrotor's obstacles) is refused when SCvx is attached, not solved without its penalty."""
    ex = pkg.examples.quadrotor
    traj = pkg.problem.TrajectoryProblem(ex.QuadrotorProblem())
    ex.define_problem(traj, "scvx", handle=handle)
    assert traj.ns > 0
    pars = pkg.scvx.Parameters(N=10, Nsub=15, iter_max=5, disc_method=pkg.ptr.FOH, q_tr=np.inf, q_exit=np.inf,
                               solver_opts={"verbose": 0}, **KW)
    with pytest.raises(pkg.lib.ScpbError, match=r"scpb_scvx_attach failed \(-4\).*no penalty for the constraint pack"):
        pkg.scvx.create(pars, traj, handle)
