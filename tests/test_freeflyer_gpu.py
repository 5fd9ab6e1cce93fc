"""GPU: BASELINE config C5 -- free-flyer PTR (freeflyer/definition.jl on the PTR loop; a new instance of the reference's
example, see scptoolbox.jl_b200/examples/freeflyer.py) against the oracle: automatic variable scaling (compute_scaling,
scp.jl:376-517) as batched bounding-box solves on the GPU cone solver, the constraint pack with packed ds/dp columns
(np = 1 + 6N), SOC(4) / LINF cones and the quadratic running cost inside the device-resident PTR loop.

Constants follow the reference's free-flyer tests (freeflyer/tests.jl:36-53: Nsub = 15, iter_max = 15, feas_tol = 1e-3,
eps = 0 => exactly iter_max iterations) with PTR's own weights (wvc = 1e3, wtr = 0.1 as in the starship PTR test)."""
import numpy as np
import pytest

from oracle import problems, ptr as optr

pytestmark = pytest.mark.gpu

TOL = dict(feastol=1e-11, abstol=1e-11, reltol=1e-11)


def _setup(pkg, handle, N, iter_max, eps=0.0):
    ex = pkg.examples.freeflyer
    mdl = ex.FreeFlyerProblem(N)
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr", handle=handle)
    pars = pkg.ptr.Parameters(N=N, Nsub=15, iter_max=iter_max, disc_method=pkg.ptr.FOH, wvc=1e3, wtr=0.1, eps_abs=eps,
                              eps_rel=eps, feas_tol=1e-3, q_tr=np.inf, q_exit=np.inf,
                              solver_opts={"verbose": 0, "maxit": 100})
    return mdl, traj, pars


def test_automatic_scaling_matches_oracle(pkg, handle):
    """compute_scaling: r, tdil and the room slacks are advised; v, omega, T, M get their boxes from min / max cone programs
    over X / U at all nodes (second-order cones => +-v_max etc.); the quaternion is unconstrained => every program is
    DUAL_INFEASIBLE and the default box [0, 1] stays (scp.jl:470-473)."""
    N = 8
    mdl, traj, pars = _setup(pkg, handle, N, 3)
    pbm = pkg.ptr.create(pars, traj, handle)
    sc = pbm.scale
    pbo = problems.FreeFlyerProblem(N)
    so = optr.Scaling(pbo, N)
    assert np.abs(sc.Sx - so.Sx).max() <= 1e-6 and np.abs(sc.cx - so.cx).max() <= 1e-6
    assert np.abs(sc.Su - so.Su).max() <= 1e-6 * so.Su.max() and np.abs(sc.cu - so.cu).max() <= 1e-6 * so.Su.max()
    assert np.abs(sc.Sp - so.Sp).max() <= 1e-9 and np.abs(sc.cp - so.cp).max() <= 1e-9
    assert np.allclose(sc.Sx[3:6], 2 * mdl.v_max, rtol=1e-6) and np.allclose(sc.cx[3:6], -mdl.v_max, rtol=1e-6)
    assert np.allclose(sc.Sx[10:13], 2 * mdl.omega_max, rtol=1e-6)
    assert np.allclose(sc.Su[0:3], 2 * mdl.T_max, rtol=1e-6) and np.allclose(sc.Su[3:6], 2 * mdl.M_max, rtol=1e-6)
    assert np.all(sc.Sx[6:10] == 1.0) and np.all(sc.cx[6:10] == 0.0)
    for i in range(6, 10):
        assert sc.computed[("x", i, 0)] in ("DUAL_INFEASIBLE", "NUMERICAL_ERROR") and sc.computed[("x", i, 1)] in ("DUAL_INFEASIBLE", "NUMERICAL_ERROR")
    assert sc.computed[("x", 3, 0)] in ("OPTIMAL", "ALMOST_OPTIMAL") and sc.computed[("u", 4, 1)] in ("OPTIMAL", "ALMOST_OPTIMAL")
    pbm.close()


def test_freeflyer_ptr_matches_oracle_ptr(pkg, handle):
    N, nb, K = 8, 2, 4
    mdl, traj, pars = _setup(pkg, handle, N, K)
    pbo = problems.FreeFlyerProblem(N)
    opars = optr.Parameters(N=N, Nsub=15, iter_max=K, wvc=1e3, wtr=0.1, eps_abs=0.0, eps_rel=0.0, feas_tol=1e-3,
                            solver_tol=1e-11)
    P = optr.PTR(pbo, opars)
    g = pbo.guess(N)
    sc = P.scale
    rng = np.random.default_rng(11)
    X0 = np.array([g[0] + (1e-3 * sc.Sx * rng.standard_normal(g[0].shape) if b else 0.0) for b in range(nb)])
    U0 = np.array([g[1] + (1e-3 * sc.Su * rng.standard_normal(g[1].shape) if b else 0.0) for b in range(nb)])
    P0 = np.array([g[2] for b in range(nb)])
    pbm = pkg.ptr.create(pars, traj, handle)
    sol = pkg.ptr.solve(pbm, (X0, U0, P0), **TOL)
    info = pbm.cone.info()
    pbm.close()
    print("freeflyer KKT", info["nk"], info["nnzL"], info["levels"], "timing", sol.timing)
    for b in range(nb):
        ref = P.solve((X0[b], U0[b], P0[b]), prefer="ipm")
        rs = ref["sol"]
        assert sol.status[b] == ref["status"] == "SCP_SOLVED", (sol.status, sol.raw_status, ref["status"])
        assert int(sol.iterations[b]) == ref["iterations"] == K
        ex = np.abs((sol.xd[b] - rs.xd) / sc.Sx).max()
        eu = np.abs((sol.ud[b] - rs.ud) / sc.Su).max()
        ep = np.abs((sol.p[b] - rs.p) / sc.Sp).max()
        dJ = abs(sol.cost[b] - rs.J_aug) / max(1.0, abs(rs.J_aug))
        print("freeflyer parity seed", b, "ex", ex, "eu", eu, "ep", ep, "dJ", dJ)
        assert dJ <= 1e-6 and max(ex, eu, ep) <= 5e-5      # 4 unconverged iterations: the figures are printed above


def test_freeflyer_c5_batch(pkg, handle):
    """C5 at its node count (N = 80, np = 481) on a 32-seed parameter sweep (r0, rf +-5 % are part of the problem data, so
    the sweep perturbs the guesses instead): every seed must end SCP_SOLVED; converged seeds are dynamically feasible
    and keep clear of the obstacles."""
    N, nb = 80, 32
    mdl, traj, pars = _setup(pkg, handle, N, 15, eps=1e-4)
    pars.eps_abs = 1e-5
    pbm = pkg.ptr.create(pars, traj, handle)
    g = traj.guess(N)
    rng = np.random.default_rng(7)
    sc = pbm.scale
    X0 = np.array([g[0] + (2e-3 * sc.Sx * rng.standard_normal(g[0].shape) if b else 0.0) for b in range(nb)])
    U0 = np.array([g[1] for b in range(nb)])
    P0 = np.array([g[2] for b in range(nb)]); P0[:, 0] *= rng.uniform(0.95, 1.05, nb)
    sol = pkg.ptr.solve(pbm, (X0, U0, P0))
    info = pbm.cone.info()
    pbm.close()
    print("freeflyer C5: nk", info["nk"], "nnzL", info["nnzL"], "levels", info["levels"], "iterations",
          sol.iterations.min(), sol.iterations.max(), "feas", int(sol.feas.sum()), "timing", sol.timing)
    assert all(s == "SCP_SOLVED" for s in sol.status), (sol.status, sol.raw_status)
    conv = sol.iterations < 15
    assert sol.feas[conv].all()
    for b in np.where(sol.feas > 0)[0]:
        for H, c in zip(mdl.obs_H, mdl.obs_c):
            d = np.linalg.norm((sol.xd[b][:, 0:3] - c) @ H.T, axis=1)
            assert d.min() >= 1.0 - 1e-3
