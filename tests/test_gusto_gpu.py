"""GPU: BASELINE config C4 -- quadrotor obstacle avoidance with GuSTO (scpb_gusto_* through the host API,
scptoolbox.jl_b200/gusto.py) against the oracle's GuSTO loop (oracle/gusto.py restating src/solvers/gusto.jl) at the
reference's own test constants (test/examples/quadrotor/tests.jl:81-145: N = 30, Nsub = 15, iter_max = 15, lambda_init =
1e4, lambda_max = 1e9, rho in (0.1, 0.9), beta = 2, gamma_fail = 5, eta in [1e-3, 10] from 10, mu = 0.8 from iteration 6,
eps_abs = eps_rel = 0  =>  exactly iter_max iterations, pen = :quad, q_tr = q_exit = Inf).

Asserted: same status, same iteration count, the same accept / reject / penalty history as far as it shows in the final
trust-region radius and penalty weight (exactly), final cost and physical trajectory within the stated tolerance with both
cone solvers at 1e-11."""
import numpy as np
import pytest

from oracle import problems, ptr as optr

pytestmark = pytest.mark.gpu

TOL = dict(feastol=1e-11, abstol=1e-11, reltol=1e-11)
KW = dict(lam_init=1e4, lam_max=1e9, rho_0=0.1, rho_1=0.9, beta_sh=2.0, beta_gr=2.0, gamma_fail=5.0, eta_init=10.0,
          eta_lb=1e-3, eta_ub=10.0, mu=0.8, iter_mu=6, feas_tol=1e-3)


def _setup(pkg, handle, N, iter_max, eps=0.0):
    ex = pkg.examples.quadrotor
    mdl = ex.QuadrotorProblem()
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "gusto", handle=handle)
    pars = pkg.gusto.Parameters(N, 15, iter_max, pkg.ptr.FOH, KW["lam_init"], KW["lam_max"], KW["rho_0"], KW["rho_1"],
                                KW["beta_sh"], KW["beta_gr"], KW["gamma_fail"], KW["eta_init"], KW["eta_lb"], KW["eta_ub"],
                                KW["mu"], KW["iter_mu"], eps, eps, KW["feas_tol"], "quad", 100.0, np.inf, np.inf, None,
                                {"verbose": 0, "maxit": 100})
    return mdl, traj, pars


def test_correct_convex_matches_oracle(pkg, handle):
    """correct_convex! (scp.jl:275-361) of a guess that violates the input set (thrust below u_min and outside the tilt
    cone, flight time beyond tf_max): the batched GPU projection equals the oracle's, seed by seed."""
    N, nb = 12, 4
    mdl, traj, pars = _setup(pkg, handle, N, 3)
    pbm = pkg.gusto.create(pars, traj, handle)
    pbo = problems.QuadrotorProblem(N)
    so = optr.Scaling(pbo, N)
    sc = pbm.scale
    assert np.abs(sc.Su - so.Su).max() <= 1e-6 * so.Su.max() and np.abs(sc.cu - so.cu).max() <= 1e-6 * so.Su.max()
    g = pbo.guess(N)
    rng = np.random.default_rng(0)
    X0 = np.array([g[0] + 0.1 * rng.standard_normal(g[0].shape) for b in range(nb)])
    U0 = np.array([g[1] + 3.0 * rng.standard_normal(g[1].shape) for b in range(nb)])
    U0[0, :, 3] = 0.1                       # below u_min and inside |a|
    P0 = np.array([g[2] * (1 + b) for b in range(nb)])      # 1.25, 2.5, 3.75 (> tf_max), 5.0
    xd, ud, p = pkg.ptr.correct_convex(pbm, (X0, U0, P0), **TOL)
    pbm.close()
    for b in range(nb):
        xo, uo, po = optr.correct_convex(pbo, so, N, X0[b], U0[b], P0[b], tol=1e-11)
        ex = np.abs(xd[b] - xo).max(); eu = np.abs((ud[b] - uo) / so.Su).max(); ep = np.abs(p[b] - po).max()
        # the L1 projection is an LP-like problem whose minimiser need not be unique (ties along the cone surface):
        # the distance it minimises is the well-defined quantity, the point itself is only held loosely
        dist = lambda x_, u_, p_: (np.abs((x_ - X0[b]) / so.Sx).sum() + np.abs((u_ - U0[b]) / so.Su).sum() +
                                   np.abs((p_ - P0[b]) / so.Sp).sum())
        d1, d2 = dist(xd[b], ud[b], p[b]), dist(xo, uo, po)
        print("correct_convex seed", b, "ex", ex, "eu", eu, "ep", ep, "moved u by", np.abs(uo - U0[b]).max(), "dist", d1, d2)
        assert abs(d1 - d2) <= 1e-8 * max(1.0, d2)
        assert ex <= 1e-7 and eu <= 1e-3 and ep <= 1e-7
        assert p[b][0] <= pbo.tf_max + 1e-9
        for k in range(N):                   # the projected inputs satisfy the input set (definition.jl:188-252)
            a, sg = ud[b][k, 0:3], ud[b][k, 3]
            assert pbo.u_min - 1e-8 <= sg <= pbo.u_max + 1e-8 and np.linalg.norm(a) <= sg + 1e-8
            assert sg * np.cos(pbo.tilt_max) - a[2] <= 1e-8


def _oracle_gusto_worker(args):
    N, K, eps_abs, eps_rel, xd, ud, p, tol = args
    import warnings
    warnings.filterwarnings("ignore")
    from oracle import gusto as og, problems as pr, ptr as op
    pb = pr.QuadrotorProblem(N)
    P = og.GuSTO(pb, og.Parameters(N=N, Nsub=15, iter_max=K, eps_abs=eps_abs, eps_rel=eps_rel, solver_tol=tol, **KW))
    try:
        guess = op.correct_convex(pb, P.scale, N, xd, ud, p, tol=tol)      # generate_initial_guess, gusto.jl:517-526
    except RuntimeError as e:
        return f"SCP_FAILED ({e})", 0, None, None, None, np.nan, False, np.nan, np.nan
    r = P.solve(guess)
    s = r["sol"]
    return r["status"], r["iterations"], s.xd, s.ud, s.p, s.J_aug, bool(s.feas), r["eta"], r["lam"]


def _seeds(N, nb):
    import bench
    pbo = problems.QuadrotorProblem(N)
    return pbo, bench.make_seeds_c4(pbo.guess(N), nb, 0, pbo.r0, pbo.rf)


def _compare(sol, b, ref, sc, tol_x, tol_J):
    st, its, xd, ud, p, J, feas, eta, lam = ref
    ex = np.abs(sol.xd[b] - xd).max(); eu = np.abs((sol.ud[b] - ud) / sc.Su).max()
    ep = np.abs((sol.p[b] - p) / sc.Sp).max(); dJ = abs(sol.cost[b] - J) / max(1.0, abs(J))
    print("gusto parity seed", b, "iters", sol.iterations[b], its, "eta", sol.eta[b], eta, "lam", sol.lam[b], lam, "ex", ex, "eu", eu,
          "ep", ep, "dJ", dJ, "J_aug", sol.cost[b], J, "feas", sol.feas[b], feas)
    assert int(sol.iterations[b]) == its
    assert sol.eta[b] == pytest.approx(eta, rel=1e-12) and sol.lam[b] == pytest.approx(lam, rel=1e-12)
    assert bool(sol.feas[b]) == feas
    assert dJ <= tol_J and max(ex, eu, ep) <= tol_x


def test_batched_gusto_matches_oracle_gusto(pkg, handle):
    """The reference's own test configuration (eps = 0 => exactly 15 iterations), nominal guess and two SURVEY 8(d) seeds.
    With both cone solvers at 1e-11 eta / lambda are identical and J_aug and the trajectory agree closely after the 15
    forced iterations, but not to solver accuracy -- the LCvx relaxation |a| <= sigma is not
    tight everywhere at the optimum, so the acceleration profile (and with it the path) has a flat direction that the
    forced iterations keep moving along; asserted: 2e-6 on J_aug, 1e-3 on the trajectory (the seeds that stop on the
    stopping rule are compared in test_gusto_outcomes_match_oracle)."""
    import multiprocessing as mp
    N, K = 30, 15
    mdl, traj, pars = _setup(pkg, handle, N, K)
    pbo, (X, U, P) = _seeds(N, 4)
    pick = [0, 1, 3]                        # seed 2 draws tdil = 1.106 s: infeasible, see test_gusto_outcomes_match_oracle
    X0, U0, P0 = X[pick], U[pick], P[pick]
    pbm = pkg.gusto.create(pars, traj, handle)
    sol = pkg.gusto.solve(pbm, (X0, U0, P0), **TOL)
    info = pbm.cone.info()
    sc = pbm.scale
    pbm.close()
    print("quadrotor GuSTO KKT", info["nk"], info["nnzL"], info["levels"], "timing", sol.timing)
    with mp.get_context("fork").Pool(len(pick)) as pool:
        refs = pool.map(_oracle_gusto_worker, [(N, K, 0.0, 0.0, X0[b], U0[b], P0[b], 1e-11) for b in range(len(pick))], chunksize=1)
    for b in range(len(pick)):
        assert sol.status[b] == refs[b][0] == "SCP_SOLVED", (sol.status, sol.raw_status, refs[b][0])
        assert refs[b][1] == K
        _compare(sol, b, refs[b], sc, 1e-3, 2e-6)
        # the keep-out zones are respected (nonconvex feasibility of the converged trajectory)
        assert max(pbo.s(0, k + 1, sol.xd[b][k], None, sol.p[b]).max() for k in range(N)) <= 1e-3


def test_gusto_outcomes_match_oracle(pkg, handle):
    """16 SURVEY 8(d) seeds with the stopping tolerances on (eps_abs = 1e-5, eps_rel = 1e-4), seed by seed against the oracle:
    the same seeds are solved, in the same number of iterations, to the same trajectory; the same seeds fail.  GuSTO keeps
    the linearised dynamics as hard constraints, so (i) a flight-time guess below ~1.13 s makes the first subproblem
    infeasible (the straight-line guess has v = 0 and a + g = 0: no sensitivity to tdil) and (ii) guesses whose required
    velocity change exceeds the shrunken trust region enter a reject / lambda-escalation spiral that ends in a solver
    failure -- in the oracle (iteration 7-8) as in the product (iteration 3-4, its cone solver gives up earlier on the
    lambda-inflated programs).  Failure kind and iteration are therefore not compared, only the fact."""
    import multiprocessing as mp
    N, K, nb = 30, 15, 16
    mdl, traj, pars = _setup(pkg, handle, N, K)
    pars.eps_abs, pars.eps_rel = 1e-5, 1e-4
    pbo, (X0, U0, P0) = _seeds(N, nb)
    pbm = pkg.gusto.create(pars, traj, handle)
    sol = pkg.gusto.solve(pbm, (X0, U0, P0), feastol=1e-10, abstol=1e-10, reltol=1e-10)
    sc = pbm.scale
    pbm.close()
    with mp.get_context("fork").Pool(8) as pool:
        refs = pool.map(_oracle_gusto_worker, [(N, K, 1e-5, 1e-4, X0[b], U0[b], P0[b], 1e-10) for b in range(nb)], chunksize=1)
    nsolved = 0
    for b in range(nb):
        ok_o = refs[b][0] == "SCP_SOLVED"
        print("seed", b, "tdil0 %.3f" % P0[b][0], sol.status[b], int(sol.iterations[b]), "| oracle", refs[b][0], refs[b][1])
        assert (sol.status[b] == "SCP_SOLVED") == ok_o
        if ok_o:
            nsolved += 1
            _compare(sol, b, refs[b], sc, 2e-2, 2e-5)
        if P0[b][0] < 1.12:   # first subproblem infeasible: a clear case ends with the certificate (test_infeasible_guess_is_
            # reported), a marginal one (tdil = 1.106 s against the ~1.13 s limit) exhausts the iterations -- in the oracle too
            assert sol.status[b].startswith("SCP_FAILED") and int(sol.iterations[b]) == 1
    assert nsolved >= 10


def test_gusto_c4_batch(pkg, handle):
    """C4 at the bench node count (N = 60) on 64 SURVEY 8(d) seeds with the stopping tolerances on: seeds stop on their own
    schedule (frozen seeds are skipped by the device loop); every solved seed is dynamically feasible and clear of the
    obstacles; every seed whose flight-time guess is at least 1.5 s is solved (see test_gusto_outcomes_match_oracle for
    the ones below)."""
    N, nb = 60, 64
    mdl, traj, pars = _setup(pkg, handle, N, 15, eps=0.0)
    pars.eps_abs, pars.eps_rel = 1e-5, 1e-4
    pbo, (X0, U0, P0) = _seeds(N, nb)
    pbm = pkg.gusto.create(pars, traj, handle)
    sol = pkg.gusto.solve(pbm, (X0, U0, P0))
    pbm.close()
    ok = np.array([s_ == "SCP_SOLVED" for s_ in sol.status])
    its = np.asarray(sol.iterations)[ok]
    print("quadrotor C4 batch: solved", int(ok.sum()), "of", nb, "iterations min/med/max", its.min(), int(np.median(its)), its.max(),
          "timing", sol.timing, "costs", sorted(set(np.round(sol.cost[ok], 4))))
    assert ok.sum() >= 0.6 * nb
    for b in range(nb):
        if P0[b][0] >= 1.5:
            assert ok[b], (b, P0[b], sol.status[b])
        # a seed whose penalty weight ran past lambda_max stops as the reference does ("infeas", gusto.jl:1220-1227) with
        # whatever penalised point it holds; the others stopped on the convergence test and must be feasible and clear
        if ok[b] and sol.lam[b] <= KW["lam_max"]:
            assert sol.feas[b] == 1
            assert max(pbo.s(0, k + 1, sol.xd[b][k], None, sol.p[b]).max() for k in range(N)) <= 1e-3


def test_infeasible_guess_is_reported(pkg, handle):
    """A flight-time guess of 0.8 s makes the first GuSTO subproblem primal infeasible (hard linearised dynamics, see
    test_gusto_c4_batch): the seed ends SCP_FAILED with the cone solver's INFEASIBLE certificate, as ECOS would report to
    the reference (unsafe_solution, scp.jl:965-980), while the nominal seed next to it in the same batch is solved."""
    N = 30
    mdl, traj, pars = _setup(pkg, handle, N, 15)
    pbo = problems.QuadrotorProblem(N)
    g = pbo.guess(N)
    X0 = np.array([g[0], g[0]]); U0 = np.array([g[1], g[1]]); P0 = np.array([g[2], [0.8]])
    pbm = pkg.gusto.create(pars, traj, handle)
    sol = pkg.gusto.solve(pbm, (X0, U0, P0))
    pbm.close()
    print("statuses", sol.status, sol.iterations)
    assert sol.status[0] == "SCP_SOLVED" and int(sol.iterations[0]) == 15
    assert sol.status[1] == "SCP_FAILED (INFEASIBLE)" and int(sol.iterations[1]) == 1
