"""GPU: planar rendezvous with IMPULSE PTR (examples/rendezvous_planar.py) against the oracle (oracle/rendezvous.py).

  * the device deadband pack (csrc/constraints.cuh) against the oracle's restatement of or -> indicator -> sigmoid ->
    logsumexp, including the exact saturation at the sharp end of the homotopy;
  * the first PTR iteration (iter_max = 1) from the straight-line guess and from the golden file's perturbed guesses,
    at the smooth and at the sharp end of the homotopy: J_aug of the subproblem the device discretized, linearized,
    assembled and solved, within 1e-6 relative of the oracle's subproblem solved by HiGHS and by the oracle interior
    point.  The objective of an LP is determined even where its solution is not (the two exact solvers agree to 3e-7),
    so this pins the IMPULSE DLTV blocks, the deadband rows and the assembled program;
  * one PTR solve, the full 10-step warm-started homotopy sweep (tests.jl:22-95) and two steps from perturbed guesses
    against tests/golden/oracle_ptr_rendezvous.npz (scripts/make_golden_rendezvous.py; oracle interior point at 1e-11):
    every step SCP_SOLVED, stopped by the stopping rule wherever the oracle's was, J_aug within 3e-3 relative (5e-3 where
    the oracle ran into iter_max), the last sweep step dynamically feasible at the terminal condition.  Iteration counts
    and the trajectory are printed, not asserted: the subproblem LPs do not determine the trajectory.  On the very first
    subproblem from the straight-line guess two exact solvers (the oracle interior point and HiGHS) agree on the
    objective to 3e-7 but end up to 4e-3 of the advised range apart in the states and 1e-2 in the inputs
    (tests/test_oracle_rendezvous.py::test_first_subproblem_does_not_determine_the_trajectory), and every later
    subproblem is built around the previous, non-unique, solution.  The J_aug tolerance covers the spread this leaves
    after a full loop, measured on an H100: at most 2.0e-3 where both loops stop on the rule (sweep step 3), 3.3e-3 where
    the oracle runs into iter_max (perturbed seed 1, step 1);
  * seed isolation: a seed alone in a padded group, lock-step and in streamed chains, carries the bits of its solve
    alone.  Seeds that share a group with other live seeds do not (xfail below): the cone solver refines the KKT
    solutions of a whole group while one of its seeds asks for it (kkt_solve, csrc/conic_ipm.cuh), so a seed whose own
    residual is already small enough still takes its group-mates' extra refinement steps;
  * scpb_ptr_set_par between two solves gives the bits of a fresh create with the new kappa;
  * ptr.propagate (IMPULSE) of the final solution.
Both interior points run at 1e-11, as in tests/test_ptr_gpu.py: a 1e-6 comparison of two SCP loops needs subproblem
solutions tighter than that."""
import os

import numpy as np
import pytest

from oracle import rendezvous as rz

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_ptr_rendezvous.npz")
TOL = dict(feastol=1e-11, abstol=1e-11, reltol=1e-11)
N = 30
HOM = rz.Homotopy(1e-3, delta_max=5.0)
KAPPAS = [HOM(x) for x in rz.hom_grid(10)]


def _setup(pkg, handle, kappa, iter_max=30):
    ex = pkg.examples.rendezvous_planar
    mdl = ex.PlanarRendezvousProblem()
    mdl.kappa = kappa
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr")
    pbm = pkg.ptr.create(ex.ptr_parameters(N=N, iter_max=iter_max), traj, handle)
    return mdl, pbm


def _ranges():
    xrg, urg, prg = rz.PlanarRendezvousProblem(N).ranges()
    span = lambda rg: np.array([r[1] - r[0] for r in rg])
    return span(xrg), span(urg), span(prg)


ITER_MAX = 30


def _compare(tag, xd, ud, p, J, it, raw, status, g_xd, g_ud, g_p, g_J, g_it, g_status):
    """status, stopping reason and J_aug asserted; iteration count and trajectory (relative to the advised ranges)
    reported"""
    Sx, Su, Sp = _ranges()
    ex = np.abs(xd - g_xd).max(axis=0) / Sx
    eu = np.abs(ud - g_ud).max(axis=0) / Su
    ep = np.abs(p - g_p) / Sp
    msg = (f"{tag}: {status} it {it} (oracle {g_it}), J {float(J):.10e} (oracle {float(g_J):.10e}, rel "
           f"{abs(J - g_J) / abs(g_J):.1e}), dx/S {ex.max():.1e}, du/S {eu.max():.1e}, dp/S {ep.max():.1e}")
    print(msg)
    assert status == g_status == "SCP_SOLVED", msg
    if g_it < ITER_MAX:          # the oracle stopped on the rule: so must the device loop
        assert raw == 0, msg
    assert abs(J - g_J) <= (3e-3 if g_it < ITER_MAX else 5e-3) * abs(g_J), msg


def _oracle_first_subproblem(xd, ud, p, kappa):
    pb = rz.PlanarRendezvousProblem(N)
    pb.kappa = kappa
    P = rz.ImpulsePTR(pb, rz.ptr_parameters(N=N))
    ref = P.make_solution(xd, ud, p)
    J = {}
    with np.errstate(all="ignore"):
        for prefer in ("ipm", "highs"):
            sol = P.solve_subproblem(ref, prefer=prefer)[0]
            assert sol.status in ("OPTIMAL", "ALMOST_OPTIMAL"), (prefer, sol.status)
            J[prefer] = sol.J_aug
    return J


@pytest.mark.parametrize("kappa", [KAPPAS[0], KAPPAS[9]])
def test_first_iteration_cost_matches_oracle(pkg, handle, kappa):
    """one PTR iteration from the straight-line guess and the three golden perturbed guesses, as one batch"""
    g = np.load(GOLDEN)
    x0, u0, p0 = rz.PlanarRendezvousProblem(N).guess(N)
    X = np.concatenate([x0[None], g["pert_xd0"]]); U = np.concatenate([u0[None], g["pert_ud0"]])
    P = np.concatenate([p0[None], g["pert_p0"]])
    mdl, pbm = _setup(pkg, handle, kappa, iter_max=1)
    try:
        sol = pkg.ptr.solve(pbm, (X, U, P), **TOL)
    finally:
        pbm.close()
    for b in range(X.shape[0]):
        J = _oracle_first_subproblem(X[b], U[b], P[b], kappa)
        msg = f"seed {b}: device {sol.cost[b]!r}, oracle ipm {J['ipm']!r}, HiGHS {J['highs']!r}"
        print(msg)
        assert sol.status[b] == "SCP_SOLVED" and int(sol.iterations[b]) == 1, msg
        for v in J.values():
            assert abs(sol.cost[b] - v) <= 1e-6 * abs(v), msg


@pytest.mark.parametrize("kappa", [KAPPAS[0], KAPPAS[4], KAPPAS[7], KAPPAS[9]])
def test_deadband_pack_matches_oracle(pkg, handle, kappa):
    pb = rz.PlanarRendezvousProblem(N)
    pb.kappa = kappa
    handle.model_set(pkg.lib.MODEL_RENDEZVOUS2D, pb.par(), 6, 12, 1)
    rng = np.random.default_rng(int(kappa))
    B = 4
    xd = rng.standard_normal((B, N, 6))
    ud = rng.uniform(-750.0, 750.0, (B, N, 12))
    ud[0, :, 3:6] = np.linspace(-750.0, 750.0, 3 * N).reshape(N, 3)      # sweep across both deadband edges
    p = np.full((B, 1), 300.0)
    t = rz.orc.t_grid(N)
    out = handle.debug_constraints(t, xd, ud, p, 6, 1)
    assert not out["C"].any() and not out["G"].any()
    n_sat = 0
    for b in range(B):
        for k in range(N):
            a = (t[k], k + 1, xd[b, k], ud[b, k], p[b])
            s, D = pb.s(*a), pb.D(*a)
            for i in range(3):
                fr = ud[b, k, 3 + i]
                _, dOR = rz.smooth_or(fr, kappa, pb.f_db, pb.f_max)
                if dOR == 0.0:          # saturated in the oracle: the device must saturate on the same input, exactly
                    n_sat += 1
                    assert (out["s"][b, k, 2 * i:2 * i + 2] == s[2 * i:2 * i + 2]).all(), (b, k, i, fr)
                    assert (out["D"][b, k, 2 * i:2 * i + 2] == D[2 * i:2 * i + 2]).all(), (b, k, i, fr)
            assert np.abs(out["s"][b, k] - s).max() <= 1e-12 * max(1.0, np.abs(s).max()), (b, k)
            assert np.abs(out["D"][b, k] - D).max() <= 1e-10 * max(1.0, np.abs(D).max()), (b, k)
    if kappa == KAPPAS[-1]:
        assert n_sat > 0.5 * B * N * 3      # at the sharp end every fr outside the deadband is saturated


def test_single_solve_against_oracle(pkg, handle):
    """the first homotopy step (kappa = h(0)) from the problem's own straight-line guess"""
    g = np.load(GOLDEN)
    mdl, pbm = _setup(pkg, handle, KAPPAS[0])
    try:
        sol = pkg.ptr.solve(pbm, None, **TOL)
    finally:
        pbm.close()
    _compare("step 1", sol.xd[0], sol.ud[0], sol.p[0], sol.cost[0], int(sol.iterations[0]), int(sol.raw_status[0]),
             sol.status[0],
             g["xd"][0], g["ud"][0], g["p"][0], g["J_aug"][0], int(g["iterations"][0]), str(g["status"][0]))


@pytest.fixture(scope="module")
def sweep(pkg, handle):
    mdl, pbm = _setup(pkg, handle, float("nan"))
    try:
        sols = pkg.examples.rendezvous_planar.homotopy_sweep(pbm, None, n_hom=10, **TOL)
        pkg.ptr.propagate(pbm, sols[-1])
    finally:
        pbm.close()
    return mdl, sols


def test_homotopy_sweep_against_oracle(sweep):
    """tests.jl:60-82: every seed at the same kappa per step, each step warm-started from the previous solution; the last
    step ends SCP_SOLVED (the reference's assertion) and feasible, and every step is compared with the oracle sweep as
    _compare states"""
    g = np.load(GOLDEN)
    mdl, sols = sweep
    assert mdl.kappa == KAPPAS[-1]
    assert sols[-1].status[0] == "SCP_SOLVED" and sols[-1].feas[0]
    for i, s in enumerate(sols):
        _compare(f"step {i + 1}", s.xd[0], s.ud[0], s.p[0], s.cost[0], int(s.iterations[0]), int(s.raw_status[0]),
                 s.status[0],
                 g["xd"][i], g["ud"][i], g["p"][i], g["J_aug"][i], int(g["iterations"][i]), str(g["status"][i]))


def test_propagate_impulse_of_the_final_solution(pkg, handle, sweep):
    """ptr.propagate uses the problem's IMPULSE method: the same columns as scpb_propagate(IMPULSE) on the same
    trajectory, ending at the terminal condition within the feasibility tolerance (every interval restarts from its
    node, so the end point is off the last node by at most the last segment's defect)"""
    mdl, sols = sweep
    s = sols[-1]
    handle.model_set(pkg.lib.MODEL_RENDEZVOUS2D, mdl.par(), 6, 12, 1)
    tc, xc, _ = handle.propagate(s.td, s.xd, s.ud, s.p, 2 * 10 * (N - 1), method=pkg.lib.IMPULSE)
    assert s.xc.shape == xc.shape == (1, 1 + (N - 1) * 20, 6)
    assert np.array_equal(s.xc, xc)
    Sx, _, _ = _ranges()
    x_tc = np.array([0.0, 0.0, -0.1, 0.0, 0.0, 0.0])
    assert (np.abs(s.xc[0, -1] - x_tc) / Sx).max() <= 5e-3 + 1e-6
    assert (np.abs(s.xd[0, -1] - x_tc) / Sx).max() <= 1e-6


def _bits(sol, b):
    return (sol.xd[b].tobytes(), sol.ud[b].tobytes(), sol.p[b].tobytes(), sol.cost[b].tobytes(), int(sol.iterations[b]),
            int(sol.raw_status[b]))


def _two_steps(pkg, pbm, mdl, guesses, **opts):
    mdl.kappa = KAPPAS[0]
    s1 = pkg.ptr.solve(pbm, guesses, **opts)
    mdl.kappa = KAPPAS[1]
    return s1, pkg.ptr.solve(pbm, s1, **opts)


def test_perturbed_guesses_against_oracle(pkg, handle):
    """the first two homotopy steps from the golden file's seeded perturbed guesses, as one batch"""
    g = np.load(GOLDEN)
    mdl, pbm = _setup(pkg, handle, KAPPAS[0])
    try:
        steps = _two_steps(pkg, pbm, mdl, (g["pert_xd0"], g["pert_ud0"], g["pert_p0"]), **TOL)
    finally:
        pbm.close()
    for i, s in enumerate(steps):
        for b in range(g["pert_xd0"].shape[0]):
            _compare(f"seed {b} step {i + 1}", s.xd[b], s.ud[b], s.p[b], s.cost[b], int(s.iterations[b]),
                     int(s.raw_status[b]), s.status[b],
                     g["pert_xd"][b, i], g["pert_ud"][b, i], g["pert_p"][b, i], g["pert_J_aug"][b, i],
                     int(g["pert_iterations"][b, i]), str(g["pert_status"][b, i]))


def _batch_and_alone(pkg, handle, monkeypatch, chunks, B, seed):
    monkeypatch.setenv("SCPB_PTR_CHUNKS", chunks)
    X, U, P = rz.perturbed_guesses(rz.PlanarRendezvousProblem(N), B, seed=seed)
    mdl, pbm = _setup(pkg, handle, KAPPAS[0])
    try:
        batch = _two_steps(pkg, pbm, mdl, (X, U, P), group=4)
        alone = [_two_steps(pkg, pbm, mdl, (X[b:b + 1], U[b:b + 1], P[b:b + 1]), group=4) for b in range(B)]
    finally:
        pbm.close()
    return batch, alone


@pytest.mark.parametrize("chunks", ["0", "3"])
def test_seed_in_a_padded_group_equals_its_solve_alone(pkg, handle, monkeypatch, chunks):
    """B = 9 seeds in groups of 4: seed 8 shares its group with three padded lanes only.  Lock-step (SCPB_PTR_CHUNKS=0)
    and in three streamed chains its two homotopy steps carry the bits of the same seed solved alone"""
    batch, alone = _batch_and_alone(pkg, handle, monkeypatch, chunks, 9, 77)
    assert all(s == "SCP_SOLVED" for s in batch[1].status)
    for i in range(2):
        assert _bits(batch[i], 8) == _bits(alone[8][i], 0), (chunks, i)


@pytest.mark.xfail(reason="the cone solver refines a group's KKT solutions while any live seed of the group asks for it "
                          "(kkt_solve, csrc/conic_ipm.cuh): group-mates change a seed's last bits", strict=False)
def test_seeds_sharing_a_group_equal_their_solves_alone(pkg, handle, monkeypatch):
    batch, alone = _batch_and_alone(pkg, handle, monkeypatch, "0", 9, 77)
    for b in range(8):
        for i in range(2):
            assert _bits(batch[i], b) == _bits(alone[b][i], 0), (b, i)


def test_set_par_equals_a_fresh_create(pkg, handle):
    """a problem set up at kappa_0 and moved to kappa_5 by scpb_ptr_set_par (ptr.solve pushes the model's current block)
    gives the bits of a problem created at kappa_5"""
    X, U, P = rz.perturbed_guesses(rz.PlanarRendezvousProblem(N), 3, seed=5)
    mdl, pbm = _setup(pkg, handle, KAPPAS[0])
    mdl2, pbm2 = _setup(pkg, handle, KAPPAS[5])
    try:
        first = pkg.ptr.solve(pbm, (X, U, P))
        mdl.kappa = KAPPAS[5]
        moved = pkg.ptr.solve(pbm, (X, U, P))
        fresh = pkg.ptr.solve(pbm2, (X, U, P))
        with pytest.raises(pkg.ScpbError, match="npar"):
            pkg.ptr.set_parameters(pbm, np.zeros(0))
        with pytest.raises(pkg.ScpbError, match="npar"):
            pkg.ptr.set_parameters(pbm, np.zeros(65))
        with pytest.raises(pkg.ScpbError, match="shorter"):           # the dynamics block alone would zero kappa
            pkg.ptr.set_parameters(pbm, mdl.par()[:5])
    finally:
        pbm.close()
        pbm2.close()
    for b in range(3):
        assert _bits(moved, b) == _bits(fresh, b), b
    assert any(_bits(first, b) != _bits(moved, b) for b in range(3))      # kappa did change what was solved


def test_impulse_rejected_at_setup_for_a_model_without_impulse_semantics(pkg, handle, monkeypatch):
    """with the host check lifted, scpb_ptr_setup itself refuses IMPULSE for a pack without impulse semantics"""
    monkeypatch.setattr(pkg.ptr, "IMPULSE_MODELS", (pkg.lib.MODEL_DBLINT,))
    ex = pkg.examples.double_integrator
    traj = pkg.problem.TrajectoryProblem(ex.DoubleIntegratorProblem())
    ex.define_problem(traj, "ptr")
    pars = pkg.ptr.Parameters(N=10, Nsub=10, iter_max=5, disc_method=pkg.ptr.IMPULSE, wvc=1e3, wtr=0.1, eps_abs=1e-5,
                              eps_rel=1e-4, feas_tol=1e-3, q_tr=np.inf, q_exit=np.inf)
    with pytest.raises(pkg.ScpbError, match="scpb_ptr_setup.*impulse semantics"):
        pkg.ptr.create(pars, traj, handle)
