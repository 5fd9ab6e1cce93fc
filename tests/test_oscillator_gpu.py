"""GPU: the forced-oscillator deadband problem with FOH PTR (examples/oscillator.py, a model with a fixed final time: no F
column) against the oracle (oracle/oscillator.py).

  * K1 (k_discretize_foh with NF = 0): A, B-, B+, r, E, the defects and the feasibility flags against the oracle's FOH
    discretization, F all zeros; scpb_propagate against the oracle roll-out;
  * the device deadband pack (csrc/constraints.cuh, the shared SmoothOr with a scalar match) against the oracle's
    restatement of or -> indicator -> sigmoid -> logsumexp, bitwise wherever the oracle saturates;
  * the first PTR iteration (iter_max = 1) from the reference guess and from the golden file's perturbed guesses, at both
    ends of the homotopy: J_aug within 1e-6 relative of the oracle's subproblem solved by HiGHS and by the oracle interior
    point;
  * the 10-step warm-started homotopy sweep of tests.jl:60-82 and two steps from perturbed guesses against
    tests/golden/oracle_ptr_oscillator.npz (scripts/make_golden_oscillator.py; oracle interior point at 1e-11): every
    step SCP_SOLVED, stopped by the stopping rule wherever the oracle's was, the oracle's iteration count, J_aug within
    1e-9 relative and every entry of x, u and p within 1e-8.  Unlike the planar rendezvous, these subproblem LPs
    determine their solution (tests/test_oracle_oscillator.py::test_subproblems_determine_the_trajectory), so the
    trajectories are asserted.  Measured on an H100: J_aug at most 5.4e-11 relative and the trajectories at most 1.9e-10
    apart, a margin of about 20x and 50x;
  * the in-loop homotopy schedule on FOH (scpb_ptr_set_homotopy; the pack's KAPPA slot is par[5]): a schedule that
    cannot act changes no bit, lock-step and streamed; the device history obeys the rule replayed on its own improv_rel;
    the decisions match the oracle's (golden sched_* keys) while the oracle's improv_rel keeps a clear margin; streamed
    equals lock-step;
  * a seed alone in a padded group carries the bits of its solve alone;
  * SCvx and GuSTO refuse the oscillator (SCPB_ERR_UNSUPPORTED).
Both interior points run at 1e-11, as in tests/test_ptr_gpu.py."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import homotopy_update as hu
from oracle import orc
from oracle import oscillator as osc
from oracle import rendezvous as rz

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_ptr_oscillator.npz")
TOL = dict(feastol=1e-11, abstol=1e-11, reltol=1e-11)
N, ITER_MAX, N_HOM = 30, 10, 10
KAPPAS = [osc.hom()(x) for x in rz.hom_grid(N_HOM)]


def _setup(pkg, handle, kappa, iter_max=ITER_MAX, grid=None, beta=0.01):
    ex = pkg.examples.oscillator
    mdl = ex.OscillatorProblem(N)
    mdl.kappa = kappa
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr")
    if grid is not None:
        pkg.problem.problem_set_homotopy_update(traj, grid, beta)
    return mdl, traj, pkg.ptr.create(ex.ptr_parameters(N=N, iter_max=iter_max), traj, handle)


def _bits(sol, b):
    return (sol.xd[b].tobytes(), sol.ud[b].tobytes(), sol.p[b].tobytes(), sol.cost[b].tobytes(), int(sol.iterations[b]),
            int(sol.raw_status[b]))


def test_discretize_and_propagate_match_oracle(pkg, handle):
    pb = osc.OscillatorProblem(N)
    X, U, P = osc.perturbed_guesses(pb, 4, seed=3)
    U[..., 0] = np.random.default_rng(4).uniform(-0.3, 0.3, (4, N))
    X[0], U[0], P[0] = pb.guess(N)
    handle.model_set(pkg.lib.MODEL_OSCILLATOR, pb.par(), 2, 4, N)
    iS = np.array([0.5, 1.0])
    t = orc.t_grid(N)
    out = handle.discretize(t, X, U, P, iS, 5e-3, 10)
    assert not out["F"].any()
    for b in range(4):
        d = osc.discretize(pb, X[b], U[b], P[b], 10, iS, 5e-3)
        for key, ref in (("A", d.A), ("Bm", d.Bm), ("Bp", d.Bp), ("E", d.E)):
            got = out[key][b].reshape(N - 1, ref.shape[2], ref.shape[1]).transpose(0, 2, 1)
            assert np.abs(got - ref).max() <= 1e-11 * np.abs(ref).max(), (b, key)
        scale = max(np.abs(X[b]).max(), 1.0)
        assert np.abs(out["r"][b] - d.r).max() <= 1e-11 * scale, b
        assert np.abs(out["defect"][b] - d.defect).max() <= 1e-11 * scale, b
        assert bool(out["feas"][b]) == d.feas, b
    res = 2 * 10 * (N - 1)
    _, xc, _ = handle.propagate(t, X, U, P, res)
    for b in range(4):
        ref = osc.propagate(pb, X[b], U[b], P[b], res)
        assert np.abs(xc[b] - ref).max() <= 1e-8 * max(np.abs(ref).max(), 1.0), b


@pytest.mark.parametrize("step", [0, 2, 5, 9])
def test_deadband_pack_matches_oracle(pkg, handle, step):
    kappa = KAPPAS[step]
    pb = osc.OscillatorProblem(N)
    pb.kappa = kappa
    handle.model_set(pkg.lib.MODEL_OSCILLATOR, pb.par(), 2, 4, N)
    rng = np.random.default_rng(step)
    B = 4
    xd = rng.standard_normal((B, N, 2))
    ud = rng.uniform(-0.3, 0.3, (B, N, 4))
    ud[0, :, 1] = np.linspace(-0.3, 0.3, N)          # sweep across both deadband edges
    p = rng.uniform(0.0, 1.0, (B, N))
    t = orc.t_grid(N)
    out = handle.debug_constraints(t, xd, ud, p, 2, 1)
    assert not out["C"].any() and not out["G"].any()
    n_sat = 0
    for b in range(B):
        for k in range(N):
            a = (t[k], k + 1, xd[b, k], ud[b, k], p[b])
            s, D = pb.s(*a), pb.D(*a)
            if osc.smooth_or(ud[b, k, 1], kappa, pb.a_db, pb.a_max)[1] == 0.0:   # saturated in the oracle: bitwise
                n_sat += 1
                assert (out["s"][b, k] == s).all() and (out["D"][b, k] == D).all(), (b, k)
            assert np.abs(out["s"][b, k] - s).max() <= 1e-12 * max(1.0, np.abs(s).max()), (b, k)
            assert np.abs(out["D"][b, k] - D).max() <= 1e-10 * max(1.0, np.abs(D).max()), (b, k)
    if step == N_HOM - 1:
        assert n_sat > 0.5 * B * N          # at the sharp end every ar outside the deadband is saturated


def _oracle_first_subproblem(xd, ud, p, kappa):
    pb = osc.OscillatorProblem(N)
    pb.kappa = kappa
    P = osc.OscillatorPTR(pb, osc.ptr_parameters(N=N))
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
    g = np.load(GOLDEN)
    x0, u0, p0 = osc.OscillatorProblem(N).guess(N)
    X = np.concatenate([x0[None], g["pert_xd0"]]); U = np.concatenate([u0[None], g["pert_ud0"]])
    P = np.concatenate([p0[None], g["pert_p0"]])
    mdl, traj, pbm = _setup(pkg, handle, kappa, iter_max=1)
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


def _compare(tag, s, b, g_xd, g_ud, g_p, g_J, g_it, g_status):
    """status, stopping reason, J_aug, iteration count and trajectory asserted (the subproblems determine it)"""
    J, it, raw = float(s.cost[b]), int(s.iterations[b]), int(s.raw_status[b])
    dx, du, dp = np.abs(s.xd[b] - g_xd).max(), np.abs(s.ud[b] - g_ud).max(), np.abs(s.p[b] - g_p).max()
    msg = (f"{tag}: {s.status[b]} it {it} (oracle {g_it}), J {J:.12e} (oracle {float(g_J):.12e}, rel "
           f"{abs(J - g_J) / abs(g_J):.1e}), dx {dx:.1e}, du {du:.1e}, dp {dp:.1e}")
    print(msg)
    assert s.status[b] == g_status == "SCP_SOLVED", msg
    if g_it < ITER_MAX:          # the oracle stopped on the rule: so must the device loop
        assert raw == 0, msg
    assert abs(J - g_J) <= 1e-9 * abs(g_J), msg
    assert it == g_it, msg
    assert max(dx, du, dp) <= 1e-8, msg


@pytest.fixture(scope="module")
def sweep(pkg, handle):
    mdl, traj, pbm = _setup(pkg, handle, float("nan"))
    try:
        sols = pkg.examples.oscillator.homotopy_sweep(pbm, None, n_hom=N_HOM, **TOL)
    finally:
        pbm.close()
    return mdl, sols


def test_homotopy_sweep_against_oracle(sweep):
    """tests.jl:60-82: every step compared with the oracle sweep; the last step ends SCP_SOLVED (the reference's
    assertion) and feasible"""
    g = np.load(GOLDEN)
    mdl, sols = sweep
    assert mdl.kappa == KAPPAS[-1]
    assert sols[-1].status[0] == "SCP_SOLVED" and sols[-1].feas[0]
    for i, s in enumerate(sols):
        _compare(f"step {i + 1}", s, 0, g["xd"][i], g["ud"][i], g["p"][i], g["J_aug"][i], int(g["iterations"][i]),
                 str(g["status"][i]))


def test_perturbed_guesses_against_oracle(pkg, handle):
    """the first two homotopy steps from the golden file's seeded perturbed guesses, as one batch"""
    g = np.load(GOLDEN)
    mdl, traj, pbm = _setup(pkg, handle, KAPPAS[0])
    try:
        s1 = pkg.ptr.solve(pbm, (g["pert_xd0"], g["pert_ud0"], g["pert_p0"]), **TOL)
        mdl.kappa = KAPPAS[1]
        s2 = pkg.ptr.solve(pbm, s1, **TOL)
    finally:
        pbm.close()
    for i, s in enumerate((s1, s2)):
        for b in range(g["pert_xd0"].shape[0]):
            _compare(f"seed {b} step {i + 1}", s, b, g["pert_xd"][b, i], g["pert_ud"][b, i], g["pert_p"][b, i],
                     g["pert_J_aug"][b, i], int(g["pert_iterations"][b, i]), str(g["pert_status"][b, i]))


@pytest.mark.parametrize("chunks", ["0", "3"])
def test_seed_in_a_padded_group_equals_its_solve_alone(pkg, handle, monkeypatch, chunks):
    """B = 9 seeds in groups of 4: seed 8 shares its group with padding only, lock-step and in three streamed chains"""
    monkeypatch.setenv("SCPB_PTR_CHUNKS", chunks)
    X, U, P = osc.perturbed_guesses(osc.OscillatorProblem(N), 9, seed=77)
    mdl, traj, pbm = _setup(pkg, handle, KAPPAS[0])
    try:
        batch = pkg.ptr.solve(pbm, (X, U, P), group=4)
        alone = pkg.ptr.solve(pbm, (X[8:], U[8:], P[8:]), group=4)
    finally:
        pbm.close()
    assert all(s == "SCP_SOLVED" for s in batch.status)
    assert _bits(batch, 8) == _bits(alone, 0)


# ------------------------------------------------------------------ in-loop homotopy schedule on FOH
@pytest.mark.parametrize("chunks", ["0", "3"])
@pytest.mark.parametrize("kind", ["one_point", "beta_minus_inf"])
def test_a_schedule_that_cannot_act_changes_no_bit(pkg, handle, monkeypatch, chunks, kind):
    monkeypatch.setenv("SCPB_PTR_CHUNKS", chunks)
    X, U, P = osc.perturbed_guesses(osc.OscillatorProblem(N), 9, seed=31)
    mdl, traj, pbm = _setup(pkg, handle, KAPPAS[0])
    try:
        plain = pkg.ptr.solve(pbm, (X, U, P), group=4)
        if kind == "one_point":
            pkg.problem.problem_set_homotopy_update(traj, [KAPPAS[0]], 1.0)
        else:
            pkg.problem.problem_set_homotopy_update(traj, KAPPAS, -math.inf)
        sched = pkg.ptr.solve(pbm, (X, U, P), group=4)
    finally:
        pbm.close()
    assert (sched.hom_index == 0).all() and (sched.iter_max == ITER_MAX).all()
    for b in range(9):
        assert _bits(sched, b) == _bits(plain, b), (kind, chunks, b)


@pytest.fixture(scope="module")
def golden_schedule(pkg, handle):
    """the golden betas from the reference guess, one seed per group, lock-step and in three streamed chains"""
    g = np.load(GOLDEN)
    assert np.array_equal(g["sched_grid"], KAPPAS)
    mdl, traj, pbm = _setup(pkg, handle, KAPPAS[0], grid=KAPPAS)
    x0, u0, p0 = osc.OscillatorProblem(N).guess(N)
    B = g["sched_beta"].size
    guesses = (np.repeat(x0[None], B, 0), np.repeat(u0[None], B, 0), np.repeat(p0[None], B, 0))
    out = {}
    try:
        for chunks in ("0", "3"):
            os.environ["SCPB_PTR_CHUNKS"] = chunks
            out[chunks] = pkg.ptr.solve(pbm, guesses, beta=g["sched_beta"], group=1, **TOL)
    finally:
        del os.environ["SCPB_PTR_CHUNKS"]
        pbm.close()
    return g, out["0"], out["3"]


def test_schedule_history_obeys_the_rule(golden_schedule):
    g, sol, _ = golden_schedule
    for b, beta in enumerate(g["sched_beta"]):
        rule = hu.HomotopyUpdate(KAPPAS, beta, float(g["sched_worsen_tol"]), ITER_MAX)
        n = int(sol.iterations[b])
        h = sol.hom_history
        idx = []
        for k in range(1, n + 1):
            idx.append(rule.index)
            rule(k, h["improv_rel"][b, k - 1])
        print(f"beta {beta:.0e}: {sol.status[b]} status {int(sol.raw_status[b])} it {n} index {int(sol.hom_index[b])} "
              f"iter_max {int(sol.iter_max[b])} J {sol.cost[b]:.12e}; history {h['index'][b, :n].tolist()}")
        assert sol.status[b] == "SCP_SOLVED"
        assert h["index"][b, :n].tolist() == idx and (h["index"][b, n:] == -1).all()
        assert int(sol.hom_index[b]) == rule.index and int(sol.iter_max[b]) == rule.iter_max
        if int(sol.raw_status[b]) == 1:
            assert n == rule.iter_max
        else:
            assert int(sol.raw_status[b]) == 0 and n <= rule.iter_max and idx[-1] == rule.index
    assert (sol.hom_index > 0).all()          # the schedule acted on every seed


def test_schedule_decisions_match_the_oracle_where_the_margin_is_clear(golden_schedule):
    """iteration by iteration, while the oracle's improv_rel lies clearly away from both thresholds (by
    max(0.5 beta, 2e-3)), the device and the oracle take the same decision.  For beta = 1e-2 and 3e-2 the margin runs
    out at iteration 3 (improv_rel 5.5e-3).  The subproblems determine the loop, so the iteration count, the final grid
    index and J_aug (1e-9 relative) are asserted too; measured on an H100 the whole histories agree"""
    g, sol, _ = golden_schedule
    wt = float(g["sched_worsen_tol"])
    for b, beta in enumerate(g["sched_beta"]):
        margin = max(0.5 * beta, 2e-3)
        oi, di = g["sched_hist_index"][b], sol.hom_history["index"][b]
        o_imp = g["sched_hist_improv_rel"][b]
        n_o, n_d = int(g["sched_iterations"][b]), int(sol.iterations[b])
        k = 0
        while k < min(n_o, n_d):
            assert di[k] == oi[k], (beta, k, di[:k + 1], oi[:k + 1])
            if k > 0 and (abs(o_imp[k] - beta) <= margin or abs(o_imp[k] - wt) <= margin):
                break
            k += 1
        print(f"beta {beta:.0e}: decisions agree over {k} iterations; device it {n_d} index {int(sol.hom_index[b])} "
              f"J {sol.cost[b]:.12e}, oracle it {n_o} index {int(g['sched_index'][b])} "
              f"J {float(g['sched_J_aug'][b]):.12e}")
        assert k >= 2
        assert sol.status[b] == str(g["sched_status"][b]) == "SCP_SOLVED"
        assert n_d == n_o and int(sol.hom_index[b]) == int(g["sched_index"][b])
        assert abs(sol.cost[b] - g["sched_J_aug"][b]) <= 1e-9 * abs(g["sched_J_aug"][b])


def test_schedule_streamed_equals_lockstep(golden_schedule):
    g, lock, streamed = golden_schedule
    for b in range(g["sched_beta"].size):
        assert _bits(streamed, b) == _bits(lock, b), b
        assert np.array_equal(streamed.hom_history["index"][b], lock.hom_history["index"][b])
        assert int(streamed.iter_max[b]) == int(lock.iter_max[b])


# ------------------------------------------------------------------ refusals
def test_scvx_and_gusto_refuse_the_oscillator(pkg, handle):
    """SCvx has no penalty for the deadband pack (scvx_has_pack) and GuSTO no node terms for it (launch_gusto_nodes):
    both refuse with SCPB_ERR_UNSUPPORTED (-4) instead of running with the penalty rows left at zero"""
    mdl, traj, pbm = _setup(pkg, handle, KAPPAS[0])
    h, sm = pbm.handle, pbm.sm
    vp = lambda d: ctypes.cast(ctypes.byref(d), ctypes.c_void_p)
    try:
        rp = np.zeros(3, dtype=np.int32)
        z, pz = pkg.lib._f64(np.zeros(2))
        ip = rp.ctypes.data_as(pkg.lib._ip)
        sv = pkg.lib.ScvxDesc()
        sv.oeta = sm.oeta
        with pytest.raises(pkg.ScpbError, match=r"\(-4\).*no penalty for the constraint pack of model 7"):
            h._check(h.lib.scpb_scvx_attach(pbm.ptr, vp(sv), ip, ip, pz, pz), "scpb_scvx_attach")
        gv = pkg.lib.GustoDesc()
        gv.oeta, gv.olam, gv.nsq, gv.q_tr = sm.oeta, sm.olam, 0, 0
        h._check(h.lib.scpb_gusto_attach(pbm.ptr, vp(gv), ip, ip, pz, pz, pz), "scpb_gusto_attach")
        x0, u0, p0 = (pkg.lib._f64(a[None])[0] for a in traj.guess(N))
        with pytest.raises(pkg.ScpbError, match=r"\(-4\).*no device pack for model 7"):
            h._check(h.lib.scpb_gusto_solve(pbm.ptr, 1, x0.ctypes.data_as(pkg.lib._dp), u0.ctypes.data_as(pkg.lib._dp),
                                            p0.ctypes.data_as(pkg.lib._dp), None, None, None, None, None, None, None,
                                            None, None, None, None, None), "scpb_gusto_solve")
    finally:
        pbm.close()
    with pytest.raises(pkg.ScpbError, match="convex state sets"):          # the host refuses it before the device
        gp = pkg.gusto.Parameters(N, 10, 5, pkg.lib.FOH, 1.0, 1e9, 0.1, 0.9, 2.0, 2.0, 10.0, 1.0, 1e-3, 10.0, 0.8, 5,
                                  eps_abs=1e-5, eps_rel=1e-4, feas_tol=5e-3)
        pkg.gusto.create(gp, traj, handle)
