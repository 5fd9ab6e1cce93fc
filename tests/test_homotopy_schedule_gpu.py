"""GPU: the in-loop homotopy schedule (scpb_ptr_set_homotopy, k_ptr_step in csrc/ptr.cu) on the planar rendezvous
(examples/rendezvous_planar.py, IMPULSE PTR, N = 30, iter_max = 30), with kappa stepped through
Homotopy(1e-3; delta_max = 5)(LinRange(0, 1, 10)) inside one solve by the callback rule of
test/examples/rendezvous_3d/definition.jl:96-151.

  * a schedule that cannot act (one grid point, or beta = -Inf) gives the bits of a solve without one, lock-step and in
    streamed chains;
  * the recorded history obeys the rule exactly, replayed on the host (oracle/homotopy_update.py) over the device's own
    improv_rel: grid index per iteration, final index, effective iter_max, iteration count and whether the seed stopped
    on the stopping rule;
  * against the oracle loop with the same callback (tests/golden/oracle_ptr_rendezvous_schedule.npz,
    scripts/make_golden_rendezvous_schedule.py): every solve SCP_SOLVED, and the update decisions agree iteration by
    iteration for as long as the oracle's improv_rel keeps a clear margin from beta and worsen_tol.  Past that point the
    two loops may take different decisions, and trajectories, iteration counts and J_aug are printed, not asserted: the
    subproblems are LPs whose solutions are not unique (tests/test_oracle_rendezvous.py), so the two loops follow
    different, equally optimal, subproblem solutions;
  * a seed alone in a padded group equals its solve alone, and per-seed beta in one batch (one seed per group) equals
    every beta solved alone; lock-step and streamed chains give the same bits.
"""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import homotopy_update as hu
from oracle import rendezvous as rz

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_ptr_rendezvous_schedule.npz")
TOL = dict(feastol=1e-11, abstol=1e-11, reltol=1e-11)
N, ITER_MAX, N_HOM = 30, 30, 10
HOM = rz.Homotopy(1e-3, delta_max=5.0)
GRID = [HOM(x) for x in rz.hom_grid(N_HOM)]


def _setup(pkg, handle, kappa=GRID[0], grid=None, beta=0.01):
    ex = pkg.examples.rendezvous_planar
    mdl = ex.PlanarRendezvousProblem()
    mdl.kappa = kappa
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr")
    if grid is not None:
        pkg.problem.problem_set_homotopy_update(traj, grid, beta)
    pbm = pkg.ptr.create(ex.ptr_parameters(N=N, iter_max=ITER_MAX), traj, handle)
    return mdl, traj, pbm


def _bits(sol, b):
    return (sol.xd[b].tobytes(), sol.ud[b].tobytes(), sol.p[b].tobytes(), sol.cost[b].tobytes(), int(sol.iterations[b]),
            int(sol.raw_status[b]))


def _guesses(B, seed):
    return rz.perturbed_guesses(rz.PlanarRendezvousProblem(N), B, seed=seed)


@pytest.mark.parametrize("chunks", ["0", "3"])
@pytest.mark.parametrize("kind", ["one_point", "beta_minus_inf"])
def test_a_schedule_that_cannot_act_changes_no_bit(pkg, handle, monkeypatch, chunks, kind):
    monkeypatch.setenv("SCPB_PTR_CHUNKS", chunks)
    X, U, P = _guesses(9, 31)
    mdl, traj, pbm = _setup(pkg, handle)
    try:
        plain = pkg.ptr.solve(pbm, (X, U, P), group=4)
        if kind == "one_point":
            pkg.problem.problem_set_homotopy_update(traj, [GRID[0]], 1.0)
        else:
            pkg.problem.problem_set_homotopy_update(traj, GRID, -math.inf)
        sched = pkg.ptr.solve(pbm, (X, U, P), group=4)
    finally:
        pbm.close()
    assert (sched.hom_index == 0).all() and (sched.iter_max == ITER_MAX).all()
    for b in range(9):
        assert _bits(sched, b) == _bits(plain, b), (kind, chunks, b)
        n = int(sched.iterations[b])
        assert (sched.hom_history["index"][b, :n] == 0).all() and (sched.hom_history["index"][b, n:] == -1).all()


def _replay(sol, b, beta, worsen_tol=-1e-3):
    """the host rule over the device's own improv_rel: what the device must have done"""
    rule = hu.HomotopyUpdate(GRID, beta, worsen_tol, ITER_MAX)
    n = int(sol.iterations[b])
    imp = sol.hom_history["improv_rel"][b]
    idx = []
    for k in range(1, n + 1):
        idx.append(rule.index)
        rule(k, imp[k - 1])
    return rule, idx


@pytest.fixture(scope="module")
def golden_batch(pkg, handle):
    """the golden betas from the straight-line guess, one seed per group, lock-step"""
    g = np.load(GOLDEN)
    assert np.allclose(g["grid"], GRID, rtol=0, atol=0)
    mdl, traj, pbm = _setup(pkg, handle, grid=GRID)
    x0, u0, p0 = rz.PlanarRendezvousProblem(N).guess(N)
    B = g["beta"].size
    guesses = (np.repeat(x0[None], B, 0), np.repeat(u0[None], B, 0), np.repeat(p0[None], B, 0))
    os.environ["SCPB_PTR_CHUNKS"] = "0"
    try:
        sol = pkg.ptr.solve(pbm, guesses, beta=g["beta"], group=1, **TOL)
    finally:
        del os.environ["SCPB_PTR_CHUNKS"]
        pbm.close()
    return g, sol


def test_history_obeys_the_rule(golden_batch):
    g, sol = golden_batch
    for b, beta in enumerate(g["beta"]):
        rule, idx = _replay(sol, b, beta)
        n = int(sol.iterations[b])
        h = sol.hom_history
        print(f"beta {beta:.0e}: {sol.status[b]} status {int(sol.raw_status[b])} it {n} index {int(sol.hom_index[b])} "
              f"iter_max {int(sol.iter_max[b])} J {sol.cost[b]:.9e}; history {h['index'][b, :n].tolist()}")
        assert sol.status[b] == "SCP_SOLVED"
        assert h["index"][b, :n].tolist() == idx and (h["index"][b, n:] == -1).all()
        assert math.isnan(h["improv_rel"][b, 0]) and np.isfinite(h["improv_rel"][b, 1:n]).all()
        assert np.isnan(h["improv_rel"][b, n:]).all()
        assert int(sol.hom_index[b]) == rule.index and int(sol.iter_max[b]) == rule.iter_max
        if int(sol.raw_status[b]) == 1:       # ran into its own iter_max
            assert n == rule.iter_max
        else:                                 # stopped on the rule, in an iteration the callback did not act
            assert int(sol.raw_status[b]) == 0 and n <= rule.iter_max
            assert idx[-1] == rule.index
    assert (sol.hom_index > 0).any()          # the schedule did act


def test_updates_match_the_oracle_where_the_margin_is_clear(golden_batch):
    """iteration by iteration, while the oracle's improv_rel lies clearly away from both thresholds (by
    max(0.5 beta, 2e-3)), the device and the oracle take the same decision; the comparison ends at the first iteration
    without that margin"""
    g, sol = golden_batch
    wt = float(g["worsen_tol"])
    for b, beta in enumerate(g["beta"]):
        margin = max(0.5 * beta, 2e-3)
        oi, di = g["hist_index"][b], sol.hom_history["index"][b]
        o_imp, d_imp = g["hist_improv_rel"][b], sol.hom_history["improv_rel"][b]
        n_o, n_d = int(g["iterations"][b]), int(sol.iterations[b])
        k = 0
        while k < min(n_o, n_d):
            assert di[k] == oi[k], (beta, k, di[:k + 1], oi[:k + 1])
            if k > 0 and (abs(o_imp[k] - beta) <= margin or abs(o_imp[k] - wt) <= margin):
                break
            k += 1
        print(f"beta {beta:.0e}: decisions agree over {k} iterations; device it {n_d} index {int(sol.hom_index[b])} "
              f"J {sol.cost[b]:.9e}, oracle it {n_o} index {int(g['index'][b])} J {float(g['J_aug'][b]):.9e} "
              f"({str(g['status'][b])})")
        assert k >= 2
        assert sol.status[b] == str(g["status"][b]) == "SCP_SOLVED"


@pytest.mark.parametrize("chunks", ["0", "3"])
def test_seed_in_a_padded_group_equals_its_solve_alone(pkg, handle, monkeypatch, chunks):
    """B = 9 in groups of 4 with a real schedule: seed 8 shares its group with padding only"""
    monkeypatch.setenv("SCPB_PTR_CHUNKS", chunks)
    X, U, P = _guesses(9, 77)
    mdl, traj, pbm = _setup(pkg, handle, grid=GRID, beta=0.01)
    try:
        batch = pkg.ptr.solve(pbm, (X, U, P), group=4)
        alone = pkg.ptr.solve(pbm, (X[8:], U[8:], P[8:]), group=4)
    finally:
        pbm.close()
    assert _bits(batch, 8) == _bits(alone, 0)
    assert int(batch.hom_index[8]) == int(alone.hom_index[0]) and int(batch.iter_max[8]) == int(alone.iter_max[0])
    assert np.array_equal(batch.hom_history["index"][8], alone.hom_history["index"][0])
    assert batch.hom_history["improv_rel"][8].tobytes() == alone.hom_history["improv_rel"][0].tobytes()


def test_per_seed_beta_equals_each_beta_alone_and_streamed_equals_lockstep(pkg, handle, monkeypatch):
    betas = np.array([-1e-3, 3e-3, 1e-2, 3e-2, 1e-1])
    X, U, P = _guesses(1, 5)
    B = betas.size
    G = (np.repeat(X, B, 0), np.repeat(U, B, 0), np.repeat(P, B, 0))
    mdl, traj, pbm = _setup(pkg, handle, grid=GRID)
    try:
        monkeypatch.setenv("SCPB_PTR_CHUNKS", "0")
        lock = pkg.ptr.solve(pbm, G, beta=betas, group=1)
        alone = [pkg.ptr.solve(pbm, (X, U, P), beta=bt, group=1) for bt in betas]
        monkeypatch.setenv("SCPB_PTR_CHUNKS", "3")
        streamed = pkg.ptr.solve(pbm, G, beta=betas, group=1)
    finally:
        pbm.close()
    for b in range(B):
        print(f"beta {betas[b]:+.0e}: it {int(lock.iterations[b])} index {int(lock.hom_index[b])} "
              f"iter_max {int(lock.iter_max[b])} J {lock.cost[b]:.9e}")
        assert _bits(lock, b) == _bits(alone[b], 0), b
        assert _bits(streamed, b) == _bits(lock, b), b
        assert np.array_equal(streamed.hom_history["index"][b], lock.hom_history["index"][b])
        assert int(streamed.iter_max[b]) == int(lock.iter_max[b]) == int(alone[b].iter_max[0])
    assert len({int(i) for i in lock.hom_index}) > 1      # the thresholds lead to different schedules


def test_schedule_arguments_are_checked(pkg, handle):
    mdl, traj, pbm = _setup(pkg, handle)
    h = pbm.handle
    try:
        with pytest.raises(pkg.ScpbError, match="beta"):
            pkg.ptr.solve(pbm, None, beta=0.01)
        grid, pg = pkg.lib._f64(GRID)
        with pytest.raises(pkg.ScpbError, match="par\\[6\\]"):
            h._check(h.lib.scpb_ptr_set_homotopy(pbm.ptr, 6, grid.size, pg, -1e-3), "scpb_ptr_set_homotopy")
        with pytest.raises(pkg.ScpbError, match="last solve had no schedule"):
            h._check(h.lib.scpb_ptr_homotopy_result(pbm.ptr, 1, None, None, 0, None, None), "scpb_ptr_homotopy_result")
        h._check(h.lib.scpb_ptr_set_homotopy(pbm.ptr, 7, grid.size, pg, -1e-3), "scpb_ptr_set_homotopy")
        beta, pb = pkg.lib._f64([0.01, 0.02, 0.03])
        h._check(h.lib.scpb_ptr_set_homotopy_beta(pbm.ptr, 3, pb), "scpb_ptr_set_homotopy_beta")
        x0, u0, p0 = (pkg.lib._f64(a)[0] for a in traj.guess(N))
        with pytest.raises(pkg.ScpbError, match="3 update thresholds for 1 seeds"):
            h._check(h.lib.scpb_ptr_solve(pbm.ptr, 1, x0.ctypes.data_as(pkg.lib._dp), u0.ctypes.data_as(pkg.lib._dp),
                                          p0.ctypes.data_as(pkg.lib._dp), None, None, None, None, None, None, None,
                                          None, None, None), "scpb_ptr_solve")
        # SCvx and GuSTO refuse a problem with a schedule, before anything else about it (this one is IMPULSE as well)
        rp = np.zeros(2, dtype=np.int32)
        z, pz = pkg.lib._f64(np.zeros(2))
        ip = rp.ctypes.data_as(pkg.lib._ip)
        vp = lambda d: ctypes.cast(ctypes.byref(d), ctypes.c_void_p)
        sv, gv = pkg.lib.ScvxDesc(), pkg.lib.GustoDesc()
        scvx = lambda: h._check(h.lib.scpb_scvx_attach(pbm.ptr, vp(sv), ip, ip, pz, pz), "scpb_scvx_attach")
        gusto = lambda: h._check(h.lib.scpb_gusto_attach(pbm.ptr, vp(gv), ip, ip, pz, pz, pz), "scpb_gusto_attach")
        for attach in (scvx, gusto):
            with pytest.raises(pkg.ScpbError, match="in-loop homotopy schedule"):
                attach()
        h._check(h.lib.scpb_ptr_set_homotopy(pbm.ptr, -1, 0, None, 0.0), "scpb_ptr_set_homotopy")   # detach
        for attach in (scvx, gusto):
            with pytest.raises(pkg.ScpbError, match="FOH discretization only"):
                attach()
    finally:
        pbm.close()
