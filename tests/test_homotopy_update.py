"""CPU: the in-loop homotopy callback of test/examples/rendezvous_3d/definition.jl:96-151 as the oracle restates it
(oracle/homotopy_update.py), on scripted improv_rel / stop sequences, and the host side of the device schedule.

The device twin (k_ptr_step, csrc/ptr.cu) is checked against this rule on its own recorded improv_rel in
tests/test_homotopy_schedule_gpu.py."""
import math

import numpy as np
import pytest

from oracle import homotopy_update as hu

GRID = [1.0, 2.0, 4.0, 8.0]
NAN = math.nan


def _run(improv, stop, beta=0.01, iter_max=5, grid=GRID, worsen_tol=-1e-3, unsafe_at=None):
    rule = hu.HomotopyUpdate(grid, beta, worsen_tol, iter_max)
    out = hu.scripted_loop(rule, improv, stop, unsafe_at=unsafe_at)
    return rule, out


def test_nan_at_the_first_iteration_does_not_act():
    rule, (it, status, idx, itmax) = _run([NAN] + [0.5] * 10, [False] * 11)
    assert (it, status) == (5, 1)
    assert idx == [0] * 5 and itmax == [5] * 5 and rule.last_update == 1


def test_update_extends_iter_max_by_the_iterations_since_the_last_update():
    # iteration 3 acts: iter_max 5 + (3 - 1) = 7; iteration 6 acts: 7 + (6 - 3) = 10
    improv = [NAN, 0.5, 0.005, 0.5, 0.5, 0.002] + [0.5] * 10
    rule, (it, status, idx, itmax) = _run(improv, [False] * 16)
    assert idx == [0, 0, 0, 1, 1, 1, 2, 2, 2, 2]
    assert itmax == [5, 5, 7, 7, 7, 10, 10, 10, 10, 10]
    assert (it, status, rule.index, rule.last_update) == (10, 1, 2, 6)


def test_an_update_cancels_the_stop_of_its_iteration():
    # iterations 3 and 4 ask to stop but act, so the loop goes on; iteration 5 does not act and stops
    improv = [NAN, 0.5, 0.001, 0.001, 0.5]
    stop = [False, False, True, True, True]
    rule, (it, status, idx, _) = _run(improv, stop)
    assert (it, status, idx) == (5, 0, [0, 0, 0, 1, 2])


def test_the_end_of_the_grid_lets_the_stop_through():
    improv = [NAN, 0.001, 0.001, 0.001, 0.001]
    stop = [False, True, True, True, True]
    rule, (it, status, idx, itmax) = _run(improv, stop, iter_max=30)
    # three updates exhaust the four-point grid; iteration 5 cannot act and stops
    assert (it, status, idx, rule.index) == (5, 0, [0, 0, 1, 2, 3], 3)
    assert itmax == [30, 31, 32, 33, 33]


def test_one_point_grid_never_acts():
    rule, (it, status, idx, itmax) = _run([NAN, 0.001, 0.0], [False, True, True], grid=[3.0])
    assert (it, status, idx, itmax) == (2, 0, [0, 0], [5, 5])


@pytest.mark.parametrize("improv, acts", [(-1e-3, True), (np.nextafter(-1e-3, -1.0), False), (0.01, True),
                                          (np.nextafter(0.01, 1.0), False), (0.0, True), (NAN, False)])
def test_the_worsen_tol_and_beta_edges(improv, acts):
    rule = hu.HomotopyUpdate(GRID, 0.01, -1e-3, 30)
    assert rule(2, improv) is acts
    assert rule.index == (1 if acts else 0)


def test_beta_minus_infinity_never_acts():
    rule = hu.HomotopyUpdate(GRID, -math.inf, -1e-3, 30)
    assert not any(rule(k, v) for k, v in enumerate([NAN, -1e-3, 0.0, 1e-9, 0.5, -0.5], start=1))


def test_an_unsafe_subproblem_ends_before_the_callback():
    rule, (it, status, idx, itmax) = _run([NAN, 0.001, 0.001], [False] * 3, unsafe_at=3)
    assert (it, status, idx, itmax) == (3, 2, [0, 0, 1], [5, 6, 6])


def test_longest_chain_bound():
    """every update can come at the last allowed iteration: iter_max + (n_grid - 1)(iter_max - 1)"""
    M = 7
    rule = hu.HomotopyUpdate(GRID, 1.0, -1.0, M)
    k = 1
    while k <= rule.iter_max:
        rule(k, 0.5 if k == rule.iter_max else 2.0)
        k += 1
    assert k - 1 == M + (len(GRID) - 1) * (M - 1)


def test_problem_set_homotopy_update_validates_its_grid(pkg):
    traj = pkg.problem.TrajectoryProblem()
    with pytest.raises(ValueError):
        pkg.problem.problem_set_homotopy_update(traj, [], 0.01)
    with pytest.raises(ValueError):
        pkg.problem.problem_set_homotopy_update(traj, [1.0, math.inf], 0.01)
    pkg.problem.problem_set_homotopy_update(traj, GRID, 0.01)
    assert traj.hom["grid"].tolist() == GRID and traj.hom["worsen_tol"] == -1e-3
    pkg.problem.problem_set_homotopy_update(traj, None, 0.01)
    assert traj.hom is None


def test_schedules_are_refused_for_scvx_and_gusto(pkg):
    ex = pkg.examples.rendezvous_planar
    traj = pkg.problem.TrajectoryProblem(ex.PlanarRendezvousProblem())
    ex.define_problem(traj, "ptr")
    ex.homotopy_schedule(traj, 0.01)
    for algo in ("scvx", "gusto"):
        with pytest.raises(pkg.ScpbError, match="PTR only"):
            pkg.ptr.SCPProblem(ex.ptr_parameters(), traj, None, algo=algo)
