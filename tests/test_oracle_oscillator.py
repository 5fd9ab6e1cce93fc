"""CPU: the oracle's forced-oscillator deadband problem (oracle/oscillator.py, restating test/examples/oscillator and the
smooth OR chain of src/utils/helper.jl:600-807 with a scalar match) and its FOH homotopy sweep (tests.jl:22-80)."""
import math
import os

import numpy as np
import pytest
import scipy.linalg

from oracle import orc
from oracle import oscillator as osc
from oracle import rendezvous as rz

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_ptr_oscillator.npz")
KAPPAS = [osc.hom()(x) for x in rz.hom_grid(10)]


def test_homotopy_end_points():
    assert KAPPAS[0] == pytest.approx(math.log(99.0), rel=1e-15)
    assert KAPPAS[-1] == pytest.approx(math.log(99.0) / 1e-8, rel=1e-12)          # ~4.6e8, the sharp end


def test_scalar_match_is_the_sigmoid_of_one_value():
    """or(...; match = a_max - a_db, normalize = a_max - a_db): the indicator's shift is 1 - sigmoid([1]), where the
    logsumexp of one value is that value"""
    pb = osc.OscillatorProblem()
    for kappa in KAPPAS[:3]:
        OR, _ = osc.smooth_or(0.0, kappa, pb.a_db, pb.a_max)
        sg0 = 1 - 1 / (1 + math.exp(kappa * ((kappa * (-0.2) + math.log(1.0 + math.exp(0.0))) / kappa)))
        shift = 1 - (1 - 1 / (1 + math.exp(kappa * ((kappa * 1.0 + math.log(1.0)) / kappa))))
        assert OR == pytest.approx(sg0 + shift, rel=1e-14)


@pytest.mark.parametrize("kappa", [KAPPAS[0], KAPPAS[1], KAPPAS[2]])
def test_or_gradient_matches_finite_differences(kappa):
    pb = osc.OscillatorProblem()
    for ar in (-0.3, -0.12, -0.06, -0.01, 0.0, 0.03, 0.055, 0.2, 0.3):
        h = 1e-7
        OR, dOR = osc.smooth_or(ar, kappa, pb.a_db, pb.a_max)
        fd = (osc.smooth_or(ar + h, kappa, pb.a_db, pb.a_max)[0] - osc.smooth_or(ar - h, kappa, pb.a_db, pb.a_max)[0]) / (2 * h)
        assert abs(dOR - fd) <= 1e-6 * abs(fd) + 1e-8, (kappa, ar, dOR, fd)      # 1e-8: round-off of the quotient
        assert -1e-12 <= OR <= 1.0 + 1e-6       # the shift matches [a_max - a_db] alone: OR(a_max) is 1 + 1.6e-7


def test_or_saturates_exactly_at_the_sharp_end():
    """At the last homotopy step, outside the deadband, sigma rounds to exactly 1 and the gradient factor to exactly 0;
    inside it sigma rounds to 0: the values the device pack must reproduce bit for bit"""
    pb = osc.OscillatorProblem()
    for ar in (-0.3, -0.1, -0.051, 0.051, 0.1, 0.3):
        assert osc.smooth_or(ar, KAPPAS[-1], pb.a_db, pb.a_max) == (1.0, 0.0), ar
    for ar in (-0.049, 0.0, 0.049):
        OR, dOR = osc.smooth_or(ar, KAPPAS[-1], pb.a_db, pb.a_max)
        assert OR == 0.0 and abs(dOR) < 1e-100, (ar, OR, dOR)


@pytest.mark.parametrize("kappa", [KAPPAS[0], KAPPAS[2]])
def test_s_and_D_match_finite_differences(kappa):
    pb = osc.OscillatorProblem()
    pb.kappa = kappa
    u = np.array([0.17, -0.08, 0.2, 0.1])
    x, p = np.array([0.3, -0.2]), np.zeros(pb.np)
    D = pb.D(0.0, 1, x, u, p)
    h = 1e-7
    for j in range(4):
        e = np.zeros(4); e[j] = h
        fd = (pb.s(0.0, 1, x, u + e, p) - pb.s(0.0, 1, x, u - e, p)) / (2 * h)
        assert np.abs(D[:, j] - fd).max() <= 1e-6 * max(np.abs(fd).max(), 1.0), (j, D[:, j], fd)
    assert not pb.C(0.0, 1, x, u, p).any() and not pb.G(0.0, 1, x, u, p).any()


def test_general_or_reproduces_the_planar_oracle():
    """smooth_or_general with the planar deadband's arguments (two-element match, normalize = f_max + f_db) gives the
    bits of oracle/rendezvous.smooth_or, so both deadbands are restated by one OR chain"""
    pr = rz.PlanarRendezvousProblem()
    for kappa in [rz.Homotopy(1e-3, delta_max=5.0)(x) for x in rz.hom_grid(10)]:
        for fr in np.linspace(-750.0, 750.0, 61):
            got = osc.smooth_or_general([fr - pr.f_db, -pr.f_db - fr], [1.0, -1.0], kappa,
                                        [pr.f_max - pr.f_db, -pr.f_db - pr.f_max], pr.f_max + pr.f_db)
            assert got == rz.smooth_or(fr, kappa, pr.f_db, pr.f_max), (kappa, fr)


def test_jacobians_match_finite_differences():
    """A and B of the oracle model against central differences of f (definition.jl:161-236)"""
    pb = osc.OscillatorProblem()
    rng = np.random.default_rng(1)
    x, u = rng.standard_normal(2), rng.uniform(-0.3, 0.3, 4)
    h = 1e-6
    for j in range(2):
        e = np.zeros(2); e[j] = h
        fd = (pb.dynamics(x + e, u) - pb.dynamics(x - e, u)) / (2 * h)
        assert np.allclose(pb.A()[:, j], fd, rtol=1e-8, atol=1e-8)
    for j in range(4):
        e = np.zeros(4); e[j] = h
        fd = (pb.dynamics(x, u + e) - pb.dynamics(x, u - e)) / (2 * h)
        assert np.allclose(pb.B()[:, j], fd, rtol=1e-8, atol=1e-8)
    assert np.abs(pb.dynamics(x, u) - (pb.A() @ x + pb.B() @ u)).max() <= 1e-14


def test_transition_matrix_is_the_matrix_exponential():
    """the model is LTI: A_k = expm(A dt) on every segment, F_k = 0 and r_k = 0 (f = A x + B u)"""
    pb = osc.OscillatorProblem(30)
    x, u, p = pb.guess(30)
    d = osc.discretize(pb, x, u, p, 10, np.ones(2), 5e-3)
    Ac = pb.tf * np.array([[0.0, 1.0], [-1.0, -1.0]])
    t = orc.t_grid(30)
    for k in range(29):
        assert np.abs(d.A[k] - scipy.linalg.expm(Ac * (t[k + 1] - t[k]))).max() <= 1e-7
    assert not d.F.any() and np.abs(d.r).max() <= 1e-14


def test_zero_defect_on_the_rk4_rollout():
    """a trajectory that follows the discretization's own RK4 (x_k+1 = A_k x_k, u = 0) has a zero defect, and the
    reference guess (RK4 on a 1000-point grid, sampled linearly) is dynamically feasible"""
    pb = osc.OscillatorProblem(30)
    x, u, p = pb.guess(30)
    d = osc.discretize(pb, x, u, p, 10, np.ones(2), 5e-3)
    xr = np.zeros_like(x)
    xr[0] = x[0]
    for k in range(29):
        xr[k + 1] = d.A[k] @ xr[k]
    dr = osc.discretize(pb, xr, u, p, 10, np.ones(2), 5e-3)
    assert np.abs(dr.defect).max() <= 1e-14 and dr.feas
    assert d.feas and 0.0 < np.abs(d.defect).max() < 5e-3


@pytest.fixture(scope="module")
def sweep():
    pb = osc.OscillatorProblem(30)
    return osc.homotopy_sweep(pb, pb.guess(30))


def test_oracle_sweep_solves(sweep):
    """tests.jl:82, the reference's only assertion: the last homotopy step ends SCP_SOLVED; every step stops on the
    stopping criterion before iter_max"""
    assert [r["kappa"] for r in sweep] == pytest.approx(KAPPAS, rel=1e-15)
    assert all(r["status"] == "SCP_SOLVED" and r["iterations"] < 10 for r in sweep)
    s = sweep[-1]["sol"]
    assert s.feas and abs(s.xd[0] - np.array([1.0, 0.0])).max() < 1e-7


def test_golden_file_matches_live_oracle(sweep):
    g = np.load(GOLDEN)
    assert list(g["status"]) == [r["status"] for r in sweep]
    assert list(g["iterations"]) == [r["iterations"] for r in sweep]
    np.testing.assert_allclose(g["kappa"], [r["kappa"] for r in sweep], rtol=1e-15)
    np.testing.assert_allclose(g["J_aug"], [r["sol"].J_aug for r in sweep], rtol=1e-9)
    for i, r in enumerate(sweep):
        assert np.abs(g["xd"][i] - r["sol"].xd).max() <= 1e-7
        assert np.abs(g["ud"][i] - r["sol"].ud).max() <= 1e-7
        assert np.abs(g["p"][i] - r["sol"].p).max() <= 1e-7


def test_subproblems_determine_the_trajectory(sweep):
    """Unlike the planar rendezvous, the oscillator's subproblem LPs have a unique solution: on the first subproblem
    from the reference guess and on the first subproblem of every later homotopy step, the oracle interior point and
    HiGHS agree on the objective and on the trajectory to solver precision.  This is why the GPU tests assert the
    oscillator's iteration counts and trajectories against the oracle's."""
    pb = osc.OscillatorProblem(30)
    refs = [(KAPPAS[0], pb.guess(30))] + [(KAPPAS[i + 1], sweep[i]["sol"]) for i in (0, 4, 8)]
    for kappa, g in refs:
        pb.kappa = kappa
        P = osc.OscillatorPTR(pb, osc.ptr_parameters())
        ref = P.make_solution(*((g.xd, g.ud, g.p) if hasattr(g, "xd") else g))
        a = P.solve_subproblem(ref, prefer="ipm")[0]
        with np.errstate(all="ignore"):
            b = P.solve_subproblem(ref, prefer="highs")[0]
        assert a.status in ("OPTIMAL", "ALMOST_OPTIMAL") and b.status == "OPTIMAL"
        assert abs(a.J_aug - b.J_aug) <= 1e-9 * abs(b.J_aug)
        assert np.abs(a.xd - b.xd).max() <= 1e-8 and np.abs(a.ud - b.ud).max() <= 1e-8
        assert np.abs(a.p - b.p).max() <= 1e-8
