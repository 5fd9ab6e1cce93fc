"""CPU: the oracle's planar rendezvous (oracle/rendezvous.py, restating test/examples/rendezvous_planar and the smooth OR
chain of src/utils/helper.jl:600-807) and its homotopy sweep (tests.jl:22-95) with IMPULSE PTR."""
import math
import os

import numpy as np
import pytest

from oracle import rendezvous as rz

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_ptr_rendezvous.npz")
HOM = rz.Homotopy(1e-3, delta_max=5.0)
KAPPAS = [HOM(x) for x in rz.hom_grid(10)]


def test_homotopy_end_points():
    assert KAPPAS[0] == pytest.approx(math.log(99.0) / 5.0, rel=1e-15)
    assert KAPPAS[-1] == pytest.approx(math.log(99.0) / 1e-3, rel=1e-12)          # ~4.6e3, the sharp end
    assert all(b > a for a, b in zip(KAPPAS, KAPPAS[1:]))


@pytest.mark.parametrize("kappa", [KAPPAS[0], KAPPAS[2], KAPPAS[4]])
def test_or_gradient_matches_finite_differences(kappa):
    pb = rz.PlanarRendezvousProblem()
    for fr in (-600.0, -230.0, -150.0, 0.0, 90.0, 210.0, 520.0):
        h = 1e-3
        OR, dOR = rz.smooth_or(fr, kappa, pb.f_db, pb.f_max)
        fd = (rz.smooth_or(fr + h, kappa, pb.f_db, pb.f_max)[0] - rz.smooth_or(fr - h, kappa, pb.f_db, pb.f_max)[0]) / (2 * h)
        assert abs(dOR - fd) <= 1e-6 * max(abs(fd), 1e-6), (kappa, fr, dOR, fd)
        assert 0.0 <= OR <= 1.0 + 1e-12


@pytest.mark.parametrize("kappa", [KAPPAS[0], KAPPAS[3]])
def test_s_and_D_match_finite_differences(kappa):
    pb = rz.PlanarRendezvousProblem()
    pb.kappa = kappa
    rng = np.random.default_rng(3)
    u = np.zeros(12)
    u[0:3] = rng.uniform(-700, 700, 3)
    u[3:6] = [-420.0, 35.0, 260.0]
    x, p = np.zeros(6), np.array([300.0])
    D = pb.D(0.0, 1, x, u, p)
    h = 1e-3
    for j in range(12):
        e = np.zeros(12); e[j] = h
        fd = (pb.s(0.0, 1, x, u + e, p) - pb.s(0.0, 1, x, u - e, p)) / (2 * h)
        assert np.abs(D[:, j] - fd).max() <= 1e-6 * max(np.abs(fd).max(), 1.0), (j, D[:, j], fd)
    assert not pb.C(0.0, 1, x, u, p).any() and not pb.G(0.0, 1, x, u, p).any()


def test_or_saturates_exactly_at_the_sharp_end():
    """At the last homotopy step, outside the deadband, sigma rounds to exactly 1 and the gradient factor
    c = exp(kappa L + 2 log(1 - sigma)) to exactly 0: the values the device pack must reproduce bit for bit."""
    pb = rz.PlanarRendezvousProblem()
    for fr in (-750.0, -400.0, 260.0, 400.0, 750.0):
        OR, dOR = rz.smooth_or(fr, KAPPAS[-1], pb.f_db, pb.f_max)
        assert OR == 1.0 and dOR == 0.0, (fr, OR, dOR)
    for fr in (-140.0, 0.0, 140.0):        # inside the deadband sigma rounds to 0; the gradient underflows towards 0
        OR, dOR = rz.smooth_or(fr, KAPPAS[-1], pb.f_db, pb.f_max)
        assert OR == 0.0 and abs(dOR) < 1e-100, (fr, OR, dOR)
    OR, dOR = rz.smooth_or(200.0, KAPPAS[0], pb.f_db, pb.f_max)      # smooth end: a genuine slope
    assert 0.0 < OR < 1.0 and dOR > 0.0


@pytest.fixture(scope="module")
def sweep():
    pb = rz.PlanarRendezvousProblem(30)
    return rz.homotopy_sweep(pb, pb.guess(30))


def test_oracle_sweep_solves(sweep):
    """tests.jl:82, the reference's only assertion: the last homotopy step ends SCP_SOLVED; every step stops on the
    stopping criterion before iter_max."""
    assert [r["kappa"] for r in sweep] == pytest.approx(KAPPAS, rel=1e-15)
    assert sweep[-1]["status"] == "SCP_SOLVED"
    assert all(r["status"] == "SCP_SOLVED" and r["iterations"] < 30 for r in sweep)
    s = sweep[-1]["sol"]
    assert s.feas and abs(s.xd[-1] - np.array([0, 0, -0.1, 0, 0, 0])).max() < 1e-6


def test_golden_file_matches_live_oracle(sweep):
    g = np.load(GOLDEN)
    assert list(g["status"]) == [r["status"] for r in sweep]
    assert list(g["iterations"]) == [r["iterations"] for r in sweep]
    np.testing.assert_allclose(g["kappa"], [r["kappa"] for r in sweep], rtol=1e-15)
    np.testing.assert_allclose(g["J_aug"], [r["sol"].J_aug for r in sweep], rtol=1e-9)
    pb = rz.PlanarRendezvousProblem(30)
    xrg, urg, _ = pb.ranges()
    Sx = np.array([r[1] - r[0] for r in xrg]); Su = np.array([r[1] - r[0] for r in urg])
    for i, r in enumerate(sweep):
        assert (np.abs(g["xd"][i] - r["sol"].xd) <= 1e-7 * Sx).all()
        assert (np.abs(g["ud"][i][:, 0:3] - r["sol"].ud[:, 0:3]) <= 1e-7 * Su[0:3]).all()
        assert abs(g["p"][i][0] - r["sol"].p[0]) <= 1e-7 * 400.0


def test_first_subproblem_does_not_determine_the_trajectory():
    """The first PTR subproblem from the straight-line guess (kappa = h(0)) is an LP whose optimal face is not a point:
    the oracle interior point and HiGHS agree on the objective but not on the trajectory.  This is why the GPU tests
    report the sweep's trajectories against the oracle's instead of asserting them."""
    pb = rz.PlanarRendezvousProblem(30)
    pb.kappa = KAPPAS[0]
    P = rz.ImpulsePTR(pb, rz.ptr_parameters())
    ref = P.make_solution(*pb.guess(30))
    a = P.solve_subproblem(ref, prefer="ipm")[0]
    with np.errstate(all="ignore"):
        b = P.solve_subproblem(ref, prefer="highs")[0]
    assert a.status in ("OPTIMAL", "ALMOST_OPTIMAL") and b.status == "OPTIMAL"
    assert abs(a.J_aug - b.J_aug) <= 1e-6 * abs(b.J_aug)
    xrg, urg, _ = pb.ranges()
    Sx = np.array([r[1] - r[0] for r in xrg]); Su = np.array([r[1] - r[0] for r in urg])
    assert (np.abs(a.xd - b.xd) / Sx).max() > 1e-3 and (np.abs(a.ud - b.ud) / Su).max() > 1e-3
