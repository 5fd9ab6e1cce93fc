"""CPU: the product's PTR template with IMPULSE discretization (planar rendezvous, scptoolbox.jl_b200/ptr.py +
examples/rendezvous_planar.py) reproduces the oracle's IMPULSE subproblem (oracle/rendezvous.py); the descriptor and the
host refuse what the device does not implement."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import rendezvous as rz
from tests.test_ptr_template import _sources

N = 12


class _FakeHandle:
    """stand-in for the device objects so that the template can be built on a CPU-only box"""

    def __init__(self):
        self.lib = type("L", (), {"scpb_ptr_setup": staticmethod(lambda *a: 0)})()
        self.h = None

    def model_set(self, *a):
        pass

    def _check(self, rc, what):
        pass


def _product(pkg, monkeypatch, disc_method=None, model_id=None):
    ex = pkg.examples.rendezvous_planar
    traj = pkg.problem.TrajectoryProblem(ex.PlanarRendezvousProblem())
    ex.define_problem(traj, "ptr")
    if model_id is not None:
        traj.model_id = model_id
    pars = ex.ptr_parameters(N=N)
    if disc_method is not None:
        pars.disc_method = disc_method
    monkeypatch.setattr(pkg.lib, "ConeProblem", lambda *a, **k: type("C", (), {"c": None, "close": lambda s: None})())
    return traj, pars


@pytest.mark.parametrize("step", [0, 9])
def test_impulse_template_matches_oracle_subproblem(pkg, monkeypatch, step):
    """W @ src equals the oracle's IMPULSE subproblem at the smooth (kappa = h(0)) and the sharp (h(1)) end of the
    homotopy, with the sources filled from the oracle's IMPULSE DLTV and its s / D."""
    kappa = rz.Homotopy(1e-3, delta_max=5.0)(rz.hom_grid(10)[step])
    pbo = rz.PlanarRendezvousProblem(N)
    pbo.kappa = kappa
    X, U, P = rz.perturbed_guesses(pbo, 1, seed=11)
    U[0, :, 0:3] = np.random.default_rng(5).uniform(-400, 400, (N, 3))
    opt = rz.ImpulsePTR(pbo, rz.ptr_parameters(N=N))
    ref = opt.make_solution(X[0], U[0], P[0])
    ocp = opt.build(ref)[0].compile()
    traj, pars = _product(pkg, monkeypatch)
    traj.mdl.kappa = kappa
    pbm = pkg.ptr.SCPProblem(pars, traj, _FakeHandle(), l1_block=0)   # the reference's exact (NormOneBridge) program
    assert pbm.desc.method == pkg.lib.IMPULSE
    cp, sm = pbm.cp, pbm.sm
    assert not any(sm.oBp <= c < sm.oF for c in pbm.W.indices)         # no Bp source: no u_{k+1} in the dynamics rows
    vals = pbm.W @ _sources(sm, pbo, opt, ref)
    n, p_, m = cp["n"], cp["p"], cp["m"]
    assert (n, p_, m, cp["l"]) == (ocp["c"].size, ocp["A"].shape[0], ocp["G"].shape[0], ocp["l"])
    A = sp.csr_matrix((vals[:cp["nnzA"]], cp["A"].indices, cp["A"].indptr), shape=(p_, n))
    G = sp.csr_matrix((vals[cp["nnzA"]:cp["nnzA"] + cp["nnzG"]], cp["G"].indices, cp["G"].indptr), shape=(m, n))
    tol = 1e-12
    assert abs(A - ocp["A"]).max() <= tol * max(1.0, abs(ocp["A"]).max())
    assert abs(G - ocp["G"]).max() <= tol * max(1.0, abs(ocp["G"]).max())
    c = vals[cp["off_c"]:cp["off_c"] + n]; b = vals[cp["off_b"]:cp["off_b"] + p_]; h = vals[cp["off_h"]:cp["off_h"] + m]
    assert np.abs(c - ocp["c"]).max() <= tol * max(1.0, np.abs(ocp["c"]).max())
    assert np.abs(b - ocp["b"]).max() <= tol * max(1.0, np.abs(ocp["b"]).max())
    assert np.abs(h - ocp["h"]).max() <= tol * max(1.0, np.abs(ocp["h"]).max())
    assert abs(vals[-1] - ocp["c0"]) <= tol
    # the device parameter block carries the current kappa
    assert pkg.problem.model_parameters(traj)[7] == kappa


def test_impulse_needs_a_model_with_impulse_semantics(pkg, monkeypatch):
    traj, pars = _product(pkg, monkeypatch, model_id=pkg.lib.MODEL_QUADROTOR)
    with pytest.raises(pkg.ScpbError, match="impulse semantics"):
        pkg.ptr.SCPProblem(pars, traj, _FakeHandle())


def test_scvx_and_gusto_refuse_impulse(pkg, monkeypatch):
    traj, _ = _product(pkg, monkeypatch)
    kw = dict(eps_abs=1e-5, eps_rel=1e-4, feas_tol=5e-3)
    sp_ = pkg.scvx.Parameters(N=N, Nsub=10, iter_max=5, disc_method=pkg.lib.IMPULSE, lam=5e2, rho_0=0.0, rho_1=0.1,
                              rho_2=0.7, beta_sh=2.0, beta_gr=2.0, eta_init=1.0, eta_lb=1e-8, eta_ub=10.0, q_tr=np.inf,
                              q_exit=np.inf, **kw)
    with pytest.raises(pkg.ScpbError, match="PTR only"):
        pkg.scvx.create(sp_, traj, _FakeHandle())
    gp = pkg.gusto.Parameters(N, 10, 5, pkg.lib.IMPULSE, 1.0, 1e9, 0.1, 0.9, 2.0, 2.0, 10.0, 1.0, 1e-3, 10.0, 0.8, 5,
                              **kw)
    with pytest.raises(pkg.ScpbError, match="PTR only"):
        pkg.gusto.create(gp, traj, _FakeHandle())


def test_zero_descriptor_means_foh(pkg):
    """method is the last field of scpb_ptr_desc: the earlier fields keep their offsets and a zero-initialised
    descriptor keeps FOH."""
    d = pkg.lib.PtrDesc()
    assert d.method == pkg.lib.FOH == 0
    assert pkg.lib.PtrDesc._fields_[-1][0] == "method"
    assert pkg.lib.PtrDesc.method.offset == 28 * 4 + 3 * 8
    assert ctypes.sizeof(pkg.lib.PtrDesc) == 28 * 4 + 3 * 8 + 8        # padded to the 8-byte alignment of the doubles


def test_homotopy_helper_matches_oracle(pkg):
    h, ho = pkg.homotopy.Homotopy(1e-3, delta_max=5.0), rz.Homotopy(1e-3, delta_max=5.0)
    for x in rz.hom_grid(10):
        assert h(x) == ho(x)
    assert h(1.0) == pytest.approx(np.log(99.0) / 1e-3, rel=1e-12)
