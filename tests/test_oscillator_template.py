"""CPU: the product's PTR template for a model with a fixed final time (the oscillator, scptoolbox.jl_b200/ptr.py +
examples/oscillator.py) reproduces the oracle's FOH subproblem (oracle/oscillator.py), and carries no F term."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oscillator as osc
from oracle import rendezvous as rz
from tests.test_ptr_template import _sources
from tests.test_rendezvous_template import _FakeHandle

N = 12


def _product(pkg, monkeypatch, kappa):
    ex = pkg.examples.oscillator
    mdl = ex.OscillatorProblem(N)
    mdl.kappa = kappa
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr")
    monkeypatch.setattr(pkg.lib, "ConeProblem", lambda *a, **k: type("C", (), {"c": None, "close": lambda s: None})())
    return traj, ex.ptr_parameters(N=N)


@pytest.mark.parametrize("step", [0, 9])
def test_foh_template_matches_oracle_subproblem(pkg, monkeypatch, step):
    """W @ src equals the oracle's FOH subproblem at the smooth (kappa = h(0)) and the sharp (h(1)) end of the homotopy,
    with the sources filled from the oracle's DLTV and its s / D"""
    kappa = osc.hom()(rz.hom_grid(10)[step])
    pbo = osc.OscillatorProblem(N)
    pbo.kappa = kappa
    X, U, P = osc.perturbed_guesses(pbo, 1, seed=11)
    U[0, :, 0] = np.random.default_rng(5).uniform(-0.3, 0.3, N)
    opt = osc.OscillatorPTR(pbo, osc.ptr_parameters(N=N))
    ref = opt.make_solution(X[0], U[0], P[0])
    ocp = opt.build(ref)[0].compile()
    traj, pars = _product(pkg, monkeypatch, kappa)
    pbm = pkg.ptr.SCPProblem(pars, traj, _FakeHandle(), l1_block=0)   # the reference's exact (NormOneBridge) program
    assert pbm.desc.method == pkg.lib.FOH
    cp, sm = pbm.cp, pbm.sm
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
    assert pkg.problem.model_parameters(traj)[5] == kappa      # the device parameter block carries the current kappa


def test_template_has_no_F_term(pkg, monkeypatch):
    """fcols = (): the source map has an empty F block and the descriptor says nf = 0 (scpb_ptr_setup refuses an nf that
    differs from the model pack's)"""
    traj, pars = _product(pkg, monkeypatch, osc.hom()(0.0))
    assert traj.fcols == []
    pbm = pkg.ptr.SCPProblem(pars, traj, _FakeHandle())
    sm = pbm.sm
    assert sm.nf == 0 and sm.oF == sm.or_ and pbm.desc.nf == 0
    assert sm.ng == 1 and pbm.desc.ng == 1 and pbm.desc.np == N


def test_parameters_are_staged(pkg, monkeypatch):
    """l1r_k is a stage-k variable of the elimination order (problem_advise_parameter_stage), not a border one"""
    traj, pars = _product(pkg, monkeypatch, osc.hom()(0.0))
    pbm = pkg.ptr.SCPProblem(pars, traj, _FakeHandle())
    vp = pbm.template.blocks["p"][0]
    assert list(pbm.cp["var_stage"][vp:vp + N]) == list(range(N))


def test_product_guess_matches_oracle(pkg):
    ex = pkg.examples.oscillator
    traj = pkg.problem.TrajectoryProblem(ex.OscillatorProblem(30))
    ex.define_problem(traj, "ptr")
    x, u, p = traj.guess(30)
    xo, uo, po = osc.OscillatorProblem(30).guess(30)
    assert np.array_equal(x, xo) and np.array_equal(u, uo) and np.array_equal(p, po)
