"""Split targets of the scalar factorisation and substitutions: the partial sums of a level live in shared memory when
they fit, and in global memory otherwise (SCPB_GLOBAL_SLOTS=1 forces that).  Both places are summed in the same slot
order, so the results must be bitwise equal: on the bench-size starship KKT (N = 100) and on the N = 31 starship SOC
subproblems.  The hybrid program's top panels scatter into their ancestors with atomics, so its last bits change from run
to run; with it, both places must agree with the CPU interpreter of the same programs."""
import numpy as np
import pytest

from tests import helpers
from tests.test_conic_seeds_gpu import KTOL, starship_soc_subproblems

pytestmark = pytest.mark.gpu


def _variant(monkeypatch, hybrid):
    monkeypatch.setenv("SCPB_SUPERNODAL", "0")
    monkeypatch.setenv("SCPB_HYBRID", str(hybrid))


def _both(monkeypatch, run):
    """run() with the slots in shared memory, then with the global slots"""
    monkeypatch.delenv("SCPB_GLOBAL_SLOTS", raising=False)
    a = run()
    monkeypatch.setenv("SCPB_GLOBAL_SLOTS", "1")
    b = run()
    monkeypatch.delenv("SCPB_GLOBAL_SLOTS")
    return a, b


def _same_bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.tobytes() == b.tobytes(), (what, np.abs(a - b).max())


@pytest.mark.parametrize("hybrid", [0, 3])
def test_bench_kkt_device_solve_shared_and_global_slots(handle, pkg, monkeypatch, hybrid):
    """One assemble + factor + solve of the bench-shaped KKT (product template, N = 100) through the device programs,
    with the slots in shared memory and in global memory (bitwise equal without the hybrid program), against the CPU
    interpreter of the same programs."""
    _variant(monkeypatch, hybrid)
    ex = pkg.examples.starship
    mdl = ex.StarshipProblem(); mdl.hs = 100.0
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr", handle=handle)
    N = 100
    pars = pkg.ptr.Parameters(N=N, Nsub=20, iter_max=5, disc_method=pkg.ptr.FOH, wvc=1e3, wtr=0.1, eps_abs=1e-5,
                              eps_rel=1e-4, feas_tol=5e-3, q_tr=np.inf, q_exit=np.inf)
    pbm = pkg.ptr.create(pars, traj, handle)
    cp = pbm.cp
    rng = np.random.default_rng(5)
    A, G = cp["A"], cp["G"]
    nb = 4
    Av = rng.uniform(0.5, 1.5, (nb, A.nnz)); Gv = rng.uniform(0.5, 1.5, (nb, G.nnz))
    wm = rng.uniform(0.5, 2.0, (nb, cp["l"]))
    rhs = rng.standard_normal((nb, cp["n"] + cp["p"]))
    (s1, b1), (s2, b2) = _both(monkeypatch, lambda: pbm.cone.debug_kkt_solve_dev(Av, Gv, wm, 1e-9, rhs))
    if not hybrid:
        _same_bits(s1, s2, "solution")
    assert (b1 == 0).all() and (b2 == 0).all()
    if hybrid:
        assert pbm.cone.info()["hybrid"]["cut_used"] == hybrid
    for k in range(nb):
        if hybrid:
            ref, _ = pkg.lib.debug_kkt_solve(A, G, cp["l"], [], pbm.perm, Av[k], Gv[k], wm[k], 1e-9, rhs[k],
                                             delta_dyn=1e-12, hybrid_cut=hybrid)
        else:
            ref, _ = pkg.lib.debug_kkt_solve(A, G, cp["l"], [], pbm.perm, Av[k], Gv[k], wm[k], 1e-9, rhs[k],
                                             delta_dyn=1e-12)
        for s in (s1, s2):
            assert np.abs(s[k] - ref).max() <= 1e-8 * max(1.0, np.abs(ref).max()), (k, np.abs(s[k] - ref).max())
    pbm.close()


@pytest.mark.parametrize("q_tr", [1, 2, 4])
def test_soc_subproblem_solves_shared_and_global_slots(handle, pkg, monkeypatch, q_tr):
    """Full cone solves of the N = 31 starship subproblems (L1, SOC and GEOM trust regions; the programs of
    tests/golden/oracle_soc_subproblems.npz) give the same bits with the slots in shared and in global memory."""
    _variant(monkeypatch, 0)
    N = 31
    subs = starship_soc_subproblems(N, 6, q_tr, seed=N + q_tr)
    cp0 = subs[0]["cp"]
    Apat, Avals = helpers.union_pattern([s["cp"]["A"] for s in subs])
    Gpat, Gvals = helpers.union_pattern([s["cp"]["G"] for s in subs])
    perm = pkg.ordering.stage_order(Apat, Gpat, helpers.labels_from_program(subs[0]["prg"], N), N)
    cone = pkg.lib.ConeProblem(handle, Apat, Gpat, cp0["l"], cp0["q"], perm=perm)
    c = np.array([s["cp"]["c"] for s in subs]); b = np.array([s["cp"]["b"] for s in subs])
    h = np.array([s["cp"]["h"] for s in subs])
    o1, o2 = _both(monkeypatch, lambda: cone.solve(Avals, Gvals, c, b, h, group=2, **KTOL))
    cone.close()
    for key in ("x", "y", "z", "s", "pobj", "dobj", "status", "iters"):
        _same_bits(o1[key], o2[key], key)
    assert (o1["status"] == 0).all(), o1["status"]
