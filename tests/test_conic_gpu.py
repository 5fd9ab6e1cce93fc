"""GPU parity: batched interior-point solver (scpb_cone_solve through the C ABI) vs the CPU oracle.

Tolerances (fp64): objective 1e-6 relative to max(1,|obj|) against HiGHS / the oracle IPM (the solver
targets ECOS' 1e-8 and returns its best iterate when the fp64 factorisation floors slightly above it),
primal/dual residuals <= 1e-6 relative, and -- where the optimum is unique (random programs) -- x within
1e-4 of the oracle solution.
"""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import conic
from tests import helpers

pytestmark = pytest.mark.gpu


def _feasible_program(rng, n, p, l, soc, dens=0.35):
    m = l + sum(soc)
    A = sp.random(p, n, density=dens, random_state=rng.integers(1 << 30), format="csr")
    A = (A + sp.csr_matrix((np.ones(p), (np.arange(p), rng.permutation(n)[:p])), shape=(p, n))).tocsr()
    G = sp.random(m, n, density=dens, random_state=rng.integers(1 << 30), format="csr")
    G = (G + sp.csr_matrix((np.ones(m), (np.arange(m), rng.integers(0, n, m))), shape=(m, n))).tocsr()
    # box rows make the problem bounded
    G = sp.vstack([G[:l], sp.eye(n), -sp.eye(n), G[l:]]).tocsr()
    l2 = l + 2 * n
    A.sort_indices(); G.sort_indices()

    def interior(k):
        v = rng.uniform(0.5, 2.0, l2)
        parts = [v]
        for q in soc:
            w = rng.standard_normal(q); w[0] = np.linalg.norm(w[1:]) + rng.uniform(0.5, 1.5)
            parts.append(w)
        return np.concatenate(parts)

    x0, s0, z0, y0 = rng.standard_normal(n), interior(0), interior(1), rng.standard_normal(p)
    h = G @ x0 + s0
    b = A @ x0
    c = -(A.T @ y0) - (G.T @ z0)
    return A, G, l2, c, b, h


def _kkt_check(A, G, l, soc, c, b, h, x, y, z, s):
    pres = max(np.abs(A @ x - b).max(initial=0.0), np.abs(G @ x + s - h).max(initial=0.0))
    dres = np.abs(c + A.T @ y + G.T @ z).max()
    return pres, dres


@pytest.mark.parametrize("seed,n,p,l,soc", [(0, 10, 3, 8, []), (1, 16, 5, 10, [3, 4]), (2, 24, 8, 6, [5, 3, 3]),
                                            (3, 12, 0, 9, [4])])
def test_random_programs_match_oracle(handle, pkg, seed, n, p, l, soc):
    rng = np.random.default_rng(seed)
    nb = 5
    A, G, l2, c0, b0, h0 = _feasible_program(np.random.default_rng(1000 * seed + 7), n, p, l, soc)
    # batch: same pattern, different values and data per seed, each with its own strictly feasible
    # primal/dual certificate (so every instance is feasible and bounded)
    Av, Gv, cs, bs, hs = [A.data.copy()], [G.data.copy()], [c0], [b0], [h0]
    for k in range(1, nb):
        Ak = sp.csr_matrix((A.data * (1 + 0.2 * rng.standard_normal(A.nnz)), A.indices, A.indptr), shape=A.shape)
        x0, y0 = rng.standard_normal(n), rng.standard_normal(p)
        s0, z0 = [rng.uniform(0.5, 2.0, l2)], [rng.uniform(0.5, 2.0, l2)]
        for q in soc:
            for lst in (s0, z0):
                w = rng.standard_normal(q); w[0] = np.linalg.norm(w[1:]) + rng.uniform(0.5, 1.5)
                lst.append(w)
        s0, z0 = np.concatenate(s0), np.concatenate(z0)
        Av.append(Ak.data); Gv.append(G.data.copy())
        hs.append(G @ x0 + s0); bs.append(Ak @ x0); cs.append(-(Ak.T @ y0) - (G.T @ z0))
    Av, Gv, cs, hs = np.array(Av), np.array(Gv), np.array(cs), np.array(hs)
    bs = np.array(bs).reshape(nb, p)
    cone = pkg.lib.ConeProblem(handle, A, G, l2, soc, perm=pkg.ordering.rcm_order(A, G))
    out = cone.solve(Av, Gv, cs, bs, hs)
    for k in range(nb):
        Ak = sp.csr_matrix((Av[k], A.indices, A.indptr), shape=A.shape)
        cp = dict(c=cs[k], c0=0.0, A=Ak, b=bs[k], G=G, h=hs[k], l=l2, q=list(soc))
        ref = conic.solve_ipm(cp, tol=1e-9)
        assert ref["status"] in ("OPTIMAL", "ALMOST_OPTIMAL")
        assert out["status"][k] == 0, (k, out["status"], out["iters"])
        assert abs(out["pobj"][k] - ref["obj"]) <= 1e-6 * max(1.0, abs(ref["obj"]))
        pres, dres = _kkt_check(Ak, G, l2, soc, cs[k], bs[k], hs[k], out["x"][k], out["y"][k], out["z"][k], out["s"][k])
        assert pres <= 1e-6 * max(1.0, np.abs(hs[k]).max()) and dres <= 1e-6 * max(1.0, np.abs(cs[k]).max())
        assert np.abs(out["x"][k] - ref["z"]).max() <= 1e-4 * max(1.0, np.abs(ref["z"]).max())
        assert (out["s"][k][:l2] > -1e-9).all() and (out["z"][k][:l2] > -1e-9).all()
    cone.close()


@pytest.mark.parametrize("N,group", [(12, 0), (31, 2), (31, 4), (100, 2)])
def test_starship_ptr_subproblem_matches_highs(handle, pkg, N, group):
    """The reference's own subproblem (starship PTR, q_tr = Inf => LP): batch of perturbed references."""
    nb = 6
    pb, P, subs = helpers.starship_subproblems(N, nb, seed=N)
    Apat, Avals = helpers.union_pattern([s["cp"]["A"] for s in subs])
    Gpat, Gvals = helpers.union_pattern([s["cp"]["G"] for s in subs])
    lab = helpers.labels_from_program(subs[0]["prg"], N)
    perm = pkg.ordering.stage_order(Apat, Gpat, lab, N)
    cone = pkg.lib.ConeProblem(handle, Apat, Gpat, subs[0]["cp"]["l"], [], perm=perm)
    info = cone.info()
    assert info["nnzL"] < 40 * info["nk"] and info["levels"] < 200, info
    c = np.array([s["cp"]["c"] for s in subs]); b = np.array([s["cp"]["b"] for s in subs])
    h = np.array([s["cp"]["h"] for s in subs])
    out = cone.solve(Avals, Gvals, c, b, h, group=group)
    for k, sub in enumerate(subs):
        ref = conic.solve_highs(sub["cp"], tol=1e-9)
        assert ref["status"] == "OPTIMAL"
        assert out["status"][k] == 0, (out["status"], out["iters"])     # OPTIMAL at ECOS' tolerances, every seed
        want = ref["obj"] - sub["cp"]["c0"]
        assert abs(out["pobj"][k] - want) <= 1e-7 * max(1.0, abs(want)), (k, out["pobj"][k], want)
        assert abs(out["pobj"][k] - out["dobj"][k]) <= 2e-7 * max(1.0, abs(want))
        x = out["x"][k]
        cpk = sub["cp"]
        assert np.abs(cpk["A"] @ x - cpk["b"]).max() <= 1e-7 * max(1.0, np.abs(cpk["b"]).max())
        assert (cpk["G"] @ x - cpk["h"]).max() <= 1e-7 * max(1.0, np.abs(cpk["h"]).max())
    assert out["iters"].max() <= 45
    cone.close()


def _dense_kkt(A, G, l, soc, wm, delta):
    n, p = A.shape[1], A.shape[0]
    blocks = [np.diag(wm[:l])] if l else []
    o = l
    for q in soc:
        blocks.append(wm[o:o + q * q].reshape(q, q)); o += q * q
    import scipy.linalg as sla
    Wm = sla.block_diag(*blocks) if blocks else np.zeros((0, 0))
    Gd, Ad = G.toarray(), A.toarray()
    H = Gd.T @ Wm @ Gd + delta * np.eye(n)
    return np.block([[H, Ad.T], [Ad, -delta * np.eye(p)]])


def _variant(monkeypatch, sn):
    """kernel variant: "1" supernodal panels, "0" scalar level-scheduled programs, "hN" hybrid program with cut N"""
    monkeypatch.setenv("SCPB_SUPERNODAL", "1" if sn == "1" else "0")
    monkeypatch.setenv("SCPB_HYBRID", sn[1:] if sn.startswith("h") else "0")


@pytest.mark.parametrize("sn", ["1", "0", "h1", "h2"])
@pytest.mark.parametrize("seed,n,p,l,soc", [(0, 12, 4, 9, []), (1, 20, 7, 15, [3, 4]), (2, 30, 10, 25, [5]),
                                            (4, 15, 5, 0, [3, 3, 4])])
def test_device_kkt_solve_matches_dense(handle, pkg, monkeypatch, sn, seed, n, p, l, soc):
    """One reduced-KKT assemble + factor + solve through the kernel's own code path (supernodal panels held in
    registers, conic_sn.cuh; the scalar level-scheduled programs with SCPB_SUPERNODAL=0; the hybrid program that runs
    the top of the elimination tree as in-place panels, SCPB_HYBRID=<cut>) against numpy."""
    _variant(monkeypatch, sn)
    rng = np.random.default_rng(seed)
    m = l + sum(soc)
    A = sp.random(p, n, density=0.4, random_state=rng.integers(1 << 30), format="csr")
    A = (A + sp.csr_matrix((np.ones(p), (np.arange(p), rng.permutation(n)[:p])), shape=(p, n))).tocsr()
    G = sp.random(m, n, density=0.4, random_state=rng.integers(1 << 30), format="csr")
    G = (G + sp.csr_matrix((np.ones(m), (np.arange(m), rng.integers(0, n, m))), shape=(m, n))).tocsr()
    G = sp.vstack([G[:l], sp.eye(n), G[l:]]).tocsr()
    l2 = l + n
    A.sort_indices(); G.sort_indices()
    nb = 3
    delta = 1e-7
    for perm in (None, pkg.ordering.rcm_order(A, G)):
        cone = pkg.lib.ConeProblem(handle, A, G, l2, soc, perm=perm)
        Av = np.array([A.data * (1 + 0.1 * rng.standard_normal(A.nnz)) for _ in range(nb)])
        Gv = np.array([G.data * (1 + 0.1 * rng.standard_normal(G.nnz)) for _ in range(nb)])
        wms, rhs = [], rng.standard_normal((nb, n + p))
        for k in range(nb):
            w = list(rng.uniform(0.1, 10.0, l2))
            for q in soc:
                M = rng.standard_normal((q, q))
                w += list((M @ M.T + q * np.eye(q)).ravel())
            wms.append(w)
        wms = np.array(wms)
        sol, bad = cone.debug_kkt_solve_dev(Av, Gv, wms, delta, rhs)
        for k in range(nb):
            Ak = sp.csr_matrix((Av[k], A.indices, A.indptr), shape=A.shape)
            Gk = sp.csr_matrix((Gv[k], G.indices, G.indptr), shape=G.shape)
            want = np.linalg.solve(_dense_kkt(Ak, Gk, l2, soc, wms[k], delta), rhs[k])
            assert bad[k] == 0
            assert np.abs(sol[k] - want).max() <= 1e-7 * max(1.0, np.abs(want).max()), (sn, k)
        cone.close()


@pytest.mark.parametrize("sn", ["1", "0", "h3", "h6", "h9"])
def test_device_kkt_solve_on_the_product_template(handle, pkg, monkeypatch, sn):
    """The bench-shaped KKT (product template with the L1 lowering, stage ordering, N = 24): the device factorisation and
    substitutions agree with the CPU interpreter of the same programs, seed by seed."""
    _variant(monkeypatch, sn)
    ex = pkg.examples.starship
    mdl = ex.StarshipProblem(); mdl.hs = 100.0
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr", handle=handle)
    N = 24
    pars = pkg.ptr.Parameters(N=N, Nsub=20, iter_max=5, disc_method=pkg.ptr.FOH, wvc=1e3, wtr=0.1, eps_abs=1e-5,
                              eps_rel=1e-4, feas_tol=5e-3, q_tr=np.inf, q_exit=np.inf)
    pbm = pkg.ptr.create(pars, traj, handle)
    cp = pbm.cp
    rng = np.random.default_rng(1)
    A, G = cp["A"], cp["G"]
    nb = 5
    Av = rng.uniform(0.5, 1.5, (nb, A.nnz)); Gv = rng.uniform(0.5, 1.5, (nb, G.nnz))
    wm = rng.uniform(0.5, 2.0, (nb, cp["l"]))
    rhs = rng.standard_normal((nb, cp["n"] + cp["p"]))
    sol, bad = pbm.cone.debug_kkt_solve_dev(Av, Gv, wm, 1e-9, rhs)
    for k in range(nb):
        ref, info = pkg.lib.debug_kkt_solve(A, G, cp["l"], [], pbm.perm, Av[k], Gv[k], wm[k], 1e-9, rhs[k], delta_dyn=1e-12)
        assert bad[k] == 0
        assert np.abs(sol[k] - ref).max() <= 1e-8 * max(1.0, np.abs(ref).max()), (sn, k, np.abs(sol[k] - ref).max())
    if sn.startswith("h"):   # the hybrid variant really ran (it needs the shared-memory vector, which N = 24 has)
        assert pbm.cone.info()["hybrid"]["cut_used"] == int(sn[1:]), pbm.cone.info()["hybrid"]
    pbm.close()


def test_infeasibility_certificates(handle, pkg):
    """termination_status values the reference branches on (program.jl:427-428; scp.jl:470-473 DUAL_INFEASIBLE while
    computing the scaling, :975 unsafe_solution): an infeasible and an unbounded program in the same batch as a solvable
    one must come back INFEASIBLE / DUAL_INFEASIBLE / OPTIMAL, seed by seed."""
    # variables (x1, x2); rows: -x1 <= h1, -x2 <= h2, x1 + x2 <= h3 ; equality x1 - x2 = b
    A = sp.csr_matrix(np.array([[1.0, -1.0]]))
    G = sp.csr_matrix(np.array([[-1.0, 0.0], [0.0, -1.0], [1.0, 1.0]]))
    cone = pkg.lib.ConeProblem(handle, A, G, 3, [])
    Av = np.tile(A.data, (3, 1)); Gv = np.tile(G.data, (3, 1))
    c = np.array([[1.0, 1.0], [1.0, 1.0], [-1.0, -1.0]])
    b = np.array([[0.0], [0.0], [0.0]])
    h = np.array([[0.0, 0.0, 2.0],        # solvable: min x1+x2, x >= 0, x1 + x2 <= 2, x1 = x2 -> 0
                  [-2.0, -2.0, 1.0],      # infeasible: x1 >= 2, x2 >= 2, x1 + x2 <= 1
                  [0.0, 0.0, 2.0]])       # seed 2 becomes unbounded below by dropping the cap (huge h3 is not enough):
    Gv[2, -2:] = 0.0                      # ... zero the row x1 + x2 <= h3 -> min -(x1+x2), x >= 0, x1 = x2: unbounded
    out = cone.solve(Av, Gv, c, b, h)
    assert list(out["status"]) == [0, 4, 5], (out["status"], out["iters"])
    assert abs(out["pobj"][0]) < 1e-7
    y, z = out["y"][1], out["z"][1]       # the returned (y, z) is the certificate, up to scale
    Ad, Gd = A.toarray(), G.toarray()
    nrm = -(b[1] @ y + h[1] @ z)
    assert nrm > 0 and np.abs(Ad.T @ y + Gd.T @ z).max() <= 1e-6 * nrm and (z > -1e-9 * nrm).all()
    x = out["x"][2]
    G2 = Gd.copy(); G2[2] = 0.0
    assert c[2] @ x < 0 and np.abs(Ad @ x).max() <= 1e-6 * abs(c[2] @ x) and (G2 @ x).max() <= 1e-6 * abs(c[2] @ x)
    cone.close()


def test_cone_error_paths(handle, pkg):
    A = sp.csr_matrix(np.array([[1.0, 1.0]])); G = sp.csr_matrix(-np.eye(2))
    with pytest.raises(pkg.ScpbError):
        pkg.lib.ConeProblem(handle, A, G, 1, [2])           # cone sizes do not add up to m
    with pytest.raises(pkg.ScpbError):
        pkg.lib.ConeProblem(handle, A, G, 2, [], perm=[0, 0, 1])  # not a permutation
    cone = pkg.lib.ConeProblem(handle, A, G, 2, [])
    out = cone.solve([[1.0, 1.0]], [G.data], [[1.0, 2.0]], [[1.0]], [[0.0, 0.0]])   # min x1+2x2, x1+x2=1, x>=0
    assert out["status"][0] == 0 and abs(out["pobj"][0] - 1.0) < 1e-7
    assert np.abs(out["x"][0] - [1.0, 0.0]).max() < 1e-6
    cone.close()


def test_global_memory_sweep_fallback(handle, pkg, monkeypatch):
    """Problems whose substitution vector does not fit shared memory take the global-memory sweeps (kkt_ldl_solve);
    SCPB_NO_VSMEM forces that path on a small problem so that it stays covered."""
    monkeypatch.setenv("SCPB_NO_VSMEM", "1")
    test_starship_ptr_subproblem_matches_highs(handle, pkg, 12, 0)
    test_random_programs_match_oracle(handle, pkg, 1, 16, 5, 10, [3, 4])
