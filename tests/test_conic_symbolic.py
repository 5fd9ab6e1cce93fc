"""CPU: the solver's index programs (assembly, level-scheduled LDL', substitutions) executed by the
host interpreter (scpb_debug_kkt_solve) must solve the reduced KKT system exactly like a dense solve."""
import numpy as np
import pytest
import scipy.sparse as sp


def _random_program(rng, n, p, l, soc_dims, dens=0.3):
    m = l + sum(soc_dims)
    A = sp.random(p, n, density=dens, random_state=rng.integers(1 << 30), format="csr")
    A = (A + sp.csr_matrix((np.ones(p), (np.arange(p), rng.permutation(n)[:p])), shape=(p, n))).tocsr()
    G = sp.random(m, n, density=dens, random_state=rng.integers(1 << 30), format="csr")
    G = (G + sp.csr_matrix((np.ones(m), (np.arange(m), rng.integers(0, n, m))), shape=(m, n))).tocsr()
    A.sort_indices(); G.sort_indices()
    return A, G


def _dense_kkt(A, G, l, soc_dims, wm, delta):
    n, p = A.shape[1], A.shape[0]
    W2 = np.zeros((G.shape[0], G.shape[0]))
    W2[np.arange(l), np.arange(l)] = wm[:l]
    off, wo = l, l
    for q in soc_dims:
        W2[off:off + q, off:off + q] = wm[wo:wo + q * q].reshape(q, q)
        off += q; wo += q * q
    Gd, Ad = G.toarray(), A.toarray()
    H = Gd.T @ W2 @ Gd + delta * np.eye(n)
    return np.block([[H, Ad.T], [Ad, -delta * np.eye(p)]])


@pytest.mark.parametrize("seed,n,p,l,soc", [(0, 12, 4, 9, []), (1, 20, 7, 15, [3, 4]), (2, 30, 10, 25, [5]),
                                            (3, 8, 0, 10, []), (4, 15, 5, 0, [3, 3, 4])])
def test_kkt_programs_match_dense_solve(pkg, seed, n, p, l, soc):
    rng = np.random.default_rng(seed)
    A, G = _random_program(rng, n, p, l, soc)
    m = G.shape[0]
    wm = list(rng.uniform(0.1, 10.0, l))
    for q in soc:
        M = rng.standard_normal((q, q))
        wm += list((M @ M.T + q * np.eye(q)).ravel())
    wm = np.array(wm)
    delta = 1e-7
    K = _dense_kkt(A, G, l, soc, wm, delta)
    rhs = rng.standard_normal(n + p)
    want = np.linalg.solve(K, rhs)
    for perm in (None, rng.permutation(n + p).astype(np.int32), pkg.ordering.rcm_order(A, G)):
        sol, info = pkg.lib.debug_kkt_solve(A, G, l, soc, perm, A.data, G.data, wm, delta, rhs)
        assert np.abs(sol - want).max() <= 1e-7 * max(1.0, np.abs(want).max()), info   # cond(K) ~ 1/delta
        assert info["levels"] >= 1 and info["nnzL"] >= A.nnz
        # the supernodal program (dense panels; the next kernel generation) solves the same system
        sol2, info2 = pkg.lib.debug_kkt_solve(A, G, l, soc, perm, A.data, G.data, wm, delta, rhs, supernodal=True)
        assert np.abs(sol2 - want).max() <= 1e-7 * max(1.0, np.abs(want).max()), info2
        assert info2["nnzL"] == info["nnzL"] and info2["sn_levels"] <= info["levels"]
        assert info2["supernodes"] <= n + p and info2["panel_doubles"] >= info["nnzL"] + n + p
        assert info2["max_width"] <= 12      # supernodes are cut at CONIC_SN_WMAX columns (one panel row per lane)


def test_stage_order_keeps_fill_small(pkg):
    """Chain-structured program: stage ordering must give O(N) fill and O(log N + const) levels."""
    rng = np.random.default_rng(5)
    N, nx, nu = 40, 4, 2
    nv = N * (nx + nu) + 1                       # states, inputs, one global parameter
    xi = lambda k, i: k * (nx + nu) + i
    ui = lambda k, i: k * (nx + nu) + nx + i
    gp = nv - 1
    rows, cols, vals = [], [], []
    r = 0
    for k in range(N - 1):                        # dynamics rows couple stage k and k+1 and the parameter
        for i in range(nx):
            for j in range(nx):
                rows.append(r); cols.append(xi(k, j)); vals.append(rng.standard_normal())
            for j in range(nu):
                rows.append(r); cols.append(ui(k, j)); vals.append(rng.standard_normal())
            rows.append(r); cols.append(xi(k + 1, i)); vals.append(-1.0)
            rows.append(r); cols.append(gp); vals.append(rng.standard_normal())
            r += 1
    A = sp.csr_matrix((vals, (rows, cols)), shape=(r, nv))
    G = sp.vstack([sp.eye(nv), -sp.eye(nv)]).tocsr()      # box constraints
    stage = np.concatenate([np.repeat(np.arange(N), nx + nu), [-1]])
    perm = pkg.ordering.stage_order(A, G, stage, N)
    l = G.shape[0]
    wm = rng.uniform(0.5, 2.0, l)
    rhs = rng.standard_normal(nv + r)
    sol, info = pkg.lib.debug_kkt_solve(A, G, l, [], perm, A.data, G.data, wm, 1e-8, rhs)
    K = _dense_kkt(A, G, l, [], wm, 1e-8)
    assert np.abs(K @ sol - rhs).max() < 1e-6
    assert info["nnzL"] < 40 * (nv + r), info
    assert info["levels"] < 12 * (nx + nu) + 8 * nx, info
    # natural order (variables first, then rows) is far worse on the same pattern
    _, info_nat = pkg.lib.debug_kkt_solve(A, G, l, [], None, A.data, G.data, wm, 1e-8, rhs)
    assert info_nat["nnzL"] > 2 * info["nnzL"]


def test_supernodal_program_on_the_starship_kkt(pkg):
    """The reference's starship PTR subproblem under the product's stage ordering: the supernodal schedule must need far
    fewer dependent steps than the scalar one (22 vs 88 at N = 100, profiles/r1_supernode_study.txt) with small panels,
    and solve the KKT system like the scalar program does."""
    from tests import helpers
    N = 16
    pb, P, subs = helpers.starship_subproblems(N, 1, seed=3)
    cp = subs[0]["cp"]
    A, G, l = cp["A"].tocsr(), cp["G"].tocsr(), cp["l"]
    lab = helpers.labels_from_program(subs[0]["prg"], N)
    perm = pkg.ordering.stage_order(A, G, lab, N)
    rng = np.random.default_rng(0)
    wm = rng.uniform(0.5, 2.0, l)
    rhs = rng.standard_normal(A.shape[1] + A.shape[0])
    s1, i1 = pkg.lib.debug_kkt_solve(A, G, l, [], perm, A.data, G.data, wm, 1e-9, rhs, delta_dyn=1e-7)
    s2, i2 = pkg.lib.debug_kkt_solve(A, G, l, [], perm, A.data, G.data, wm, 1e-9, rhs, delta_dyn=1e-7, supernodal=True)
    assert np.abs(s1 - s2).max() <= 1e-8 * max(1.0, np.abs(s1).max())
    # (this is the reference's NormOneBridge form, whose dense L1 blocks give wider supernodes than the product's lowering)
    assert i2["sn_levels"] * 2 <= i1["levels"] and i2["max_rows"] <= 64 and i2["max_width"] <= 12, (i1, i2)


def test_supernodal_program_on_the_product_template(pkg, monkeypatch):
    """The bench-shaped KKT (product template with the L1 lowering, stage ordering, N = 24): the scalar program and the
    supernodal interpreter give the same solution and every panel fits a lane group (<= 32 rows, <= 12 columns), so the
    device runs the supernodal kernels (tests/test_conic_gpu.py checks those against this interpreter)."""
    ex = pkg.examples.starship
    mdl = ex.StarshipProblem(); mdl.hs = 100.0
    traj = pkg.problem.TrajectoryProblem(mdl)
    ex.define_problem(traj, "ptr", handle=None)
    N = 24
    pars = pkg.ptr.Parameters(N=N, Nsub=20, iter_max=5, disc_method=pkg.ptr.FOH, wvc=1e3, wtr=0.1, eps_abs=1e-5,
                              eps_rel=1e-4, feas_tol=5e-3, q_tr=np.inf, q_exit=np.inf)

    class FakeHandle:
        def model_set(self, *a): pass
    monkeypatch.setattr(pkg.lib, "ConeProblem", lambda *a, **k: type("C", (), {"c": None, "close": lambda s: None})())
    fake = FakeHandle(); fake.lib = type("L", (), {"scpb_ptr_setup": staticmethod(lambda *a: 0)})(); fake.h = None
    fake._check = lambda rc, what: None
    pbm = pkg.ptr.SCPProblem(pars, traj, fake, l1_block=4)
    cp = pbm.cp
    rng = np.random.default_rng(1)
    A, G = cp["A"], cp["G"]
    Av = rng.uniform(0.5, 1.5, A.nnz); Gv = rng.uniform(0.5, 1.5, G.nnz); wm = rng.uniform(0.5, 2.0, cp["l"])
    rhs = rng.standard_normal(cp["n"] + cp["p"])
    args = (A, G, cp["l"], [], pbm.perm, Av, Gv, wm, 1e-9, rhs)
    s1, i1 = pkg.lib.debug_kkt_solve(*args, delta_dyn=1e-7)
    s2, i2 = pkg.lib.debug_kkt_solve(*args, delta_dyn=1e-7, supernodal=True)
    scale = max(1.0, np.abs(s1).max())
    assert np.abs(s1 - s2).max() <= 1e-8 * scale
    assert i2["sn_levels"] * 3 <= i1["levels"] and i2["max_rows"] <= 32 and i2["max_width"] <= 10, (i1, i2)
    # hybrid program: scalar programs below the cut + one bridge level, in-place panels above; same solution, and the
    # dependent steps (scalar levels + top supernodal levels) stay well below the scalar level count
    for cut in (3, 6, 9):
        s3, i3 = pkg.lib.debug_kkt_solve(*args, delta_dyn=1e-7, hybrid_cut=cut)
        assert np.abs(s1 - s3).max() <= 1e-8 * scale, (cut, np.abs(s1 - s3).max())
        assert i3["scalar_levels"] == i1["levels"] and i3["levels"] + i3["top_levels"] <= 0.6 * i1["levels"], (cut, i3)
        assert i3["top_levels"] == i2["sn_levels"] - cut and i3["top_supernodes"] > 0
    # targets too long for one item are split over several; the interpreter applies their partial sums through the
    # slots the device uses and rejects a slot numbering that does not cover each split target's items in its level
    assert i1["split_items"] > 0, i1


def test_native_rcm_order(pkg):
    """scpb_order_rcm (csrc/ordering.cu; used by the MathOptInterface shim, julia/SCPToolboxB200.jl): a permutation of the
    KKT nodes with every equality row behind its variables, and a fill within 10 % of the scipy heuristic of
    ordering.rcm_order (and not above the emission order's) on the rocket PTR subproblem (SOC cones)."""
    import ctypes as C
    from oracle import problems, ptr as optr
    N = 12
    pbo = problems.RocketProblem(N)
    xd, ud, p = problems.test_trajectory(pbo, 1, N, seed=3)
    P = optr.PTR(pbo, optr.Parameters(N=N, Nsub=15, iter_max=5, wvc=1e3, wtr=0.1, eps_abs=1e-5, eps_rel=1e-4, feas_tol=1e-3))
    prg, _ = P.build(P.make_solution(xd[0], ud[0], p[0]))
    cp = prg.compile()
    A = cp["A"].tocsr(); G = cp["G"].tocsr(); A.sort_indices(); G.sort_indices()
    n, pp, m = A.shape[1], A.shape[0], G.shape[0]
    L = pkg.lib.load()
    perm = np.zeros(n + pp, dtype=np.int32)
    keep = [np.ascontiguousarray(x, dtype=np.int32) for x in (A.indptr, A.indices, G.indptr, G.indices, cp["q"])]
    ptr = [k.ctypes.data_as(pkg.lib._ip) for k in keep]
    rc = L.scpb_order_rcm(n, pp, m, ptr[0], ptr[1], ptr[2], ptr[3], cp["l"], len(cp["q"]), ptr[4], perm.ctypes.data_as(pkg.lib._ip))
    assert rc == 0
    assert sorted(perm.tolist()) == list(range(n + pp))
    pos = np.empty(n + pp, dtype=int); pos[perm] = np.arange(n + pp)
    for r in range(pp):
        cols = A.indices[A.indptr[r]:A.indptr[r + 1]]
        assert pos[n + r] > pos[cols].max()
    assert L.scpb_order_rcm(n, pp, m, ptr[0], ptr[1], ptr[2], ptr[3], cp["l"] + 1, len(cp["q"]), ptr[4], perm.ctypes.data_as(pkg.lib._ip)) != 0
    rng = np.random.default_rng(0)
    nwm = cp["l"] + sum(int(q) ** 2 for q in cp["q"])
    wm = np.zeros(nwm); wm[:cp["l"]] = rng.uniform(0.5, 2.0, cp["l"])
    o = cp["l"]
    for q in cp["q"]:
        wm[o:o + q * q] = np.eye(q).ravel(); o += q * q
    rhs = rng.standard_normal(n + pp)
    fill = {}
    for name, pr in (("native", perm), ("scipy", pkg.ordering.rcm_order(A, G)), ("natural", np.arange(n + pp, dtype=np.int32))):
        sol, info = pkg.lib.debug_kkt_solve(A, G, cp["l"], cp["q"], pr, A.data, G.data, wm, 1e-9, rhs)
        fill[name] = info["nnzL"]
        K = sp.bmat([[1e-9 * sp.eye(n) + G.T @ sp.block_diag([sp.diags(wm[:cp["l"]])] + [sp.eye(int(q)) for q in cp["q"]]) @ G, A.T],
                     [A, -1e-9 * sp.eye(pp)]]).tocsc()
        assert np.abs(K @ sol - rhs).max() <= 1e-6 * np.abs(rhs).max()
    print("nnzL", fill)
    assert fill["native"] <= 1.1 * fill["scipy"] and fill["native"] <= fill["natural"]
