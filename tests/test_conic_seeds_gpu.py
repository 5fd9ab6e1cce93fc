"""The batched cone solver seed by seed: second-order cones of the shapes the product emits, explicit seed-group sizes,
padded and mixed groups.

(a) Known-answer programs built from a chosen primal-dual optimum (LP rows active or inactive; second-order cones
    interior, at the apex or on the boundary), so that the exact answer is known by construction.  A CPU test checks
    the constructions against the oracle interior point.
(b) The starship PTR subproblems with second-order-cone trust regions (q_tr = 1, 2, 4) against the oracle.
(c) One device KKT solve whose SOC blocks are Nesterov-Todd scalings of interior (s, z) pairs, against numpy.
(d) Seed groups: group sizes 1 to 8 (IPM_MAXG), both CTA sizes, padded last groups and more groups than SMs; seeds with
    different outcomes in one group; bitwise independence of a seed from padded lanes and from NaN-data group-mates.
"""
import os

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import conic, problems, ptr as optr
from tests import helpers

gpu = pytest.mark.gpu

# device tolerances of the subproblem solves.  The known-answer programs run at the library default (ECOS' 1e-8): asked
# for 1e-9, the device stalls between 1e-9 and 1e-7 on the programs with boundary cones (the oracle reaches 1e-10) and
# returns ALMOST_OPTIMAL; x is then still within 1e-7 of the constructed optimum
KTOL = dict(feastol=1e-9, abstol=1e-9, reltol=1e-9)
OPTIMAL, NUMERICAL, PINF, DINF = 0, 2, 4, 5


# ------------------------------------------------------------------ known-answer construction
def _pattern(rng, n, p, m, dens):
    """Random sparsity patterns of A (p x n) and G (m x n); every row has an entry, every A row a distinct pivot column."""
    A = sp.random(p, n, density=dens, random_state=rng.integers(1 << 30), format="csr")
    A = (A + sp.csr_matrix((np.ones(p), (np.arange(p), rng.permutation(n)[:p])), shape=(p, n))).tocsr()
    G = sp.random(m, n, density=dens, random_state=rng.integers(1 << 30), format="csr")
    G = (G + sp.csr_matrix((np.ones(m), (np.arange(m), rng.integers(0, n, m))), shape=(m, n))).tocsr()
    A.sort_indices(); G.sort_indices()
    return A, G


def _soc_point(rng, q):
    """A point of int SOC(q)."""
    w = rng.standard_normal(q)
    w[0] = np.linalg.norm(w[1:]) + rng.uniform(0.5, 1.5)
    return w


def _known_answer(rng, A, G, l, soc, states=None):
    """Values on the patterns of A and G plus (c, b, h) whose optimum is a drawn (x*, y*, z*, s*).

    LP row: s > 0, z = 0 or s = 0, z > 0.  SOC: interior (s in int K, z = 0), apex (s = 0, z in int K) or boundary
    (s = t (1, v), z = tau (1, -v), |v| = 1; v = +-1 for q = 2).  Strict complementarity holds everywhere.  x* is unique
    when the rows with s* = 0 stacked with A have rank n: every optimal x satisfies them with equality (complementary
    slackness with z*).  Draws again until that holds."""
    n, p, m = A.shape[1], A.shape[0], G.shape[0]
    for _ in range(100):
        Av = A.data * rng.uniform(0.5, 1.5, A.nnz) * rng.choice([-1.0, 1.0], A.nnz)
        Gv = G.data * rng.uniform(0.5, 1.5, G.nnz) * rng.choice([-1.0, 1.0], G.nnz)
        Ak = sp.csr_matrix((Av, A.indices, A.indptr), shape=A.shape)
        Gk = sp.csr_matrix((Gv, G.indices, G.indptr), shape=G.shape)
        s, z = np.zeros(m), np.zeros(m)
        tight = np.zeros(m, dtype=bool)
        act = rng.random(l) < 0.5
        s[:l] = np.where(act, 0.0, rng.uniform(0.5, 2.0, l))
        z[:l] = np.where(act, rng.uniform(0.5, 2.0, l), 0.0)
        tight[:l] = act
        o = l
        for k, q in enumerate(soc):
            st = states[k] if states is not None else rng.choice(["interior", "apex", "boundary"])
            if st == "interior":
                s[o:o + q] = _soc_point(rng, q)
            elif st == "apex":
                z[o:o + q] = _soc_point(rng, q)
                tight[o:o + q] = True
            else:
                v = rng.standard_normal(q - 1)
                v /= np.linalg.norm(v)
                t, tau = rng.uniform(0.5, 2.0, 2)
                s[o:o + q] = t * np.concatenate([[1.0], v])
                z[o:o + q] = tau * np.concatenate([[1.0], -v])
            o += q
        rows = sp.vstack([Ak, Gk[np.flatnonzero(tight)]]).toarray()
        if np.linalg.matrix_rank(rows) < n:
            continue
        x, y = rng.standard_normal(n), rng.standard_normal(p)
        h = Gk @ x + s
        b = Ak @ x
        c = -(Ak.T @ y) - (Gk.T @ z)
        return dict(A=Ak, G=Gk, Av=Av, Gv=Gv, c=c, b=b, h=h, x=x, y=y, z=z, s=s, obj=float(c @ x), l=l, q=list(soc),
                    tight=tight)
    raise AssertionError("no instance with a unique primal optimum")


def _spmv_ld(M, v):
    """M v in long double for a CSR matrix M."""
    M = sp.csr_matrix(M)
    prod = M.data.astype(np.longdouble) * v[M.indices]
    out = np.zeros(M.shape[0], dtype=np.longdouble)
    np.add.at(out, np.repeat(np.arange(M.shape[0]), np.diff(M.indptr)), prod)
    return out


def _kkt_residuals(kp, x, y, z, s):
    """Primal and dual residuals and the complementarity gap, in long double."""
    L = np.longdouble
    A, G = kp["A"], kp["G"]
    x, y, z, s = (np.asarray(v, dtype=L) for v in (x, y, z, s))
    b, h, c = (np.asarray(kp[k], dtype=L) for k in ("b", "h", "c"))
    pres = max(np.abs(_spmv_ld(A, x) - b).max(initial=L(0)), np.abs(_spmv_ld(G, x) + s - h).max(initial=L(0)))
    dres = np.abs(c + _spmv_ld(A.T, y) + _spmv_ld(G.T, z)).max(initial=L(0))
    return float(pres), float(dres), float(s @ z)


def _cone_margin(l, soc, u):
    """Smallest interior margin of u over the cones (LP: value; SOC: u0 - |u1|), in long double."""
    u = np.asarray(u, dtype=np.longdouble)
    mg = [u[:l].min()] if l else []
    o = l
    for q in soc:
        mg.append(u[o] - np.sqrt(np.sum(u[o + 1:o + q] ** 2)))
        o += q
    return float(min(mg))


def _check_kkt(kp, x, y, z, s, pobj, tol=1e-7, what=""):
    """Residuals, gap and cone membership of a returned (x, y, z, s); residuals relative to the data norms the solver
    uses, the gap relative to the objective."""
    pres, dres, gap = _kkt_residuals(kp, x, y, z, s)
    sb = max(1.0, np.linalg.norm(kp["b"]), np.linalg.norm(kp["h"]))
    sc = max(1.0, np.linalg.norm(kp["c"]))
    assert pres <= tol * sb and dres <= tol * sc, (what, pres, dres)
    assert abs(gap) <= tol * max(1.0, abs(pobj)), (what, gap)
    assert _cone_margin(kp["l"], kp["q"], s) >= -1e-9 * max(1.0, np.abs(s).max()), what
    assert _cone_margin(kp["l"], kp["q"], z) >= -1e-9 * max(1.0, np.abs(z).max()), what


def _check_known_answer(kp, x, obj, what=""):
    assert abs(obj - kp["obj"]) <= 1e-7 * max(1.0, abs(kp["obj"])), (what, obj, kp["obj"])
    assert np.abs(x - kp["x"]).max() <= 1e-6 * max(1.0, np.abs(kp["x"]).max()), (what, np.abs(x - kp["x"]).max())


# name, n, p, l, soc dims, state of every cone (None: drawn), pattern density
KNOWN = {
    "soc2": (10, 2, 4, [2] * 12, None, 0.3),
    "qtr4_set": (12, 3, 8, [2, 3, 4, 9, 11], None, 0.3),
    "qtr4_set_no_boundary": (12, 3, 8, [2, 3, 4, 9, 11], ["apex", "interior", "apex", "interior", "apex"], 0.3),
    "soc11x40": (60, 10, 0, [11] * 40, None, 0.08),
    "soc64_boundary": (20, 4, 30, [64], ["boundary"], 0.2),
    "soc64_apex": (20, 4, 6, [64], ["apex"], 0.2),
    "soc2x1500": (150, 10, 20, [2] * 1500, None, 0.012),
}


def _program(name, seed=0, nb=1):
    """nb known-answer instances of one named program, sharing one pattern."""
    n, p, l, soc, states, dens = KNOWN[name]
    rng = np.random.default_rng(seed)
    A, G = _pattern(rng, n, p, l + sum(soc), dens)
    return A, G, l, soc, [_known_answer(rng, A, G, l, soc, states) for _ in range(nb)]


def _stack(kps):
    return (np.array([k["Av"] for k in kps]), np.array([k["Gv"] for k in kps]), np.array([k["c"] for k in kps]),
            np.array([k["b"] for k in kps]).reshape(len(kps), -1), np.array([k["h"] for k in kps]))


@pytest.mark.parametrize("name", sorted(KNOWN))
def test_known_answer_constructions_against_the_oracle(name):
    """The constructions themselves: the oracle interior point finds the constructed optimum (CPU)."""
    A, G, l, soc, kps = _program(name)
    kp = kps[0]
    assert np.linalg.matrix_rank(sp.vstack([kp["A"], kp["G"][np.flatnonzero(kp["tight"])]]).toarray()) == A.shape[1]
    # the constructed point itself is optimal: feasible, dual feasible, zero gap, in the cones
    _check_kkt(kp, kp["x"], kp["y"], kp["z"], kp["s"], kp["obj"], tol=1e-12, what="construction")
    cp = dict(c=kp["c"], c0=0.0, A=kp["A"], b=kp["b"], G=kp["G"], h=kp["h"], l=l, q=list(soc))
    ref = conic.solve_ipm(cp, tol=1e-10)
    assert ref["status"] == "OPTIMAL", ref["status"]
    _check_known_answer(kp, ref["z"], ref["obj"], "oracle")
    _check_kkt(kp, ref["z"], ref["y_eq"], ref["z_ineq"], ref["s"], ref["obj"], what="oracle")


@gpu
@pytest.mark.parametrize("name", sorted(KNOWN))
def test_known_answer_programs_on_the_device(handle, pkg, name):
    """Every cone shape the product emits (q = 2, the q_tr = 4 set, many q = 11, one q = 64, more cones than the CTA
    has threads): the device finds the constructed optimum."""
    nb = 3
    A, G, l, soc, kps = _program(name, seed=1, nb=nb)
    cone = pkg.lib.ConeProblem(handle, A, G, l, soc, perm=pkg.ordering.rcm_order(A, G))
    out = cone.solve(*_stack(kps))
    cone.close()
    for k, kp in enumerate(kps):
        assert out["status"][k] == OPTIMAL, (name, k, out["status"], out["iters"])
        _check_known_answer(kp, out["x"][k], out["pobj"][k], (name, k))
        _check_kkt(kp, out["x"][k], out["y"][k], out["z"][k], out["s"][k], out["pobj"][k], what=(name, k))


# ------------------------------------------------------------------ the product's own SOC subproblems
SUB_CASES = [(q_tr, N) for q_tr in (1, 2, 4) for N in (12, 31)]
SUB_NB = 6
SUB_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_soc_subproblems.npz")


def starship_soc_subproblems(N, nb, q_tr, seed):
    """helpers.starship_subproblems with the trust-region norm passed through (q_tr = 1: L1, 2: SOC, 4: squared
    two-norm through the GEOM cone): nb first PTR subproblems around perturbed initial guesses."""
    pb = problems.StarshipProblem(N)
    g = pb.guess(N)
    pars = optr.Parameters(N=N, Nsub=30, iter_max=15, wvc=1e3, wtr=0.1, eps_abs=1e-5, eps_rel=1e-4, feas_tol=5e-3,
                           q_tr=q_tr)
    P = optr.PTR(pb, pars)
    rng = np.random.default_rng(seed)
    sc = P.scale
    subs = []
    for b in range(nb):
        xd = g[0] + (0.02 * sc.Sx * rng.standard_normal(g[0].shape) if b else 0.0)
        ud = g[1] + (0.02 * sc.Su * rng.standard_normal(g[1].shape) if b else 0.0)
        p = g[2] * (1 + (0.05 * rng.uniform(-1, 1, g[2].shape) if b else 0.0))
        prg, _ = P.build(P.make_solution(xd, ud, p))
        subs.append(dict(prg=prg, cp=prg.compile()))
    return subs


def _golden_subproblems():
    """The oracle interior point's answers (conic.solve_ipm, tol = 1e-10) to the subproblems above, precomputed by
    scripts/make_golden_soc_subproblems.py: a run of the oracle on all of them takes minutes."""
    return np.load(SUB_GOLDEN)


@pytest.mark.parametrize("q_tr", [1, 2, 4])
def test_golden_subproblem_answers_are_the_oracles(q_tr):
    """The stored oracle answers still are what the oracle computes (CPU; the first two seeds at N = 12)."""
    gold = _golden_subproblems()
    subs = starship_soc_subproblems(12, 2, q_tr, seed=12 + q_tr)
    for k, sub in enumerate(subs):
        ref = conic.solve_ipm(sub["cp"], tol=1e-10)
        assert ref["status"] == str(gold[f"status_q{q_tr}_N12"][k])
        assert abs(ref["obj"] - gold[f"obj_q{q_tr}_N12"][k]) <= 1e-12 * max(1.0, abs(ref["obj"]))


@gpu
@pytest.mark.parametrize("group", [0, 2])
@pytest.mark.parametrize("q_tr,N", SUB_CASES)
def test_starship_soc_subproblems_match_the_oracle(handle, pkg, q_tr, N, group):
    """PTR subproblems with L1 / SOC / GEOM trust regions (SOC dimensions 2, 3, 4, 9 and 11), stage ordering."""
    subs = starship_soc_subproblems(N, SUB_NB, q_tr, seed=N + q_tr)
    gold = _golden_subproblems()
    cp0 = subs[0]["cp"]
    Apat, Avals = helpers.union_pattern([s["cp"]["A"] for s in subs])
    Gpat, Gvals = helpers.union_pattern([s["cp"]["G"] for s in subs])
    perm = pkg.ordering.stage_order(Apat, Gpat, helpers.labels_from_program(subs[0]["prg"], N), N)
    cone = pkg.lib.ConeProblem(handle, Apat, Gpat, cp0["l"], cp0["q"], perm=perm)
    c = np.array([s["cp"]["c"] for s in subs]); b = np.array([s["cp"]["b"] for s in subs])
    h = np.array([s["cp"]["h"] for s in subs])
    out = cone.solve(Avals, Gvals, c, b, h, group=group, **KTOL)
    cone.close()
    for k, sub in enumerate(subs):
        cpk = sub["cp"]
        assert str(gold[f"status_q{q_tr}_N{N}"][k]) in ("OPTIMAL", "ALMOST_OPTIMAL")
        assert out["status"][k] == OPTIMAL, (k, out["status"], out["iters"])
        want = gold[f"obj_q{q_tr}_N{N}"][k] - cpk["c0"]
        assert abs(out["pobj"][k] - want) <= 1e-7 * max(1.0, abs(want)), (k, out["pobj"][k], want)
        _check_kkt(dict(cpk, q=list(cpk["q"])), out["x"][k], out["y"][k], out["z"][k], out["s"][k], out["pobj"][k],
                   what=k)


# ------------------------------------------------------------------ device KKT solve with NT-scaled SOC blocks
def _nt_winv2(rng, l, soc):
    """W^-2 in the solver's layout (LP weights, then the dense q x q SOC blocks) from the oracle's Nesterov-Todd scaling
    of an interior (s, z) pair."""
    K = conic._Cones(l, soc)
    s = np.concatenate([rng.uniform(0.1, 10.0, l)] + [_soc_point(rng, q) * rng.uniform(0.1, 10.0) for q in soc])
    z = np.concatenate([rng.uniform(0.1, 10.0, l)] + [_soc_point(rng, q) * rng.uniform(0.1, 10.0) for q in soc])
    _, Wi, _ = K.nt(s, z)
    Wi = Wi.toarray()
    W2i = Wi @ Wi   # W is symmetric: W^-2 = (W'W)^-1 = Wi Wi
    w = [np.diag(W2i)[:l]]
    o = l
    for q in soc:
        w.append(W2i[o:o + q, o:o + q].ravel())
        o += q
    return np.concatenate(w)


@gpu
@pytest.mark.parametrize("sn", ["0", "1", "h1", "h2"])
@pytest.mark.parametrize("seed,n,p,l,soc", [(0, 14, 4, 6, [2] * 5 + [11] * 2), (1, 24, 6, 10, [11] * 6),
                                            (2, 40, 5, 0, [2] * 1200)])
def test_device_kkt_solve_with_nt_soc_blocks(handle, pkg, monkeypatch, sn, seed, n, p, l, soc):
    """The reduced KKT system assembled from Nesterov-Todd SOC blocks (dimensions 2 and 11, and more cones than the CTA
    has threads) against a dense numpy solve, for every kernel variant."""
    from tests.test_conic_gpu import _dense_kkt, _variant
    _variant(monkeypatch, sn)
    rng = np.random.default_rng(seed)
    m = l + sum(soc)
    A, G = _pattern(rng, n, p, m, min(0.4, 6.0 / n))
    G = sp.vstack([G[:l], sp.eye(n), G[l:]]).tocsr()   # n more LP rows keep G' W^-2 G definite
    G.sort_indices()
    l2 = l + n
    nb = 3
    delta = 1e-7
    cone = pkg.lib.ConeProblem(handle, A, G, l2, soc, perm=pkg.ordering.rcm_order(A, G))
    Av = np.array([A.data * rng.uniform(0.5, 1.5, A.nnz) for _ in range(nb)])
    Gv = np.array([G.data * rng.uniform(0.5, 1.5, G.nnz) for _ in range(nb)])
    wms = np.array([_nt_winv2(rng, l2, soc) for _ in range(nb)])
    rhs = rng.standard_normal((nb, n + p))
    sol, bad = cone.debug_kkt_solve_dev(Av, Gv, wms, delta, rhs)
    cone.close()
    for k in range(nb):
        Ak = sp.csr_matrix((Av[k], A.indices, A.indptr), shape=A.shape)
        Gk = sp.csr_matrix((Gv[k], G.indices, G.indptr), shape=G.shape)
        want = np.linalg.solve(_dense_kkt(Ak, Gk, l2, soc, wms[k], delta), rhs[k])
        assert bad[k] == 0
        assert np.abs(sol[k] - want).max() <= 1e-7 * max(1.0, np.abs(want).max()), (sn, k, np.abs(sol[k] - want).max())


# ------------------------------------------------------------------ seed groups and isolation
# the q_tr = 4 cone set without boundary cones: the device converges to 1e-12 on it, so that comparisons between runs
# are not limited by the floor the boundary cones put near 1e-8
GEOM_PROGRAM = "qtr4_set_no_boundary"
_BATCH = {}


def _batch(B):
    """B known-answer seeds of one program (the q_tr = 4 cone set with LP rows, no boundary cones), one pattern."""
    if B not in _BATCH:
        _BATCH[B] = _program(GEOM_PROGRAM, seed=7, nb=B)
    return _BATCH[B]


def _seed(out, k):
    return {key: out[key][k] for key in ("x", "y", "z", "s", "pobj", "dobj", "status", "iters")}


def _bitwise_equal(a, b):
    return all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in ("x", "y", "z", "s", "pobj", "dobj", "iters"))


def _diff(a, b):
    return {k: float(np.abs(np.asarray(a[k], float) - np.asarray(b[k], float)).max()) for k in ("x", "pobj", "iters")}


@gpu
@pytest.mark.parametrize("threads", [512, 1024])
@pytest.mark.parametrize("group", [1, 2, 4, 8])
def test_seed_group_geometry(handle, pkg, group, threads):
    """B = 1, G + 1 (a padded last group) and 267 (more groups than the H100's 132 SMs for G <= 2; not a multiple of G):
    every seed finds its constructed optimum and matches a solve of that seed alone at the same group size and CTA size.
    Active group-mates share the refinement loop of the KKT solves (conic_ipm.cuh, kkt_solve: the group refines again
    while one of its active seeds asks for it), so a seed's last bits may depend on them: against the solve alone the
    status is equal and the objective agrees to 1e-9 relative."""
    opts = dict(group=group, threads=threads)
    A, G, l, soc, kps = _batch(267)
    cone = pkg.lib.ConeProblem(handle, A, G, l, soc, perm=pkg.ordering.rcm_order(A, G))
    alone = {}
    for B in (1, group + 1, 267):
        out = cone.solve(*_stack(kps[:B]), **opts)
        for k in range(B):
            kp = kps[k]
            assert out["status"][k] == OPTIMAL, (B, k, out["status"][k], out["iters"][k])
            _check_known_answer(kp, out["x"][k], out["pobj"][k], (B, k))
            _check_kkt(kp, out["x"][k], out["y"][k], out["z"][k], out["s"][k], out["pobj"][k], what=(B, k))
            if k not in alone:
                alone[k] = cone.solve(*_stack([kp]), **opts)
            one = alone[k]
            assert out["status"][k] == one["status"][0], (B, k)
            assert abs(out["pobj"][k] - one["pobj"][0]) <= 1e-9 * max(1.0, abs(one["pobj"][0])), (B, k)
    assert cone.info()["group"] == group
    cone.close()


def _mixed_program():
    """test_conic_gpu.test_infeasibility_certificates' program: x = (x1, x2); -x1 <= h1, -x2 <= h2, x1 + x2 <= h3;
    x1 - x2 = b.  Seed kinds: OPTIMAL (objective 0), primal infeasible, unbounded, NaN data."""
    A = sp.csr_matrix(np.array([[1.0, -1.0]]))
    G = sp.csr_matrix(np.array([[-1.0, 0.0], [0.0, -1.0], [1.0, 1.0]]))
    kinds = {
        "O": (G.data, [1.0, 1.0], [0.0, 0.0, 2.0]),
        "P": (G.data, [1.0, 1.0], [-2.0, -2.0, 1.0]),
        "D": (np.concatenate([G.data[:-2], [0.0, 0.0]]), [-1.0, -1.0], [0.0, 0.0, 2.0]),
        "N": (G.data, [1.0, 1.0], [0.0, np.nan, 2.0]),
    }
    return A, G, kinds


def _mixed_batch(order):
    A, G, kinds = _mixed_program()
    Gv = np.array([kinds[k][0] for k in order]); c = np.array([kinds[k][1] for k in order])
    h = np.array([kinds[k][2] for k in order])
    return np.tile(A.data, (len(order), 1)), Gv, c, np.zeros((len(order), 1)), h


def _check_mixed(A, G, order, out):
    Ad, Gd = A.toarray(), G.toarray()
    want = dict(O=OPTIMAL, P=PINF, D=DINF, N=NUMERICAL)
    assert [int(s) for s in out["status"]] == [want[k] for k in order], (order, out["status"], out["iters"])
    for k, kind in enumerate(order):
        y, z, x = out["y"][k], out["z"][k], out["x"][k]
        if kind == "O":
            assert abs(out["pobj"][k]) < 1e-7 and np.abs(x).max() < 1e-6
        elif kind == "P":   # (y, z) certifies infeasibility: A'y + G'z = 0, z >= 0, b'y + h'z < 0
            nrm = -(np.array([-2.0, -2.0, 1.0]) @ z)
            assert nrm > 0 and np.abs(Ad.T @ y + Gd.T @ z).max() <= 1e-6 * nrm and (z > -1e-9 * nrm).all(), k
        elif kind == "D":   # x certifies unboundedness: A x = 0, G2 x <= 0, c'x < 0
            G2 = Gd.copy(); G2[2] = 0.0
            cx = -x.sum()
            assert cx < 0 and np.abs(Ad @ x).max() <= 1e-6 * abs(cx) and (G2 @ x).max() <= 1e-6 * abs(cx), k


@gpu
@pytest.mark.parametrize("group", [2, 4, 8])
def test_mixed_outcomes_in_one_group(handle, pkg, group):
    """OPTIMAL, infeasible, unbounded and NaN-data seeds in every pairing (at G = 2 each of the six pairs is a group;
    at G = 4 and 8 every group holds all four kinds): each seed keeps its own status and certificate."""
    A, G, _ = _mixed_program()
    order = "OPDNODPNONPD"
    cone = pkg.lib.ConeProblem(handle, A, G, 3, [])
    out = cone.solve(*_mixed_batch(order), group=group)
    cone.close()
    _check_mixed(A, G, order, out)


@gpu
@pytest.mark.parametrize("threads", [512, 1024])
@pytest.mark.parametrize("group", [2, 4, 8])
def test_a_seed_is_bitwise_independent_of_padding_and_nan_mates(handle, pkg, group, threads):
    """A seed whose group-mates are padded lanes or NaN-data seeds gives the same bits as its solve as the only real
    seed of the group (B = 1: its group-mates are padded copies of it).  Padded lanes run as frozen copies of seed
    B - 1, and a NaN seed stops at its first residual check; neither may steer the refinement of the others."""
    opts = dict(group=group, threads=threads, **KTOL)
    A, G, l, soc, kps = _batch(4)
    Av, Gv, c, b, h = _stack(kps[:2])
    nan = dict(Av=Av[1].copy(), Gv=Gv[1].copy(), c=c[1].copy(), b=b[1].copy(), h=h[1].copy())
    nan["h"][len(nan["h"]) // 2] = np.nan
    cone = pkg.lib.ConeProblem(handle, A, G, l, soc, perm=pkg.ordering.rcm_order(A, G))
    ref = _seed(cone.solve(Av[:1], Gv[:1], c[:1], b[:1], h[:1], **opts), 0)
    assert ref["status"] == OPTIMAL
    # seed 0 followed by one NaN seed: the rest of the group is padding (copies of the NaN seed)
    # ... and a NaN seed in front of it, so that it is not the first lane of its group
    for pos in (0, 1):
        rows = [None] * 2
        rows[pos] = (Av[0], Gv[0], c[0], b[0], h[0])
        rows[1 - pos] = (nan["Av"], nan["Gv"], nan["c"], nan["b"], nan["h"])
        out = cone.solve(*(np.array(col) for col in zip(*rows)), **opts)
        assert out["status"][1 - pos] == NUMERICAL, out["status"]
        got = _seed(out, pos)
        assert _bitwise_equal(got, ref), (pos, _diff(got, ref))
    cone.close()


@gpu
def test_reused_buffers_give_the_bits_of_a_fresh_problem(handle, pkg):
    """B = 4 and then B = 3 on one ConeProblem (the device buffers are reused, the padded lane now copies seed 2) equal
    B = 3 on a fresh ConeProblem, bit for bit, at G = 4."""
    A, G, l, soc, kps = _batch(4)
    perm = pkg.ordering.rcm_order(A, G)
    cone = pkg.lib.ConeProblem(handle, A, G, l, soc, perm=perm)
    cone.solve(*_stack(kps[:4]), group=4, **KTOL)
    out = cone.solve(*_stack(kps[:3]), group=4, **KTOL)
    cone.close()
    fresh = pkg.lib.ConeProblem(handle, A, G, l, soc, perm=perm)
    want = fresh.solve(*_stack(kps[:3]), group=4, **KTOL)
    fresh.close()
    for k in range(3):
        assert _bitwise_equal(_seed(out, k), _seed(want, k)), (k, _diff(_seed(out, k), _seed(want, k)))


# ------------------------------------------------------------------ the PTR loop with SOC trust regions
@gpu
@pytest.mark.xfail(reason="ends 1e-4..1e-3 (ex(phys)) away from the oracle loop like q_tr = 4 (test_zz_unvalidated_gpu.py) "
                          "although every subproblem's cone solve matches the oracle: not localised beyond the PTR loop "
                          "with a non-LINF trust region", strict=False)
@pytest.mark.parametrize("q_tr", [1, 2])
def test_ptr_with_soc_trust_regions_matches_the_oracle_loop(pkg, handle, q_tr):
    """The batched PTR loop with L1 (q_tr = 1) and SOC (q_tr = 2) trust regions, which need no GEOM cone, against the
    oracle loop: 5 forced iterations of the starship problem (tests/test_zz_unvalidated_gpu.py runs q_tr = 4 the same
    way).  Every subproblem starts the interior point cold (the PTR loop's default; warm starts are opt-in), so
    SCPB_NO_WARM=1 would change nothing.  Measured on an H100: q_tr = 1 ex(phys) 8.1e-4, dJ 3.0e-4; q_tr = 2 ex(phys)
    1.2e-4, dJ 6.0e-6; q_tr = 4 ex(phys) 6.3e-4, dJ 1.0e-4; 5 iterations and SCP_SOLVED on both sides every time."""
    from tests.test_ptr_gpu import _setup
    N, Nsub, K = 12, 60, 5
    mdl, traj, pars = _setup(pkg, handle, N, Nsub, iter_max=K)
    pars.q_tr = q_tr
    pars.eps_abs = 0.0
    pars.eps_rel = 0.0
    pbo = problems.StarshipProblem(N)
    g = pbo.guess(N)
    mdl.hs = pbo.hs
    P = optr.PTR(pbo, optr.Parameters(N=N, Nsub=Nsub, iter_max=K, wvc=1e3, wtr=0.1, eps_abs=0.0, eps_rel=0.0,
                                      feas_tol=5e-3, q_tr=q_tr, solver_tol=1e-10))
    X0, U0, P0 = np.array([g[0]]), np.array([g[1]]), np.array([g[2]])
    pbm = pkg.ptr.create(pars, traj, handle)
    sol = pkg.ptr.solve(pbm, (X0, U0, P0), feastol=1e-10, abstol=1e-10, reltol=1e-10)
    pbm.close()
    ref = P.solve((X0[0], U0[0], P0[0]), prefer="ipm")
    rs = ref["sol"]
    ex7 = np.abs((sol.xd[0][:, :7] - rs.xd[:, :7]) / P.scale.Sx[:7]).max()
    dJ = abs(sol.cost[0] - rs.J_aug) / max(1.0, abs(rs.J_aug))
    print("q_tr", q_tr, "iterations", sol.iterations[0], ref["iterations"], "ex(phys)", ex7, "dJ", dJ,
          sol.status[0], ref["status"])
    assert sol.status[0] == ref["status"] == "SCP_SOLVED" and int(sol.iterations[0]) == ref["iterations"] == K
    assert ex7 <= 1e-4 and dJ <= 1e-6
