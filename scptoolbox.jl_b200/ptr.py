"""PTR -- host-side mirror of src/solvers/ptr.jl for the GPU path.

  Parameters           ptr.jl:57-71
  create(pars, traj)   ptr.jl:148-195 + SCPProblem / compute_scaling (scp.jl:140-157, 376-517)
  solve(pbm, guesses)  ptr.jl:448-532, for a BATCH of initial guesses in lock step on the GPU

`create` builds the subproblem once, symbolically (Subproblem ctor ptr.jl:213-293, add_dynamics! scp.jl:657-674,
add_convex_*! :685-734, add_nonconvex_constraints! :744-794, add_bcs! :808-895, add_trust_region! ptr.jl:565-743,
add_cost! :753-895) with device-computed quantities as symbolic sources, compiles it to the shared sparsity
pattern + fill matrix W, orders the KKT system stage-wise and hands everything to libscpb.  `solve` is one C-ABI
call (scpb_ptr_solve) that runs discretize! -> formulate -> solve -> discretize! -> stopping test on the device.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import lib, ordering
from .parser import ConicTemplate, Expr, Lin, matvec
from .problem import model_parameters

FOH, IMPULSE = lib.FOH, lib.IMPULSE
IMPULSE_MODELS = (lib.MODEL_RENDEZVOUS2D,)     # device packs with impulse semantics (csrc/models.cuh)


@dataclass
class Parameters:            # ptr.jl:57-71
    N: int
    Nsub: int
    iter_max: int
    disc_method: int
    wvc: float
    wtr: float
    eps_abs: float
    eps_rel: float
    feas_tol: float
    q_tr: float
    q_exit: float
    solver: object = None            # kept for signature compatibility (the solver is libscpb)
    solver_opts: dict = None         # {"verbose":.., "maxit":..} as in the reference tests


class SCPScaling:
    """SCPScaling + compute_scaling (scp.jl:39-49, 376-517): x = S*xh + c maps the bounding box of every variable onto
    [0, 1].  A variable with an advised range (problem_advise_scale!) uses it; for the others the reference solves
    2*(nx + nu + 2*np) tiny cone programs  min / max z_i  over the convex sets X (states, parameters) and U (inputs,
    parameters) imposed at every time node (scp.jl:439-481).  Here those programs share one sparsity pattern per set,
    so they are ONE batched call of the GPU cone solver each (only the cost vector differs per seed); a program that
    comes back DUAL_INFEASIBLE (unbounded variable) or NUMERICAL_ERROR keeps the default box [0, 1] (scp.jl:470-473)."""

    def __init__(self, traj, handle=None, t=None):
        zero_tol = np.sqrt(np.finfo(float).eps)
        nx, nu, np_ = traj.nx, traj.nu, traj.np
        box = {"x": np.tile([0.0, 1.0], (nx, 1)), "u": np.tile([0.0, 1.0], (nu, 1)), "p": np.tile([0.0, 1.0], (np_, 1))}
        adv = {"x": traj.xrg, "u": traj.urg, "p": traj.prg}
        for k_ in box:
            for i, r in enumerate(adv[k_]):
                if r is not None:
                    box[k_][i] = r
        self.computed = {}        # (block, index, 0 = min / 1 = max) -> cone status name, for the boxes that were solved
        missing = {k_: [i for i, r in enumerate(adv[k_]) if r is None] for k_ in box}
        # the reference's four passes, in its order: x over X, u over U, p over X, p over U (a later pass overwrites)
        passes = [("x", traj.X, "X"), ("u", traj.U, "U"), ("p", traj.X, "X"), ("p", traj.U, "U")]
        cache = {}
        for blk, cset, tag in passes:
            if not missing[blk] or cset is None:
                continue              # no set: every program is unbounded -> default box (what ECOS reports, :470)
            if handle is None or t is None:
                raise lib.ScpbError(f"no scaling advice for {blk}{missing[blk]}: the bounding-box solves need a device handle")
            if tag not in cache:
                cache[tag] = self._set_program(traj, cset, tag, t)
            self._bbox_pass(handle, cache[tag], blk, missing[blk], box[blk])

        def mk(b):
            S = b[:, 1] - b[:, 0]
            S = np.where(S < zero_tol, 1.0, S)
            return S, b[:, 0].copy()

        self.Sx, self.cx = mk(box["x"])
        self.Su, self.cu = mk(box["u"])
        self.Sp, self.cp = mk(box["p"])

    @staticmethod
    def _set_program(traj, cset, tag, t):
        """plain (unscaled) variables x, u, p; the set imposed at every node k on the SAME variables (scp.jl:446-455)"""
        prg = ConicTemplate(1)
        x = prg.new_variable(traj.nx, "x")
        u = prg.new_variable(traj.nu, "u")
        p = prg.new_variable(traj.np, "p")
        for k in range(len(t)):
            if tag == "X":
                cset(prg, t[k], k + 1, x, p)
            else:
                cset(prg, t[k], k + 1, u, p)
        cp = prg.compile()
        vals = np.asarray(cp["W"] @ np.ones(1)).ravel()
        return dict(prg=prg, cp=cp, vals=vals)

    def _bbox_pass(self, handle, prog, blk, idx, box):
        cp, vals, prg = prog["cp"], prog["vals"], prog["prg"]
        n, p_, m = cp["n"], cp["p"], cp["m"]
        if m == 0 and p_ == 0:
            return
        off = prg.blocks[blk][0]
        nb = 2 * len(idx)
        Av = np.tile(vals[:cp["nnzA"]], (nb, 1)); Gv = np.tile(vals[cp["nnzA"]:cp["nnzA"] + cp["nnzG"]], (nb, 1))
        b = np.tile(vals[cp["off_b"]:cp["off_b"] + p_], (nb, 1)); h = np.tile(vals[cp["off_h"]:cp["off_h"] + m], (nb, 1))
        c = np.zeros((nb, n))
        for q, i in enumerate(idx):
            c[2 * q, off + i] = 1.0         # min z_i
            c[2 * q + 1, off + i] = -1.0    # max z_i
        cone = lib.ConeProblem(handle, cp["A"], cp["G"], cp["l"], cp["soc_dims"], perm=ordering.rcm_order(cp["A"], cp["G"]))
        try:
            out = cone.solve(Av, Gv, c, b, h)
        finally:
            cone.close()
        for q, i in enumerate(idx):
            for j in range(2):
                st = int(out["status"][2 * q + j])
                self.computed[(blk, i, j)] = lib.CONE_STATUS.get(st, "?")
                if st in (0, 3):                                   # OPTIMAL / ALMOST_OPTIMAL
                    box[i, j] = (1.0 if j == 0 else -1.0) * out["pobj"][2 * q + j]
                elif st not in (5, 2):                             # DUAL_INFEASIBLE / NUMERICAL_ERROR keep the default
                    raise lib.ScpbError(f"Solver failed during variable scaling ({lib.CONE_STATUS.get(st, st)})")


def t_grid(N):
    """RealVector(LinRange(0, 1, N)) with Julia's lerpi arithmetic (scp.jl:147)."""
    j = np.arange(N, dtype=np.float64) / float(N - 1)
    return (1.0 - j) * 0.0 + j * 1.0


def trapz(f, grid):          # helper.jl:560-568
    F = Expr()
    for k in range(len(grid) - 1):
        d = grid[k + 1] - grid[k]
        F = F + (f[k + 1] + f[k]) * (0.5 * d)
    return F


class SourceMap:
    """Layout of the per-seed source vector (see include/scpb.h, scpb_ptr_desc)."""

    def __init__(self, N, nx, nu, np_, ns, nf, ng=None):
        M = N - 1
        ng = np_ if ng is None else ng       # packed columns of ds/dp per node (csrc/constraints.cuh)
        o = 1
        self.oA = o; o += M * nx * nx
        self.oBm = o; o += M * nx * nu
        self.oBp = o; o += M * nx * nu
        self.oF = o; o += M * nx * nf
        self.or_ = o; o += M * nx
        self.oE = o; o += M * nx * nx
        self.oC = o; o += N * ns * nx
        self.oD = o; o += N * ns * nu
        self.oG = o; o += N * ns * ng
        self.ors = o; o += N * ns
        self.oxh = o; o += N * nx
        self.ouh = o; o += N * nu
        self.oph = o; o += np_
        self.oeta = o; o += 1          # SCvx / GuSTO trust-region radius (scvx.jl:245, gusto.jl:229); unused by PTR
        self.olam = o; o += 1          # GuSTO: lambda, the soft-penalty weight (gusto.jl:228)
        self.nsrc = o
        self.N, self.nx, self.nu, self.np, self.ns, self.nf, self.ng = N, nx, nu, np_, ns, nf, ng

    def mat(self, off, k, rows, cols, colmajor=True, mask=None):
        blk = rows * cols
        M = [[None] * cols for _ in range(rows)]
        for i in range(rows):
            for j in range(cols):
                if mask is not None and not mask[i, j]:
                    continue
                e = (i + rows * j) if colmajor else (i * cols + j)
                M[i][j] = Lin.src(off + k * blk + e)
        return M

    def vec(self, off, k, n):
        return [Lin.src(off + k * n + i) for i in range(n)]


class SCPProblem:
    """pbm returned by create(): template, device objects, scaling."""

    def __init__(self, pars, traj, handle, l1_block=4, algo="ptr"):
        self.pars, self.traj, self.handle = pars, traj, handle
        self.l1_block = l1_block
        self.algo = algo
        self.t = t_grid(pars.N)
        traj.scp = pars
        if pars.disc_method not in (FOH, IMPULSE):
            raise lib.ScpbError(f"unknown discretization method {pars.disc_method}")
        if pars.disc_method == IMPULSE and algo != "ptr":
            raise lib.ScpbError(f"IMPULSE discretization is implemented for PTR only, not for {algo}")
        if pars.disc_method == IMPULSE and traj.model_id not in IMPULSE_MODELS:
            raise lib.ScpbError(f"IMPULSE discretization needs a model pack with impulse semantics (model {traj.model_id} "
                                "has none)")
        if getattr(traj, "hom", None) is not None and algo != "ptr":
            raise lib.ScpbError(f"an in-loop homotopy schedule is implemented for PTR only, not for {algo}")
        self.scale = SCPScaling(traj, handle, self.t)
        self._build()

    # ------------------------------------------------------------------ template (ptr.jl:213-293, 565-895)
    def _build(self):
        pars, traj, sc, t = self.pars, self.traj, self.scale, self.t
        N, nx, nu, np_ = pars.N, traj.nx, traj.nu, traj.np
        ns, nf = traj.ns, len(traj.fcols)
        gcols = traj.gcols if getattr(traj, "gcols", None) else (lambda k: list(range(np_)))
        ng = len(gcols(0)) if ns else np_
        sm = SourceMap(N, nx, nu, np_, ns, nf, ng)
        traj.ocp = None
        self.sm = sm
        prg = ConicTemplate(sm.nsrc, l1_block=self.l1_block)
        x = prg.new_variable((nx, N), "x", sc.Sx, sc.cx, stage="col")
        u = prg.new_variable((nu, N), "u", sc.Su, sc.cu, stage="col")
        p = prg.new_variable(np_, "p", sc.Sp, sc.cp, stage=(traj.p_stage(N) if traj.p_stage else None))
        vd = prg.new_variable((nx, N - 1), "vd", stage="col")
        scvx = self.algo == "scvx"
        if not scvx:            # PTR: the trust-region radii are variables (ptr.jl:246-249); SCvx: eta is data
            eta_x = prg.new_variable(N, "eta_x", stage="idx")
            eta_u = prg.new_variable(N, "eta_u", stage="idx")
            eta_p = prg.new_variable(1, "eta_p", stage=None)
        else:                   # scvx.jl:263-264: the penalty epigraph variables are created with the subproblem
            P = prg.new_variable(N, "P", stage="idx")
            Pf = prg.new_variable(2, "Pf", stage=None)
        # add_dynamics! / state_update! (discretization.jl:424-497).  IMPULSE (:469-494): one input block, no u_{k+1}
        # term; u_N stays a variable of the cost, U and the trust region
        from .problem import dltv_masks
        mA, mB, mE = dltv_masks(traj)
        impulse = pars.disc_method == IMPULSE
        for k in range(N - 1):
            A = sm.mat(sm.oA, k, nx, nx, mask=mA)
            Bm = sm.mat(sm.oBm, k, nx, nu, mask=mB)
            E = sm.mat(sm.oE, k, nx, nx, mask=mE)
            r = sm.vec(sm.or_, k, nx)
            Fp = sm.mat(sm.oF, k, nx, nf)
            if impulse:
                rhs = [a + b + d for a, b, d in zip(matvec(A, x[:, k]), matvec(Bm, u[:, k]), matvec(E, vd[:, k]))]
            else:
                Bp = sm.mat(sm.oBp, k, nx, nu, mask=mB)
                rhs = [a + b + c + d for a, b, c, d in zip(matvec(A, x[:, k]), matvec(Bm, u[:, k]),
                                                           matvec(Bp, u[:, k + 1]), matvec(E, vd[:, k]))]
            Fpv = matvec(Fp, [p[j] for j in traj.fcols])
            prg.zero([x[i, k + 1] - (rhs[i] + Fpv[i] + Expr(None, r[i])) for i in range(nx)], "dynamics")
        # convex state / input constraints (scp.jl:685-734)
        if traj.X is not None:
            for k in range(N):
                traj.X(prg, t[k], k + 1, x[:, k], p)
        if traj.U is not None:
            for k in range(N):
                traj.U(prg, t[k], k + 1, u[:, k], p)
        # nonconvex constraints (scp.jl:744-794)
        vs = None
        if ns:
            vs = prg.new_variable((ns, N), "vs", stage="col")
            for k in range(N):
                Cm, Dm, Gm = traj.s_struct(t[k], k + 1)
                Cs = sm.mat(sm.oC, k, ns, nx, colmajor=False, mask=Cm)
                Ds = sm.mat(sm.oD, k, ns, nu, colmajor=False, mask=Dm)
                Gs = sm.mat(sm.oG, k, ns, ng, colmajor=False, mask=Gm)
                rs = sm.vec(sm.ors, k, ns)
                lhs = [a + b + c for a, b, c in zip(matvec(Cs, x[:, k]), matvec(Ds, u[:, k]),
                                                    matvec(Gs, [p[j] for j in gcols(k)]))]
                prg.nonpos([lhs[i] + Expr(None, rs[i]) - vs[i, k] for i in range(ns)], "path_ncvx")
        # boundary conditions, relaxed (scp.jl:808-895); affine g => exact linearisation
        vic = vtc = None
        g_ic, g_tc = [], []
        if traj.gic is not None:
            g_ic = g = traj.gic(x[:, 0], p)
            vic = prg.new_variable(len(g), "vic", stage=0)
            prg.zero([g[i] + vic[i] for i in range(len(g))], "initial_condition")
        if traj.gtc is not None:
            g_tc = g = traj.gtc(x[:, N - 1], p)
            vtc = prg.new_variable(len(g), "vtc", stage=N - 1)
            prg.zero([g[i] + vtc[i] for i in range(len(g))], "terminal_condition")
        # trust region (ptr.jl:565-743)
        q = pars.q_tr
        cone = {1: prg.l1, 2: prg.soc, 4: prg.soc, np.inf: prg.linf}[q]

        def bound(d_lq, eta, name, stage):
            """d_lq <= eta, or for q_tr = 4 the squared two-norm trust region d_lq^2 <= eta (ptr.jl:604-630): |d_lq| <= w
            (a two-entry SOC) and geomean(eta, 1) >= w (GEOM)."""
            if q == 4:
                w = prg.new_variable(1, f"w_{name}_{prg.nvar}", stage=stage)
                prg.soc([w[0], d_lq], name)
                prg.geom([w[0], eta, 1.0], name)
            else:
                prg.nonpos([d_lq - eta])

        dp_lq = prg.new_variable(1, "dp_lq", stage=None)
        ph_ref = sm.vec(sm.oph, 0, np_)
        cone([dp_lq[0]] + [(p[i] - sc.cp[i]) * (1.0 / sc.Sp[i]) - Expr(None, ph_ref[i]) for i in range(np_)],
             "parameter_trust_region")
        if not scvx:
            bound(dp_lq[0], eta_p[0], "parameter_trust_region", None)
        dx_lq = prg.new_variable(N, "dx_lq", stage="idx")
        for k in range(N):
            xr = sm.vec(sm.oxh, k, nx)
            cone([dx_lq[k]] + [(x[i, k] - sc.cx[i]) * (1.0 / sc.Sx[i]) - Expr(None, xr[i]) for i in range(nx)],
                 "state_trust_region")
            if not scvx:
                bound(dx_lq[k], eta_x[k], "state_trust_region", k)
        du_lq = prg.new_variable(N, "du_lq", stage="idx")
        for k in range(N):
            ur = sm.vec(sm.ouh, k, nu)
            cone([du_lq[k]] + [(u[i, k] - sc.cu[i]) * (1.0 / sc.Su[i]) - Expr(None, ur[i]) for i in range(nu)],
                 "input_trust_region")
            if not scvx:
                bound(du_lq[k], eta_u[k], "input_trust_region", k)
        if scvx:                # trust_region_bound (scvx.jl:649-674): dx_lq[k] + du_lq[k] + dp_lq <= eta
            eta_src = Expr(None, Lin.src(sm.oeta))
            for k in range(N):
                if q == 4:      # scvx.jl:646-662: |(dx_lq, du_lq, dp_lq)|_2 <= w (SOC), geomean(eta, 1) >= w (GEOM)
                    w = prg.new_variable(1, f"w_tr_{k}", stage=k)
                    prg.soc([w[0], dx_lq[k], du_lq[k], dp_lq[0]], "trust_region_bound")
                    prg.geom([w[0], eta_src, 1.0], "trust_region_bound")
                else:
                    prg.nonpos([dx_lq[k] + du_lq[k] + dp_lq[0] - eta_src], "trust_region_bound")
        # cost (ptr.jl:753-895, scp.jl:552-601)
        J = Expr()
        traj.ocp = prg          # a convex (non-affine) running cost adds its epigraph to the program (parser.sumsq)
        if traj.phi is not None:
            J = J + traj.phi(x[:, N - 1], p)
        if traj.Gamma is not None:
            J = J + trapz([traj.Gamma(t[k], k + 1, x[:, k], u[:, k], p) for k in range(N)], t)
        traj.ocp = None
        prg.add_cost(J)
        self.J_orig, self.g_ic, self.g_tc = J, list(g_ic), list(g_tc)     # rows re-evaluated by SCvx (nonlinear cost)
        if not scvx:
            prg.add_cost((trapz(list(eta_x), t) + trapz(list(eta_u), t) + eta_p[0]) * pars.wtr)
        if not scvx:
            P = prg.new_variable(N, "P", stage="idx")
            Pf = prg.new_variable(2, "Pf", stage=None)
        for k in range(N):
            if k < N - 1:
                E = sm.mat(sm.oE, k, nx, nx, mask=mE)
                Ev = matvec(E, vd[:, k])
                prg.l1([P[k]] + list(Ev) + (list(vs[:, k]) if vs is not None else []), "vd_vs_penalty", stage=k)
            elif vs is not None:
                prg.l1([P[k]] + list(vs[:, k]), "vd_vs_penalty", stage=k)
            else:
                prg.zero([P[k]])
        if vic is not None:
            prg.l1([Pf[0]] + list(vic), "vic_penalty", stage=0)
        else:
            prg.zero([Pf[0]])
        if vtc is not None:
            prg.l1([Pf[1]] + list(vtc), "vtc_penalty", stage=N - 1)
        else:
            prg.zero([Pf[1]])
        prg.add_cost((trapz(list(P), t) + Pf[0] + Pf[1]) * (pars.lam if scvx else pars.wvc))
        self._finish(prg)

    def _finish(self, prg):
        """compile the template, order the KKT system stage-wise, create the device objects"""
        pars, traj, sc, sm = self.pars, self.traj, self.scale, self.sm
        N, nx, nu, np_ = pars.N, traj.nx, traj.nu, traj.np
        ns, nf, ng = sm.ns, sm.nf, sm.ng
        self.template = prg
        self.cp = cp = prg.compile()
        # one extra W row for the cost constant c0
        import scipy.sparse as sp
        c0 = cp["cost_const"]
        row = sp.csr_matrix((list(c0.t.values()), ([0] * len(c0.t), list(c0.t.keys()))), shape=(1, sm.nsrc))
        self.W = sp.vstack([cp["W"], row]).tocsr()
        self.W.sort_indices()
        self.nval = self.W.shape[0]
        # ---- device objects ----
        h = self.handle
        h.model_set(traj.model_id, model_parameters(traj), nx, nu, np_)
        self.perm = ordering.stage_order(cp["A"], cp["G"], cp["var_stage"], N)
        self.cone = lib.ConeProblem(h, cp["A"], cp["G"], cp["l"], cp["soc_dims"], perm=self.perm)
        d = lib.PtrDesc()
        d.N, d.Nsub, d.nx, d.nu, d.np, d.ns, d.nf = N, pars.Nsub, nx, nu, np_, ns, nf
        for k_ in ("nsrc", "oA", "oBm", "oBp", "oF", "or_", "oE", "oC", "oD", "oG", "ors", "oxh", "ouh", "oph"):
            setattr(d, k_, getattr(sm, k_))
        d.nval = self.nval
        d.ng = ng
        d.vx, d.vu, d.vp = prg.blocks["x"][0], prg.blocks["u"][0], prg.blocks["p"][0]
        d.q_exit = {np.inf: 0, 1: 1, 2: 2}[pars.q_exit]
        d.iter_max = pars.iter_max
        d.eps_abs, d.eps_rel, d.feas_tol = pars.eps_abs, pars.eps_rel, pars.feas_tol
        d.method = pars.disc_method
        self.desc = d
        scale = np.concatenate([sc.Sx, sc.Su, sc.Sp, sc.cx, sc.cu, sc.cp, 1.0 / sc.Sx])
        self._keep = [np.ascontiguousarray(self.W.indptr, dtype=np.int32),
                      np.ascontiguousarray(self.W.indices, dtype=np.int32),
                      np.ascontiguousarray(self.W.data, dtype=np.float64),
                      np.ascontiguousarray(scale, dtype=np.float64), np.ascontiguousarray(self.t)]
        ptr = C.c_void_p()
        k = self._keep
        rc = h.lib.scpb_ptr_setup(h.h, self.cone.c, C.cast(C.byref(d), C.c_void_p), k[0].ctypes.data_as(lib._ip),
                                  k[1].ctypes.data_as(lib._ip), k[2].ctypes.data_as(lib._dp),
                                  k[3].ctypes.data_as(lib._dp), k[4].ctypes.data_as(lib._dp), C.byref(ptr))
        h._check(rc, "scpb_ptr_setup")
        self.ptr = ptr

    def close(self):
        if getattr(self, "ptr", None) is not None and self.ptr.value:
            self.handle.lib.scpb_ptr_free(self.ptr)
            self.ptr = C.c_void_p()
        if getattr(self, "cone", None) is not None:
            self.cone.close()


@dataclass
class SCPBatchSolution:      # batched SCPSolution (scp.jl:105-119)
    status: list
    iterations: np.ndarray
    cost: np.ndarray
    td: np.ndarray
    xd: np.ndarray
    ud: np.ndarray
    p: np.ndarray
    deviation: np.ndarray
    feas: np.ndarray
    timing: dict
    raw_status: np.ndarray
    tc: np.ndarray = None       # continuous-time grid and state trajectory xc (B, res, nx): filled by propagate()
    xc: np.ndarray = None
    hom_index: np.ndarray = None    # in-loop homotopy schedule: final grid index per seed (B,),
    iter_max: np.ndarray = None     # effective iter_max per seed (B,; without a schedule the configured one),
    hom_history: dict = None        # {"index", "improv_rel"} (B, cap): per iteration the grid index the subproblem was
                                    # built with and its improv_rel (-1 / NaN after the seed's last iteration)


def create(pars: Parameters, traj, handle, l1_block=4) -> SCPProblem:
    """PTR.create (ptr.jl:148-195).  l1_block: see parser.ConicTemplate (0 reproduces the reference's exact
    NormOneBridge cone program; the default 4 is an equivalent, sparser lowering for the GPU factorisation)."""
    return SCPProblem(pars, traj, handle, l1_block=l1_block)


def set_parameters(pbm: SCPProblem, par=None):
    """Replace the model parameter block the device problem uses (scpb_ptr_set_par); None: the model's current block."""
    par, pp = lib._f64(model_parameters(pbm.traj) if par is None else par)
    pbm.handle._check(pbm.handle.lib.scpb_ptr_set_par(pbm.ptr, pp, par.size), "scpb_ptr_set_par")


def homotopy_history_length(pbm: SCPProblem):
    """the most iterations a seed can run under the problem's schedule: every update extends its iter_max by the
    iterations since the previous one, so iter_max + (n_grid - 1)(iter_max - 1)"""
    n, it = pbm.traj.hom["grid"].size, pbm.pars.iter_max
    return it + (n - 1) * max(it - 1, 0)


def set_homotopy(pbm: SCPProblem, B, beta=None):
    """Push the problem's in-loop homotopy schedule (problem_set_homotopy_update) and the per-seed thresholds of the next
    solve to the device (scpb_ptr_set_homotopy, scpb_ptr_set_homotopy_beta); a problem without one detaches it."""
    h, hom = pbm.handle, getattr(pbm.traj, "hom", None)
    if hom is None:
        if beta is not None:
            raise lib.ScpbError("beta is the update threshold of a homotopy schedule, and the problem has none "
                                "(problem_set_homotopy_update)")
        h._check(h.lib.scpb_ptr_set_homotopy(pbm.ptr, 0, 0, None, 0.0), "scpb_ptr_set_homotopy")
        return
    slot = -1 if hom["par_index"] is None else hom["par_index"]        # -1: the slot the pack reads its parameter from
    grid, pg = lib._f64(hom["grid"])
    h._check(h.lib.scpb_ptr_set_homotopy(pbm.ptr, int(slot), grid.size, pg, hom["worsen_tol"]), "scpb_ptr_set_homotopy")
    b = np.ascontiguousarray(np.broadcast_to(np.asarray(hom["beta"] if beta is None else beta, dtype=np.float64), (B,)))
    b, pb = lib._f64(b)
    h._check(h.lib.scpb_ptr_set_homotopy_beta(pbm.ptr, B, pb), "scpb_ptr_set_homotopy_beta")


def guess_arrays(pbm: SCPProblem, guesses):
    """guesses = (xd0 (B,N,nx), ud0 (B,N,nu), p0 (B,np)), an earlier batch solution (a warm start, solve(pbm, warm),
    scp.jl:532-539: its discrete trajectory is the initial guess) or None (the problem's own guess, one seed) ->
    contiguous float64 arrays"""
    traj, N = pbm.traj, pbm.pars.N
    if guesses is None:
        x0, u0, p0 = traj.guess(N)
        guesses = (x0[None], u0[None], p0[None])
    if hasattr(guesses, "xd") and hasattr(guesses, "ud"):
        guesses = (guesses.xd, guesses.ud, guesses.p)
    xd0, ud0, p0 = (np.ascontiguousarray(g, dtype=np.float64) for g in guesses)
    B = xd0.shape[0]
    assert xd0.shape == (B, N, traj.nx) and ud0.shape == (B, N, traj.nu) and p0.shape == (B, traj.np)
    return xd0, ud0, p0


def run_solve(pbm: SCPProblem, fn, guesses, cone_opts, n_extra=0, n_timing=8):
    """One call of the C solve fn (scpb_ptr_solve, scpb_scvx_solve or scpb_gusto_solve) on the guess arrays: the batch
    solution and the n_extra per-seed outputs that follow feas (SCvx: eta; GuSTO: eta, lambda).  The cone options are
    the reference's (nref = equil = -1, solver_opts["maxit"]) with the keyword arguments on top."""
    h, pars = pbm.handle, pbm.pars
    xd0, ud0, p0 = guesses
    B = xd0.shape[0]
    o = lib.ConeOpts()
    o.nref = -1
    o.equil = -1
    if pars.solver_opts and "maxit" in pars.solver_opts:
        o.maxit = int(pars.solver_opts["maxit"])
    for k_, v in cone_opts.items():
        setattr(o, k_, v)
    xd, ud, p = np.empty_like(xd0), np.empty_like(ud0), np.empty_like(p0)
    status = np.zeros(B, dtype=np.int32); iters = np.zeros(B, dtype=np.int32); feas = np.zeros(B, dtype=np.int32)
    J = np.empty(B); dev = np.empty(B); extras = [np.empty(B) for _ in range(n_extra)]; timing = np.zeros(n_timing)
    dp = lambda a: a.ctypes.data_as(lib._dp)
    ip = lambda a: a.ctypes.data_as(lib._ip)
    rc = fn(pbm.ptr, B, dp(xd0), dp(ud0), dp(p0), C.cast(C.byref(o), C.c_void_p), dp(xd), dp(ud), dp(p), ip(status),
            ip(iters), dp(J), dp(dev), ip(feas), *[dp(e) for e in extras], dp(timing))
    h._check(rc, fn.__name__)
    # scp.jl:221-222: anything but an unsafe solver status is reported solved
    names = ["SCP_SOLVED" if s_ in (0, 1) else f"SCP_FAILED ({lib.CONE_STATUS.get((int(s_) - 2) // 16, '?')})"
             for s_ in status]
    tm = dict(discretize=timing[0], formulate=timing[1], solve=timing[2], overhead=timing[3], total=timing[4],
              lockstep_iterations=int(timing[5]), ipm_iterations=int(timing[6]))
    if n_timing > 8:        # PTR: streamed chains and the initial discretize!
        tm.update(chunks=int(timing[7]), initial_discretize=timing[8])
    return SCPBatchSolution(names, iters, J, pbm.t, xd, ud, p, dev, feas, tm, status), extras


def solve(pbm: SCPProblem, guesses=None, beta=None, **cone_opts) -> SCPBatchSolution:
    """PTR.solve (ptr.jl:448-532) for a batch: guesses = (xd0 (B,N,nx), ud0 (B,N,nu), p0 (B,np));
    None => the problem's own guess (one seed).  The model's parameter block is read again here, as the reference's
    closures read the model at call time: a parameter changed between two solves (a homotopy step) takes effect
    without a new create.
    beta: update threshold of the problem's in-loop homotopy schedule, a scalar or one per seed (None: the one given to
    problem_set_homotopy_update), so a sweep over thresholds is one batch."""
    traj, pars, h = pbm.traj, pbm.pars, pbm.handle
    set_parameters(pbm)
    g = guess_arrays(pbm, guesses)
    B = g[0].shape[0]
    set_homotopy(pbm, B, beta)
    sol, _ = run_solve(pbm, h.lib.scpb_ptr_solve, g, cone_opts, n_timing=10)
    sol.iter_max = np.full(B, pars.iter_max, dtype=np.int32)
    if getattr(traj, "hom", None) is not None:
        cap = homotopy_history_length(pbm)
        sol.hom_index = np.zeros(B, dtype=np.int32)
        hidx, himp = np.zeros((B, cap), dtype=np.int32), np.zeros((B, cap))
        ip = lambda a: a.ctypes.data_as(lib._ip)
        rc = h.lib.scpb_ptr_homotopy_result(pbm.ptr, B, ip(sol.hom_index), ip(sol.iter_max), cap, ip(hidx),
                                            himp.ctypes.data_as(lib._dp))
        h._check(rc, "scpb_ptr_homotopy_result")
        sol.hom_history = {"index": hidx, "improv_rel": himp}
    return sol


def correct_convex(pbm: SCPProblem, guesses, **cone_opts):
    """correct_convex! (scp.jl:275-361) for a batch of guesses: the closest trajectory, in the scaled L1 sense, that
    satisfies the convex path constraints X and U at every node -- what GuSTO and SCvx apply to the initial guess
    (gusto.jl:517-526, scvx.jl:563).  One template (sources = the guess), one batched call of the GPU cone solver."""
    traj, pars, sc, h, t = pbm.traj, pbm.pars, pbm.scale, pbm.handle, pbm.t
    N, nx, nu, np_ = pars.N, traj.nx, traj.nu, traj.np
    xd0 = np.ascontiguousarray(guesses[0], dtype=np.float64)
    ud0 = np.ascontiguousarray(guesses[1], dtype=np.float64)
    p0 = np.ascontiguousarray(guesses[2], dtype=np.float64)
    B = xd0.shape[0]
    cc = getattr(pbm, "_cc", None)
    if cc is None:
        ox, ou, op = 1, 1 + N * nx, 1 + N * nx + N * nu
        prg = ConicTemplate(op + np_, l1_block=0)
        x = prg.new_variable((nx, N), "x", sc.Sx, sc.cx, stage="col")
        u = prg.new_variable((nu, N), "u", sc.Su, sc.cu, stage="col")
        p = prg.new_variable(np_, "p", sc.Sp, sc.cp, stage=(traj.p_stage(N) if traj.p_stage else None))
        for k in range(N):
            if traj.X is not None:
                traj.X(prg, t[k], k + 1, x[:, k], p)
            if traj.U is not None:
                traj.U(prg, t[k], k + 1, u[:, k], p)
        ex = prg.new_variable(N, "tau_x", stage="idx"); eu = prg.new_variable(N, "tau_u", stage="idx")
        ep = prg.new_variable(1, "tau_p", stage=None)
        for k in range(N):
            prg.l1([ex[k]] + [(x[i, k] - Expr(None, Lin.src(ox + k * nx + i))) * (1.0 / sc.Sx[i]) for i in range(nx)],
                   "x_variation", stage=k)
            prg.l1([eu[k]] + [(u[i, k] - Expr(None, Lin.src(ou + k * nu + i))) * (1.0 / sc.Su[i]) for i in range(nu)],
                   "u_variation", stage=k)
        prg.l1([ep[0]] + [(p[i] - Expr(None, Lin.src(op + i))) * (1.0 / sc.Sp[i]) for i in range(np_)], "p_variation", stage=-1)
        J = Expr()
        for k in range(N):
            J = J + ex[k] + eu[k]
        prg.add_cost(J + ep[0])
        cp = prg.compile()
        perm = ordering.stage_order(cp["A"], cp["G"], cp["var_stage"], N)
        cc = pbm._cc = dict(prg=prg, cp=cp, perm=perm)
    prg, cp = cc["prg"], cc["cp"]
    src = np.concatenate([np.ones((B, 1)), xd0.reshape(B, -1), ud0.reshape(B, -1), p0], axis=1)
    vals = np.asarray((cp["W"] @ src.T).T)
    n, p_, m, nA, nG = cp["n"], cp["p"], cp["m"], cp["nnzA"], cp["nnzG"]
    cone = lib.ConeProblem(h, cp["A"], cp["G"], cp["l"], cp["soc_dims"], perm=cc["perm"])
    try:
        out = cone.solve(vals[:, :nA], vals[:, nA:nA + nG], vals[:, cp["off_c"]:cp["off_c"] + n],
                         vals[:, cp["off_b"]:cp["off_b"] + p_], vals[:, cp["off_h"]:cp["off_h"] + m], **cone_opts)
    finally:
        cone.close()
    bad = [int(s_) for s_ in out["status"] if s_ not in (0, 3)]
    if bad:
        raise lib.ScpbError("Solver failed to find the closest initial guess that satisfies the convex constraints "
                            f"({lib.CONE_STATUS.get(bad[0], bad[0])})")
    z = out["x"]
    vx, vu, vp = prg.blocks["x"][0], prg.blocks["u"][0], prg.blocks["p"][0]
    xd = z[:, vx:vx + N * nx].reshape(B, N, nx) * sc.Sx + sc.cx
    ud = z[:, vu:vu + N * nu].reshape(B, N, nu) * sc.Su + sc.cu
    pp = z[:, vp:vp + np_] * sc.Sp + sc.cp
    return np.ascontiguousarray(xd), np.ascontiguousarray(ud), np.ascontiguousarray(pp)


def propagate(pbm: SCPProblem, sol: SCPBatchSolution, res=None) -> SCPBatchSolution:
    """The continuous-time part of SCPSolution (scp.jl:228-236): xc = propagate(last_sol, pbm; res = 2*Nsub*(N-1))
    (discretization.jl:515-562) for every seed of the batch, on the device.  The reference only propagates solved
    trajectories; here failed seeds are propagated as well (their xc is simply not meaningful)."""
    pars = pbm.pars
    res = int(res) if res is not None else 2 * pars.Nsub * (pars.N - 1)
    pbm.handle.model_set(pbm.traj.model_id, model_parameters(pbm.traj), pbm.traj.nx, pbm.traj.nu, pbm.traj.np)
    sol.tc, sol.xc, sec = pbm.handle.propagate(pbm.t, sol.xd, sol.ud, sol.p, res, method=pars.disc_method)
    sol.timing["propagate"] = sec
    return sol
