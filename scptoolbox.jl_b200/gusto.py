"""GuSTO -- host-side mirror of src/solvers/gusto.jl for the GPU path (pen = :quad).

  Parameters           gusto.jl:58-85
  create(pars, traj)   gusto.jl:146-205 + the shared SCPProblem machinery (ptr.py)
  solve(pbm, guesses)  gusto.jl:425-502 for a BATCH of initial guesses in lock step on the GPU

Subproblem (Subproblem ctor gusto.jl:218-287; add_cost! :534-553; dynamics and boundary conditions UN-relaxed :452-454):
  * original cost (gusto.jl:570-677): terminal cost + trapezoid rule of the convex input quadratic u' S u;
  * state penalty (gusto.jl:725-867): every nonconvex path constraint s_i(x_k, p), linearised at the reference by the
    device constraint pack, enters through the quadratic soft penalty lambda max(0, .)^2 (soft_penalty :936-995:
    u >= 0, f_lin + u - v <= 0, cost lambda v^2);
  * soft trust region (gusto.jl:1056-1164): |x^_k - x^_ref,k|_q <= dx_lq[k], |p^ - p^_ref|_q <= dp_lq,
    dx_lq[k] + dp_lq - (eta + tr[k]) <= 0 and the same soft penalty on tr[k].
The quadratic terms reach the linear-objective cone solver as one rotated second-order cone per node and cost group,
q >= sum_i v_i^2 with the cost lambda q (JuMP lowers ECOS' quadratic objectives to the same cone; keeping lambda out of
the cone keeps its entries O(1): with sqrt(lambda) v inside, q reaches 1e4..1e6 in the first iterations and every such
cone sits at relative distance ~4/q from its boundary, which wrecks the Nesterov-Todd scaling).  lambda and eta are
PER-SEED device sources, so one compiled template serves every seed and every iteration.
The loop body on the device (csrc/ptr.cu, scpb_gusto_*): nonconvex costs J, J_st of the new iterate, the convexification
error rho (cost error + dynamics error, update_trust_region! :1245-1293), the trust-region / penalty update rule
(update_rule! :1310-1427 incl. the mu-shrink of :268) and the stopping rule (:1203-1231).

Not mirrored: convex state sets X through cone indicators (gusto.jl:871-900; none of the BASELINE GuSTO configs has X),
the softplus penalty (EXP cone), q_tr = 4, a parameter-dependent S."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import lib
from .parser import ConicTemplate, Expr, Lin, matvec
from .ptr import FOH, SCPBatchSolution, SCPProblem, SourceMap, guess_arrays, run_solve, trapz  # noqa: F401
from .scvx import _rows_matrix


@dataclass
class Parameters:            # gusto.jl:58-85
    N: int
    Nsub: int
    iter_max: int
    disc_method: int
    lam_init: float
    lam_max: float
    rho_0: float
    rho_1: float
    beta_sh: float
    beta_gr: float
    gamma_fail: float
    eta_init: float
    eta_lb: float
    eta_ub: float
    mu: float
    iter_mu: int
    eps_abs: float
    eps_rel: float
    feas_tol: float
    pen: str = "quad"
    hom: float = 100.0
    q_tr: float = np.inf
    q_exit: float = np.inf
    solver: object = None
    solver_opts: dict = None


class GuSTOProblem(SCPProblem):
    def __init__(self, pars, traj, handle, l1_block=4):
        if pars.pen != "quad":
            raise lib.ScpbError("GuSTO: only the quadratic soft penalty is implemented (pen = 'quad')")
        if pars.q_tr not in (1, 2, np.inf):
            raise lib.ScpbError("GuSTO: q_tr must be 1, 2 or Inf")
        if traj.X is not None:
            raise lib.ScpbError("GuSTO: convex state sets (X) through cone indicators are not implemented")
        super().__init__(pars, traj, handle, l1_block=l1_block, algo="gusto")

    # ------------------------------------------------------------------ template (gusto.jl:218-287, 534-1190)
    def _build(self):
        pars, traj, sc, t = self.pars, self.traj, self.scale, self.t
        N, nx, nu, np_ = pars.N, traj.nx, traj.nu, traj.np
        ns, nf = traj.ns, len(traj.fcols)
        gcols = traj.gcols if getattr(traj, "gcols", None) else (lambda k: list(range(np_)))
        ng = len(gcols(0)) if ns else np_
        sm = SourceMap(N, nx, nu, np_, ns, nf, ng)
        self.sm = sm
        prg = ConicTemplate(sm.nsrc, l1_block=self.l1_block)
        x = prg.new_variable((nx, N), "x", sc.Sx, sc.cx, stage="col")
        u = prg.new_variable((nu, N), "u", sc.Su, sc.cu, stage="col")
        p = prg.new_variable(np_, "p", sc.Sp, sc.cp, stage=(traj.p_stage(N) if traj.p_stage else None))
        lam = Lin.src(sm.olam)                   # lambda, per seed
        eta = Expr(None, Lin.src(sm.oeta))       # trust-region radius, per seed
        # ---- original cost: terminal + trapz of u' S u (S constant, PSD) ----
        S = np.asarray(traj.S(t[0], 1, None), dtype=float)
        self.S = S
        w, V = np.linalg.eigh(S)
        L_run = []
        for k in range(N):
            rows = []
            for i in range(nu):
                if w[i] > 1e-14:
                    e = Expr()
                    for j in range(nu):
                        if V[j, i] != 0.0:
                            e = e + u[j, k] * float(np.sqrt(w[i]) * V[j, i])
                    rows.append(e)
            L_run.append(prg.sumsq(rows, "run_cost", stage=k) if rows else Expr())
        L = trapz(L_run, t)
        traj.ocp = prg
        if traj.phi is not None:
            L = L + traj.phi(x[:, N - 1], p)
        traj.ocp = None
        # ---- state penalty: linearised nonconvex constraints, quadratic soft penalty ----
        L_st_nodes = []
        for k in range(N):
            vs = []
            if ns:
                Cm, Dm, Gm = traj.s_struct(t[k], k + 1)
                Cs = sm.mat(sm.oC, k, ns, nx, colmajor=False, mask=Cm)
                Gs = sm.mat(sm.oG, k, ns, ng, colmajor=False, mask=Gm)
                rs = sm.vec(sm.ors, k, ns)
                lhs = [a + b for a, b in zip(matvec(Cs, x[:, k]), matvec(Gs, [p[j] for j in gcols(k)]))]
                uu = prg.new_variable(ns, f"su{k}", stage=k)
                vv = prg.new_variable(ns, f"sv{k}", stage=k)
                for i in range(ns):
                    prg.nonpos([-uu[i]])
                    prg.nonpos([lhs[i] + Expr(None, rs[i]) + uu[i] - vv[i]], "soft_path")
                    vs.append(vv[i])
            L_st_nodes.append(prg.sumsq(vs, "state_penalty", stage=k) if vs else Expr())
        L_st = trapz(L_st_nodes, t).scale_lin(lam)
        # ---- soft trust region ----
        q = pars.q_tr
        cone = {1: prg.l1, 2: prg.soc, np.inf: prg.linf}[q]
        tr = prg.new_variable(N, "tr", stage="idx")
        dx_lq = prg.new_variable(N, "dx_lq", stage="idx")
        dp_lq = prg.new_variable(1, "dp_lq", stage=None)
        ph_ref = sm.vec(sm.oph, 0, np_)
        cone([dp_lq[0]] + [(p[i] - sc.cp[i]) * (1.0 / sc.Sp[i]) - Expr(None, ph_ref[i]) for i in range(np_)],
             "parameter_trust_region")
        tu = prg.new_variable(N, "tu", stage="idx")
        tv = prg.new_variable(N, "tv", stage="idx")
        L_tr_nodes = []
        for k in range(N):
            xr = sm.vec(sm.oxh, k, nx)
            cone([dx_lq[k]] + [(x[i, k] - sc.cx[i]) * (1.0 / sc.Sx[i]) - Expr(None, xr[i]) for i in range(nx)],
                 "state_trust_region")
            prg.nonpos([dx_lq[k] + dp_lq[0] - (tr[k] + eta)], "trust_region_bound")
            prg.nonpos([-tu[k]])
            prg.nonpos([tr[k] + tu[k] - tv[k]])
            L_tr_nodes.append(prg.sumsq([tv[k]], "trust_penalty", stage=k))
        L_tr1 = trapz(L_tr_nodes, t)               # L_tr / lambda
        L_tr = L_tr1.scale_lin(lam)
        prg.add_cost(L); prg.add_cost(L_st); prg.add_cost(L_tr)
        # ---- dynamics, un-relaxed ----
        from .problem import dltv_masks
        mA, mB, _ = dltv_masks(traj)
        for k in range(N - 1):
            A = sm.mat(sm.oA, k, nx, nx, mask=mA)
            Bm = sm.mat(sm.oBm, k, nx, nu, mask=mB)
            Bp = sm.mat(sm.oBp, k, nx, nu, mask=mB)
            r = sm.vec(sm.or_, k, nx)
            Fp = sm.mat(sm.oF, k, nx, nf)
            rhs = [a + b + c for a, b, c in zip(matvec(A, x[:, k]), matvec(Bm, u[:, k]), matvec(Bp, u[:, k + 1]))]
            Fpv = matvec(Fp, [p[j] for j in traj.fcols])
            prg.zero([x[i, k + 1] - (rhs[i] + Fpv[i] + Expr(None, r[i])) for i in range(nx)], "dynamics")
        # ---- convex input constraints (hard), boundary conditions (un-relaxed, affine) ----
        if traj.U is not None:
            for k in range(N):
                traj.U(prg, t[k], k + 1, u[:, k], p)
        if traj.gic is not None:
            prg.zero(list(traj.gic(x[:, 0], p)), "initial_condition")
        if traj.gtc is not None:
            prg.zero(list(traj.gtc(x[:, N - 1], p)), "terminal_condition")
        self.J_orig, self.g_ic, self.g_tc = L, [], []
        self._finish(prg)
        # ---- device loop data: J = affine row + weighted squares over (x, u, p); L_tr over the solver variables ----
        Lx = Expr.lift(L)
        aff_t, rows, wts = {}, [], []
        for v, coef in Lx.t.items():
            if v in prg.sq_log:                      # epigraph variable q of a sumsq: J takes the squares themselves
                if not set(coef.t) <= {0}:
                    raise lib.ScpbError("GuSTO: the original cost must not depend on device sources")
                for r in prg.sq_log[v]:
                    rows.append(r); wts.append(coef.t.get(0, 0.0))
            else:
                aff_t[v] = coef
        qrows = [Expr(aff_t, Lx.c)] + rows + [Expr.lift(L_tr1)]
        self.Q = _rows_matrix(qrows, self.cp["n"])
        self.Q_w = np.ascontiguousarray(wts if wts else [0.0], dtype=np.float64)
        d = lib.GustoDesc()
        for k_ in ("lam_init", "lam_max", "rho_0", "rho_1", "beta_sh", "beta_gr", "gamma_fail", "eta_init", "eta_lb",
                   "eta_ub", "mu"):
            setattr(d, k_, float(getattr(pars, k_)))
        d.iter_mu = int(pars.iter_mu)
        d.q_tr = {np.inf: 0, 1: 1, 2: 2}[pars.q_tr]
        d.oeta, d.olam, d.nsq = sm.oeta, sm.olam, len(rows)
        self.gdesc = d
        qm = self.Q
        h = self.handle
        rc = h.lib.scpb_gusto_attach(self.ptr, C.cast(C.byref(d), C.c_void_p), qm[0].ctypes.data_as(lib._ip),
                                     qm[1].ctypes.data_as(lib._ip), qm[2].ctypes.data_as(lib._dp),
                                     qm[3].ctypes.data_as(lib._dp), self.Q_w.ctypes.data_as(lib._dp))
        h._check(rc, "scpb_gusto_attach")


def create(pars: Parameters, traj, handle, l1_block=4) -> GuSTOProblem:
    """GuSTO.create (gusto.jl:146-205)."""
    return GuSTOProblem(pars, traj, handle, l1_block=l1_block)


def solve(pbm: GuSTOProblem, guesses=None, project_guess=True, **cone_opts) -> SCPBatchSolution:
    """GuSTO.solve (gusto.jl:425-502) for a batch: guesses = (xd0 (B,N,nx), ud0 (B,N,nu), p0 (B,np)).  As in
    generate_initial_guess (gusto.jl:517-526) the guesses are first projected onto the convex path constraints
    (correct_convex!, scp.jl:275-361) -- one batched call of the GPU cone solver."""
    from .ptr import correct_convex
    if hasattr(guesses, "xd") and hasattr(guesses, "ud"):      # a warm start from an earlier batch solution
        project_guess = False                                   # gusto.jl:434-438: is not re-projected
    g = guess_arrays(pbm, guesses)
    if project_guess:
        g = correct_convex(pbm, g)
    sol, (eta, lam) = run_solve(pbm, pbm.handle.lib.scpb_gusto_solve, g, cone_opts, n_extra=2)
    sol.eta, sol.lam = eta, lam
    return sol
