"""SCvx -- host-side mirror of src/solvers/scvx.jl for the GPU path.

  Parameters           scvx.jl:57-81
  create(pars, traj)   scvx.jl:160-205 + the shared SCPProblem machinery (ptr.py)
  solve(pbm, guesses)  scvx.jl:460-546 for a BATCH of initial guesses in lock step on the GPU

The subproblem template is the PTR one with the SCvx differences (ptr.py, `algo == "scvx"`): no trust-region
variables -- the radius eta is per-seed data on the device (a template source) --, the trust-region bound
dx_lq[k] + du_lq[k] + dp_lq <= eta (scvx.jl:649-674), penalty weight lambda (scvx.jl:804-901).  The loop body adds
what PTR does not need: the NONLINEAR augmented cost J = L + lambda (trapz(|defect|_1 + |s^+|_1) + |g_ic|_1 + |g_tc|_1)
of every candidate (actual_cost_penalty!, scvx.jl:919-951), the ratio test and the accept / reject / radius rule
(update_trust_region! / update_rule, scvx.jl:745-770, 1000-1045).  The rows that J needs besides the device packs --
original cost and affine boundary conditions -- are compiled from the same closures into a small sparse matrix Q.
Not mirrored: correct_convex! of the initial guess (scvx.jl:563): guesses are used as they are.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import scipy.sparse as sp

from . import lib
from .ptr import FOH, SCPBatchSolution, SCPProblem  # noqa: F401


@dataclass
class Parameters:            # scvx.jl:57-81
    N: int
    Nsub: int
    iter_max: int
    disc_method: int
    lam: float
    rho_0: float
    rho_1: float
    rho_2: float
    beta_sh: float
    beta_gr: float
    eta_init: float
    eta_lb: float
    eta_ub: float
    eps_abs: float
    eps_rel: float
    feas_tol: float
    q_tr: float
    q_exit: float
    solver: object = None
    solver_opts: dict = None
    wvc: float = 0.0             # unused (shared template code reads pars.lam for SCvx)
    wtr: float = 0.0


def _rows_matrix(exprs, nvar):
    """Affine expressions with constant coefficients -> (CSR over the solver variables, constants)."""
    rp, ci, v, c0 = [0], [], [], []
    for e in exprs:
        for k in sorted(e.t):
            lin = e.t[k]
            if not set(lin.t) <= {0}:
                raise lib.ScpbError("SCvx: original cost / boundary conditions must not depend on device sources")
            w = lin.t.get(0, 0.0)
            if w != 0.0:
                ci.append(k); v.append(w)
        if not set(e.c.t) <= {0}:
            raise lib.ScpbError("SCvx: original cost / boundary conditions must not depend on device sources")
        c0.append(e.c.t.get(0, 0.0))
        rp.append(len(ci))
    return (np.array(rp, dtype=np.int32), np.array(ci, dtype=np.int32), np.array(v, dtype=np.float64),
            np.array(c0, dtype=np.float64))


class SCvxProblem(SCPProblem):
    def __init__(self, pars, traj, handle, l1_block=4):
        super().__init__(pars, traj, handle, l1_block=l1_block, algo="scvx")
        from .parser import Expr
        rows = [Expr.lift(self.J_orig)] + [Expr.lift(g) for g in self.g_ic] + [Expr.lift(g) for g in self.g_tc]
        self.Q = _rows_matrix(rows, self.cp["n"])
        self.n_ic, self.n_tc = len(self.g_ic), len(self.g_tc)
        d = lib.ScvxDesc()
        for k_ in ("lam", "rho_0", "rho_1", "rho_2", "beta_sh", "beta_gr", "eta_init", "eta_lb", "eta_ub"):
            setattr(d, k_, float(getattr(pars, k_)))
        d.oeta, d.n_ic, d.n_tc = self.sm.oeta, self.n_ic, self.n_tc
        self.sdesc = d
        q = self.Q
        self._keepq = q
        h = handle
        rc = h.lib.scpb_scvx_attach(self.ptr, C.cast(C.byref(d), C.c_void_p), q[0].ctypes.data_as(lib._ip),
                                    q[1].ctypes.data_as(lib._ip), q[2].ctypes.data_as(lib._dp),
                                    q[3].ctypes.data_as(lib._dp))
        h._check(rc, "scpb_scvx_attach")


def create(pars: Parameters, traj, handle, l1_block=4) -> SCvxProblem:
    """SCvx.create (scvx.jl:160-205)."""
    return SCvxProblem(pars, traj, handle, l1_block=l1_block)


def solve(pbm: SCvxProblem, guesses=None, **cone_opts) -> SCPBatchSolution:
    """SCvx.solve (scvx.jl:460-546) for a batch: guesses = (xd0 (B,N,nx), ud0 (B,N,nu), p0 (B,np))."""
    traj, pars, h = pbm.traj, pbm.pars, pbm.handle
    if guesses is None:
        x0, u0, p0 = traj.guess(pars.N)
        guesses = (x0[None], u0[None], p0[None])
    if hasattr(guesses, "xd") and hasattr(guesses, "ud"):      # warm start from an earlier batch solution (solve(pbm, warm),
        guesses = (guesses.xd, guesses.ud, guesses.p)           # scp.jl:532-539: its discrete trajectory is the initial guess)
    xd0 = np.ascontiguousarray(guesses[0], dtype=np.float64)
    ud0 = np.ascontiguousarray(guesses[1], dtype=np.float64)
    p0 = np.ascontiguousarray(guesses[2], dtype=np.float64)
    B, N = xd0.shape[0], pars.N
    assert xd0.shape == (B, N, traj.nx) and ud0.shape == (B, N, traj.nu) and p0.shape == (B, traj.np)
    o = lib.ConeOpts()
    o.nref = -1
    o.equil = -1
    if pars.solver_opts and "maxit" in pars.solver_opts:
        o.maxit = int(pars.solver_opts["maxit"])
    for k_, v in cone_opts.items():
        setattr(o, k_, v)
    xd, ud, p = np.empty_like(xd0), np.empty_like(ud0), np.empty_like(p0)
    status = np.zeros(B, dtype=np.int32); iters = np.zeros(B, dtype=np.int32); feas = np.zeros(B, dtype=np.int32)
    J = np.empty(B); dev = np.empty(B); eta = np.empty(B); timing = np.zeros(8)
    dp = lambda a: a.ctypes.data_as(lib._dp)
    ip = lambda a: a.ctypes.data_as(lib._ip)
    rc = h.lib.scpb_scvx_solve(pbm.ptr, B, dp(xd0), dp(ud0), dp(p0), C.cast(C.byref(o), C.c_void_p), dp(xd), dp(ud),
                               dp(p), ip(status), ip(iters), dp(J), dp(dev), ip(feas), dp(eta), dp(timing))
    h._check(rc, "scpb_scvx_solve")
    names = []
    for s_ in status:
        if s_ in (0, 1):
            names.append("SCP_SOLVED")
        else:
            names.append(f"SCP_FAILED ({lib.CONE_STATUS.get((int(s_) - 2) // 16, '?')})")
    tm = dict(discretize=timing[0], formulate=timing[1], solve=timing[2], overhead=timing[3], total=timing[4],
              lockstep_iterations=int(timing[5]), ipm_iterations=int(timing[6]))
    sol = SCPBatchSolution(names, iters, J, pbm.t, xd, ud, p, dev, feas, tm, status)
    sol.eta = eta
    return sol
