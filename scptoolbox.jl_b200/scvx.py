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
from .ptr import FOH, SCPBatchSolution, SCPProblem, guess_arrays, run_solve  # noqa: F401


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
    sol, (eta,) = run_solve(pbm, pbm.handle.lib.scpb_scvx_solve, guess_arrays(pbm, guesses), cone_opts, n_extra=1)
    sol.eta = eta
    return sol
