"""TrajectoryProblem -- host-side mirror of src/parser/problem.jl (struct :64-121, setters :241-659).

The reference stores Julia closures for the dynamics and constraints; a GPU kernel cannot call them, so
here the *dynamics* (f, A, B, F) and the *nonconvex constraints* (s, C, D, G) are selected as device
packs (csrc/models.cuh, csrc/constraints.cuh) by `problem_set_dynamics!` / `problem_set_s!`, while
everything that only shapes the cone program -- convex sets X / U, boundary conditions, cost, scaling
advice, the initial guess -- keeps the reference's closure style and is evaluated once, symbolically,
when the subproblem template is built (parser.py).
"""
from __future__ import annotations

import numpy as np


class TrajectoryProblem:
    def __init__(self, mdl=None):
        self.mdl = mdl
        self.nx = self.nu = self.np = 0
        self.xrg, self.urg, self.prg = [], [], []
        self.model_id = 0
        self.model_par = None
        self.fcols = [0]
        self.A_struct = None
        self.B_struct = None
        self.p_stage = None
        self.guess = None
        self.phi = None          # terminal cost  phi(x_expr, p_expr, pbm) -> Expr     (problem.jl:365-368)
        self.S = None            # GuSTO: input quadratic penalty S(t,k,p,pbm) of the running cost   (problem.jl:405)
        self.Gamma = None        # running cost   Gamma(t,k,x,u,p,pbm) -> Expr          (problem.jl:392-394)
        self.X = None            # X(t,k,x,p,pbm,ocp): emits cone rows into ocp        (problem.jl:487-523)
        self.U = None            # U(t,k,u,p,pbm,ocp)                                  (problem.jl:534-543)
        self.ns = 0
        self.s_struct = None     # (Cmask, Dmask, Gmask) structural non-zeros of the constraint pack
        self.gcols = None        # gcols(k) -> parameter indices of the pack's packed ds/dp columns at node k (None: all)
        self.ocp = None          # the program under construction while the cost closures run (see ptr.SCPProblem._build)
        self.gic = None          # affine boundary conditions g(x_expr, p_expr, pbm) -> list[Expr]
        self.gtc = None
        self.scp = None
        self.hom = None          # in-loop homotopy schedule (problem_set_homotopy_update)


def problem_set_dims(pbm, nx, nu, np_):
    """problem_set_dims! (problem.jl:241-249)"""
    pbm.nx, pbm.nu, pbm.np = nx, nu, np_
    pbm.xrg = [None] * nx
    pbm.urg = [None] * nu
    pbm.prg = [None] * np_


def problem_advise_scale(pbm, which, idx, rg):
    """problem_advise_scale! (problem.jl:262-282)"""
    if rg[1] < rg[0]:
        raise ValueError("min must be less than max")
    tgt = {"state": pbm.xrg, "input": pbm.urg, "parameter": pbm.prg}[which]
    for i in (idx if hasattr(idx, "__iter__") else [idx]):
        tgt[i] = (float(rg[0]), float(rg[1]))


def problem_set_guess(pbm, guess):
    """problem_set_guess! (problem.jl:316-319)"""
    pbm.guess = lambda N: guess(N, pbm)


def problem_set_terminal_cost(pbm, phi):
    pbm.phi = lambda x, p: phi(x, p, pbm)


def problem_set_running_cost(pbm, SGamma, algo="ptr"):
    """problem_set_running_cost! (problem.jl:390-418).  SCvx / PTR: the running cost Gamma(t, k, x, u, p, pbm).  GuSTO: the
    input quadratic penalty S(t, k, p, pbm) of the running cost u' S u (convex: constant in p); the input-affine and
    additive terms l and g of the GuSTO cost (problem.jl:395-400) are not mirrored."""
    if algo == "gusto":
        pbm.S = lambda t, k, p: SGamma(t, k, p, pbm)
    else:
        pbm.Gamma = lambda t, k, x, u, p: SGamma(t, k, x, u, p, pbm)


def problem_set_dynamics(pbm, model_id, par, fcols=(0,), A_struct=None, B_struct=None):
    """problem_set_dynamics! (problem.jl:425-450): selects the device pack that evaluates f, A, B, F.
    par: the pack's parameter block, or a callable returning it, evaluated at every solve and propagate (the reference's
    closures read the model when they are called, so a model parameter changed between two solves takes effect).
    fcols: parameter index of each active (time-dilation) column of F.
    A_struct / B_struct: optional structural non-zero patterns of df/dx (nx x nx) and df/du (nx x nu); the
    discrete-time blocks inherit the reachability closure (Phi = closure(I + A), B_k = Phi*B, E_k ~ Phi), which
    removes structurally zero coefficients from the dynamics rows of the subproblem."""
    pbm.model_id = int(model_id)
    pbm.model_par = par if callable(par) else np.asarray(par, dtype=np.float64)
    pbm.fcols = list(fcols)
    pbm.A_struct = None if A_struct is None else np.asarray(A_struct, bool)
    pbm.B_struct = None if B_struct is None else np.asarray(B_struct, bool)


def model_parameters(pbm):
    """the current parameter block of the device packs (problem_set_dynamics)"""
    return np.asarray(pbm.model_par() if callable(pbm.model_par) else pbm.model_par, dtype=np.float64)


def dltv_masks(pbm):
    """Structural patterns (A_k, B_k, E_k) implied by A_struct/B_struct; None = dense."""
    if getattr(pbm, "A_struct", None) is None:
        return None, None, None
    nx = pbm.nx
    R = np.eye(nx, dtype=bool) | pbm.A_struct
    for _ in range(nx):                       # transitive closure
        R = R | ((R.astype(int) @ R.astype(int)) > 0)
    Bm = None if pbm.B_struct is None else ((R.astype(int) @ pbm.B_struct.astype(int)) > 0)
    return R, Bm, R


def problem_set_X(pbm, X):
    pbm.X = lambda ocp, t, k, x, p: X(t, k, x, p, pbm, ocp)


def problem_set_U(pbm, U):
    pbm.U = lambda ocp, t, k, u, p: U(t, k, u, p, pbm, ocp)


def problem_set_s(pbm, ns, struct, gcols=None):
    """problem_set_s! (problem.jl:560-587): the constraint pack of the selected model evaluates s, C, D, G on the
    device; struct(t, k, pbm) -> (Cmask, Dmask, Gmask) gives their structural non-zeros at node k
    (row-major ns x nx / nu / np).  Node-dependent structure keeps e.g. phase-switch rows from coupling a
    parameter to every stage."""
    pbm.ns = int(ns)
    pbm.s_struct = lambda t, k: struct(t, k, pbm)
    pbm.gcols = gcols        # packed ds/dp: gcols(k) lists the parameters the pack's NG columns refer to at node k


def problem_advise_parameter_stage(pbm, stage_of):
    """GPU-specific ordering advice: stage_of(N) -> list (len np) with the time node a parameter is tied to, or
    -1 for a genuinely global parameter (used only for the elimination order of the KKT factorisation)."""
    pbm.p_stage = stage_of


def problem_set_homotopy_update(pbm, grid, beta, worsen_tol=-1e-3, par_index=None):
    """The declarative twin of a problem_set_callback! (problem.jl:645-659) that steps the constraint pack's homotopy
    parameter through `grid` inside one PTR solve, as test/examples/rendezvous_3d/definition.jl:96-151 does.  After the
    stopping rule of iteration `iter`, a seed updates when beta >= improv_rel >= worsen_tol and the grid is not
    exhausted: the parameter takes the next grid value, iter_max grows by iter - last_update, and a stop asked for in
    that iteration is cancelled.  Runs on the device, per seed (csrc/ptr.cu, k_ptr_step); every solve restarts each seed
    from grid[0] and the configured iter_max.
    beta: the default update threshold (ptr.solve(..., beta=...) overrides it per solve or per seed).
    par_index: the parameter slot the pack reads the homotopy parameter from (None: the pack's own; the device refuses
    any other slot).
    grid = None removes the schedule."""
    if grid is None:
        pbm.hom = None
        return
    grid = np.ascontiguousarray(grid, dtype=np.float64).ravel()
    if grid.size == 0 or not np.isfinite(grid).all():
        raise ValueError("the homotopy grid must be a non-empty list of finite values")
    pbm.hom = dict(grid=grid, beta=float(beta), worsen_tol=float(worsen_tol), par_index=par_index)


def problem_set_bc(pbm, kind, g):
    """problem_set_bc! (problem.jl:600-627) for affine boundary conditions g(x, p) = 0."""
    if kind == "ic":
        pbm.gic = lambda x, p: g(x, p, pbm)
    else:
        pbm.gtc = lambda x, p: g(x, p, pbm)
