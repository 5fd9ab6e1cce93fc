"""Forced harmonic oscillator with an input deadband, on the GPU API (PTR, FOH discretization, fixed final time).

Model and trajectory data: test/examples/oscillator/parameters.jl:69-115; problem definition:
test/examples/oscillator/definition.jl (dims :37-45, scaling advice :47-69, guess :71-114, cost :116-142, dynamics
:161-236, convex sets :238-368, deadband :370-444, initial condition :446-473); solve: tests.jl:22-80.

State x = [r v], input u = [aa ar l1aa l1adiff] (applied and reference acceleration, |aa| and |aa - ar|), parameter
p = [l1r_1 .. l1r_N] (one slack l1r_k >= |r_k| per node, read by the running cost at its own node only).  The horizon
tf = 10 s is fixed: the dynamics do not read p, F = 0 and the problem has no time-dilation column (fcols = ()).  The
deadband constraint aa = OR(ar) ar is a smooth OR whose sharpness kappa is stepped through a homotopy; each step is
warm-started from the previous solution (homotopy_sweep), or stepped inside one solve by the in-loop schedule
(homotopy_schedule)."""
from __future__ import annotations

import numpy as np

from .. import lib, ptr
from ..homotopy import Homotopy
from ..problem import (TrajectoryProblem, problem_advise_parameter_stage, problem_advise_scale, problem_set_bc,
                       problem_set_dims, problem_set_dynamics, problem_set_guess, problem_set_homotopy_update,
                       problem_set_running_cost, problem_set_s, problem_set_U, problem_set_X)

ID_R, ID_V = 0, 1
ID_AA, ID_AR, ID_L1AA, ID_L1ADIFF = 0, 1, 2, 3


class OscillatorProblem:
    """parameters.jl:69-115"""

    def __init__(self, N=30):
        self.N = N
        self.zeta, self.omega0 = 0.5, 1.0      # damping ratio, natural frequency [rad/s]
        self.a_db, self.a_max = 0.05, 0.3      # deadband and maximum acceleration [m/s^2]
        self.r0, self.v0 = 1.0, 0.0            # initial position [m] and velocity [m/s]
        self.tf = 10.0                         # trajectory duration [s]
        self.kappa = float("nan")              # sigmoid sharpness kappa1, set by the homotopy before every solve
        self.alpha, self.gamma = 0.06, 1e-1    # control usage weight, weight of the deadband relaxation

    def par(self):
        """device parameter block: zeta, omega0, tf (dynamics pack, csrc/models.cuh), then a_db, a_max, kappa (constraint
        pack, csrc/constraints.cuh)"""
        return np.array([self.zeta, self.omega0, self.tf, self.a_db, self.a_max, self.kappa])

    def dynamics(self, x, u):
        """f(t, k >= 0, x, u, p) (definition.jl:161-192)"""
        f = np.zeros(2)
        f[ID_V] = u[ID_AA]
        f[ID_R] = x[ID_V]
        f[ID_V] += -self.omega0 ** 2 * x[ID_R] - 2 * self.zeta * self.omega0 * x[ID_V]
        return f * self.tf


def _rk4(f, x0, tspan):
    """rk4_generic(f, x0; tspan, full = true) (src/utils/helper.jl:411-424, 451-501)"""
    X = np.zeros((len(tspan), len(x0)))
    X[0] = x0
    for k in range(1, len(tspan)):
        t, x = tspan[k - 1], X[k - 1]
        h = tspan[k] - t
        k1 = f(t, x)
        k2 = f(t + h / 2, x + h / 2 * k1)
        k3 = f(t + h / 2, x + h / 2 * k2)
        k4 = f(t + h, x + h * k3)
        X[k] = x + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
    return X


def _linterp(t, F, grid):
    """linterp(t, f_cps, t_grid) (src/utils/helper.jl:107-118); F[k] is the value at grid[k]"""
    t = max(grid[0], min(grid[-1], t))
    k = max(int(np.sum(t > grid)), 1)
    c = (grid[k] - t) / (grid[k] - grid[k - 1])
    return c * F[k - 1] + (1 - c) * F[k]


def define_problem(pbm: TrajectoryProblem, algo: str = "ptr"):
    mdl = pbm.mdl
    N = mdl.N
    problem_set_dims(pbm, 2, 4, N)

    # scaling advice (definition.jl:47-69)
    problem_advise_scale(pbm, "state", ID_R, (-mdl.r0, mdl.r0))
    problem_advise_scale(pbm, "state", ID_V, (-mdl.v0, mdl.v0))
    problem_advise_scale(pbm, "input", ID_AA, (-mdl.a_max, mdl.a_max))
    problem_advise_scale(pbm, "input", ID_AR, (-mdl.a_max, mdl.a_max))
    problem_advise_scale(pbm, "input", ID_L1AA, (0.0, mdl.a_max))
    problem_advise_scale(pbm, "input", ID_L1ADIFF, (0.0, 2 * mdl.a_max))
    problem_advise_scale(pbm, "parameter", range(N), (0.0, mdl.r0))
    # l1r_k appears at node k only (cost, X): a stage-k variable keeps it out of the dense border of the KKT ordering
    problem_advise_parameter_stage(pbm, lambda N_: list(range(N_)))

    def guess(N_, pbm_):        # definition.jl:71-114: the uncontrolled RK4 roll-out, sampled linearly at the nodes
        m_ = pbm_.mdl
        t_grid, tau = ptr.t_grid(1000), ptr.t_grid(N_)
        X = _rk4(lambda t, x: m_.dynamics(x, np.zeros(4)), np.array([m_.r0, m_.v0]), t_grid)
        x = np.array([_linterp(tau[k], X, t_grid) for k in range(N_)])
        return x, np.zeros((N_, 4)), np.abs(x[:, ID_R])

    problem_set_guess(pbm, guess)

    def Gamma(t, k, x, u, p, pbm_):      # definition.jl:116-142; k is 1-based
        m_ = pbm_.mdl
        f = p[k - 1] / m_.r0
        f = f + u[ID_L1AA] * m_.alpha / m_.a_max
        return f + u[ID_L1ADIFF] * m_.gamma / m_.a_max

    problem_set_running_cost(pbm, Gamma, algo)

    # dynamics pack (definition.jl:161-236): fixed final time, no F column; the parameter block is read at every solve,
    # so a new kappa takes effect
    As = np.array([[False, True], [True, True]])
    Bs = np.zeros((2, 4), bool)
    Bs[ID_V, ID_AA] = True
    problem_set_dynamics(pbm, lib.MODEL_OSCILLATOR, lambda: pbm.mdl.par(), fcols=(), A_struct=As, B_struct=Bs)

    def X(t, k, x, p, pbm_, ocp):      # definition.jl:240-272: |r_k| <= l1r_k
        ocp.l1([p[k - 1], x[ID_R]], "abs_r")

    problem_set_X(pbm, X)

    def U(t, k, u, p, pbm_, ocp):      # definition.jl:274-365
        m_ = pbm_.mdl
        aa, ar, l1aa, l1adiff = u[ID_AA], u[ID_AR], u[ID_L1AA], u[ID_L1ADIFF]
        ocp.nonpos([aa - m_.a_max], "accel_bounds")
        ocp.nonpos([-m_.a_max - aa], "accel_bounds")
        ocp.nonpos([ar - m_.a_max], "accel_bounds")
        ocp.nonpos([-m_.a_max - ar], "accel_bounds")
        ocp.l1([l1aa, aa], "accel_bounds")
        ocp.l1([l1adiff, aa - ar], "accel_bounds")

    problem_set_U(pbm, U)

    def s_struct(t, k, pbm_):          # deadband (definition.jl:370-444): D is +-1 on aa and -+dOR/dar on ar only
        Cm = np.zeros((2, 2), bool); Dm = np.zeros((2, 4), bool); Gm = np.zeros((2, 1), bool)
        Dm[:, [ID_AA, ID_AR]] = True
        return Cm, Dm, Gm

    problem_set_s(pbm, 2, s_struct, gcols=lambda k: [k])    # the pack's one ds/dp column is the node's own (zero) slack

    def gic(x, p, pbm_):               # definition.jl:446-473
        m_ = pbm_.mdl
        return [x[ID_R] - m_.r0, x[ID_V] - m_.v0]

    problem_set_bc(pbm, "ic", gic)


def ptr_parameters(N=30, Nsub=10, iter_max=10, solver_opts=None):
    """the reference's PTR configuration (tests.jl:24-58): FOH, q_tr = q_exit = Inf, every subproblem an LP"""
    return ptr.Parameters(N=N, Nsub=Nsub, iter_max=iter_max, disc_method=ptr.FOH, wvc=1e2, wtr=1e-3,
                          eps_abs=-np.inf, eps_rel=1e-3 / 100, feas_tol=5e-3, q_tr=np.inf, q_exit=np.inf,
                          solver_opts=solver_opts or {"verbose": 0})


def homotopy_sweep(pbm, guesses=None, n_hom=10, hom=None, **cone_opts):
    """tests.jl:60-80 for a batch: kappa = hom(LinRange(0, 1, n_hom)[i]) for every seed at step i (default
    Homotopy(1e-8)), each step warm-started from the previous step's batch solution (PTR.solve(pbm, warm)).
    guesses: (xd0, ud0, p0) batch or None (the problem's own guess).  Returns the list of batch solutions."""
    hom = hom or Homotopy(1e-8)
    grid = ptr.t_grid(n_hom)
    sols, warm = [], guesses
    for i in range(n_hom):
        pbm.traj.mdl.kappa = hom(grid[i])
        warm = ptr.solve(pbm, warm, **cone_opts)
        sols.append(warm)
    return sols


def homotopy_schedule(traj, beta, n_hom=10, hom=None, worsen_tol=-1e-3):
    """Step kappa through hom(LinRange(0, 1, n_hom)) (default Homotopy(1e-8)) inside ONE PTR solve: a seed moves to the
    next value when its relative cost improvement lies in [worsen_tol, beta] (problem_set_homotopy_update).  Call before
    ptr.create or between solves; ptr.solve(..., beta=[...]) then sweeps the threshold over a batch."""
    hom = hom or Homotopy(1e-8)
    problem_set_homotopy_update(traj, [hom(x) for x in ptr.t_grid(n_hom)], beta, worsen_tol)
