"""Planar spacecraft rendezvous with impulsive RCS thrust and a thrust deadband, on the GPU API (PTR, IMPULSE
discretization).

Vehicle, environment and trajectory data: test/examples/rendezvous_planar/parameters.jl:80-152; problem definition:
test/examples/rendezvous_planar/definition.jl (dims :36-41, scaling advice :43-92, guess :94-124, cost :126-144, dynamics
:146-242, input set :244-335, deadband :337-413, boundary conditions :415-475); solve: tests.jl:22-95.

State x = [r(2) v(2) theta omega], input u = [f(3) fr(3) l1f(3) l1feq(3)] (thrust of the three RCS pods, their reference
values, |f| and |f - fr|), parameter p = [tdil].  Every variable carries scaling advice, so no bounding-box solve is
needed.  The deadband constraint f = OR(fr) fr is a smooth OR whose sharpness kappa is stepped through a homotopy; each
step is warm-started from the previous solution (homotopy_sweep), or stepped inside one solve by the in-loop schedule
(homotopy_schedule, the pattern of test/examples/rendezvous_3d/definition.jl:96-151)."""
from __future__ import annotations

import math

import numpy as np

from .. import lib, ptr
from ..homotopy import Homotopy
from ..parser import Expr
from ..problem import (TrajectoryProblem, problem_advise_scale, problem_set_bc, problem_set_dims, problem_set_dynamics,
                       problem_set_guess, problem_set_homotopy_update, problem_set_running_cost, problem_set_s,
                       problem_set_U)

ID_F, ID_FR, ID_L1F, ID_L1FEQ = range(0, 3), range(3, 6), range(6, 9), range(9, 12)


class PlanarRendezvousProblem:
    """parameters.jl:80-152"""

    def __init__(self):
        mu, Re = 3.986e14, 6378e3              # [m^3/s^2], [m]
        R = Re + 400e3                         # orbit radius
        self.n = math.sqrt(mu / (R * R * R))   # mean motion (Julia's R^3 is R*R*R)
        self.m, self.J, self.lu, self.lv = 30e3, 1e5, 0.6, 2.1
        self.f_max, self.f_db = 750.0, 200.0
        self.r0, self.v0 = np.array([100.0, 10.0]), np.array([0.0, 0.0])
        self.th0, self.om0 = 180.0 * math.pi / 180.0, 0.0
        self.vf = 0.1
        self.tf_min, self.tf_max = 100.0, 500.0
        self.kappa = float("nan")              # sigmoid sharpness, set by the homotopy before every solve
        self.gamma = 3e-1

    def par(self):
        """device parameter block: m, J, lu, lv, n (dynamics pack, csrc/models.cuh), then f_db, f_max, kappa (constraint
        pack, csrc/constraints.cuh)"""
        return np.array([self.m, self.J, self.lu, self.lv, self.n, self.f_db, self.f_max, self.kappa])


def define_problem(pbm: TrajectoryProblem, algo: str = "ptr"):
    mdl = pbm.mdl
    problem_set_dims(pbm, 6, 12, 1)

    # scaling advice (definition.jl:43-92)
    rx0, ry0, vx0, vy0 = mdl.r0[0], mdl.r0[1], mdl.v0[0], mdl.v0[1]
    tmin, one = mdl.tf_min, 1.0 * math.pi / 180.0
    adv = [(0.0, max(rx0, 1.0)), (min(ry0, -0.1), max(ry0, 0.1)),
           (min(vx0, -rx0 / tmin, -0.1), min(vx0, 0.1)), (min(vy0, -ry0 / tmin, -0.1), max(vy0, -ry0 / tmin, 0.1)),
           (min(mdl.th0, -one), max(mdl.th0, one)),
           (min(-mdl.th0 / tmin, mdl.om0, -one), max(-mdl.th0 / tmin, mdl.om0, one))]
    for i, rg in enumerate(adv):
        problem_advise_scale(pbm, "state", i, rg)
    for i in list(ID_F) + list(ID_FR):
        problem_advise_scale(pbm, "input", i, (-mdl.f_max, mdl.f_max))
    for i in ID_L1F:
        problem_advise_scale(pbm, "input", i, (0.0, mdl.f_max))
    for i in ID_L1FEQ:
        problem_advise_scale(pbm, "input", i, (0.0, 2 * mdl.f_max))
    problem_advise_scale(pbm, "parameter", 0, (mdl.tf_min, mdl.tf_max))

    def guess(N, pbm_):          # definition.jl:94-124: straight line, idle thrusters
        m_ = pbm_.mdl
        p = np.array([0.5 * (m_.tf_min + m_.tf_max)])
        x0 = np.concatenate([m_.r0, -m_.r0 / p[0], [m_.th0, -m_.th0 / p[0]]])
        xf = np.zeros(6)
        xf[2:4] = x0[2:4]
        xf[5] = x0[5]
        t = ptr.t_grid(N)
        x = np.array([(1.0 - t[k]) * x0 + (1 - (1.0 - t[k])) * xf for k in range(N)])   # linterp, helper.jl:107-118
        return x, np.zeros((N, 12)), p

    problem_set_guess(pbm, guess)

    def Gamma(t, k, x, u, p, pbm_):      # definition.jl:126-144: L1 thrust + gamma * L1 deadband relaxation
        m_ = pbm_.mdl
        l1f, l1feq = Expr(), Expr()
        for i in ID_L1F:
            l1f = l1f + u[i]
        for i in ID_L1FEQ:
            l1feq = l1feq + u[i]
        return l1f / m_.f_max + (l1feq * m_.gamma) / m_.f_max

    problem_set_running_cost(pbm, Gamma, algo)

    # dynamics pack (definition.jl:146-242); the parameter block is read at every solve, so a new kappa takes effect
    As = np.zeros((6, 6), bool); Bs = np.zeros((6, 12), bool)
    for i, j in [(0, 2), (1, 3), (3, 1), (2, 3), (3, 2), (2, 4), (3, 4), (4, 5)]:
        As[i, j] = True
    Bs[[2, 3, 5], 0:3] = True
    problem_set_dynamics(pbm, lib.MODEL_RENDEZVOUS2D, lambda: pbm.mdl.par(), fcols=(0,), A_struct=As, B_struct=Bs)

    def U(t, k, u, p, pbm_, ocp):      # definition.jl:244-335
        m_ = pbm_.mdl
        for i in range(3):
            f, fr, l1f, l1feq = u[ID_F[i]], u[ID_FR[i]], u[ID_L1F[i]], u[ID_L1FEQ[i]]
            ocp.nonpos([l1f - m_.f_max], "thrust_absval_max")
            ocp.nonpos([fr - m_.f_max], "thrust_refval_max")
            ocp.nonpos([-fr - m_.f_max], "thrust_refval_min")
            ocp.l1([l1f, f], "thrust_absval")
            ocp.l1([l1feq, f - fr], "thrust_absval")
        ocp.nonpos([p[0] - m_.tf_max], "min_time_bound")
        ocp.nonpos([m_.tf_min - p[0]], "max_time_bound")

    problem_set_U(pbm, U)

    def s_struct(t, k, pbm_):          # deadband (definition.jl:337-413): D is +-1 on f_i and -+dOR/dfr on fr_i only
        Cm = np.zeros((6, 6), bool); Dm = np.zeros((6, 12), bool); Gm = np.zeros((6, 1), bool)
        for i in range(3):
            Dm[2 * i:2 * i + 2, [ID_F[i], ID_FR[i]]] = True
        return Cm, Dm, Gm

    problem_set_s(pbm, 6, s_struct)

    def gic(x, p, pbm_):               # definition.jl:415-443
        m_ = pbm_.mdl
        rhs = np.concatenate([m_.r0, m_.v0, [m_.th0, m_.om0]])
        return [x[i] - rhs[i] for i in range(6)]

    def gtc(x, p, pbm_):               # definition.jl:445-472: at rest at the port, approaching at vf along xh
        m_ = pbm_.mdl
        rhs = [0.0, 0.0, -m_.vf * 1.0, -m_.vf * 0.0, 0.0, 0.0]
        return [x[i] - rhs[i] for i in range(6)]

    problem_set_bc(pbm, "ic", gic)
    problem_set_bc(pbm, "tc", gtc)


def ptr_parameters(N=30, Nsub=10, iter_max=30, solver_opts=None):
    """the reference's PTR configuration (tests.jl:31-58): IMPULSE, q_tr = q_exit = Inf, every subproblem an LP"""
    return ptr.Parameters(N=N, Nsub=Nsub, iter_max=iter_max, disc_method=ptr.IMPULSE, wvc=5e2, wtr=3e-2,
                          eps_abs=-np.inf, eps_rel=1e-3 / 100, feas_tol=5e-3, q_tr=np.inf, q_exit=np.inf,
                          solver_opts=solver_opts or {"verbose": 0})


def homotopy_sweep(pbm, guesses=None, n_hom=10, hom=None, **cone_opts):
    """tests.jl:60-79 for a batch: kappa = hom(LinRange(0, 1, n_hom)[i]) for every seed at step i (default
    Homotopy(1e-3; delta_max = 5)), each step warm-started from the previous step's batch solution (PTR.solve(pbm,
    warm)).  guesses: (xd0, ud0, p0) batch or None (the problem's own guess).  Returns the list of batch solutions."""
    hom = hom or Homotopy(1e-3, delta_max=5.0)
    grid = ptr.t_grid(n_hom)
    sols, warm = [], guesses
    for i in range(n_hom):
        pbm.traj.mdl.kappa = hom(grid[i])
        warm = ptr.solve(pbm, warm, **cone_opts)
        sols.append(warm)
    return sols


def homotopy_schedule(traj, beta, n_hom=10, hom=None, worsen_tol=-1e-3):
    """Step kappa through hom(LinRange(0, 1, n_hom)) (default Homotopy(1e-3; delta_max = 5)) inside ONE PTR solve: a seed
    moves to the next value when its relative cost improvement lies in [worsen_tol, beta] (problem_set_homotopy_update).
    Call before ptr.create or between solves; ptr.solve(..., beta=[...]) then sweeps the threshold over a batch."""
    hom = hom or Homotopy(1e-3, delta_max=5.0)
    problem_set_homotopy_update(traj, [hom(x) for x in ptr.t_grid(n_hom)], beta, worsen_tol)
