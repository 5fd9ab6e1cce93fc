"""Quadrotor obstacle avoidance (BASELINE config C4) on the GPU API, in its GuSTO flavour.

Vehicle, environment and trajectory data: test/examples/quadrotor/parameters.jl:96-135; problem definition:
test/examples/quadrotor/definition.jl (dims :40-45, scaling advice :47-58, guess :60-91, cost :93-138, dynamics :140-186,
input set :188-252, obstacles :254-294, boundary conditions :296-360).

State x = [r(3) v(3)], input u = [a(3) sigma], parameter p = [tdil].  Only tdil carries scaling advice: the other
variables are scaled by the automatic bounding-box solves of compute_scaling (ptr.SCPScaling); r and v have no convex
set at all, so they keep the default box (scp.jl:470-473)."""
from __future__ import annotations

import math

import numpy as np

from .. import lib
from ..parser import Expr
from ..problem import (TrajectoryProblem, problem_advise_scale, problem_set_bc, problem_set_dims, problem_set_dynamics,
                       problem_set_guess, problem_set_running_cost, problem_set_s, problem_set_terminal_cost,
                       problem_set_U)


class QuadrotorProblem:
    """parameters.jl:96-135"""

    def __init__(self):
        self.g = np.array([0.0, 0.0, -9.81])
        self.u_max, self.u_min, self.tilt_max = 23.2, 0.6, math.radians(60)
        self.obs_H = [np.diag([2.0, 2.0, 0.0]), np.diag([1.5, 1.5, 0.0])]
        self.obs_c = [np.array([1.0, 2.0, 0.0]), np.array([2.0, 5.0, 0.0])]
        self.n_obs = 2
        self.r0, self.v0 = np.zeros(3), np.zeros(3)
        self.rf, self.vf = np.array([2.5, 6.0, 0.0]), np.zeros(3)
        self.tf_min, self.tf_max = 0.0, 2.5
        self.gamma = 0.0

    def par(self):
        """device parameter block: g (dynamics pack, csrc/models.cuh), then 2 x {H column-major, c} (constraint pack)"""
        ob = []
        for H, c in zip(self.obs_H, self.obs_c):
            ob += list(H.flatten(order="F")) + list(c)
        return np.concatenate([self.g, ob])


def define_problem(pbm: TrajectoryProblem, algo: str = "gusto", handle=None):
    mdl = pbm.mdl
    problem_set_dims(pbm, 6, 4, 1)
    problem_advise_scale(pbm, "parameter", 0, (mdl.tf_min, mdl.tf_min + 1.0 * (mdl.tf_max - mdl.tf_min)))

    def guess(N, pbm_):          # definition.jl:60-91
        m_ = pbm_.mdl
        x0 = np.concatenate([m_.r0, m_.v0]); xf = np.concatenate([m_.rf, m_.vf])
        x = np.array([(1 - k / (N - 1)) * x0 + (k / (N - 1)) * xf for k in range(N)])
        hover = np.concatenate([-m_.g, [np.linalg.norm(m_.g)]])
        return x, np.tile(hover, (N, 1)), np.array([0.5 * (m_.tf_min + m_.tf_max)])

    problem_set_guess(pbm, guess)

    def phi(x, p, pbm_):         # definition.jl:96-103: gamma (tdil / tdil_max)^2
        m_ = pbm_.mdl
        if m_.gamma == 0.0:
            return Expr()
        return pbm_.ocp.sumsq([p[0] * (1.0 / m_.tf_max)], "time_cost", stage=-1) * m_.gamma

    problem_set_terminal_cost(pbm, phi)
    if algo == "gusto":          # definition.jl:122-133: S[sigma, sigma] = (1 - gamma) / |g|^2

        def S(t, k, p, pbm_):
            m_ = pbm_.mdl
            S_ = np.zeros((4, 4))
            S_[3, 3] = (1 - m_.gamma) / np.linalg.norm(m_.g) ** 2
            return S_

        problem_set_running_cost(pbm, S, "gusto")
    else:                        # definition.jl:106-120: (1 - gamma) (sigma / |g|)^2

        def Gamma(t, k, x, u, p, pbm_):
            m_ = pbm_.mdl
            return pbm_.ocp.sumsq([u[3] * (1.0 / np.linalg.norm(m_.g))], "input_energy", stage=k - 1) * (1 - m_.gamma)

        problem_set_running_cost(pbm, Gamma)

    # dynamics pack (definition.jl:140-186): r' = tdil v, v' = tdil (a + g)
    As = np.zeros((6, 6), bool); Bs = np.zeros((6, 4), bool)
    As[0:3, 3:6] = np.eye(3, dtype=bool)
    Bs[3:6, 0:3] = np.eye(3, dtype=bool)
    problem_set_dynamics(pbm, lib.MODEL_QUADROTOR, mdl.par(), fcols=(0,), A_struct=As, B_struct=Bs)

    def U(t, k, u, p, pbm_, ocp):    # definition.jl:188-252
        m_ = pbm_.mdl
        a, sg = u[0:3], u[3]
        ocp.nonpos([m_.u_min - sg], "min_accel")
        ocp.nonpos([sg - m_.u_max], "max_accel")
        ocp.soc([sg, a[0], a[1], a[2]], "lcvx_equality")
        ocp.nonpos([sg * math.cos(m_.tilt_max) - a[2]], "max_tilt")
        ocp.nonpos([p[0] - m_.tf_max], "max_duration")
        ocp.nonpos([m_.tf_min - p[0]], "min_duration")

    problem_set_U(pbm, U)

    # obstacles (definition.jl:254-294): device pack Constr<QUADROTOR>, s_i = 1 - |H_i (r - c_i)|
    def s_struct(t, k, pbm_):
        Cm = np.zeros((2, 6), bool); Dm = np.zeros((2, 4), bool); Gm = np.zeros((2, 1), bool)
        Cm[:, 0:2] = True            # H has no z-row / column: ds/dr_z is structurally zero
        return Cm, Dm, Gm

    problem_set_s(pbm, mdl.n_obs, s_struct)

    def gic(x, p, pbm_):
        rhs = np.concatenate([pbm_.mdl.r0, pbm_.mdl.v0])
        return [x[i] - rhs[i] for i in range(6)]

    def gtc(x, p, pbm_):
        rhs = np.concatenate([pbm_.mdl.rf, pbm_.mdl.vf])
        return [x[i] - rhs[i] for i in range(6)]

    problem_set_bc(pbm, "ic", gic)
    problem_set_bc(pbm, "tc", gtc)
