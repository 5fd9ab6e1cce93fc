"""Double integrator with friction as a free-final-time, minimum-time PTR problem (BASELINE config C1) on the GPU API.

The reference ships this plant only as a fixed-time LCvx program (test/examples/double_integrator/definition.jl:38-118
on parameters.jl:50-64: f = [x2; u - g], travel distance s, two parameter choices).  The SCP form is a NEW definition
on the same data: x = [position, velocity], |u| <= u_max = 2 (the outer bound of definition.jl:60-65), p = [tf],
dynamics pack SCPB_MODEL_DBLINT = tf [x2; u - g], rest-to-rest over the distance s, cost tf.  The continuous-time
optimum is the bang-bang law of the maximum principle (cf. solve_mp, definition.jl:137-294) and is known in closed
form (t_opt), which pins the whole SCP chain against an analytic answer."""
from __future__ import annotations

import math

import numpy as np

from .. import lib
from ..parser import Expr
from ..problem import (TrajectoryProblem, problem_advise_scale, problem_set_bc, problem_set_dims, problem_set_dynamics,
                       problem_set_guess, problem_set_terminal_cost, problem_set_U, problem_set_X)


class DoubleIntegratorProblem:
    """parameters.jl:50-64"""

    def __init__(self, choice: int = 1):
        assert choice in (1, 2)
        self.g = 0.1 if choice == 1 else 0.6
        self.s = 47.0 if choice == 1 else 30.0
        self.T = 10.0
        self.u_max = 2.0
        self.tf_min, self.tf_max = 1.0, 30.0

    def par(self):
        return np.array([self.g])

    def t_opt(self):
        """(minimum time, switching time): accelerate with u_max - g, brake with u_max + g"""
        a1, a2 = self.u_max - self.g, self.u_max + self.g
        t1 = math.sqrt(2 * self.s * a2 / (a1 * (a1 + a2)))
        return t1 * (1 + a1 / a2), t1


def define_problem(pbm: TrajectoryProblem, algo: str = "ptr", handle=None):
    mdl = pbm.mdl
    problem_set_dims(pbm, 2, 1, 1)
    problem_advise_scale(pbm, "state", 0, (0.0, mdl.s))
    problem_advise_scale(pbm, "state", 1, (0.0, 2.0 * mdl.s / 8.0))
    problem_advise_scale(pbm, "input", 0, (-mdl.u_max, mdl.u_max))
    problem_advise_scale(pbm, "parameter", 0, (mdl.tf_min, mdl.tf_max))
    problem_set_terminal_cost(pbm, lambda x, p, pbm_: p[0] * (1.0 / pbm_.mdl.T))
    As = np.zeros((2, 2), bool); As[0, 1] = True
    Bs = np.zeros((2, 1), bool); Bs[1, 0] = True
    problem_set_dynamics(pbm, lib.MODEL_DBLINT, mdl.par(), fcols=(0,), A_struct=As, B_struct=Bs)

    def X(t, k, x, p, pbm_, ocp):
        ocp.nonpos([p[0] - pbm_.mdl.tf_max], "max_time")
        ocp.nonpos([pbm_.mdl.tf_min - p[0]], "min_time")

    def U(t, k, u, p, pbm_, ocp):
        ocp.l1([Expr.lift(pbm_.mdl.u_max), u[0]], "input_bound")

    problem_set_X(pbm, X)
    problem_set_U(pbm, U)
    problem_set_bc(pbm, "ic", lambda x, p, pbm_: [x[0] - 0.0, x[1] - 0.0])
    problem_set_bc(pbm, "tc", lambda x, p, pbm_: [x[0] - pbm_.mdl.s, x[1] - 0.0])

    def guess(N, pbm_):
        m_ = pbm_.mdl
        tau = np.arange(N) / (N - 1)
        xg = np.zeros((N, 2)); ug = np.zeros((N, 1))
        xg[:, 0] = tau * m_.s
        xg[:, 1] = m_.s / m_.T
        return xg, ug, np.array([m_.T])

    problem_set_guess(pbm, guess)
