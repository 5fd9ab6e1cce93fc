"""Mars powered-descent guidance as a free-final-time PTR problem (BASELINE config C2) on the GPU API.

The reference ships this vehicle only as a single-shot LCvx program (test/examples/rocket_landing/definition.jl:33-140
on parameters.jl:78-150); the SCP form is a NEW definition on the same data: state x = [r(3) v(3) z = ln m], input
u = [a(3) xi] (thrust acceleration and its slack), parameter p = [tf], dynamics pack SCPB_MODEL_ROCKET =
tf (A_c x + B_c u + p_c) (parameters.jl:110-121), the constraints of definition.jl:93-131 with the mass profile z0
evaluated on a NOMINAL flight time (every constraint stays convex in (x, u, p): the thrust-magnitude bounds
mu = rho exp(-z0) are node constants), terminal cost -z_N (maximum final mass), no nonconvex path constraint.
It is the SOC-constrained PTR case of the test suite: two second-order cones per node (thrust slack, speed limit)
inside the SCP loop."""
from __future__ import annotations

import math

import numpy as np

from .. import lib
from ..parser import Expr
from ..problem import (TrajectoryProblem, problem_advise_scale, problem_set_bc, problem_set_dims, problem_set_dynamics,
                       problem_set_guess, problem_set_terminal_cost, problem_set_U, problem_set_X)


class RocketProblem:
    """parameters.jl:78-150"""

    def __init__(self):
        ex, ey, ez = np.eye(3)
        self.g = -3.7114 * ez
        th = 30 * math.pi / 180
        T_sidereal_mars = 24.6229 * 3600
        self.omega = (2 * math.pi / T_sidereal_mars) * (ex * math.cos(th) + ey * 0 + ez * math.sin(th))
        self.m_dry, self.m_wet, self.Isp = 1505.0, 1905.0, 225.0
        n_eng = 6
        self.phi = 27 * math.pi / 180
        T_max = 3.1e3
        self.rho_min = n_eng * 0.3 * T_max * math.cos(self.phi)
        self.rho_max = n_eng * 0.8 * T_max * math.cos(self.phi)
        self.gamma_gs = 86 * math.pi / 180
        self.gamma_p = 40 * math.pi / 180
        self.v_max = 500 * 1e3 / 3600
        self.r0 = (2 * ex + 0 * ey + 1.5 * ez) * 1e3
        self.v0 = 80 * ex + 30 * ey - 75 * ez
        self.alpha = 1 / (self.Isp * 9.807 * math.cos(self.phi))
        self.tf_min, self.tf_max, self.tf_nom = 50.0, 110.0, 75.0
        cg, sg = math.cos(self.gamma_gs), math.sin(self.gamma_gs)
        self.H_gs = np.array([[cg, 0, -sg], [-cg, 0, -sg], [0, cg, -sg], [0, -cg, -sg]])

    def par(self):
        """device parameter block of SCPB_MODEL_ROCKET (csrc/models.cuh): g(3), omega(3), alpha"""
        return np.concatenate([self.g, self.omega, [self.alpha]])

    def z0(self, tau):
        return math.log(self.m_wet - self.alpha * self.rho_max * tau * self.tf_nom)

    def z1(self, tau):
        return math.log(self.m_wet - self.alpha * self.rho_min * tau * self.tf_nom)


def define_problem(pbm: TrajectoryProblem, algo: str = "ptr", handle=None):
    mdl = pbm.mdl
    problem_set_dims(pbm, 7, 4, 1)
    amax = mdl.rho_max / mdl.m_dry
    xr = [(-500.0, 2500.0), (-500.0, 500.0), (0.0, 1600.0), (-100.0, 100.0), (-100.0, 100.0), (-100.0, 100.0),
          (math.log(mdl.m_dry), math.log(mdl.m_wet))]
    for i, r in enumerate(xr):
        problem_advise_scale(pbm, "state", i, r)
    lat = amax * math.sin(mdl.gamma_p)
    for i, r in enumerate([(-lat, lat), (-lat, lat), (0.0, amax), (0.0, amax)]):
        problem_advise_scale(pbm, "input", i, r)
    problem_advise_scale(pbm, "parameter", 0, (mdl.tf_min, mdl.tf_max))

    def phi(x, p, pbm):     # fraction of the propellant budget spent (maximum final mass)
        m_ = pbm.mdl
        dz = math.log(m_.m_wet) - math.log(m_.m_dry)
        return (x[6] - math.log(m_.m_wet)) * (-1.0 / dz)

    problem_set_terminal_cost(pbm, phi)
    # df/dx, df/du structure of f = tf (A_c x + B_c u + p_c): r' = v, v' = -w x (w x r) - 2 w x v + a, z' = -alpha xi
    As = np.zeros((7, 7), bool); Bs = np.zeros((7, 4), bool)
    As[0:3, 3:6] = np.eye(3, dtype=bool)
    As[3:6, 0:6] = True
    Bs[3:6, 0:3] = np.eye(3, dtype=bool); Bs[6, 3] = True
    problem_set_dynamics(pbm, lib.MODEL_ROCKET, mdl.par(), fcols=(0,), A_struct=As, B_struct=Bs)

    def X(t, k, x, p, pbm, ocp):
        m_ = pbm.mdl
        r, v, z = x[0:3], x[3:6], x[6]
        ocp.nonpos([m_.z0(t) - z], "mass_lower")
        ocp.nonpos([z - m_.z1(t)], "mass_upper")
        for i in range(4):
            ocp.nonpos([r[0] * m_.H_gs[i, 0] + r[1] * m_.H_gs[i, 1] + r[2] * m_.H_gs[i, 2]], "glide_slope")
        ocp.soc([Expr.lift(m_.v_max), v[0], v[1], v[2]], "max_speed")
        if k == pbm.scp.N:
            ocp.nonpos([math.log(m_.m_dry) - z], "dry_mass")
        ocp.nonpos([p[0] - m_.tf_max], "max_time")
        ocp.nonpos([m_.tf_min - p[0]], "min_time")

    def U(t, k, u, p, pbm, ocp):
        m_ = pbm.mdl
        a, xi = u[0:3], u[3]
        ocp.soc([xi, a[0], a[1], a[2]], "lcvx_equality")
        ocp.nonpos([xi * math.cos(m_.gamma_p) - a[2]], "pointing")
        mu_min, mu_max = m_.rho_min * math.exp(-m_.z0(t)), m_.rho_max * math.exp(-m_.z0(t))
        ocp.nonpos([mu_min - xi], "min_thrust")
        ocp.nonpos([xi - mu_max], "max_thrust")

    problem_set_X(pbm, X)
    problem_set_U(pbm, U)

    def gic(x, p, pbm):
        m_ = pbm.mdl
        rhs = list(m_.r0) + list(m_.v0) + [math.log(m_.m_wet)]
        return [x[i] - rhs[i] for i in range(7)]

    def gtc(x, p, pbm):
        return [x[i] - 0.0 for i in range(6)]

    problem_set_bc(pbm, "ic", gic)
    problem_set_bc(pbm, "tc", gtc)

    def guess(N, pbm_):
        m_ = pbm_.mdl
        tau = np.arange(N) / (N - 1)
        xg = np.zeros((N, 7)); ug = np.zeros((N, 4))
        for k in range(N):
            xg[k, 0:3] = (1 - tau[k]) * m_.r0
            xg[k, 3:6] = (1 - tau[k]) * m_.v0
            xg[k, 6] = (1 - tau[k]) * math.log(m_.m_wet) + tau[k] * math.log(0.5 * (m_.m_dry + m_.m_wet))
            ug[k, 0:3] = -m_.g
            ug[k, 3] = np.linalg.norm(m_.g)
        return xg, ug, np.array([m_.tf_nom])

    problem_set_guess(pbm, guess)
