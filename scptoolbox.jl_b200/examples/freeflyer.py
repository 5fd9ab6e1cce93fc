"""6-DoF free-flyer in the space station as a PTR problem (BASELINE config C5) on the GPU API.

Vehicle, environment and trajectory data: test/examples/freeflyer/parameters.jl:105-190; problem definition:
test/examples/freeflyer/definition.jl (dims :42-49, scaling advice :52-67, guess :84-167, cost :170-222,
convex sets :286-375, nonconvex constraints :376-442, boundary conditions :455-520).  The reference runs this example
with SCvx and GuSTO only (test/runtests.jl:31-60); the PTR instance is the same problem on the same closures, with the
SCvx flavour of the running cost (a convex quadratic of the input, lowered to one second-order cone per node).

State x = [r(3) v(3) q(4, scalar last) omega(3)], input u = [T(3) M(3)], parameters p = [tdil, delta(6 rooms x N nodes)]:
delta[i, k] is the slack of room i's signed-distance function at node k, so np = 1 + 6 N and every nonconvex row couples
a node only to its own six slacks (packed ds/dp columns, csrc/constraints.cuh).  Only r, tdil and delta carry scaling
advice: v, q, omega, T and M are scaled by the automatic bounding-box solves of compute_scaling (ptr.SCPScaling)."""
from __future__ import annotations

import math

import numpy as np

from .. import lib
from ..parser import Expr
from ..problem import (TrajectoryProblem, problem_advise_parameter_stage, problem_advise_scale, problem_set_bc,
                       problem_set_dims, problem_set_dynamics, problem_set_guess, problem_set_running_cost,
                       problem_set_s, problem_set_terminal_cost, problem_set_U, problem_set_X)


def room(offset, width, height, depth, yaw=0.0, pitch=0.0, roll=0.0):
    """Hyperrectangle(offset, width, height, depth; yaw, pitch, roll) (src/utils/hyperrectangle.jl:85-138): returns the
    centre c and half-widths s of the axis-aligned box."""
    cd = lambda a: math.cos(math.radians(a))
    sd = lambda a: math.sin(math.radians(a))
    lo = np.array([-width / 2, -height / 2, 0.0]); hi = np.array([width / 2, height / 2, depth])
    Rz = np.array([[cd(yaw), -sd(yaw), 0], [sd(yaw), cd(yaw), 0], [0, 0, 1]])
    Ry = np.array([[cd(pitch), 0, sd(pitch)], [0, 1, 0], [-sd(pitch), 0, cd(pitch)]])
    Rx = np.array([[1, 0, 0], [0, cd(roll), -sd(roll)], [0, sd(roll), cd(roll)]])
    R = Rz @ Ry @ Rx
    lr, ur = R @ lo, R @ hi
    l = np.minimum(lr, ur) + np.asarray(offset, float)
    u = np.maximum(lr, ur) + np.asarray(offset, float)
    return (u + l) / 2, (u - l) / 2


# quaternions, scalar last (src/utils/quaternion.jl)
def q_from_axis_angle(alpha, axis):
    a = np.asarray(axis, float); a = a / np.linalg.norm(a)
    return np.concatenate([a * math.sin(alpha / 2), [math.cos(alpha / 2)]])


def q_mul(q, p):            # quaternion.jl:190-214: skew(q, :L) * vec(p)
    qv, qw, pv, pw = q[:3], q[3], p[:3], p[3]
    return np.concatenate([qw * pv + np.cross(qv, pv) + qv * pw, [qw * pw - qv @ pv]])


def q_conj(q):
    return np.concatenate([-q[:3], [q[3]]])


def q_log(q):               # quaternion.jl:277-282
    nv = np.linalg.norm(q[:3])
    return 2 * math.atan2(nv, q[3]), q[:3] / nv


def slerp(q0, q1, tau):     # quaternion.jl:483-490
    tau = max(0.0, min(1.0, tau))
    da, dax = q_log(q_mul(q_conj(q0), q1))
    return q_mul(q0, q_from_axis_angle(tau * da, dax))


class FreeFlyerProblem:
    """parameters.jl:105-190"""

    def __init__(self, N: int):
        self.N = N
        z_iss = 4.75
        self.obs_H = [np.diag([1.0, 1.0, 1.0]) / 0.3] * 3
        self.obs_c = [np.array([8.5, -0.15, 5.0]), np.array([11.2, 1.84, 5.0]), np.array([11.3, 3.8, 4.8])]
        self.rooms = [room([6.0, 0.0, z_iss], 1.0, 1.0, 1.5, pitch=90.0),
                      room([7.5, 0.0, z_iss], 2.0, 2.0, 4.0, pitch=90.0),
                      room([11.5, 0.0, z_iss], 1.25, 1.25, 0.5, pitch=90.0),
                      room([10.75, -1.0, z_iss], 1.5, 1.5, 1.5, yaw=-90.0, pitch=90.0),
                      room([10.75, 1.0, z_iss], 1.5, 1.5, 1.5, yaw=90.0, pitch=90.0),
                      room([10.75, 2.5, z_iss], 2.5, 2.5, 4.5, yaw=90.0, pitch=90.0)]
        self.n_iss, self.n_obs = 6, 3
        self.np = 1 + self.n_iss * N
        self.v_max, self.omega_max = 0.4, math.radians(1)
        self.T_max, self.M_max = 20e-3, 1e-4
        self.mass = 7.2
        self.J = np.diag([0.1083, 0.1083, 0.1083])
        self.r0 = np.array([6.5, -0.2, 5.0]); self.v0 = np.array([0.035, 0.035, 0.0])
        self.q0 = q_from_axis_angle(math.radians(-40), [0.0, 1.0, 1.0]); self.w0 = np.zeros(3)
        self.rf = np.array([11.3, 6.0, 4.5]); self.vf = np.zeros(3)
        self.qf = q_from_axis_angle(0.0, [0.0, 0.0, 1.0]); self.wf = np.zeros(3)
        self.tf_min, self.tf_max = 60.0, 200.0
        self.gamma, self.hom, self.eps_sdf = 0.0, 50.0, 1e-4

    def id_delta(self, i, k):
        """0-based parameter index of delta[i, k] (reshape(p[id_delta], n_iss, :), column-major)"""
        return 1 + i + self.n_iss * k

    def par(self):
        """device parameter block: dynamics pack (mass, J, Jinv; csrc/models.cuh) then the constraint pack's data
        (hom, 3 x {H column-major, c}; csrc/constraints.cuh)"""
        ob = []
        for H, c in zip(self.obs_H, self.obs_c):
            ob += list(H.flatten(order="F")) + list(c)
        return np.concatenate([[self.mass], self.J.flatten(order="F"), np.linalg.inv(self.J).flatten(order="F"),
                               [self.hom], ob])


def define_problem(pbm: TrajectoryProblem, algo: str = "ptr", handle=None):
    mdl = pbm.mdl
    N = mdl.N
    problem_set_dims(pbm, 13, 6, mdl.np)
    # set_scale! (definition.jl:52-67)
    lo, hi = np.minimum(mdl.r0, mdl.rf), np.maximum(mdl.r0, mdl.rf)
    for i in range(3):
        problem_advise_scale(pbm, "state", i, (lo[i], hi[i]))
    problem_advise_scale(pbm, "parameter", 0, (mdl.tf_min, mdl.tf_max))
    for i in range(1, mdl.np):
        problem_advise_scale(pbm, "parameter", i, (-100.0, 1.0))

    # set_cost! (definition.jl:170-222)
    def phi(x, p, pbm_):
        m_ = pbm_.mdl
        J = Expr()
        for i in range(1, m_.np):
            J = J + p[i] * (-m_.eps_sdf)
        if m_.gamma != 0.0:
            J = J + pbm_.ocp.sumsq([p[0] * (1.0 / m_.tf_max)], "time_cost", stage=-1) * m_.gamma
        return J

    def Gamma(t, k, x, u, p, pbm_):
        m_ = pbm_.mdl
        q = pbm_.ocp.sumsq([u[i] * (1.0 / m_.T_max) for i in range(3)] + [u[3 + i] * (1.0 / m_.M_max) for i in range(3)],
                           "input_energy", stage=k - 1)
        return q * (1.0 - m_.gamma)

    problem_set_terminal_cost(pbm, phi)
    problem_set_running_cost(pbm, Gamma)

    # dynamics pack (definition.jl:224-284): r' = v, v' = T/m, q' = q (x) omega / 2, omega' = J^-1 (M - omega x J omega)
    As = np.zeros((13, 13), bool); Bs = np.zeros((13, 6), bool)
    As[0:3, 3:6] = np.eye(3, dtype=bool)
    As[6:10, 6:13] = True
    As[10:13, 10:13] = True
    Bs[3:6, 0:3] = np.eye(3, dtype=bool); Bs[10:13, 3:6] = True
    problem_set_dynamics(pbm, lib.MODEL_FREEFLYER, mdl.par(), fcols=(0,), A_struct=As, B_struct=Bs)

    # set_convex_constraints! (definition.jl:286-375)
    def X(t, k, x, p, pbm_, ocp):
        m_ = pbm_.mdl
        r, v, w = x[0:3], x[3:6], x[10:13]
        ocp.soc([Expr.lift(m_.v_max), v[0], v[1], v[2]], "max_lin_vel")
        ocp.soc([Expr.lift(m_.omega_max), w[0], w[1], w[2]], "max_ang_vel")
        ocp.nonpos([p[0] - m_.tf_max], "max_duration")
        ocp.nonpos([m_.tf_min - p[0]], "min_duration")
        for i in range(m_.n_iss):
            c, s_ = m_.rooms[i]
            d = p[m_.id_delta(i, k - 1)]
            ocp.linf([1.0 - d] + [(r[j] - c[j]) * (1.0 / s_[j]) for j in range(3)], f"room_sdf_{i + 1}")

    def U(t, k, u, p, pbm_, ocp):
        m_ = pbm_.mdl
        ocp.soc([Expr.lift(m_.T_max), u[0], u[1], u[2]], "max_thrust")
        ocp.soc([Expr.lift(m_.M_max), u[3], u[4], u[5]], "max_torque")

    problem_set_X(pbm, X)
    problem_set_U(pbm, U)

    # set_nonconvex_constraints! (definition.jl:376-442): device pack Constr<FREEFLYER>, ns = n_obs + 1
    ns = mdl.n_obs + 1

    def s_struct(t, k, pbm_):
        Cm = np.zeros((ns, 13), bool); Dm = np.zeros((ns, 6), bool); Gm = np.zeros((ns, mdl.n_iss), bool)
        Cm[0:mdl.n_obs, 0:3] = True
        Gm[ns - 1, :] = True
        return Cm, Dm, Gm

    problem_set_s(pbm, ns, s_struct, gcols=lambda k: [mdl.id_delta(i, k) for i in range(mdl.n_iss)])
    problem_advise_parameter_stage(pbm, lambda N_: [-1] + [k for k in range(N_) for _ in range(mdl.n_iss)])

    # set_bcs! (definition.jl:455-520)
    def gic(x, p, pbm_):
        m_ = pbm_.mdl
        rhs = np.concatenate([m_.r0, m_.v0, m_.q0, m_.w0])
        return [x[i] - rhs[i] for i in range(13)]

    def gtc(x, p, pbm_):
        m_ = pbm_.mdl
        rhs = np.concatenate([m_.rf, m_.vf, m_.qf, m_.wf])
        return [x[i] - rhs[i] for i in range(13)]

    problem_set_bc(pbm, "ic", gic)
    problem_set_bc(pbm, "tc", gtc)
    problem_set_guess(pbm, lambda N_, pbm_: initial_guess(pbm_.mdl, N_))


def initial_guess(m_, N):
    """set_guess! (definition.jl:84-167): L-shaped axis-aligned position path at constant speed, SLERP attitude with the
    matching constant body rate, idle inputs, room slacks evaluated on the path."""
    p = np.zeros(m_.np)
    flight_time = 0.5 * (m_.tf_min + m_.tf_max)
    p[0] = flight_time
    x = np.zeros((N, 13))
    speed = np.abs(m_.rf - m_.r0).sum() / flight_time
    times = np.array([(1 - k / (N - 1)) * 0.0 + (k / (N - 1)) * flight_time for k in range(N)])
    leg = np.abs(m_.rf - m_.r0) / speed
    cum = np.cumsum(leg)
    for k in range(N):
        tk = min(times[k], cum[2])        # the last node sits on the end of the last leg
        for i in range(3):
            if tk <= cum[i]:
                t0 = cum[i - 1] if i > 0 else 0.0
                tf = cum[i]
                r0 = m_.r0.copy(); r0[:i] = m_.rf[:i]
                rf = r0.copy(); rf[i] = m_.rf[i]
                c = (tf - tk) / (tf - t0)                     # linterp (helper.jl:107-118)
                x[k, 0:3] = c * r0 + (1 - c) * rf
                d = rf - r0
                x[k, 3:6] = speed * d / np.linalg.norm(d)
                break
    for k in range(N):
        x[k, 6:10] = slerp(m_.q0, m_.qf, k / (N - 1))
    ang, ax = q_log(q_mul(m_.qf, q_conj(m_.q0)))
    x[:, 10:13] = (ang / flight_time) * ax
    for i in range(m_.n_iss):
        c, s_ = m_.rooms[i]
        for k in range(N):
            p[m_.id_delta(i, k)] = 1 - np.abs((x[k, 0:3] - c) / s_).max()
    u = np.zeros((N, 6))
    return x, u, p
