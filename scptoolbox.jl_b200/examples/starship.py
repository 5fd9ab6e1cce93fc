"""Starship landing flip -- mirror of test/examples/starship_flip/{parameters,definition}.jl on the GPU API.

parameters.jl:100-212 -> StarshipProblem ; definition.jl:29-41 define_problem! ; set_scale! :50-79 ;
set_cost! :454-478 ; set_dynamics! :552-637 (device pack SCPB_MODEL_STARSHIP) ; set_convex_constraints! :639-702 ;
set_nonconvex_constraints! :704-810 (device constraint pack) ; set_bcs! :812-873 ; starship_initial_guess :97-445.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp

from .. import lib
from ..parser import ConicTemplate, Expr, matvec
from ..problem import (TrajectoryProblem, problem_advise_parameter_stage, problem_advise_scale, problem_set_bc, problem_set_dims,
                       problem_set_dynamics, problem_set_guess, problem_set_s, problem_set_terminal_cost,
                       problem_set_U, problem_set_X)


def deg2rad(d):
    return d * math.pi / 180.0


class StarshipProblem:
    """parameters.jl:100-212"""

    def __init__(self):
        g0 = 9.81
        self.g0 = g0
        rs, ls = 4.5, 50.0
        self.m = 120e3
        self.lcg, self.lcp = 0.4 * ls, 0.45 * ls
        self.J = 1 / 12 * self.m * (6 * rs ** 2 + ls ** 2)
        vterm = 85
        self.CD = self.m * g0 / vterm ** 2 * 1.2
        Isp = 330
        self.T_min1, self.T_max1 = 880e3, 2210e3
        self.T_min3, self.T_max3 = 3 * self.T_min1, 3 * self.T_max1
        self.alpha_e = -1 / (Isp * g0)
        self.delta_max = deg2rad(10.0)
        self.deltadot_max = 2 * self.delta_max
        self.rate_delay = 0.05
        self.r0 = np.array([100.0, 600.0]); self.v0 = np.array([0.0, -float(vterm)])
        self.theta0 = deg2rad(90.0); self.theta_s = deg2rad(-10.0)
        self.vs = np.array([0.0, -10.0]); self.vf = np.array([0.0, -0.1])
        self.tf_min, self.tf_max = 0.0, 40.0
        self.gamma_gs = deg2rad(27.0); self.thetamax2 = deg2rad(15.0)
        self.tau_s = 0.5
        self.hs = 100.0
        self.ey = np.array([0.0, 1.0])

    def par(self):
        """device parameter block (include/scpb.h, csrc/models.cuh + constraints.cuh)"""
        return np.array([self.m, self.J, self.lcg, self.lcp, self.CD, self.alpha_e, self.rate_delay, self.g0,
                         self.tau_s, self.rate_delay, self.deltadot_max, self.gamma_gs, self.thetamax2])


def define_problem(pbm: TrajectoryProblem, algo: str = "ptr", handle=None):
    mdl = pbm.mdl
    problem_set_dims(pbm, 8, 3, 10)
    # set_scale!
    adv = problem_advise_scale
    xr = [(-100.0, 100.0), (0.0, mdl.r0[1]), (-10.0, 10.0), (mdl.v0[1], 0.0), (0.0, mdl.theta0),
          (deg2rad(-10.0), deg2rad(10.0)), (mdl.m - 1e3, mdl.m), (-mdl.delta_max, mdl.delta_max)]
    for i, r in enumerate(xr):
        adv(pbm, "state", i, r)
    adv(pbm, "input", 0, (mdl.T_min1, mdl.T_max3))
    adv(pbm, "input", 1, (-mdl.delta_max, mdl.delta_max))
    adv(pbm, "input", 2, (-mdl.deltadot_max, mdl.deltadot_max))
    adv(pbm, "parameter", 0, (0.0, mdl.tf_max))
    adv(pbm, "parameter", 1, (0.0, mdl.tf_max))
    for i, r in enumerate(xr):
        adv(pbm, "parameter", 2 + i, r)

    # set_cost!: maximise switch altitude, minimise fuel
    def phi(x, p, pbm):
        m_ = pbm.mdl
        alt_cost = p[2 + 1] * (-1.0 / m_.hs)
        dm_cost = (0.0 - x[6]) * (1.0 / 10e3)
        return alt_cost * 0.3 + dm_cost

    problem_set_terminal_cost(pbm, phi)
    # structure of df/dx, df/du (definition.jl:582-620): x = [r(2) v(2) theta omega m delta_d], u = [T delta delta_dot]
    As = np.zeros((8, 8), bool); Bs = np.zeros((8, 3), bool)
    As[0, 2] = As[1, 3] = As[4, 5] = As[7, 7] = True
    As[2:4, 2:5] = True
    As[5, 2:5] = True
    Bs[2:4, 0:2] = True; Bs[5, 0:2] = True; Bs[6, 0] = True; Bs[7, 1] = True
    problem_set_dynamics(pbm, lib.MODEL_STARSHIP, mdl.par(), fcols=(0, 1), A_struct=As, B_struct=Bs)

    # set_convex_constraints!
    def X(t, k, x, p, pbm, ocp):
        m_ = pbm.mdl
        ocp.nonpos([x[3] * 1.0], "no_climb")
        ocp.nonpos([p[0] + p[1] - m_.tf_max], "max_time")
        ocp.nonpos([m_.tf_min - (p[0] + p[1])], "min_time")

    def U(t, k, u, p, pbm, ocp):
        m_ = pbm.mdl
        flip = t <= m_.tau_s
        T_max = m_.T_max3 if flip else m_.T_max1
        T_min = m_.T_min3 if flip else m_.T_min1
        ocp.nonpos([u[0] - T_max], "max_thrust")
        ocp.nonpos([T_min - u[0]], "min_thrust")
        ocp.l1([Expr.lift(m_.delta_max), u[1]], "gimbal")

    problem_set_X(pbm, X)
    problem_set_U(pbm, U)

    # set_nonconvex_constraints!: node-dependent structure of the device pack Constr<STARSHIP>
    ns = 7 + 2 * 8

    def phase_switch(t, N):          # definition.jl:707-714
        dt = 1 / (N - 1)
        return (mdl.tau_s - dt) + 1e-3 <= t and t <= mdl.tau_s + 1e-3

    def s_struct(t, k, pbm_):
        N = pbm_.scp.N
        Cm = np.zeros((ns, 8), bool); Dm = np.zeros((ns, 3), bool); Gm = np.zeros((ns, 10), bool)
        Cm[0, 7] = Cm[1, 7] = True
        Cm[4, 0] = Cm[4, 1] = True
        Dm[0, 1] = Dm[0, 2] = Dm[1, 1] = Dm[1, 2] = Dm[2, 2] = Dm[3, 2] = True
        psw = phase_switch(t, N)
        if psw:
            for i in range(8):
                Cm[5 + i, i] = Cm[13 + i, i] = True
                Gm[5 + i, 2 + i] = Gm[13 + i, 2 + i] = True
        if psw or t > mdl.tau_s:
            Cm[21, 4] = Cm[22, 4] = True
        return Cm, Dm, Gm

    problem_set_s(pbm, ns, s_struct)

    def p_stage(N):
        tg = np.arange(N) / (N - 1)
        ksw = [k for k in range(N) if phase_switch(tg[k], N)]
        return [-1, -1] + [ksw[0] if ksw else -1] * 8

    problem_advise_parameter_stage(pbm, p_stage)

    # set_bcs!
    def gic(x, p, pbm):
        m_ = pbm.mdl
        rhs = [m_.r0[0], m_.r0[1], m_.v0[0], m_.v0[1], m_.theta0, 0.0, 0.0]
        return [x[i] - rhs[i] for i in range(7)]

    def gtc(x, p, pbm):
        m_ = pbm.mdl
        rhs = [0.0, 0.0, m_.vf[0], m_.vf[1], 0.0, 0.0]
        return [x[i] - rhs[i] for i in range(6)]

    problem_set_bc(pbm, "ic", gic)
    problem_set_bc(pbm, "tc", gtc)
    problem_set_guess(pbm, lambda N, pbm_: starship_initial_guess(N, pbm_, handle))


# ------------------------------------------------------------------------------------------------
def _dynamics(m_, t, x, u, p, no_aero_torques=False):
    v = x[2:4]; th = x[4]; om = x[5]; dd = x[7]
    T, de = u[0], u[1]
    tdil = p[0] / m_.tau_s if t <= m_.tau_s else p[1] / (1 - m_.tau_s)
    ei = np.array([math.cos(th), math.sin(th)]); ej = np.array([-math.sin(th), math.cos(th)])
    Tv = T * (-math.sin(de) * ei + math.cos(de) * ej)
    D = -m_.CD * np.linalg.norm(v) * v
    MT = -m_.lcg * T * math.sin(de)
    MD = 0.0 if no_aero_torques else -(m_.lcp - m_.lcg) * (D @ ei)
    f = np.array([v[0], v[1], (Tv[0] + D[0]) / m_.m, (Tv[1] + D[1]) / m_.m - m_.g0, om, (MT + MD) / m_.J,
                  m_.alpha_e * T, (de - dd) / m_.rate_delay])
    return f * tdil


def _rk4(f, x0, ts):
    X = np.zeros((len(ts), x0.size)); X[0] = x0
    for k in range(1, len(ts)):
        t, h = ts[k - 1], ts[k] - ts[k - 1]
        x = X[k - 1]
        k1 = f(t, x); k2 = f(t + h / 2, x + h / 2 * k1); k3 = f(t + h / 2, x + h / 2 * k2); k4 = f(t + h, x + h * k3)
        X[k] = x + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
    return X


def _lin(a, b, n):
    j = np.arange(n) / (n - 1)
    return (1 - j) * a + j * b


def _sample(tg, X, t):
    t = max(tg[0], min(tg[-1], t))
    k = min(max(int(np.sum(t > tg)), 1), len(tg) - 1)
    c = (tg[k] - t) / (tg[k] - tg[k - 1])
    return c * X[k - 1] + (1 - c) * X[k]


def starship_initial_guess(N, pbm, handle):
    """definition.jl:97-445.  The terminal-descent SOCPs (one per candidate flight time, :395-413) are solved
    as ONE batch on the GPU cone solver instead of a sequential ECOS loop."""
    m_ = pbm.mdl
    tau = _lin(0.0, 1.0, N)
    id1 = np.where(tau <= m_.tau_s)[0]
    id2 = np.arange(id1[-1], N)
    xg = np.zeros((N, 8)); ug = np.zeros((N, 3))
    flip_ac = m_.lcg / m_.J * m_.T_min3 * math.sin(m_.delta_max)
    flip_ts = math.sqrt((m_.theta0 - m_.theta_s) / flip_ac)

    def ctrl(t):
        d = m_.delta_max if t <= flip_ts else (-m_.delta_max if t <= 2 * flip_ts else 0.0)
        return np.array([m_.T_min3, d, 0.0])

    pf = np.zeros(10); pf[0] = m_.tau_s; pf[1] = 1 - m_.tau_s
    x10 = np.zeros(8); x10[0:2] = m_.r0; x10[2:4] = m_.v0; x10[4] = m_.theta0; x10[7] = m_.delta_max
    tt = _lin(0.0, 2 * flip_ts + 10.0, 5000)
    x1 = _rk4(lambda t, x: _dynamics(m_, t, x, ctrl(t), pf, True), x10, tt)
    k0 = int(np.argmax(x1[:, 3] >= m_.vs @ m_.ey))
    tt, x1 = tt[:k0 + 1], x1[:k0 + 1]
    t1 = tt[-1]
    t_of = lambda ta: ta / m_.tau_s * t1
    for i in id1:
        xg[i] = _sample(tt, x1, t_of(tau[i])); ug[i] = ctrl(t_of(tau[i]))
    xs = _sample(tt, x1, t_of(tau[id1[-1]]))
    m_.hs = float(xs[0:2] @ m_.ey)
    tau2 = tau[id2] - tau[id2[0]]
    N2 = len(tau2)
    A_l = np.zeros((4, 4)); A_l[0, 2] = A_l[1, 3] = 1.0
    B_l = np.zeros((4, 2)); B_l[2, 0] = B_l[3, 1] = 1.0 / m_.m
    r_l = np.array([0.0, 0.0, 0.0, -m_.g0])
    dt = tau2[1] - tau2[0]

    def discretize(t2):
        td = t2 / (1 - m_.tau_s)

        def der(t, V):
            Phi = V[:16].reshape(4, 4, order="F")
            iP = np.linalg.solve(Phi, np.eye(4))
            return np.concatenate([((td * A_l) @ Phi).flatten(order="F"), (iP @ (td * B_l) * ((dt - t) / dt)).flatten(order="F"),
                                   (iP @ (td * B_l) * (t / dt)).flatten(order="F"), iP @ (td * r_l)])

        V0 = np.zeros(36); V0[:16] = np.eye(4).flatten(order="F")
        V = _rk4(der, V0, _lin(0.0, dt, 100))[-1]
        A = V[:16].reshape(4, 4, order="F")
        return A, A @ V[16:24].reshape(4, 2, order="F"), A @ V[24:32].reshape(4, 2, order="F"), A @ V[32:36]

    ztol = math.sqrt(np.finfo(float).eps)
    Sx, cx, Su, cu = np.ones(4), np.zeros(4), np.ones(2), np.zeros(2)

    def upd(S, c, i, lo, hi):
        lo, hi = min(lo, hi), max(lo, hi)
        if hi - lo > ztol:
            S[i] = hi - lo; c[i] = lo

    for i in range(4):
        upd(Sx, cx, i, 0, xs[i])
    Tmx = m_.T_max1 * math.sin(m_.thetamax2)
    upd(Su, cu, 0, -Tmx, Tmx); upd(Su, cu, 1, m_.T_min1, m_.T_max1)

    def program(t2):
        cvx = ConicTemplate(1)
        x = cvx.new_variable((4, N2), "x", Sx, cx, stage="col")
        u = cvx.new_variable((2, N2), "u", Su, cu, stage="col")
        x0 = [xs[0], xs[1], xs[2], xs[3]]; xf = [0.0, 0.0, m_.vf[0], m_.vf[1]]
        cvx.zero([x[i, 0] - x0[i] for i in range(4)]); cvx.zero([x[i, N2 - 1] - xf[i] for i in range(4)])
        A, Bm, Bp, r = discretize(t2)
        for k in range(N2 - 1):
            rhs = [a + b + c for a, b, c in zip(matvec(A, x[:, k]), matvec(Bm, u[:, k]), matvec(Bp, u[:, k + 1]))]
            cvx.zero([x[i, k + 1] - (rhs[i] + r[i]) for i in range(4)])
        for k in range(N2):
            cvx.soc([Expr.lift(m_.T_max1), u[0, k], u[1, k]])
            cvx.nonpos([m_.T_min1 - u[1, k]])
            cvx.soc([u[1, k] * (1.0 / math.cos(m_.thetamax2)), u[0, k], u[1, k]])
        for k in range(N2):
            cvx.nonpos([-x[1, k]])
        return cvx, cvx.compile()

    cands = np.arange(10.0, 41.0, 1.0)
    progs = [program(t2) for t2 in cands]
    cp0 = progs[0][1]
    one = np.ones(1)
    vals = np.array([cp["W"] @ one for _, cp in progs])
    from .. import ordering
    perm = ordering.stage_order(cp0["A"], cp0["G"], cp0["var_stage"], N2)
    cone = lib.ConeProblem(handle, cp0["A"], cp0["G"], cp0["l"], cp0["soc_dims"], perm=perm)
    nA, nG, n, p_, m = cp0["nnzA"], cp0["nnzG"], cp0["n"], cp0["p"], cp0["m"]
    out = cone.solve(vals[:, :nA], vals[:, nA:nA + nG], vals[:, cp0["off_c"]:cp0["off_c"] + n],
                     vals[:, cp0["off_b"]:cp0["off_b"] + p_], vals[:, cp0["off_h"]:cp0["off_h"] + m])
    cone.close()
    ok = np.where((out["status"] == 0) | (out["status"] == 3))[0]
    if ok.size == 0:
        raise lib.ScpbError("could not find a terminal descent time of flight")
    j = int(ok[0]); t2 = float(cands[j])
    z = out["x"][j]
    x2 = (z[:4 * N2].reshape(N2, 4) * Sx + cx).T
    T2 = (z[4 * N2:6 * N2].reshape(N2, 2) * Su + cu).T
    xg[id2, 0:2] = x2[0:2].T; xg[id2, 2:4] = x2[2:4].T
    td = t2 / (1 - m_.tau_s)
    m20 = xg[id2[0], 6]
    for k in range(N2):
        Tk = T2[:, k]; jn = id2[k]
        xg[jn, 4] = -math.atan2(Tk[0], Tk[1]); ug[jn, 0] = np.linalg.norm(Tk)
        if k > 0:
            xg[jn - 1, 5] = (xg[jn, 4] - xg[jn - 1, 4]) / ((tau2[k] - tau2[k - 1]) * td)
            f_ = m_.alpha_e * ug[id2[:k + 1], 0]; g_ = tau2[:k + 1] * td
            xg[jn, 6] = m20 + sum(0.5 * (g_[i + 1] - g_[i]) * (f_[i + 1] + f_[i]) for i in range(k))
    pg = np.zeros(10); pg[0] = t1; pg[1] = t2; pg[2:10] = xs
    return xg, ug, pg
