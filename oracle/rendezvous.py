"""Oracle planar rendezvous (test/examples/rendezvous_planar) and the IMPULSE flavour of the oracle PTR loop.
TEST INFRASTRUCTURE ONLY.

  PlanarRendezvousProblem   parameters.jl:80-152, definition.jl:22-475
  smooth_or                 or -> indicator -> sigmoid -> logsumexp (src/utils/helper.jl:600-807), in the reference's
                            operation order: at the last homotopy step the sigmoid saturates to exactly 1 and the
                            gradient factor to exactly 0, and the device pack must saturate on the same inputs
  Homotopy                  src/utils/homotopy.jl
  ImpulsePTR                oracle/ptr.PTR with discretize! (IMPULSE) and the dynamics rows of state_update!'s IMPULSE
                            branch (discretization.jl:469-494): no u_{k+1} term
"""
from __future__ import annotations

import math

import numpy as np

from . import orc
from .ptr import PTR, Parameters
from .problems import deg2rad


def _exp(v):
    """exp with IEEE overflow to +Inf (Julia's exp; math.exp raises instead)"""
    try:
        return math.exp(v)
    except OverflowError:
        return math.inf


def _logsumexp(f, df, t):
    """logsumexp(f, df; t) (helper.jl:623-651) for scalar predicates with scalar gradients (df may be None)"""
    a = max(t * fi for fi in f)
    E = 0.0
    for fi in f:
        E = E + _exp(t * fi - a)
    L = (a + math.log(E)) / t
    if df is None:
        return L, None
    dL = 0.0
    for fi, gi in zip(f, df):
        dL = dL + gi * (_exp(t * fi - a) / E)
    return L, dL


def _sigmoid(f, df, kappa):
    """sigmoid(value, gradient; kappa) (helper.jl:672-701)"""
    L, dL = _logsumexp(f, df, kappa)
    sg = 1 - 1 / (1 + _exp(kappa * L))
    if df is None:
        return sg, None
    c = _exp(kappa * L + 2 * math.log(1 - sg)) if sg < 1 else 0.0    # log(0) = -Inf -> exp = 0, as in Julia
    return sg, kappa * c * dL


def smooth_or(fr, kappa, f_db, f_max):
    """OR and dOR/dfr of the deadband predicate of one thruster (definition.jl:355-396):
    or([fr - f_db, -f_db - fr], [[1], [-1]]; kappa, match = [f_max - f_db, -f_db - f_max], normalize = f_max + f_db)"""
    nrm = f_max + f_db
    pred = [(fr - f_db) / nrm, (-f_db - fr) / nrm]
    grad = [1.0 / nrm, -1.0 / nrm]
    match = [(f_max - f_db) / nrm, (-f_db - f_max) / nrm]
    offset, _ = _sigmoid(match, None, kappa)           # indicator: y-shift matching the exact value at `match`
    dsg = 1 - offset
    sg, dOR = _sigmoid(pred, grad, kappa)
    return sg + dsg, dOR


class Homotopy:             # src/utils/homotopy.jl
    def __init__(self, delta_min, delta_max=1.0, eps=1e-2):
        self.eps, self.delta_min, self.delta_max = eps, delta_min, delta_max
        self.rho = delta_min / delta_max

    def __call__(self, x):
        return math.log(1 / self.eps - 1) / (self.rho ** x * self.delta_max)


def hom_grid(n):
    """LinRange(0.0, 1.0, n)"""
    return orc.t_grid(n)


class PlanarRendezvousProblem:
    """parameters.jl:80-152 and definition.jl:22-475 (PTR flavour)."""
    name = "rendezvous_planar"
    model_id = orc.MODEL_RENDEZVOUS2D
    nx, nu, np = 6, 12, 1
    ns = 6

    def __init__(self, N: int = 30):
        self.N = N
        mu, Re = 3.986e14, 6378e3
        R = Re + 400e3
        self.n = math.sqrt(mu / (R * R * R))
        self.m, self.J, self.lu, self.lv = 30e3, 1e5, 0.6, 2.1
        self.f_max, self.f_db = 750.0, 200.0
        self.r0, self.v0 = np.array([100.0, 10.0]), np.array([0.0, 0.0])
        self.th0, self.om0, self.vf = deg2rad(180.0), 0.0, 0.1
        self.tf_min, self.tf_max = 100.0, 500.0
        self.kappa = float("nan")
        self.gamma = 3e-1
        self.id_f, self.id_fr, self.id_l1f, self.id_l1feq = range(0, 3), range(3, 6), range(6, 9), range(9, 12)

    def par(self):
        """dynamics pack m, J, lu, lv, n, then the constraint pack f_db, f_max, kappa (include/scpb.h)"""
        return np.array([self.m, self.J, self.lu, self.lv, self.n, self.f_db, self.f_max, self.kappa])

    def orc_model(self):
        return orc.make_model(self.model_id, self.nx, self.nu, self.np, self.par()[:5])

    def ranges(self):       # set_scale!, definition.jl:43-92
        rx0, ry0, vx0, vy0 = self.r0[0], self.r0[1], self.v0[0], self.v0[1]
        tmin = self.tf_min
        xrg = [(0.0, max(rx0, 1.0)), (min(ry0, -0.1), max(ry0, 0.1)),
               (min(vx0, -rx0 / tmin, -0.1), min(vx0, 0.1)), (min(vy0, -ry0 / tmin, -0.1), max(vy0, -ry0 / tmin, 0.1)),
               (min(self.th0, deg2rad(-1.0)), max(self.th0, deg2rad(1.0))),
               (min(-self.th0 / tmin, self.om0, deg2rad(-1.0)), max(-self.th0 / tmin, self.om0, deg2rad(1.0)))]
        urg = [(-self.f_max, self.f_max)] * 6 + [(0.0, self.f_max)] * 3 + [(0.0, 2 * self.f_max)] * 3
        return xrg, urg, [(self.tf_min, self.tf_max)]

    def guess(self, N):     # set_guess!, definition.jl:94-124
        p = np.array([0.5 * (self.tf_min + self.tf_max)])
        x0 = np.concatenate([self.r0, -self.r0 / p[0], [self.th0, -self.th0 / p[0]]])
        xf = np.zeros(6)
        xf[2:4] = x0[2:4]
        xf[5] = x0[5]
        t = orc.t_grid(N)
        c = [(1.0 - t[k]) / (1.0 - 0.0) for k in range(N)]      # linterp on [0, 1], helper.jl:107-118
        x = np.array([c[k] * x0 + (1 - c[k]) * xf for k in range(N)])
        return x, np.zeros((N, 12)), p

    def cost_aff(self, x, u, p, t):     # set_cost!, definition.jl:126-144, trapezoid rule of scp.jl
        from . import conic
        from .ptr import trapz
        run = []
        for k in range(len(t)):
            r = conic.Aff()
            for i in self.id_l1f:
                r = r + u[i, k]
            r = r / self.f_max
            q = conic.Aff()
            for i in self.id_l1feq:
                q = q + u[i, k]
            run.append(r + (q * self.gamma) / self.f_max)
        return trapz(run, t)

    # nonconvex constraints, definition.jl:337-413; k is 1-based
    def s(self, t, k, x, u, p):
        s = np.zeros(self.ns)
        for i in range(3):
            f, fr = u[self.id_f[i]], u[self.id_fr[i]]
            OR, _ = smooth_or(fr, self.kappa, self.f_db, self.f_max)
            s[2 * i] = f - OR * fr
            s[2 * i + 1] = OR * fr - f
        return s

    def C(self, t, k, x, u, p):
        return np.zeros((self.ns, self.nx))

    def D(self, t, k, x, u, p):
        D = np.zeros((self.ns, self.nu))
        for i in range(3):
            fr = u[self.id_fr[i]]
            OR, dOR = smooth_or(fr, self.kappa, self.f_db, self.f_max)
            dORfr = dOR * fr + OR
            D[2 * i, self.id_f[i]] = 1.0
            D[2 * i, self.id_fr[i]] = -dORfr
            D[2 * i + 1, self.id_f[i]] = -1.0
            D[2 * i + 1, self.id_fr[i]] = dORfr
        return D

    def G(self, t, k, x, u, p):
        return np.zeros((self.ns, self.np))

    def gic(self, x, p):
        return x[0:6] - np.concatenate([self.r0, self.v0, [self.th0, self.om0]])

    def H0(self, x, p):
        return np.eye(6)

    K0 = None

    def gtc(self, x, p):
        return x[0:6] - np.array([0.0, 0.0, -self.vf * 1.0, -self.vf * 0.0, 0.0, 0.0])

    def Hf(self, x, p):
        return np.eye(6)

    Kf = None

    def emit_U(self, prg, t, k, u, p):      # set_convex_constraints!, definition.jl:244-335
        for i in range(3):
            f, fr, l1f, l1feq = u[self.id_f[i]], u[self.id_fr[i]], u[self.id_l1f[i]], u[self.id_l1feq[i]]
            prg.nonpos([l1f - self.f_max], "thrust_absval_max")
            prg.nonpos([fr - self.f_max], "thrust_refval_max")
            prg.nonpos([-fr - self.f_max], "thrust_refval_min")
            prg.l1([l1f, f], "thrust_absval")
            prg.l1([l1feq, f - fr], "thrust_absval")
        prg.nonpos([p[0] - self.tf_max], "min_time_bound")
        prg.nonpos([self.tf_min - p[0]], "max_time_bound")


def perturbed_guesses(pb, nb, seed):
    """Seeded perturbations of the straight-line guess: states moved by 2% of their advised ranges, random reference
    thrusts fr within +-300 N (across the deadband), flight time within +-10%."""
    rng = np.random.default_rng(seed)
    N = pb.N
    x, u, p = pb.guess(N)
    xrg, _, _ = pb.ranges()
    Sx = np.array([r[1] - r[0] for r in xrg])
    X = x + 0.02 * Sx * rng.standard_normal((nb, N, pb.nx))
    U = np.tile(u, (nb, 1, 1))
    U[..., 3:6] = rng.uniform(-300.0, 300.0, (nb, N, 3))
    P = p * (1 + 0.1 * rng.uniform(-1.0, 1.0, (nb, 1)))
    return X, U, P


def ptr_parameters(N=30, Nsub=10, iter_max=30, solver_tol=1e-11):
    """tests.jl:31-58"""
    return Parameters(N=N, Nsub=Nsub, iter_max=iter_max, wvc=5e2, wtr=3e-2, eps_abs=-np.inf, eps_rel=1e-3 / 100,
                      feas_tol=5e-3, q_tr=np.inf, q_exit=np.inf, solver_tol=solver_tol)


class ImpulsePTR(PTR):
    """The oracle PTR loop with IMPULSE discretization.  The constraint pack reads pb.kappa whenever a subproblem is
    built, so set_kappa between two solve() calls is the reference's `mdl.traj.kappa = hom_kappa(...)`."""

    def set_kappa(self, kappa):
        self.pb.kappa = float(kappa)

    def make_solution(self, xd, ud, p):
        d = orc.discretize_impulse(self.model, xd, ud, p, self.pars.Nsub, self.scale.iSx, self.pars.feas_tol, self.t)
        d.Bp = np.zeros_like(d.Bm)      # conic.matvec skips zeros: the dynamics rows carry no u_{k+1} term
        from .ptr import Solution
        return Solution(xd=np.array(xd, dtype=float), ud=np.array(ud, dtype=float), p=np.array(p, dtype=float),
                        dyn=d, feas=d.feas, defect=d.defect)


def homotopy_sweep(pb, guess, n_hom=10, pars=None, prefer="ipm", steps=None, verbose=False):
    """tests.jl:60-79: kappa steps through Homotopy(1e-3; delta_max = 5)(LinRange(0, 1, n_hom)), every solve warm-started
    from the previous one.  Returns one result dict (oracle/ptr.PTR.solve) per step, with 'kappa' added."""
    hom = Homotopy(1e-3, delta_max=5.0)
    grid = hom_grid(n_hom)
    P = ImpulsePTR(pb, pars or ptr_parameters(pb.N))
    out = []
    g = guess
    for i in range(n_hom if steps is None else steps):
        P.set_kappa(hom(grid[i]))
        r = P.solve(g, prefer=prefer)
        r["kappa"] = pb.kappa
        if verbose:
            print(f"[{i + 1}/{n_hom}] kappa={pb.kappa:.3e} {r['status']} it {r['iterations']} J {r['sol'].J_aug:.9e}",
                  flush=True)
        out.append(r)
        s = r["sol"]
        g = (s.xd, s.ud, s.p)
    return out
