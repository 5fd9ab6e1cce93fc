"""Oracle forced harmonic oscillator with an input deadband (test/examples/oscillator) and its FOH PTR loop with a settable
kappa.  TEST INFRASTRUCTURE ONLY.

  OscillatorProblem      parameters.jl:69-115, definition.jl:22-473 (PTR flavour): a FIXED final time, so F = 0 and the
                         dynamics read no parameter; p holds one slack l1r_k >= |r_k| per node
  smooth_or_general      or(pred, grad; kappa, match, normalize) -> indicator -> sigmoid -> logsumexp (helper.jl:760-807)
                         on the sigmoid of oracle/rendezvous.py, for a match of one value or one per predicate; with the
                         planar arguments it gives the bits of oracle/rendezvous.smooth_or (a CPU test checks this)
  smooth_or              the deadband's OR (definition.jl:381-389): a SCALAR match, so the indicator's y-shift is the
                         sigmoid of a one-element vector
  discretize, propagate  discretize! (FOH, discretization.jl:160-217, 235-286, 354-406) and propagate (:515-562) for this
                         LTI model, restated in numpy: the C oracle's model table has no pack with F = 0
  OscillatorPTR          oracle/ptr.PTR (FOH) on that discretization, whose constraint rows read pb.kappa when a
                         subproblem is built
  OscillatorCallbackPTR  the same loop with the in-loop homotopy callback of oracle/homotopy_update.py
  homotopy_sweep         tests.jl:60-80: kappa = Homotopy(1e-8)(LinRange(0, 1, 10)[i]), every solve warm-started
"""
from __future__ import annotations

import numpy as np

from . import homotopy_update as hu
from . import orc
from .ptr import PTR, Parameters, Scaling, Solution
from .rendezvous import Homotopy, _sigmoid, hom_grid

MODEL_OSCILLATOR = 7        # SCPB_MODEL_OSCILLATOR, include/scpb.h


def smooth_or_general(pred, grad, kappa, match, normalize):
    """or(pred, grad; kappa, match, normalize) (helper.jl:760-807) of scalar predicates with scalar gradients: OR and
    its gradient.  match is one value (the indicator then takes the sigmoid of a one-element vector) or one per
    predicate."""
    match = list(match) if hasattr(match, "__len__") else [match]
    m = [v / normalize for v in match]
    f = [v / normalize for v in pred]
    g = [v / normalize for v in grad]
    offset, _ = _sigmoid(m, None, kappa)               # indicator: y-shift matching the exact value at `match`
    dsg = 1 - offset
    sg, dOR = _sigmoid(f, g, kappa)
    return sg + dsg, dOR


def smooth_or(ar, kappa, a_db, a_max):
    """OR and dOR/dar of the deadband predicate (definition.jl:381-389, 415-427):
    or([ar - a_db, -a_db - ar], [[1], [-1]]; kappa, match = a_max - a_db, normalize = a_max - a_db)"""
    return smooth_or_general([ar - a_db, -a_db - ar], [1.0, -1.0], kappa, a_max - a_db, a_max - a_db)


def hom():
    """the homotopy of tests.jl:61: Homotopy(1e-8), kappa from log(99) ~ 4.6 to 4.6e8"""
    return Homotopy(1e-8)


def rk4(f, x0, tspan):
    """rk4_generic(f, x0; tspan, full = true) (helper.jl:411-424, 451-501): the states at every point of tspan"""
    X = np.zeros((len(tspan), len(x0)))
    X[0] = x0
    for k in range(1, len(tspan)):
        t, tp, x = tspan[k - 1], tspan[k], X[k - 1]
        h = tp - t
        k1 = f(t, x)
        k2 = f(t + h / 2, x + h / 2 * k1)
        k3 = f(t + h / 2, x + h / 2 * k2)
        k4 = f(t + h, x + h * k3)
        X[k] = x + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
    return X


def linterp(t, F, grid):
    """linterp(t, f_cps, t_grid) (helper.jl:107-118), F[k] the value at grid[k]"""
    t = max(grid[0], min(grid[-1], t))
    k = max(int(np.sum(t > grid)), 1)          # get_interval, 1-based: the interval [grid[k-1], grid[k]] 0-based
    c = (grid[k] - t) / (grid[k] - grid[k - 1])
    return c * F[k - 1] + (1 - c) * F[k]


class OscillatorProblem:
    """parameters.jl:69-115 and definition.jl:22-473 (PTR flavour).  Indices are 0-based; the k the reference hands the
    closures is 1-based."""
    name = "oscillator"
    model_id = MODEL_OSCILLATOR
    nx, nu = 2, 4
    ns = 2

    def __init__(self, N: int = 30):
        self.N = N
        self.np = N                                     # id_l1r = 1:N
        self.zeta, self.omega0 = 0.5, 1.0
        self.a_db, self.a_max = 0.05, 0.3
        self.r0, self.v0, self.tf = 1.0, 0.0, 10.0
        self.kappa = float("nan")                       # kappa1, set by the homotopy before every solve
        self.alpha, self.gamma = 0.06, 1e-1
        self.id_r, self.id_v = 0, 1
        self.id_aa, self.id_ar, self.id_l1aa, self.id_l1adiff = 0, 1, 2, 3

    def par(self):
        """dynamics pack zeta, omega0, tf, then the constraint pack a_db, a_max, kappa (include/scpb.h)"""
        return np.array([self.zeta, self.omega0, self.tf, self.a_db, self.a_max, self.kappa])

    def ranges(self):       # set_scale!, definition.jl:47-69
        xrg = [(-self.r0, self.r0), (-self.v0, self.v0)]
        urg = [(-self.a_max, self.a_max)] * 2 + [(0.0, self.a_max), (0.0, 2 * self.a_max)]
        return xrg, urg, [(0.0, self.r0)] * self.N

    def dynamics(self, x, u):
        """dynamics(t, k >= 0, x, u, p) (definition.jl:161-192)"""
        f = np.zeros(2)
        f[1] = u[0]
        f[0] = x[1]
        f[1] += -self.omega0 ** 2 * x[0] - 2 * self.zeta * self.omega0 * x[1]
        return f * self.tf

    def A(self):
        """df/dx (definition.jl:203-213), constant"""
        A = np.zeros((2, 2))
        A[self.id_r, self.id_v] = 1.0
        A[self.id_v, self.id_r] = -self.omega0 ** 2
        A[self.id_v, self.id_v] = -2 * self.zeta * self.omega0
        return A * self.tf

    def B(self):
        """df/du (definition.jl:215-226, k >= 0), constant"""
        B = np.zeros((2, self.nu))
        B[self.id_v, self.id_aa] = 1.0
        return B * self.tf

    def guess(self, N):     # set_guess!, definition.jl:71-114
        x0 = np.array([self.r0, self.v0])
        t_grid, tau = orc.t_grid(1000), orc.t_grid(N)
        X = rk4(lambda t, x: self.dynamics(x, np.zeros(self.nu)), x0, t_grid)
        x = np.array([linterp(tau[k], X, t_grid) for k in range(N)])
        p = np.array([abs(x[k, self.id_r]) for k in range(N)])      # norm(x[id_r, k], 1)
        return x, np.zeros((N, self.nu)), p

    def cost_aff(self, x, u, p, t):     # set_cost!, definition.jl:116-142, trapezoid rule of scp.jl
        from .ptr import trapz
        run = []
        for k in range(len(t)):
            f = p[k] / self.r0
            f = f + u[self.id_l1aa, k] * self.alpha / self.a_max
            f = f + u[self.id_l1adiff, k] * self.gamma / self.a_max
            run.append(f)
        return trapz(run, t)

    # nonconvex constraints, definition.jl:370-444; k is 1-based
    def s(self, t, k, x, u, p):
        aa, ar = u[self.id_aa], u[self.id_ar]
        OR, _ = smooth_or(ar, self.kappa, self.a_db, self.a_max)
        return np.array([aa - OR * ar, OR * ar - aa])

    def C(self, t, k, x, u, p):
        return np.zeros((self.ns, self.nx))

    def D(self, t, k, x, u, p):
        ar = u[self.id_ar]
        OR, dOR = smooth_or(ar, self.kappa, self.a_db, self.a_max)
        dORar = dOR * ar + OR
        D = np.zeros((self.ns, self.nu))
        D[0, self.id_aa], D[0, self.id_ar] = 1.0, -dORar
        D[1, self.id_aa], D[1, self.id_ar] = -1.0, dORar
        return D

    def G(self, t, k, x, u, p):
        return np.zeros((self.ns, self.np))

    def gcols(self, k):     # the device pack's packed ds/dp column at node k (0-based): the node's own slack
        return [k]

    def gic(self, x, p):    # set_bcs!, definition.jl:446-473
        return x[0:2] - np.array([self.r0, self.v0])

    def H0(self, x, p):
        return np.eye(2)

    K0 = None
    gtc = None

    def emit_X(self, prg, t, k, x, p):      # set_convex_constraints!, definition.jl:240-272
        prg.l1([p[k - 1], x[self.id_r]], "abs_r")

    def emit_U(self, prg, t, k, u, p):      # definition.jl:274-365
        aa, ar, l1aa, l1adiff = u[self.id_aa], u[self.id_ar], u[self.id_l1aa], u[self.id_l1adiff]
        prg.nonpos([aa - self.a_max], "accel_bounds")
        prg.nonpos([-self.a_max - aa], "accel_bounds")
        prg.nonpos([ar - self.a_max], "accel_bounds")
        prg.nonpos([-self.a_max - ar], "accel_bounds")
        prg.l1([l1aa, aa], "accel_bounds")
        prg.l1([l1adiff, aa - ar], "accel_bounds")


def _linrange_at(a, b, j, d):
    """LinRange(a, b, d + 1)[j + 1] with Julia's lerpi arithmetic"""
    t = j / d
    return (1.0 - t) * a + t * b


def discretize(pb, xd, ud, p, Nsub, iSx_diag, feas_tol, tg=None) -> orc.DLTV:
    """discretize! (FOH) for one trajectory, xd (N, nx), ud (N, nu): RK4 (helper.jl:411-424) over
    LinRange(t_k, t_k+1, Nsub) of V = [x; Phi; PB-; PB+; Pr; PE] with derivs_foh (discretization.jl:235-286), then
    set_update_matrices (:354-406) and the defects (:205-210).  F = 0: the model has no time-dilation parameter, so
    the PF block is empty and the returned F is all zeros (nx x np)."""
    xd, ud = np.asarray(xd, dtype=float), np.asarray(ud, dtype=float)
    N, nx, nu = xd.shape[0], pb.nx, pb.nu
    tg = orc.t_grid(N) if tg is None else np.asarray(tg, dtype=float)
    Ac, Bc = pb.A(), pb.B()
    sizes = [nx, nx * nx, nx * nu, nx * nu, nx, nx * nx]          # x, Phi, PB-, PB+, Pr, PE (column-major blocks)
    offs = np.cumsum([0] + sizes)
    unpack = lambda V: [V[offs[i]:offs[i + 1]].reshape(-1, 1 if i in (0, 4) else sizes[i] // nx, order="F")
                        for i in range(6)]
    M = N - 1
    out = dict(A=np.zeros((M, nx, nx)), Bm=np.zeros((M, nx, nu)), Bp=np.zeros((M, nx, nu)), F=np.zeros((M, nx, pb.np)),
               r=np.zeros((M, nx)), E=np.zeros((M, nx, nx)), defect=np.zeros((M, nx)))
    feas = True
    for k in range(M):
        t1, t2, uk, ukp1 = tg[k], tg[k + 1], ud[k], ud[k + 1]

        def derivs(t, V):
            x, Phi = unpack(V)[0][:, 0], unpack(V)[1]
            ts = max(t1, min(t2, t))
            cc = (t2 - ts) / (t2 - t1)
            u = cc * uk + (1.0 - cc) * ukp1
            sm, sp = (t2 - t) / (t2 - t1), (t - t1) / (t2 - t1)
            f = pb.dynamics(x, u)
            r = f - Ac @ x - Bc @ u
            iPhi = np.linalg.inv(Phi)
            blocks = [f, Ac @ Phi, iPhi @ (sm * Bc), iPhi @ (sp * Bc), iPhi @ r, iPhi]
            return np.concatenate([np.asarray(b).ravel(order="F") for b in blocks])

        V = np.zeros(offs[-1])
        V[0:nx] = xd[k]
        V[offs[1]:offs[2]] = np.eye(nx).ravel(order="F")
        for j in range(1, Nsub):
            t, tp = _linrange_at(t1, t2, j - 1, Nsub - 1), _linrange_at(t1, t2, j, Nsub - 1)
            h = tp - t
            k1 = derivs(t, V)
            k2 = derivs(t + h / 2, V + h / 2 * k1)
            k3 = derivs(t + h / 2, V + h / 2 * k2)
            k4 = derivs(t + h, V + h * k3)
            V = V + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
        x, Phi, PBm, PBp, Pr, PE = unpack(V)
        out["A"][k], out["Bm"][k], out["Bp"][k] = Phi, Phi @ PBm, Phi @ PBp
        out["r"][k], out["E"][k] = (Phi @ Pr)[:, 0], Phi @ PE
        out["defect"][k] = xd[k + 1] - x[:, 0]
        if np.abs(np.asarray(iSx_diag) * out["defect"][k]).max() > feas_tol:
            feas = False
    return orc.DLTV(out["A"], out["Bm"], out["Bp"], out["F"], out["r"], out["E"], out["defect"], feas)


def propagate(pb, xd, ud, p, res):
    """propagate(sol, pbm; res) (discretization.jl:515-562, FOH branch): RK4 of f over LinRange(0, 1, res) from xd[0],
    the input linearly interpolated over the whole time grid; (res, nx)"""
    xd, ud = np.asarray(xd, dtype=float), np.asarray(ud, dtype=float)
    tg = orc.t_grid(xd.shape[0])
    X = np.zeros((res, pb.nx))
    X[0] = xd[0]
    for j in range(1, res):
        t, tp = _linrange_at(0.0, 1.0, j - 1, res - 1), _linrange_at(0.0, 1.0, j, res - 1)
        h, x = tp - t, X[j - 1]
        k1 = pb.dynamics(x, linterp(t, ud, tg))
        k2 = pb.dynamics(x + h / 2 * k1, linterp(t + h / 2, ud, tg))
        k3 = pb.dynamics(x + h / 2 * k2, linterp(t + h / 2, ud, tg))
        k4 = pb.dynamics(x + h * k3, linterp(t + h, ud, tg))
        X[j] = x + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
    return X


def perturbed_guesses(pb, nb, seed):
    """Seeded perturbations of the reference guess: states moved by 2% of their scale (the advised range; 1 for the
    velocity, whose advised range is empty), random reference accelerations ar within +-a_max (across the deadband) and
    the slacks l1r_k = |r_k| of the moved states."""
    rng = np.random.default_rng(seed)
    N = pb.N
    x, u, _ = pb.guess(N)
    xrg, _, _ = pb.ranges()
    Sx = np.array([r[1] - r[0] for r in xrg])
    Sx[Sx < np.sqrt(np.finfo(float).eps)] = 1.0
    X = x + 0.02 * Sx * rng.standard_normal((nb, N, pb.nx))
    U = np.tile(u, (nb, 1, 1))
    U[..., pb.id_ar] = rng.uniform(-pb.a_max, pb.a_max, (nb, N))
    P = np.abs(X[..., pb.id_r])
    return X, U, P


def ptr_parameters(N=30, Nsub=10, iter_max=10, solver_tol=1e-11):
    """tests.jl:24-58: FOH, q_tr = q_exit = Inf"""
    return Parameters(N=N, Nsub=Nsub, iter_max=iter_max, wvc=1e2, wtr=1e-3, eps_abs=-np.inf, eps_rel=1e-3 / 100,
                      feas_tol=5e-3, q_tr=np.inf, q_exit=np.inf, solver_tol=solver_tol)


class OscillatorPTR(PTR):
    """The oracle FOH PTR loop on the numpy discretization above.  The constraint rows read pb.kappa whenever a
    subproblem is built, so set_kappa between two solve() calls is the reference's `mdl.traj.κ1 = hom_κ1(...)`."""

    def __init__(self, pb, pars: Parameters):      # oracle/ptr.PTR.__init__ without the C model
        self.pb, self.pars = pb, pars
        self.scale = Scaling(pb, pars.N)
        self.t = orc.t_grid(pars.N)

    def make_solution(self, xd, ud, p):
        d = discretize(self.pb, xd, ud, p, self.pars.Nsub, self.scale.iSx, self.pars.feas_tol, self.t)
        return Solution(xd=np.array(xd, dtype=float), ud=np.array(ud, dtype=float), p=np.array(p, dtype=float),
                        dyn=d, feas=d.feas, defect=d.defect)

    def set_kappa(self, kappa):
        self.pb.kappa = float(kappa)


class OscillatorCallbackPTR(OscillatorPTR):
    """OscillatorPTR with the in-loop homotopy callback (oracle/homotopy_update.py)."""
    solve_with_schedule = hu.CallbackPTR.solve_with_schedule


def homotopy_sweep(pb, guess, n_hom=10, pars=None, prefer="ipm", steps=None, verbose=False):
    """tests.jl:60-80: kappa steps through Homotopy(1e-8)(LinRange(0, 1, n_hom)), every solve warm-started from the
    previous one.  Returns one result dict (oracle/ptr.PTR.solve) per step, with 'kappa' added."""
    h = hom()
    grid = hom_grid(n_hom)
    P = OscillatorPTR(pb, pars or ptr_parameters(pb.N))
    out = []
    g = guess
    for i in range(n_hom if steps is None else steps):
        P.set_kappa(h(grid[i]))
        r = P.solve(g, prefer=prefer)
        r["kappa"] = pb.kappa
        if verbose:
            print(f"[{i + 1}/{n_hom}] kappa={pb.kappa:.3e} {r['status']} it {r['iterations']} J {r['sol'].J_aug:.9e}",
                  flush=True)
        out.append(r)
        s = r["sol"]
        g = (s.xd, s.ud, s.p)
    return out

