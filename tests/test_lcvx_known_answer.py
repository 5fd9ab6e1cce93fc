"""The reference's one numeric known answer for a CONE program: the lossless-convexification double integrator
(test/examples/double_integrator/definition.jl:38-118) against the maximum-principle solution `solve_mp` (:137-294).

    min  sum_k sigma2_k dt   s.t.  x_{k+1} = A x_k + B- u_k + B+ u_{k+1} + w,  x_1 = 0,  x_N = (s, 0),
         1 <= sigma_k <= 2,  |u_k| <= sigma_k  (L1 cone),  geomean(sigma2_k, 1) >= sigma_k  (GEOM cone, :89-92)

with the FOH data of parameters.jl:49-77 (N = 50, T = 10; friction g = 0.1 / 0.6 and travel s = 47 / 30 for the two parameter
sets).  The GEOM cone over two entries is the rotated second-order cone sigma2 * 1 >= sigma^2, i.e. the standard cone
|(2 sigma, sigma2 - 1)|_2 <= sigma2 + 1 -- the form MathOptInterface's bridges hand to ECOS.  `solve_mp` is restated below
(adjoint p(t) = c (t - ts), input law mp_input, RK4 roll-out, nested 25 x 25 grid search on (c, ts)): an ANALYTIC optimum, so
the SOC code paths of the oracle interior point and of the CUDA solver are checked against something neither of them
produced.  The two solutions differ by the first-order-hold discretisation (dt = 0.2 s; the input law has corners where it
saturates), which is what the tolerances below are: measured 0.046 / 0.056 on u at the interior nodes, 1.6e-3 / 4e-3 on the
states, 1.6e-3 / 1.0e-2 relative on the cost (the second parameter set pays for its backed-off end nodes)."""
import numpy as np
import pytest

from oracle import conic

N, T = 50, 10.0
DT = T / (N - 1)
PARS = {1: (0.1, 47.0, (-3.0, -1.0), (4.5, 5.5)), 2: (0.6, 30.0, (-1.5, -0.5), (6.5, 7.5))}   # g, s, c range, ts range


def mp_input(p):                                   # definition.jl:225-243
    if p > 4: return 2.0
    if p >= 2: return p / 2
    if p >= 0: return 1.0
    if p >= -2: return -1.0
    if p >= -4: return p / 2
    return -2.0


def mp_sim(g, s, c, ts):                           # definition.jl:259-294
    f = lambda t, x: np.array([x[1], mp_input(c * (t - ts)) - g])
    crit = sorted(tc for tc in (ts + a / c for a in (4, 2, 0, -2, -4)) if 0 <= tc <= T)
    knots = [0.0] + crit + [T]
    x = np.zeros(2)
    ts_all, xs_all = [], []
    for a, b in zip(knots[:-1], knots[1:]):
        grid = np.linspace(a, b, 100)
        for k in range(99):                         # rk4 (helper.jl:411-424)
            t, h = grid[k], grid[k + 1] - grid[k]
            k1 = f(t, x); k2 = f(t + h / 2, x + h / 2 * k1); k3 = f(t + h / 2, x + h / 2 * k2); k4 = f(t + h, x + h * k3)
            ts_all.append(t); xs_all.append(x.copy())
            x = x + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
    ts_all.append(T); xs_all.append(x.copy())
    return float(np.linalg.norm(x - np.array([s, 0.0]))), np.array(ts_all), np.array(xs_all)


def solve_mp(choice):                              # definition.jl:137-222 (grid refinement of the shooting parameters)
    g, s, (c0, c1), (t0, t1) = PARS[choice]
    cg, tg = np.linspace(c0, c1, 25), np.linspace(t0, t1, 25)
    for _ in range(10):
        err = np.array([[mp_sim(g, s, c, ts)[0] for c in cg] for ts in tg])
        i, j = np.unravel_index(np.argmin(err[1:-1, 1:-1]), (23, 23))
        i += 1; j += 1
        if err[i, j] <= 1e-2:
            break
        cg, tg = np.linspace(cg[j - 1], cg[j + 1], 25), np.linspace(tg[i - 1], tg[i + 1], 25)
    c, ts = cg[j], tg[i]
    e, tt, xx = mp_sim(g, s, c, ts)
    assert e <= 1e-2
    return c, ts, tt, xx


def lcvx_program(choice):
    """The cone program of solve_lcvx in the oracle's modelling layer; returns (compiled program, index of u, of sigma2)."""
    g, s = PARS[choice][:2]
    A = np.array([[1.0, DT], [0.0, 1.0]])
    Bm = np.array([DT * DT / 3, DT / 2]); Bp = np.array([DT * DT / 6, DT / 2])      # parameters.jl:63-73 in closed form
    w = np.array([-g * DT * DT / 2, -g * DT])
    P = conic.ConeProgram()
    x = P.new_variable((2, N), "x"); u = P.new_variable((1, N), "u")
    sg = P.new_variable((1, N), "sigma"); s2 = P.new_variable((1, N), "sigma2")
    P.zero([x[0, 0], x[1, 0]])
    P.zero([x[0, N - 1] - s, x[1, N - 1]])
    for k in range(N):
        P.nonpos([sg[0, k] - 2.0]); P.nonpos([1.0 - sg[0, k]])
        P.l1([sg[0, k], u[0, k]])
        P.geom([sg[0, k], s2[0, k], 1.0])          # GEOM (sigma; sigma2, 1), definition.jl:80-83
        if k < N - 1:
            for i in range(2):
                P.zero([x[i, k + 1] - (x[0, k] * A[i, 0] + x[1, k] * A[i, 1] + u[0, k] * Bm[i] + u[0, k + 1] * Bp[i] + w[i])])
    cost = conic.Aff()
    for k in range(N):
        cost = cost + s2[0, k] * DT
    P.add_cost(cost)
    return P.compile(), P.raw_index("u")[0], P.raw_index("sigma2")[0], P.raw_index("x")[0]


def _check_against_mp(choice, z, cost, iu, ix, tol_u, tol_J):
    c, ts, tt, xx = solve_mp(choice)
    tk = np.linspace(0.0, T, N)
    u_mp = np.array([mp_input(c * (t - ts)) for t in tk])
    # cost of the analytic solution: int max(|u|, 1)^2 dt  (sigma = max(|u|, 1) at the optimum, sigma2 = sigma^2)
    fine = np.linspace(0.0, T, 200001)
    J_mp = np.trapz(np.array([max(abs(mp_input(c * (t - ts))), 1.0) ** 2 for t in fine]), fine)
    # interior nodes only: the first and last input act through half a hold interval (B- u_1, B+ u_N) but pay a full
    # rectangle of cost, so the discrete optimum backs them off (u_1 = 1.15 instead of 2 for parameter set 2)
    eu = np.abs(z[iu + 1:iu + N - 1] - u_mp[1:-1]).max()
    x_mp = np.array([np.interp(tk, tt, xx[:, i]) for i in range(2)])
    ex = np.abs(z[ix:ix + 2 * N].reshape(N, 2).T - x_mp).max() / max(1.0, np.abs(x_mp).max())
    # the program's cost is the rectangle rule over the N nodes (definition.jl:107-110): compare like with like
    J_rect = float(np.sum(np.maximum(np.abs(u_mp), 1.0) ** 2) * DT)
    print(f"choice {choice}: c {c:.4f} ts {ts:.4f}  |u - u_mp|_inf {eu:.3e}  x rel {ex:.3e}  cost {cost:.6f}  J_mp(rect) {J_rect:.6f}  J_mp(int) {J_mp:.6f}")
    assert eu <= tol_u and ex <= 5e-3
    assert abs(cost - J_rect) <= tol_J * J_rect


@pytest.mark.parametrize("choice", [1, 2])
def test_oracle_interior_point_reproduces_the_maximum_principle_solution(choice):
    cp, iu, is2, ix = lcvx_program(choice)
    r = conic.solve_ipm(cp, tol=1e-10)
    assert r["status"] == "OPTIMAL"
    _check_against_mp(choice, r["z"], r["obj"], iu, ix, 0.08, 2e-2)


@pytest.mark.gpu
def test_cuda_cone_solver_reproduces_the_maximum_principle_solution(pkg, handle):
    """Both parameter sets as one batch of two seeds through scpb_cone_solve (they share the pattern; b and h differ)."""
    cps = [lcvx_program(ch) for ch in (1, 2)]
    cp0 = cps[0][0]
    for cp, *_ in cps[1:]:
        assert (cp["A"].indices == cp0["A"].indices).all() and (cp["G"].indices == cp0["G"].indices).all()
    cone = pkg.lib.ConeProblem(handle, cp0["A"], cp0["G"], cp0["l"], cp0["q"], perm=pkg.ordering.rcm_order(cp0["A"], cp0["G"]))
    A0, G0 = cp0["A"].tocsr(), cp0["G"].tocsr()
    for cp, *_ in cps:
        cp["A"].sort_indices(); cp["G"].sort_indices()
    out = cone.solve(np.array([cp["A"].data for cp, *_ in cps]), np.array([cp["G"].data for cp, *_ in cps]),
                     np.array([cp["c"] for cp, *_ in cps]), np.array([cp["b"] for cp, *_ in cps]),
                     np.array([cp["h"] for cp, *_ in cps]))
    cone.close()
    print("statuses", out["status"], "iterations", out["iters"])
    # OPTIMAL or ALMOST_OPTIMAL (measured: the solver's floor on these SOC programs sits near 1e-9, at 1e-10 it reports
    # ALMOST_OPTIMAL after 15-16 iterations); what counts is the agreement with the oracle and the analytic optimum below
    assert all(int(s_) in (0, 3) for s_ in out["status"]), (out["status"], out["iters"])
    for b, (cp, iu, is2, ix) in enumerate(cps):
        ref = conic.solve_ipm(cp, tol=1e-10)
        cost = float(cp["c"] @ out["x"][b]) + cp["c0"]
        # against the oracle's interior point: the same optimum of the same (strictly convex in sigma2, u) program
        print("seed", b, "cost", cost, ref["obj"], "max |u - u_oracle|", np.abs(out["x"][b][iu:iu + N] - ref["z"][iu:iu + N]).max())
        assert abs(cost - ref["obj"]) <= 1e-6 * max(1.0, abs(ref["obj"]))
        assert np.abs(out["x"][b][iu:iu + N] - ref["z"][iu:iu + N]).max() <= 3e-4   # both solvers at 1e-8 / 1e-10
        # ... and against the analytic optimum
        _check_against_mp(b + 1, out["x"][b], cost, iu, ix, 0.08, 2e-2)
