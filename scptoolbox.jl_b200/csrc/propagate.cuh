// propagate.cuh -- final continuous-time propagation of a converged SCP solution.
//
// Replaces propagate(sol, pbm; res) (src/solvers/discretization.jl:515-562, FOH branch :533-538), called once per
// trajectory by SCPSolution (src/solvers/scp.jl:231-232 with res = 2*Nsub*(N-1)): classic RK4 (helper.jl:411-424,
// 451-501) of the nonlinear dynamics over tc = LinRange(0, 1, res), the input linearly interpolated over the WHOLE
// time grid (helper.jl:84-118), integration actions after every step (helper.jl:492-496).  The reference's k(t)
// helper always evaluates to N (discretization.jl:530); no shipped model reads it.
//
// The integration is an initial-value problem: sequential in time, independent across seeds -> one thread per seed.
// It runs once per solve (19 800 steps for the starship bench configuration), not once per SCP iteration.
// Time arithmetic uses the round-to-nearest intrinsics in the reference's operation order (same reason as in
// discretize.cuh: the starship model switches phase on `t <= tau_s`).
#pragma once
#include "models.cuh"

struct PropArgs {
    int B, N, res;
    const double *t_grid;   // [N]
    const double *xd;       // [B][N][nx]  (only node 0 is read)
    const double *ud;       // [B][N][nu]
    const double *p;        // [B][np]
    int np;
    double *xc;             // [B][res][nx]  = Julia's nx x res column-major matrix per seed
    ModelPar par;
};

template <class M>
__global__ void __launch_bounds__(32) k_propagate_foh(const PropArgs a)
{
    constexpr int NX = M::NX, NU = M::NU, NF = M::NF, NPD = M::NPD;
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    const double *ud = a.ud + (size_t)b * a.N * NU;
    double *xc = a.xc + (size_t)b * a.res * NX;
    double X[NX], pp[at_least_1(NPD)];
#pragma unroll
    for (int i = 0; i < NX; i++) { X[i] = a.xd[(size_t)b * a.N * NX + i]; xc[i] = X[i]; }
#pragma unroll
    for (int i = 0; i < NPD; i++) pp[i] = a.p[(size_t)b * a.np + i];
    const double tg0 = a.t_grid[0], tgN = a.t_grid[a.N - 1];
    const int d = a.res - 1;

    // u(t): saturate t to the grid, interval k with t_grid[k-1] < t <= t_grid[k] (first/last interval at the ends),
    // c = (t_k - t)/(t_k - t_{k-1}),  u = c u_{k-1} + (1-c) u_k        (helper.jl:84-118)
    auto input_at = [&](double t, double *u) {
        const double ts = fmax(tg0, fmin(tgN, t));
        int lo = 0, hi = a.N;            // number of grid points strictly below ts
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ts > a.t_grid[mid]) lo = mid + 1; else hi = mid;
        }
        int k = lo;
        if (k == 0) k = 1;
        if (k > a.N - 1) k = a.N - 1;
        const double tk = a.t_grid[k], tkm = a.t_grid[k - 1];
        const double c = __ddiv_rn(__dsub_rn(tk, ts), __dsub_rn(tk, tkm)), omc = __dsub_rn(1.0, c);
#pragma unroll
        for (int i = 0; i < NU; i++)
            u[i] = __dadd_rn(__dmul_rn(c, ud[(size_t)(k - 1) * NU + i]), __dmul_rn(omc, ud[(size_t)k * NU + i]));
    };
    auto rhs = [&](double t, const double *x, const double *u, double *f) {
        double A[NX * NX], Bu[NX * NU], Fc[at_least_1(NF) * NX];   // Jacobians are dead code here and removed by the compiler
        M::eval(a.par, t, x, u, pp, f, A, Bu, Fc);
    };

    for (int j = 1; j <= d; j++) {
        // tc = LinRange(0, 1, res): lerpi(j, d, 0, 1) = (1 - j/d)*0 + (j/d)*1
        const double f0 = __ddiv_rn((double)(j - 1), (double)d), f1 = __ddiv_rn((double)j, (double)d);
        const double t = __dadd_rn(__dmul_rn(__dsub_rn(1.0, f0), 0.0), __dmul_rn(f0, 1.0));
        const double tp = __dadd_rn(__dmul_rn(__dsub_rn(1.0, f1), 0.0), __dmul_rn(f1, 1.0));
        const double h = __dsub_rn(tp, t), hh = __ddiv_rn(h, 2.0);
        const double tm = __dadd_rn(t, hh), te = __dadd_rn(t, h);
        double u[NU], k1[NX], k2[NX], k3[NX], k4[NX], xt[NX];
        input_at(t, u);
        rhs(t, X, u, k1);
#pragma unroll
        for (int i = 0; i < NX; i++) xt[i] = X[i] + hh * k1[i];
        input_at(tm, u);
        rhs(tm, xt, u, k2);
#pragma unroll
        for (int i = 0; i < NX; i++) xt[i] = X[i] + hh * k2[i];
        rhs(tm, xt, u, k3);
#pragma unroll
        for (int i = 0; i < NX; i++) xt[i] = X[i] + h * k3[i];
        input_at(te, u);
        rhs(te, xt, u, k4);
#pragma unroll
        for (int i = 0; i < NX; i++) X[i] = X[i] + h / 6.0 * (k1[i] + 2.0 * k2[i] + 2.0 * k3[i] + k4[i]);
        M::post_step(X);
#pragma unroll
        for (int i = 0; i < NX; i++) xc[(size_t)j * NX + i] = X[i];
    }
}

// IMPULSE branch (discretization.jl:539-558): every interval is integrated on its own from the impulse-updated state
// x_k + f(t_k, -k, x_k, u_k, p) with the thrusters idle, on LinRange(t_k, t_k+1, subres), subres = ceil(res / (N - 1));
// the output holds xd[:, 1] followed by the subres columns of every interval: 1 + (N - 1) * subres columns per seed.
// One thread per (seed, interval): the intervals are independent initial-value problems.
template <class M>
__global__ void __launch_bounds__(64) k_propagate_impulse(const PropArgs a, int subres)
{
    constexpr int NX = M::NX, NU = M::NU, NF = M::NF, NPD = M::NPD;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int nseg = a.N - 1;
    if (i >= (long long)a.B * nseg) return;
    const int b = (int)(i / nseg), k = (int)(i % nseg);
    const size_t ncol = 1 + (size_t)nseg * subres;
    double *xc = a.xc + (size_t)b * ncol * NX;
    double X[NX], uk[NU], u0[NU], pp[at_least_1(NPD)], jump[NX], Bj[NX * NU];
#pragma unroll
    for (int j = 0; j < NX; j++) X[j] = a.xd[((size_t)b * a.N + k) * NX + j];
#pragma unroll
    for (int j = 0; j < NU; j++) { uk[j] = a.ud[((size_t)b * a.N + k) * NU + j]; u0[j] = 0.0; }
#pragma unroll
    for (int j = 0; j < NPD; j++) pp[j] = a.p[(size_t)b * a.np + j];
    if (k == 0) {
#pragma unroll
        for (int j = 0; j < NX; j++) xc[j] = X[j];
    }
    const double t1 = a.t_grid[k], t2 = a.t_grid[k + 1];
    if constexpr (M::IMPULSE) {
        M::eval_impulse(a.par, t1, X, uk, pp, jump, Bj);
#pragma unroll
        for (int j = 0; j < NX; j++) X[j] += jump[j];
    }
    double *out = xc + (1 + (size_t)k * subres) * NX;
#pragma unroll
    for (int j = 0; j < NX; j++) out[j] = X[j];
    const int d = subres - 1;
    for (int q = 1; q <= d; q++) {
        const double f0 = __ddiv_rn((double)(q - 1), (double)d), f1 = __ddiv_rn((double)q, (double)d);
        const double t = __dadd_rn(__dmul_rn(__dsub_rn(1.0, f0), t1), __dmul_rn(f0, t2));
        const double tp = __dadd_rn(__dmul_rn(__dsub_rn(1.0, f1), t1), __dmul_rn(f1, t2));
        const double h = __dsub_rn(tp, t), hh = __ddiv_rn(h, 2.0);
        const double tm = __dadd_rn(t, hh), te = __dadd_rn(t, h);
        double k1[NX], k2[NX], k3[NX], k4[NX], xt[NX], A[NX * NX], Bu[NX * NU], Fc[at_least_1(NF) * NX];
        M::eval(a.par, t, X, u0, pp, k1, A, Bu, Fc);
#pragma unroll
        for (int j = 0; j < NX; j++) xt[j] = X[j] + hh * k1[j];
        M::eval(a.par, tm, xt, u0, pp, k2, A, Bu, Fc);
#pragma unroll
        for (int j = 0; j < NX; j++) xt[j] = X[j] + hh * k2[j];
        M::eval(a.par, tm, xt, u0, pp, k3, A, Bu, Fc);
#pragma unroll
        for (int j = 0; j < NX; j++) xt[j] = X[j] + h * k3[j];
        M::eval(a.par, te, xt, u0, pp, k4, A, Bu, Fc);
#pragma unroll
        for (int j = 0; j < NX; j++) X[j] = X[j] + h / 6.0 * (k1[j] + 2.0 * k2[j] + 2.0 * k3[j] + k4[j]);
        M::post_step(X);
#pragma unroll
        for (int j = 0; j < NX; j++) out[(size_t)q * NX + j] = X[j];
    }
}
