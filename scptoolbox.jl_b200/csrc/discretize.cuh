// discretize.cuh -- K1: batched, segment-parallel RK4 + variational-equation kernel.
//
// Replaces discretize!/derivs_foh/set_update_matrices (src/solvers/discretization.jl:160-406)
// and rk4_generic/rk4_core_step/linterp (src/utils/helper.jl:451-501, 411-424, 107-118).
//
// Work decomposition: one warp per (seed b, segment k) -- the B*(N-1) items are
// independent (discretization.jl:182 only reads ref.xd/ud/p).  Inside the warp the augmented
// propagation vector V = [x; Phi; PB-; PB+; PF; Pr; PE] is laid out COLUMN-PER-LANE:
//   lanes 0..NX-1      hold the columns of Phi,
//   following lanes    hold the quadrature columns (int Phi^-1 B s-, int Phi^-1 B s+,
//                      int Phi^-1 F[:,active], int Phi^-1 r, int Phi^-1 E),
//   every lane         carries a redundant copy of the state x (NX doubles) so that the model
//                      pack is evaluated without any exchange.
// A stage evaluation is: model eval (registers) -> A*Phi column (registers, structural zeros
// folded) -> ONE warp-wide Gauss-Jordan elimination with partial pivoting on [Phi | RHS] where
// every lane owns one column (pivot column broadcast by shuffles), which yields Phi^-1*RHS for all
// quadrature columns at once (the reference forms inv(Phi) by LU and multiplies, :267-273).
// Only F's active columns are propagated (np may be 481 for the free-flyer, SURVEY section 7).
//
// Time arithmetic (sub-grid nodes, stage times, sigma-/sigma+, linterp weight) uses the
// round-to-nearest intrinsics in exactly the reference's operation order so that comparisons
// such as `t <= tau_s` inside a model pack see bit-identical t values.
#pragma once
#include "models.cuh"

struct OutView {
    double *ptr;
    long long sB, sK, sE;  // strides (in doubles) over seed-in-group, segment, element
    long long sGrp = 0;    // stride over seed groups
    int Gq = 1;            // seeds per group: address = (b/Gq)*sGrp + (b%Gq)*sB + k*sK + e*sE
    __host__ __device__ long long at(int b, int k, long long e) const
    {
        return (long long)(b / Gq) * sGrp + (long long)(b % Gq) * sB + (long long)k * sK + e * sE;
    }
};

struct DiscArgs {
    int B, N, Nsub;
    int np;                 // full parameter dimension (row length of p and of dense F)
    int f_packed;           // 1: F holds only the NF active columns; 0: dense nx*np (Julia layout)
    const double *t_grid;   // [N]
    const double *xd;       // [B][N][nx]
    const double *ud;       // [B][N][nu]
    const double *p;        // [B][np]
    long long xsB, xsK, xsE;  // strides of xd
    long long usB, usK, usE;  // strides of ud
    long long psB, psE;       // strides of p
    const double *iSx;      // [nx]
    OutView A, Bm, Bp, F, r, E, defect;
    double *dnorm;          // [B][N-1]  ||iSx*defect||_inf per segment
    int *status;            // device word, OR-ed with 1 on a singular pivot
    const int *skip;        // nullable [B]: seeds marked non-zero are left untouched (SCP seeds that have stopped)
    int b0 = 0, nb = 0;     // chunk of seeds [b0, b0 + nb) this launch works on (nb = 0: all B); arrays stay indexed by seed
    ModelPar par;
};

__device__ __forceinline__ double shfl_d(double v, int src)
{
    return __shfl_sync(0xffffffffu, v, src);
}

// IMP = 1: IMPULSE discretization (discretization.jl:186-193, 304-340, 384-390): the segment starts from the
// impulse-updated state x_k + f(t_k, -k, x_k, u_k, p), coasts with u = 0, and B_k = A_k * B(t_k, -k, x_k, u_k, p) (one
// input block: Bm; Bp is written as zero).  Phi, F, r and E columns are the FOH ones evaluated at u = 0.
// MB: resident 128-thread blocks per SM the register allocation is held to (2: 255 registers; 3: 168; 4: 128, each step
// with more spill code) -- more warps per scheduler to hide the fixed-latency chains of the stage (scpb_api.cu: launch_disc)
template <class M, int IMP, int MB = 2>
__global__ void __launch_bounds__(128, MB) k_discretize_foh(const DiscArgs a)
{
    constexpr int NX = M::NX, NU = M::NU, NF = M::NF, NPD = M::NPD;
    constexpr int C = NX + 2 * NU + NF + 1 + NX;  // columns of [Phi PB- PB+ PF Pr PE]
    constexpr int CPL = (C + 31) / 32;            // columns per lane
    constexpr int QSZ = (NU + NF + 1) * NX;       // per-warp stash of B, Fc, r

    extern __shared__ double smem[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nseg = a.N - 1;
    if (gw >= (long long)(a.nb > 0 ? a.nb : a.B) * nseg) return;
    const int b = a.b0 + (int)(gw / nseg), k = (int)(gw % nseg);
    if (b >= a.B) return;
    if (a.skip && a.skip[b]) return;     // warp-uniform: the whole warp works on seed b
    double *Q = smem + wib * QSZ;

    // ---- column bookkeeping for this lane ----
    int qoff[CPL], ej[CPL], scl[CPL];
    bool act[CPL];
#pragma unroll
    for (int s = 0; s < CPL; s++) {
        const int c = lane + 32 * s;
        qoff[s] = -1; ej[s] = -1; scl[s] = 0; act[s] = (c < C);
        if (c >= NX && c < NX + NU) { qoff[s] = (c - NX) * NX; scl[s] = 1; }
        else if (c >= NX + NU && c < NX + 2 * NU) { qoff[s] = (c - NX - NU) * NX; scl[s] = 2; }
        else if (c >= NX + 2 * NU && c < NX + 2 * NU + NF) qoff[s] = (NU + (c - NX - 2 * NU)) * NX;
        else if (c == NX + 2 * NU + NF) qoff[s] = (NU + NF) * NX;
        else if (c > NX + 2 * NU + NF && c < C) ej[s] = c - (NX + 2 * NU + NF + 1);
    }
    const bool phi_lane = (lane < NX);

    // ---- inputs ----
    const double t1 = a.t_grid[k], t2 = a.t_grid[k + 1];
    const double dts = __dsub_rn(t2, t1);
    double uk[NU], ukp1[NU], pp[at_least_1(NPD)];
    double xv[NX], xb[NX], xs[NX];
#pragma unroll
    for (int i = 0; i < NX; i++) xv[i] = a.xd[b * a.xsB + k * a.xsK + i * a.xsE];
#pragma unroll
    for (int i = 0; i < NU; i++) {
        uk[i] = a.ud[b * a.usB + k * a.usK + i * a.usE];
        ukp1[i] = a.ud[b * a.usB + (k + 1) * a.usK + i * a.usE];
    }
#pragma unroll
    for (int i = 0; i < NPD; i++) pp[i] = a.p[b * a.psB + i * a.psE];
    if constexpr (IMP) {
        static_assert(M::IMPULSE, "this model pack has no impulse semantics");
        double jump[NX], Bj[NX * NU];
        M::eval_impulse(a.par, t1, xv, uk, pp, jump, Bj);
#pragma unroll
        for (int i = 0; i < NX; i++) xv[i] += jump[i];
    }

    // V0 = [x_k; vec(I); 0]  (discretization.jl:177-185)
    double colv[CPL][NX], phib[NX], phis[NX];
#pragma unroll
    for (int s = 0; s < CPL; s++)
#pragma unroll
        for (int r = 0; r < NX; r++) colv[s][r] = (s == 0 && phi_lane && r == lane) ? 1.0 : 0.0;

    int bad = 0;
    const int d = a.Nsub - 1;
    for (int j = 1; j <= d; j++) {
        // t_subgrid = LinRange(t1, t2, Nsub): lerpi(j, d, a, b) = (1 - j/d) a + (j/d) b
        const double fr0 = __ddiv_rn((double)(j - 1), (double)d), fr1 = __ddiv_rn((double)j, (double)d);
        const double ta = __dadd_rn(__dmul_rn(__dsub_rn(1.0, fr0), t1), __dmul_rn(fr0, t2));
        const double tb = __dadd_rn(__dmul_rn(__dsub_rn(1.0, fr1), t1), __dmul_rn(fr1, t2));
        const double h = __dsub_rn(tb, ta);
        const double hh = __ddiv_rn(h, 2.0);
#pragma unroll
        for (int i = 0; i < NX; i++) { xb[i] = xv[i]; xs[i] = xv[i]; }
#pragma unroll
        for (int r = 0; r < NX; r++) { phib[r] = colv[0][r]; phis[r] = colv[0][r]; }

#pragma unroll 1
        for (int st = 0; st < 4; st++) {
            const double t = (st == 0) ? ta : ((st == 3) ? __dadd_rn(ta, h) : __dadd_rn(ta, hh));
            const double wst = (st == 2) ? h : hh;                       // next stage: x + wst*k
            const double wac = (st == 0 || st == 3) ? h / 6.0 : h / 3.0; // accumulate

            // linterp on the 2-node span (helper.jl:107-118) and FOH weights (discretization.jl:252-253)
            const double tsat = fmax(t1, fmin(t2, t));
            const double cc = __ddiv_rn(__dsub_rn(t2, tsat), dts);
            const double omc = __dsub_rn(1.0, cc);
            const double sgm = __ddiv_rn(__dsub_rn(t2, t), dts);
            const double sgp = __ddiv_rn(__dsub_rn(t, t1), dts);
            double u[NU];
#pragma unroll
            for (int i = 0; i < NU; i++) u[i] = IMP ? 0.0 : cc * uk[i] + omc * ukp1[i];

            double f[NX], A[NX * NX], Bu[NX * NU], Fc[at_least_1(NF) * NX];
            M::eval(a.par, t, xs, u, pp, f, A, Bu, Fc);

            // r = f - A x - B u - F p
            double rr[NX];
#pragma unroll
            for (int i = 0; i < NX; i++) {
                double s = f[i];
#pragma unroll
                for (int c2 = 0; c2 < NX; c2++) s -= A[i + NX * c2] * xs[c2];
#pragma unroll
                for (int c2 = 0; c2 < NU; c2++) s -= Bu[i + NX * c2] * u[c2];
#pragma unroll
                for (int c2 = 0; c2 < NF; c2++) s -= Fc[c2 * NX + i] * pp[M::fcol(c2)];
                rr[i] = s;
            }
            if (lane == 0) {
#pragma unroll
                for (int i = 0; i < NX * NU; i++) Q[i] = Bu[i];
#pragma unroll
                for (int i = 0; i < NX * NF; i++) Q[NX * NU + i] = Fc[i];
#pragma unroll
                for (int i = 0; i < NX; i++) Q[NX * (NU + NF) + i] = rr[i];
            }
            __syncwarp();

            // d(Phi col)/dt = A * Phi col
            double dphi[NX];
#pragma unroll
            for (int i = 0; i < NX; i++) {
                double s = 0.0;
#pragma unroll
                for (int c2 = 0; c2 < NX; c2++) s += A[i + NX * c2] * phis[c2];
                dphi[i] = s;
            }

            // working columns of [Phi | RHS]
            double w[CPL][NX];
#pragma unroll
            for (int s = 0; s < CPL; s++) {
#pragma unroll
                for (int r = 0; r < NX; r++) {
                    double v = 0.0;
                    if (s == 0 && phi_lane) v = phis[r];
                    else if (qoff[s] >= 0) v = Q[qoff[s] + r];
                    else if (ej[s] == r) v = 1.0;
                    w[s][r] = v;
                }
            }
            __syncwarp();

            // Gauss-Jordan with partial pivoting, one column per lane
#pragma unroll
            for (int i = 0; i < NX; i++) {
                int piv = i;
                double pm = fabs(w[0][i]);
#pragma unroll
                for (int r = i + 1; r < NX; r++) {
                    const double av = fabs(w[0][r]);
                    if (av > pm) { pm = av; piv = r; }
                }
                piv = __shfl_sync(0xffffffffu, piv, i);
#pragma unroll
                for (int s = 0; s < CPL; s++)
#pragma unroll
                    for (int r = i + 1; r < NX; r++)
                        if (piv == r) { const double tq = w[s][i]; w[s][i] = w[s][r]; w[s][r] = tq; }
                double ci[NX];
#pragma unroll
                for (int r = 0; r < NX; r++) ci[r] = shfl_d(w[0][r], i);
                if (ci[i] == 0.0) bad = 1;
                const double inv = 1.0 / ci[i];
#pragma unroll
                for (int s = 0; s < CPL; s++) {
                    const double tq = w[s][i] * inv;
                    w[s][i] = tq;
#pragma unroll
                    for (int r = 0; r < NX; r++)
                        if (r != i) w[s][r] = fma(-ci[r], tq, w[s][r]);
                }
            }

            // accumulate and form the next stage state
#pragma unroll
            for (int i = 0; i < NX; i++) {
                xv[i] = fma(wac, f[i], xv[i]);
                xs[i] = fma(wst, f[i], xb[i]);
            }
#pragma unroll
            for (int s = 0; s < CPL; s++) {
                const double sc = (scl[s] == 1) ? sgm : ((scl[s] == 2) ? sgp : 1.0);
#pragma unroll
                for (int r = 0; r < NX; r++) {
                    const double kv = (s == 0 && phi_lane) ? dphi[r] : sc * w[s][r];
                    colv[s][r] = fma(wac, kv, colv[s][r]);
                }
            }
#pragma unroll
            for (int r = 0; r < NX; r++) phis[r] = fma(wst, dphi[r], phib[r]);
        }
        M::post_step(xv);  // integration actions act on V[idx] after every step (helper.jl:492-496)
    }

    if constexpr (IMP) {   // B_k = A_k * B(t_k, -k, x_k, u_k, p): the input columns carry the jump Jacobian into the product
        double xk[NX], jump[NX], Bj[NX * NU];
#pragma unroll
        for (int i = 0; i < NX; i++) xk[i] = a.xd[b * a.xsB + k * a.xsK + i * a.xsE];
        M::eval_impulse(a.par, t1, xk, uk, pp, jump, Bj);
#pragma unroll
        for (int s = 0; s < CPL; s++) {
            const int c = lane + 32 * s;
            if (scl[s] == 1) {
#pragma unroll
                for (int r = 0; r < NX; r++) colv[s][r] = Bj[(c - NX) * NX + r];
            } else if (scl[s] == 2) {
#pragma unroll
                for (int r = 0; r < NX; r++) colv[s][r] = 0.0;
            }
        }
    }
    // ---- set_update_matrices (discretization.jl:354-406): A_k = Phi, X_k = A_k * XV ----
    double outc[CPL][NX];
#pragma unroll
    for (int s = 0; s < CPL; s++)
#pragma unroll
        for (int r = 0; r < NX; r++) outc[s][r] = 0.0;
#pragma unroll
    for (int i = 0; i < NX; i++) {
#pragma unroll
        for (int r = 0; r < NX; r++) {
            const double ph = shfl_d(colv[0][r], i);
#pragma unroll
            for (int s = 0; s < CPL; s++) outc[s][r] = fma(ph, colv[s][i], outc[s][r]);
        }
    }
#pragma unroll
    for (int s = 0; s < CPL; s++) {
        const int c = lane + 32 * s;
        if (!act[s]) continue;
        const OutView *ov;
        long long e0;
        bool raw = false;
        if (c < NX) { ov = &a.A; e0 = (long long)c * NX; raw = true; }
        else if (c < NX + NU) { ov = &a.Bm; e0 = (long long)(c - NX) * NX; }
        else if (c < NX + 2 * NU) { ov = &a.Bp; e0 = (long long)(c - NX - NU) * NX; }
        else if (c < NX + 2 * NU + NF) {
            const int jf = c - NX - 2 * NU;
            ov = &a.F;
            e0 = (long long)(a.f_packed ? jf : M::fcol(jf)) * NX;
        }
        else if (c == NX + 2 * NU + NF) { ov = &a.r; e0 = 0; }
        else { ov = &a.E; e0 = (long long)(c - (NX + 2 * NU + NF + 1)) * NX; }
        if (ov->ptr == nullptr) continue;
        double *dst = ov->ptr + ov->at(b, k, e0);
#pragma unroll
        for (int r = 0; r < NX; r++) dst[r * ov->sE] = raw ? colv[s][r] : outc[s][r];
    }

    // ---- defect and feasibility norm (discretization.jl:205-210) ----
    if (lane == 0) {
        double nrm = 0.0;
#pragma unroll
        for (int i = 0; i < NX; i++) {
            const double xn = a.xd[b * a.xsB + (k + 1) * a.xsK + i * a.xsE];
            const double df = xn - xv[i];
            if (a.defect.ptr) a.defect.ptr[a.defect.at(b, k, i)] = df;
            const double av = fabs(a.iSx[i] * df);
            if (av > nrm || av != av) nrm = av;
        }
        a.dnorm[(long long)b * nseg + k] = nrm;
        if (bad) atomicOr(a.status, 1);
    }
}

// feas[b] = all_k !(dnorm[b][k] > feas_tol)   (NaN compares false, as in the reference)
static __global__ void k_feas_reduce(const double *dnorm, int B, int nseg, double feas_tol, int *feas, const int *skip,
                                     int b0 = 0, int nb = 0)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= (nb > 0 ? nb : B)) return;
    const int b = b0 + q;
    if (b >= B) return;
    if (skip && skip[b]) return;
    int ok = 1;
    for (int k = 0; k < nseg; k++)
        if (dnorm[(long long)b * nseg + k] > feas_tol) ok = 0;
    feas[b] = ok;
}
