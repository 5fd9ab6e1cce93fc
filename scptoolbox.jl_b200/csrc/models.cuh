// models.cuh -- device model packs: the device (sm_90a) twins of the user closures traj.f/A/B/F
// (reference: src/parser/problem.jl:432-450 wrappers; model sources cited per pack).
//
// A pack is a struct of compile-time sizes and one __forceinline__ eval() that fills
// f, A (col-major NX*NX), B (col-major NX*NU) and the NF *active* columns of F.  In every
// example of the reference F has a single non-zero column per evaluation, the time-dilation
// column F[:, id_t] = f / p[id_t] (starship definition.jl:626-633, quadrotor :177-183,
// freeflyer :273-281); packs therefore expose only those NF columns and the parameter
// index each one belongs to (fcol).  Structural zeros are written as literals so that the
// fully unrolled consumers constant-fold them away.
// A model with a fixed final time has no time-dilation column: NF = 0, F = 0 (oscillator), and a pack may read no
// parameter at all (NPD = 0).  Consumers size their F and p buffers with at_least_1() and never read them then.
#pragma once
#include <cuda_runtime.h>
#include "../../include/scpb.h"

struct ModelPar {
    double v[SCPB_MAX_PAR];
};

// length of a per-model buffer of n elements: C++ has no zero-length arrays, so an empty one keeps one unread element
__host__ __device__ constexpr int at_least_1(int n) { return n > 0 ? n : 1; }

template <int ID>
struct Model;

// ---------------------------------------------------------------- double integrator
// f = p0 * [x2; u - g]   (dynamics of double_integrator/parameters.jl:64, free final time)
template <>
struct Model<SCPB_MODEL_DBLINT> {
    static constexpr int NX = 2, NU = 1, NF = 1, NPD = 1;
    __device__ static constexpr int fcol(int) { return 0; }
    __device__ __forceinline__ static void eval(const ModelPar &P, double, const double *x, const double *u,
                                                const double *p, double *f, double *A, double *B, double *Fc)
    {
        const double g = P.v[0];
        const double f0 = x[1], f1 = u[0] - g;
        f[0] = p[0] * f0;
        f[1] = p[0] * f1;
        A[0] = 0.0; A[1] = 0.0; A[2] = p[0]; A[3] = 0.0;
        B[0] = 0.0; B[1] = p[0];
        Fc[0] = f0; Fc[1] = f1;
    }
    static constexpr bool IMPULSE = false;
    __device__ __forceinline__ static void post_step(double *) {}
};

// ---------------------------------------------------------------- rocket (Mars PDG, LTI)
// f = p0 * (A_c x + B_c u + p_c), rocket_landing/parameters.jl:110-121
template <>
struct Model<SCPB_MODEL_ROCKET> {
    static constexpr int NX = 7, NU = 4, NF = 1, NPD = 1;
    __device__ static constexpr int fcol(int) { return 0; }
    __device__ __forceinline__ static void eval(const ModelPar &P, double, const double *x, const double *u,
                                                const double *p, double *f, double *A, double *B, double *Fc)
    {
        const double g0 = P.v[0], g1 = P.v[1], g2 = P.v[2];
        const double w0 = P.v[3], w1 = P.v[4], w2 = P.v[5];
        const double alpha = P.v[6];
        // S = skew(w); Ac[3:6,0:3] = -S*S ; Ac[3:6,3:6] = -2 S
        const double S[3][3] = {{0.0, -w2, w1}, {w2, 0.0, -w0}, {-w1, w0, 0.0}};
        double Ac[7][7];
#pragma unroll
        for (int i = 0; i < 7; i++)
#pragma unroll
            for (int j = 0; j < 7; j++) Ac[i][j] = 0.0;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            Ac[i][3 + i] = 1.0;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                double s2 = 0.0;
#pragma unroll
                for (int k = 0; k < 3; k++) s2 += S[i][k] * S[k][j];
                Ac[3 + i][j] = -s2;
                Ac[3 + i][3 + j] = -2.0 * S[i][j];
            }
        }
        const double pc[7] = {0.0, 0.0, 0.0, g0, g1, g2, 0.0};
        const double td = p[0];
#pragma unroll
        for (int i = 0; i < 7; i++) {
            double s = pc[i];
#pragma unroll
            for (int j = 0; j < 7; j++) s += Ac[i][j] * x[j];
            if (i >= 3 && i < 6) s += u[i - 3];
            if (i == 6) s += -alpha * u[3];
            Fc[i] = s;
            f[i] = td * s;
        }
#pragma unroll
        for (int j = 0; j < 7; j++)
#pragma unroll
            for (int i = 0; i < 7; i++) A[i + 7 * j] = td * Ac[i][j];
#pragma unroll
        for (int i = 0; i < 28; i++) B[i] = 0.0;
        B[3 + 7 * 0] = td;
        B[4 + 7 * 1] = td;
        B[5 + 7 * 2] = td;
        B[6 + 7 * 3] = -alpha * td;
    }
    static constexpr bool IMPULSE = false;
    __device__ __forceinline__ static void post_step(double *) {}
};

// ---------------------------------------------------------------- starship landing flip
// starship_flip/definition.jl:498-637; parameters.jl:100-212
template <>
struct Model<SCPB_MODEL_STARSHIP> {
    static constexpr int NX = 8, NU = 3, NF = 2, NPD = 2;
    __device__ static constexpr int fcol(int j) { return j; }
    __device__ __forceinline__ static void eval(const ModelPar &P, double t, const double *x, const double *u,
                                                const double *p, double *f, double *A, double *B, double *Fc)
    {
        const double m = P.v[0], J = P.v[1], lcg = P.v[2], lcp_ = P.v[3], CD = P.v[4];
        const double ae = P.v[5], rd = P.v[6], g0 = P.v[7], taus = P.v[8];
        const double v0 = x[2], v1 = x[3], th = x[4], om = x[5], dd = x[7];
        const double T = u[0], de = u[1];
        const bool ph1 = (t <= taus);  // definition.jl:521 -- t carries Julia's exact LinRange arithmetic
        const double tdil = ph1 ? p[0] / taus : p[1] / (1.0 - taus);
        const double leng = -lcg, lcp = lcp_ - lcg;
        double sth, cth, sde, cde;
        sincos(th, &sth, &cth);
        sincos(de, &sde, &cde);
        const double ei0 = cth, ei1 = sth, ej0 = -sth, ej1 = cth;
        const double d0 = -sde * ei0 + cde * ej0;  // thrust direction
        const double d1 = -sde * ei1 + cde * ej1;
        const double nv = sqrt(v0 * v0 + v1 * v1);
        const double D0 = -CD * nv * v0, D1 = -CD * nv * v1;
        const double MT = leng * T * sde;
        const double MD = -lcp * (D0 * ei0 + D1 * ei1);
        double fr[8];
        fr[0] = v0;
        fr[1] = v1;
        fr[2] = (T * d0 + D0) / m;
        fr[3] = (T * d1 + D1) / m - g0;
        fr[4] = om;
        fr[5] = (MT + MD) / J;
        fr[6] = ae * T;
        fr[7] = (de - dd) / rd;
#pragma unroll
        for (int i = 0; i < 8; i++) f[i] = fr[i] * tdil;
        // F[:, id_t] = f / p[id_t]
        const double ip = ph1 ? 1.0 / p[0] : 1.0 / p[1];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const double c = f[i] * ip;
            Fc[i] = ph1 ? c : 0.0;
            Fc[8 + i] = ph1 ? 0.0 : c;
        }
        // A = df/dx
        const double G00 = -CD * (nv + v0 * v0 / nv);
        const double G01 = -CD * (v0 * v1 / nv);
        const double G11 = -CD * (nv + v1 * v1 / nv);
        const double dTv0 = T * (-sde * ej0 - cde * ei0);
        const double dTv1 = T * (-sde * ej1 - cde * ei1);
        const double gMD0 = -lcp * (G00 * ei0 + G01 * ei1);
        const double gMD1 = -lcp * (G01 * ei0 + G11 * ei1);
        const double dthMD = -lcp * (D0 * ej0 + D1 * ej1);
#pragma unroll
        for (int i = 0; i < 64; i++) A[i] = 0.0;
        A[0 + 8 * 2] = tdil;
        A[1 + 8 * 3] = tdil;
        A[2 + 8 * 2] = tdil * (G00 / m);
        A[2 + 8 * 3] = tdil * (G01 / m);
        A[3 + 8 * 2] = tdil * (G01 / m);
        A[3 + 8 * 3] = tdil * (G11 / m);
        A[2 + 8 * 4] = tdil * (dTv0 / m);
        A[3 + 8 * 4] = tdil * (dTv1 / m);
        A[4 + 8 * 5] = tdil;
        A[5 + 8 * 2] = tdil * (gMD0 / J);
        A[5 + 8 * 3] = tdil * (gMD1 / J);
        A[5 + 8 * 4] = tdil * (dthMD / J);
        A[7 + 8 * 7] = tdil * (-1.0 / rd);
        // B = df/du
#pragma unroll
        for (int i = 0; i < 24; i++) B[i] = 0.0;
        B[2 + 8 * 0] = tdil * (d0 / m);
        B[3 + 8 * 0] = tdil * (d1 / m);
        B[2 + 8 * 1] = tdil * (T * (-cde * ei0 - sde * ej0) / m);
        B[3 + 8 * 1] = tdil * (T * (-cde * ei1 - sde * ej1) / m);
        B[5 + 8 * 0] = tdil * (leng * sde / J);
        B[5 + 8 * 1] = tdil * (leng * T * cde / J);
        B[6 + 8 * 0] = tdil * ae;
        B[7 + 8 * 1] = tdil * (1.0 / rd);
    }
    static constexpr bool IMPULSE = false;
    __device__ __forceinline__ static void post_step(double *) {}
};

// ---------------------------------------------------------------- quadrotor
// quadrotor/definition.jl:140-186:  f = p0 * [v; u[0:3] + g]
template <>
struct Model<SCPB_MODEL_QUADROTOR> {
    static constexpr int NX = 6, NU = 4, NF = 1, NPD = 1;
    __device__ static constexpr int fcol(int) { return 0; }
    __device__ __forceinline__ static void eval(const ModelPar &P, double, const double *x, const double *u,
                                                const double *p, double *f, double *A, double *B, double *Fc)
    {
        const double td = p[0];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            Fc[i] = x[3 + i];
            Fc[3 + i] = u[i] + P.v[i];
        }
#pragma unroll
        for (int i = 0; i < 6; i++) f[i] = td * Fc[i];
#pragma unroll
        for (int i = 0; i < 36; i++) A[i] = 0.0;
#pragma unroll
        for (int i = 0; i < 3; i++) A[i + 6 * (3 + i)] = td;
#pragma unroll
        for (int i = 0; i < 24; i++) B[i] = 0.0;
#pragma unroll
        for (int i = 0; i < 3; i++) B[(3 + i) + 6 * i] = td;
    }
    static constexpr bool IMPULSE = false;
    __device__ __forceinline__ static void post_step(double *) {}
};

// ---------------------------------------------------------------- 6-DoF free-flyer
// freeflyer/definition.jl:224-284, quaternion algebra src/utils/quaternion.jl:190-214
// (scalar-last quaternion), integration action definition.jl:69-82 (renormalise q).
template <>
struct Model<SCPB_MODEL_FREEFLYER> {
    static constexpr int NX = 13, NU = 6, NF = 1, NPD = 1;
    __device__ static constexpr int fcol(int) { return 0; }
    __device__ __forceinline__ static void eval(const ModelPar &P, double, const double *x, const double *u,
                                                const double *p, double *f, double *A, double *B, double *Fc)
    {
        const double mass = P.v[0];
        const double *J = &P.v[1], *Ji = &P.v[10];
        const double td = p[0];
        const double q0 = x[6], q1 = x[7], q2 = x[8], qw = x[9];
        const double o0 = x[10], o1 = x[11], o2 = x[12];
        // skew(q) (left) = [w I + [v]x, v; -v', w]
        const double SL[4][4] = {{qw, -q2, q1, q0}, {q2, qw, -q0, q1}, {-q1, q0, qw, q2}, {-q0, -q1, -q2, qw}};
        // skew(Quaternion(omega), :R) = [-[o]x, o; -o', 0]
        const double SR[4][4] = {{0.0, o2, -o1, o0}, {-o2, 0.0, o0, o1}, {o1, -o0, 0.0, o2}, {-o0, -o1, -o2, 0.0}};
        double Jw[3];
#pragma unroll
        for (int i = 0; i < 3; i++) Jw[i] = J[i + 0] * o0 + J[i + 3] * o1 + J[i + 6] * o2;
        const double c0 = o1 * Jw[2] - o2 * Jw[1];
        const double c1 = o2 * Jw[0] - o0 * Jw[2];
        const double c2 = o0 * Jw[1] - o1 * Jw[0];
        const double rh[3] = {u[3] - c0, u[4] - c1, u[5] - c2};
#pragma unroll
        for (int i = 0; i < 3; i++) {
            Fc[i] = x[3 + i];
            Fc[3 + i] = u[i] / mass;
            Fc[10 + i] = Ji[i + 0] * rh[0] + Ji[i + 3] * rh[1] + Ji[i + 6] * rh[2];
        }
#pragma unroll
        for (int i = 0; i < 4; i++) Fc[6 + i] = 0.5 * (SL[i][0] * o0 + SL[i][1] * o1 + SL[i][2] * o2);
#pragma unroll
        for (int i = 0; i < 13; i++) f[i] = td * Fc[i];
        // A
#pragma unroll
        for (int i = 0; i < 169; i++) A[i] = 0.0;
#pragma unroll
        for (int i = 0; i < 3; i++) A[i + 13 * (3 + i)] = td;
#pragma unroll
        for (int i = 0; i < 4; i++) {
#pragma unroll
            for (int j = 0; j < 4; j++) A[(6 + i) + 13 * (6 + j)] = td * 0.5 * SR[i][j];
#pragma unroll
            for (int j = 0; j < 3; j++) A[(6 + i) + 13 * (10 + j)] = td * 0.5 * SL[i][j];
        }
        // dfw/dw = -Jinv (skew(o) J - skew(J o))
        const double So[3][3] = {{0.0, -o2, o1}, {o2, 0.0, -o0}, {-o1, o0, 0.0}};
        const double SJ[3][3] = {{0.0, -Jw[2], Jw[1]}, {Jw[2], 0.0, -Jw[0]}, {-Jw[1], Jw[0], 0.0}};
        double Mm[3][3];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++)
                Mm[i][j] = So[i][0] * J[0 + 3 * j] + So[i][1] * J[1 + 3 * j] + So[i][2] * J[2 + 3 * j] - SJ[i][j];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++)
                A[(10 + i) + 13 * (10 + j)] =
                    -td * (Ji[i + 0] * Mm[0][j] + Ji[i + 3] * Mm[1][j] + Ji[i + 6] * Mm[2][j]);
        // B
#pragma unroll
        for (int i = 0; i < 78; i++) B[i] = 0.0;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            B[(3 + i) + 13 * i] = td * (1.0 / mass);
#pragma unroll
            for (int j = 0; j < 3; j++) B[(10 + i) + 13 * (3 + j)] = td * Ji[i + 3 * j];
        }
    }
    static constexpr bool IMPULSE = false;
    __device__ __forceinline__ static void post_step(double *x)
    {
        const double n = sqrt(x[6] * x[6] + x[7] * x[7] + x[8] * x[8] + x[9] * x[9]);
#pragma unroll
        for (int i = 0; i < 4; i++) x[6 + i] = x[6 + i] / n;
    }
};

// ---------------------------------------------------------------- planar rendezvous with impulsive RCS thrust
// rendezvous_planar/definition.jl:147-243, parameters.jl:87-111.  x = [r(2) v(2) theta omega]; u[0..2] = (f-, f+, f0),
// the other nine inputs (references, absolute values) do not enter the dynamics; p = [tdil]; par: m, J, lu, lv, n.
// The reference calls f / B with a NEGATIVE segment index for the impulse (discretization.jl:191, 389): the jump of
// (v, omega) and its input Jacobian, not scaled by the time dilation -> eval_impulse().
template <>
struct Model<SCPB_MODEL_RENDEZVOUS2D> {
    static constexpr int NX = 6, NU = 12, NF = 1, NPD = 1;
    static constexpr bool IMPULSE = true;
    __device__ static constexpr int fcol(int) { return 0; }
    __device__ __forceinline__ static void eval(const ModelPar &P, double, const double *x, const double *u,
                                                const double *p, double *f, double *A, double *B, double *Fc)
    {
        const double ms = P.v[0], J = P.v[1], lu = P.v[2], lv = P.v[3], n = P.v[4];
        const double th = x[4], fm = u[0], fp = u[1], f0 = u[2], tdil = p[0];
        double sth, cth;
        sincos(th, &sth, &cth);
        const double uh0 = -cth, uh1 = sth, vh0 = -sth, vh1 = -cth;
        double g[6];
        g[0] = x[2]; g[1] = x[3];
        g[2] = ((fm + fp) * uh0 + f0 * vh0) / ms + 2.0 * n * x[3];
        g[3] = ((fm + fp) * uh1 + f0 * vh1) / ms + (3.0 * n * n * x[1] - 2.0 * n * x[2]);
        g[4] = x[5];
        g[5] = ((fp - fm) * lv - f0 * lu) / J;
#pragma unroll
        for (int i = 0; i < 6; i++) { Fc[i] = g[i]; f[i] = g[i] * tdil; }
#pragma unroll
        for (int i = 0; i < 36; i++) A[i] = 0.0;
        A[0 + 6 * 2] = tdil; A[1 + 6 * 3] = tdil;
        A[3 + 6 * 1] = 3.0 * n * n * tdil;
        A[2 + 6 * 3] = 2.0 * n * tdil; A[3 + 6 * 2] = -2.0 * n * tdil;
        A[2 + 6 * 4] = ((fm + fp) * sth + f0 * (-cth)) / ms * tdil;   // d uh/d th = (sin, cos), d vh/d th = (-cos, sin)
        A[3 + 6 * 4] = ((fm + fp) * cth + f0 * sth) / ms * tdil;
        A[4 + 6 * 5] = tdil;
#pragma unroll
        for (int i = 0; i < 72; i++) B[i] = 0.0;
        B[2 + 6 * 0] = uh0 / ms * tdil; B[3 + 6 * 0] = uh1 / ms * tdil; B[5 + 6 * 0] = -lv / J * tdil;
        B[2 + 6 * 1] = uh0 / ms * tdil; B[3 + 6 * 1] = uh1 / ms * tdil; B[5 + 6 * 1] = lv / J * tdil;
        B[2 + 6 * 2] = vh0 / ms * tdil; B[3 + 6 * 2] = vh1 / ms * tdil; B[5 + 6 * 2] = -lu / J * tdil;
    }
    // the impulse at a node: jump[NX] = f(t, -k, x, u, p), Bj = B(t, -k, x, u, p) (col-major NX*NU)
    __device__ __forceinline__ static void eval_impulse(const ModelPar &P, double, const double *x, const double *u,
                                                        const double *, double *jump, double *Bj)
    {
        const double ms = P.v[0], J = P.v[1], lu = P.v[2], lv = P.v[3];
        const double th = x[4], fm = u[0], fp = u[1], f0 = u[2];
        double sth, cth;
        sincos(th, &sth, &cth);
        const double uh0 = -cth, uh1 = sth, vh0 = -sth, vh1 = -cth;
#pragma unroll
        for (int i = 0; i < 6; i++) jump[i] = 0.0;
        jump[2] = ((fm + fp) * uh0 + f0 * vh0) / ms;
        jump[3] = ((fm + fp) * uh1 + f0 * vh1) / ms;
        jump[5] = ((fp - fm) * lv - f0 * lu) / J;
#pragma unroll
        for (int i = 0; i < 72; i++) Bj[i] = 0.0;
        Bj[2 + 6 * 0] = uh0 / ms; Bj[3 + 6 * 0] = uh1 / ms; Bj[5 + 6 * 0] = -lv / J;
        Bj[2 + 6 * 1] = uh0 / ms; Bj[3 + 6 * 1] = uh1 / ms; Bj[5 + 6 * 1] = lv / J;
        Bj[2 + 6 * 2] = vh0 / ms; Bj[3 + 6 * 2] = vh1 / ms; Bj[5 + 6 * 2] = -lu / J;
    }
    __device__ __forceinline__ static void post_step(double *) {}
};

// ---------------------------------------------------------------- forced harmonic oscillator with an input deadband
// oscillator/definition.jl:161-236, parameters.jl:69-115.  x = [r v]; u[0] = aa, the applied acceleration (the reference
// acceleration ar and the two one-norm slacks do not enter the dynamics); p = [l1r_1 .. l1r_N] is not read.
//   f = tf [v; aa - w0^2 r - 2 zeta w0 v]
// over the FIXED horizon tf: F = 0, so the pack has no active F column (NF = 0) and reads no parameter (NPD = 0).
// par: zeta, omega0, tf.  The reference's impulse branch (k < 0) is not mirrored: its test runs FOH.
template <>
struct Model<SCPB_MODEL_OSCILLATOR> {
    static constexpr int NX = 2, NU = 4, NF = 0, NPD = 0;
    static constexpr bool IMPULSE = false;
    __device__ static constexpr int fcol(int) { return 0; }
    __device__ __forceinline__ static void eval(const ModelPar &P, double, const double *x, const double *u,
                                                const double *, double *f, double *A, double *B, double *)
    {
        const double zeta = P.v[0], w0 = P.v[1], tf = P.v[2];
        const double k = -(w0 * w0), c = 2.0 * zeta * w0;
        f[0] = x[1] * tf;
        f[1] = (u[0] + (k * x[0] - c * x[1])) * tf;
        A[0] = 0.0; A[1] = k * tf; A[2] = tf; A[3] = -c * tf;
#pragma unroll
        for (int i = 0; i < 8; i++) B[i] = 0.0;
        B[1] = tf;
    }
    __device__ __forceinline__ static void post_step(double *) {}
};

// ---------------------------------------------------------------- host dispatch on the model id
template <class M>
struct ModelId;
template <int ID>
struct ModelId<Model<ID>> { static constexpr int value = ID; };

// calls f(Model<id>()) and returns true; false for an id without a pack.  Every per-model switch goes through here,
// so a new model is one more case.
template <class F>
bool with_model(int id, F &&f)
{
    switch (id) {
    case SCPB_MODEL_DBLINT: f(Model<SCPB_MODEL_DBLINT>()); return true;
    case SCPB_MODEL_ROCKET: f(Model<SCPB_MODEL_ROCKET>()); return true;
    case SCPB_MODEL_STARSHIP: f(Model<SCPB_MODEL_STARSHIP>()); return true;
    case SCPB_MODEL_QUADROTOR: f(Model<SCPB_MODEL_QUADROTOR>()); return true;
    case SCPB_MODEL_FREEFLYER: f(Model<SCPB_MODEL_FREEFLYER>()); return true;
    case SCPB_MODEL_RENDEZVOUS2D: f(Model<SCPB_MODEL_RENDEZVOUS2D>()); return true;
    case SCPB_MODEL_OSCILLATOR: f(Model<SCPB_MODEL_OSCILLATOR>()); return true;
    default: return false;
    }
}
