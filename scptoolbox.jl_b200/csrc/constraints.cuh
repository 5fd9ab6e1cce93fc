// constraints.cuh -- device packs for the nonconvex path constraints s(t,k,x,u,p) <= 0 and their Jacobians
// C = ds/dx, D = ds/du, G = ds/dp  (the device twins of traj.s/C/D/G, src/parser/problem.jl:560-587,
// consumed by add_nonconvex_constraints!, src/solvers/scp.jl:744-794).
// Outputs are dense, row-major: s[NS], C[NS][NX], D[NS][NU], G[NS][NG]; entries that are structurally zero
// for a pack are simply never referenced by the host template.  G is PACKED: it holds NG columns and gcol(k, j) names
// the parameter each one belongs to at node k (0-based).  For most packs NG = np and gcol(k, j) = j; the free-flyer
// has np = 1 + 6N parameters of which only the six room-SDF slacks of node k enter s at that node
// (freeflyer/definition.jl:398-424), so its G has six columns instead of 481.
#pragma once
#include <type_traits>
#include <math_constants.h>
#include "models.cuh"

template <int ID>
struct Constr {
    static constexpr int NS = 0;
};

// parameter slot of a pack's homotopy parameter (its KAPPA), or -1 for a pack without one
template <class CP, class = void>
struct HomSlot { static constexpr int value = -1; };
template <class CP>
struct HomSlot<CP, std::void_t<decltype(CP::KAPPA)>> { static constexpr int value = CP::KAPPA; };

// the constraint pack of model ID; Constr<0> (no constraints) for a model without one
template <int ID>
using PackOf = std::conditional_t<(Constr<ID>::NS > 0), Constr<ID>, Constr<0>>;

// calls f(PackOf<id>()) when has_pack, f(Constr<0>()) otherwise or for an unknown id
template <class F>
void with_constr(int id, bool has_pack, F &&f)
{
    if (!has_pack || !with_model(id, [&](auto m) { f(PackOf<ModelId<decltype(m)>::value>()); })) f(Constr<0>());
}

// the pack at node k; a pack with a homotopy parameter takes it from *kap (a seed's own value) unless kap is null
template <class CP>
__device__ __forceinline__ void constr_eval(const ModelPar &P, const double *kap, double t, int N, int k, const double *x,
                                            const double *u, const double *p, double *s, double *C, double *D, double *G)
{
    if constexpr (HomSlot<CP>::value >= 0) CP::eval_kappa(P, kap ? *kap : P.v[CP::KAPPA], t, N, k, x, u, p, s, C, D, G);
    else CP::eval(P, t, N, k, x, u, p, s, C, D, G);
}

// starship_flip/definition.jl:704-810.  par: [9] rate_delay, [10] deltadot_max, [11] gamma_gs, [12] thetamax2,
// [8] tau_s (shared with the dynamics pack).
template <>
struct Constr<SCPB_MODEL_STARSHIP> {
    static constexpr int NS = 23, NX = 8, NU = 3, NP = 10, NG = 10;
    __device__ static constexpr int gcol(int, int j) { return j; }
    __device__ static void eval(const ModelPar &P, double t, int N, int, const double *x, const double *u, const double *p,
                                double *s, double *C, double *D, double *G)
    {
        const double taus = P.v[8], rd = P.v[9], ddmax = P.v[10], cgs = cos(P.v[11]), thmax = P.v[12];
        // phase_switch / phase2, definition.jl:707-721
        const double dt = 1.0 / (double)(N - 1), tol = 1e-3;
        const bool psw = ((taus - dt) + tol <= t) && (t <= taus + tol);
        const bool ph2 = psw || (t > taus);
        for (int i = 0; i < NS; i++) s[i] = 0.0;
        for (int i = 0; i < NS * NX; i++) C[i] = 0.0;
        for (int i = 0; i < NS * NU; i++) D[i] = 0.0;
        for (int i = 0; i < NS * NP; i++) G[i] = 0.0;
        const double r0 = x[0], r1 = x[1], th = x[4], dd = x[7], de = u[1], ddot = u[2];
        s[0] = (de - dd) - ddot * rd;
        s[1] = ddot * rd - (de - dd);
        s[2] = ddot - ddmax;
        s[3] = -ddmax - ddot;
        const double nr = sqrt(r0 * r0 + r1 * r1);
        s[4] = nr * cgs - r1;
        C[0 * NX + 7] = -1.0;
        C[1 * NX + 7] = 1.0;
        const bool tiny = nr < 1.4901161193847656e-08;  // sqrt(eps)
        C[4 * NX + 0] = (tiny ? 0.0 : r0 / nr) * cgs;
        C[4 * NX + 1] = (tiny ? 0.0 : r1 / nr) * cgs - 1.0;
        D[0 * NU + 1] = 1.0;  D[0 * NU + 2] = -rd;
        D[1 * NU + 1] = -1.0; D[1 * NU + 2] = rd;
        D[2 * NU + 2] = 1.0;
        D[3 * NU + 2] = -1.0;
        if (psw) {
            for (int i = 0; i < NX; i++) {
                s[5 + i] = p[2 + i] - x[i];
                s[13 + i] = x[i] - p[2 + i];
                C[(5 + i) * NX + i] = -1.0;
                C[(13 + i) * NX + i] = 1.0;
                G[(5 + i) * NP + 2 + i] = 1.0;
                G[(13 + i) * NP + 2 + i] = -1.0;
            }
        }
        if (ph2) {
            s[21] = th - thmax;
            s[22] = -thmax - th;
            C[21 * NX + 4] = 1.0;
            C[22 * NX + 4] = -1.0;
        }
    }
};

// shared helper: ellipsoidal keep-out zones  s_i = 1 - |H_i (r - c_i)|,  ds_i/dr = -(H_i' H_i)(r - c_i) / |H_i (r - c_i)|
// (src/utils/ellipsoid.jl:99-118; quadrotor/definition.jl:237-262, freeflyer/definition.jl:380-404).
// par block per obstacle: H (3x3 column-major), c (3).
__device__ __forceinline__ void ellipsoid_rows(const double *ob, int nobs, const double *r, double *s, double *C, int NX)
{
    for (int i = 0; i < nobs; i++) {
        const double *H = ob + 12 * i, *c = H + 9;
        const double d0 = r[0] - c[0], d1 = r[1] - c[1], d2 = r[2] - c[2];
        double y[3];
        for (int a = 0; a < 3; a++) y[a] = H[a + 3 * 0] * d0 + H[a + 3 * 1] * d1 + H[a + 3 * 2] * d2;
        const double E = sqrt(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]);
        s[i] = 1.0 - E;
        for (int b = 0; b < 3; b++) {          // (H'H d)_b = sum_a H[a,b] y_a
            const double g = H[0 + 3 * b] * y[0] + H[1 + 3 * b] * y[1] + H[2 + 3 * b] * y[2];
            C[i * NX + b] = -g / E;
        }
    }
}

// quadrotor/definition.jl:237-262: two ellipsoidal obstacles.  par: g(3), then 2 x {H(9), c(3)} from [3].
template <>
struct Constr<SCPB_MODEL_QUADROTOR> {
    static constexpr int NS = 2, NX = 6, NU = 4, NP = 1, NG = 1;
    __device__ static constexpr int gcol(int, int j) { return j; }
    __device__ static void eval(const ModelPar &P, double, int, int, const double *x, const double *, const double *,
                                double *s, double *C, double *D, double *G)
    {
        for (int i = 0; i < NS * NX; i++) C[i] = 0.0;
        for (int i = 0; i < NS * NU; i++) D[i] = 0.0;
        for (int i = 0; i < NS * NG; i++) G[i] = 0.0;
        ellipsoid_rows(&P.v[3], NS, x, s, C, NX);
    }
};

// freeflyer/definition.jl:376-442: three ellipsoidal obstacles and the space-station flight-space SDF
//   s_4 = -logsumexp(delta[:, k]; t = hom)  (src/utils/helper.jl:623-662), dG = -softmax weights on the six slacks of node k.
// par: mass [0], J [1..9], Jinv [10..18] (dynamics pack), hom [19], then 3 x {H(9), c(3)} from [20].
template <>
struct Constr<SCPB_MODEL_FREEFLYER> {
    static constexpr int NS = 4, NX = 13, NU = 6, NG = 6, NISS = 6, NOBS = 3;
    __device__ static constexpr int gcol(int k, int j) { return 1 + NISS * k + j; }
    __device__ static void eval(const ModelPar &P, double, int, int k, const double *x, const double *, const double *p,
                                double *s, double *C, double *D, double *G)
    {
        for (int i = 0; i < NS * NX; i++) C[i] = 0.0;
        for (int i = 0; i < NS * NU; i++) D[i] = 0.0;
        for (int i = 0; i < NS * NG; i++) G[i] = 0.0;
        ellipsoid_rows(&P.v[20], NOBS, x, s, C, NX);
        const double hom = P.v[19];
        double dl[NISS], a = -CUDART_INF;
        for (int j = 0; j < NISS; j++) { dl[j] = p[gcol(k, j)]; a = fmax(a, hom * dl[j]); }
        double E = 0.0;
        for (int j = 0; j < NISS; j++) E += exp(hom * dl[j] - a);
        s[3] = -((a + log(E)) / hom);
        for (int j = 0; j < NISS; j++) G[3 * NG + j] = -(exp(hom * dl[j] - a) / E);
    }
};

// Smooth logical OR of scalar predicates with scalar gradients, the reference's
//   or(pred, grad; kappa, match, normalize) -> indicator -> sigmoid -> logsumexp   (src/utils/helper.jl:623-807).
// The predicates, their gradients and `match` are divided by `normalize`; the indicator shifts the sigmoid by
// 1 - sigmoid(match) so that the OR is exact at the predicates' values `match` (one value or one per predicate).  Every
// step keeps the reference's operation order, with no contraction into fma: at the sharp end of a homotopy
// sigma = 1 - 1/(1 + exp(kappa L)) rounds to exactly 1 and the gradient factor c = exp(kappa L + 2 log(1 - sigma)) to
// exactly 0, and a rearranged formula would not saturate on the same inputs.  The shift depends on kappa only, so it is
// computed once per (seed, node) by the constructor.
template <int NM>
struct SmoothOr {
    double kap, nrm, shift;
    // sigmoid(f[, g]; kappa) of n predicates: the value, and with g its gradient *dsg
    template <int n>
    __device__ __forceinline__ static double sigmoid(const double (&f)[n], const double *g, double kap, double *dsg)
    {
        double a = __dmul_rn(kap, f[0]);
#pragma unroll
        for (int i = 1; i < n; i++) a = fmax(a, __dmul_rn(kap, f[i]));
        double e[n], E = 0.0;
#pragma unroll
        for (int i = 0; i < n; i++) {
            e[i] = exp(__dsub_rn(__dmul_rn(kap, f[i]), a));
            E = i == 0 ? e[0] : __dadd_rn(E, e[i]);
        }
        const double L = __ddiv_rn(__dadd_rn(a, log(E)), kap);
        const double kL = __dmul_rn(kap, L);
        const double sg = __dsub_rn(1.0, __ddiv_rn(1.0, __dadd_rn(1.0, exp(kL))));
        if (g) {
            double dL = 0.0;
#pragma unroll
            for (int i = 0; i < n; i++) {
                const double t = __dmul_rn(g[i], __ddiv_rn(e[i], E));
                dL = i == 0 ? t : __dadd_rn(dL, t);
            }
            const double c = exp(__dadd_rn(kL, __dmul_rn(2.0, log(__dsub_rn(1.0, sg)))));
            *dsg = __dmul_rn(__dmul_rn(kap, c), dL);
        }
        return sg;
    }
    __device__ __forceinline__ SmoothOr(double kappa, double normalize, const double (&match)[NM])
        : kap(kappa), nrm(normalize)
    {
        double m[NM];
#pragma unroll
        for (int i = 0; i < NM; i++) m[i] = __ddiv_rn(match[i], nrm);
        shift = __dsub_rn(1.0, sigmoid(m, nullptr, kap, nullptr));
    }
    // OR and dOR of the predicates pred with gradients grad (both before normalisation)
    template <int NP>
    __device__ __forceinline__ void operator()(const double (&pred)[NP], const double (&grad)[NP], double &OR,
                                               double &dOR) const
    {
        double f[NP], g[NP];
#pragma unroll
        for (int i = 0; i < NP; i++) { f[i] = __ddiv_rn(pred[i], nrm); g[i] = __ddiv_rn(grad[i], nrm); }
        OR = __dadd_rn(sigmoid(f, g, kap, &dOR), shift);
    }
};

// rendezvous_planar/definition.jl:337-413: the RCS deadband.  For thruster i, with the smooth OR of the predicates
// "reference thrust above / below the deadband",
//   s_2i = f_i - OR(fr_i) fr_i,   s_2i+1 = OR(fr_i) fr_i - f_i,   D = +-1 on f_i, -+(dOR/dfr fr_i + OR) on fr_i,
// OR = or([fr - f_db, -f_db - fr], [1, -1]; kappa, match = [f_max - f_db, -f_db - f_max], normalize = f_max + f_db).
// At the sharp end of the homotopy (kappa ~ 4.6e3) it saturates exactly (SmoothOr).
// par: m, J, lu, lv, n (dynamics pack) [0..4], then f_db [5], f_max [6], kappa [7].
// KAPPA names the slot of the homotopy parameter: eval_kappa takes kappa as an argument, so the PTR loop can pass each
// seed's own value of an in-loop homotopy schedule (scpb_ptr_set_homotopy) without copying the parameter block.
template <>
struct Constr<SCPB_MODEL_RENDEZVOUS2D> {
    static constexpr int NS = 6, NX = 6, NU = 12, NG = 1, KAPPA = 7;
    __device__ static constexpr int gcol(int, int j) { return j; }
    __device__ static void eval(const ModelPar &P, double t, int N, int k, const double *x, const double *u,
                                const double *p, double *s, double *C, double *D, double *G)
    {
        eval_kappa(P, P.v[KAPPA], t, N, k, x, u, p, s, C, D, G);
    }
    __device__ static void eval_kappa(const ModelPar &P, double kap, double, int, int, const double *, const double *u,
                                      const double *, double *s, double *C, double *D, double *G)
    {
        const double fdb = P.v[5], fmx = P.v[6];
        const SmoothOr<2> smooth_or(kap, __dadd_rn(fmx, fdb), {__dsub_rn(fmx, fdb), __dsub_rn(-fdb, fmx)});
        for (int i = 0; i < NS * NX; i++) C[i] = 0.0;
        for (int i = 0; i < NS * NU; i++) D[i] = 0.0;
        for (int i = 0; i < NS * NG; i++) G[i] = 0.0;
        for (int i = 0; i < 3; i++) {
            const double f = u[i], fr = u[3 + i];
            double OR, dOR;
            smooth_or({__dsub_rn(fr, fdb), __dsub_rn(-fdb, fr)}, {1.0, -1.0}, OR, dOR);
            const double ORfr = __dmul_rn(OR, fr);
            const double dORfr = __dadd_rn(__dmul_rn(dOR, fr), OR);
            s[2 * i] = __dsub_rn(f, ORfr);
            s[2 * i + 1] = __dsub_rn(ORfr, f);
            D[(2 * i) * NU + i] = 1.0;
            D[(2 * i) * NU + 3 + i] = -dORfr;
            D[(2 * i + 1) * NU + i] = -1.0;
            D[(2 * i + 1) * NU + 3 + i] = dORfr;
        }
    }
};

// oscillator/definition.jl:370-444: the input deadband.  With the smooth OR of the predicates "reference acceleration
// above / below the deadband",
//   s_0 = aa - OR(ar) ar,   s_1 = OR(ar) ar - aa,   D = +-1 on aa, -+(dOR/dar ar + OR) on ar,
// OR = or([ar - a_db, -a_db - ar], [1, -1]; kappa, match = a_max - a_db, normalize = a_max - a_db): a SCALAR match, so
// the indicator's shift is the sigmoid of one value (logsumexp of a single term).  C and G are zero; G is packed to the
// node's own parameter l1r_k (NG = 1), which s does not read.
// par: zeta, omega0, tf (dynamics pack) [0..2], then a_db [3], a_max [4], kappa [5] (KAPPA, as for the rendezvous).
template <>
struct Constr<SCPB_MODEL_OSCILLATOR> {
    static constexpr int NS = 2, NX = 2, NU = 4, NG = 1, KAPPA = 5;
    __device__ static constexpr int gcol(int k, int) { return k; }
    __device__ static void eval(const ModelPar &P, double t, int N, int k, const double *x, const double *u,
                                const double *p, double *s, double *C, double *D, double *G)
    {
        eval_kappa(P, P.v[KAPPA], t, N, k, x, u, p, s, C, D, G);
    }
    __device__ static void eval_kappa(const ModelPar &P, double kap, double, int, int, const double *, const double *u,
                                      const double *, double *s, double *C, double *D, double *G)
    {
        const double adb = P.v[3], amx = P.v[4];
        const double span = __dsub_rn(amx, adb);
        const SmoothOr<1> smooth_or(kap, span, {span});
        for (int i = 0; i < NS * NX; i++) C[i] = 0.0;
        for (int i = 0; i < NS * NU; i++) D[i] = 0.0;
        for (int i = 0; i < NS * NG; i++) G[i] = 0.0;
        const double aa = u[0], ar = u[1];
        double OR, dOR;
        smooth_or({__dsub_rn(ar, adb), __dsub_rn(-adb, ar)}, {1.0, -1.0}, OR, dOR);
        const double ORar = __dmul_rn(OR, ar);
        const double dORar = __dadd_rn(__dmul_rn(dOR, ar), OR);
        s[0] = __dsub_rn(aa, ORar);
        s[1] = __dsub_rn(ORar, aa);
        D[0 * NU + 0] = 1.0;
        D[0 * NU + 1] = -dORar;
        D[1 * NU + 0] = -1.0;
        D[1 * NU + 1] = dORar;
    }
};
