// conic_ipm.cuh -- batched primal-dual interior-point solver for
//     min c'x  s.t.  A x = b,  G x + s = h,  s in K = R+^l x SOC(q_1) x ... x SOC(q_nsoc)
// Replaces solve!(prg) = JuMP.optimize! -> ECOS (src/parser/program.jl:419-424) for a batch of
// seeds that share one sparsity pattern.  Algorithm family: the one ECOS implements (Mehrotra
// predictor-corrector, Nesterov-Todd scaling, static + dynamic regularisation of a quasi-definite
// KKT system, iterative refinement) -- ECOS is an unvendored dependency of the reference, so this
// is written from the published algorithm (Domahidi et al. 2013; CVXOPT conelp), not from its code.
//
// Execution model: seeds are independent, so ALL synchronisation is kept inside a CTA.
// One persistent CTA owns a group of G seeds and runs the complete interior-point solve for them:
// residual SpMVs, cone scaling, KKT assembly, numeric LDL', triangular solves, line search.
// Every sparse operation is a "gather program" generated on the host from the shared pattern
// (conic_symbolic.h); data arrays are group-blocked [group][entry][G] so the G lanes that execute
// the same program step touch adjacent doubles.  The factorisation and the substitutions are
// level-scheduled on the elimination tree: a level costs one __syncthreads, never a grid sync.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>

#include "conic_sn.cuh"

struct IpmProgram {  // device copies of ConeSymbolic index arrays
    int n, p, m, l, nsoc, nk, nnzL, nlevels, nwm, nnzA, nnzG;
    const int *soc_dim, *soc_off, *soc_woff;
    const int *A_rp, *A_ci, *G_rp, *G_ci;
    const int *At_rp, *At_ri, *At_vi, *Gt_rp, *Gt_ri, *Gt_vi;
    const int *iperm;
    const int *L_cp, *L_ri, *Lr_rp, *Lr_pos, *Lr_col;
    const int *lvl_ptr, *lvl_nodes;
    const int *as_ptr, *as_a, *as_b, *as_c, *as_src, *as_sign;
    const int4 *fw_item, *bw_item;
    const int4 *fwp_item, *bwp_item, *fa_item, *fb_item;
    SnProgram sn;            // supernodal program (used when IpmData.sn is set)
    HyProgram hy;            // top supernodes of the hybrid program (kernel variant SN = 2; the scalar program arrays of
                             // this struct are then the hybrid ones and nlevels counts the low levels + the bridge level)
    int ysize;               // doubles per seed of the Y array: max(nnzL + nk, supernodal panels)
    const int *sn_pos;       // target id -> panel offset
    const int *fa_lvl, *fa_R, *fb_lvl;
    const int *fwp_lvl, *bwp_lvl, *fwp_R, *bwp_R;
    const int2 *Lr_pc, *ft_op;
    const int4 *fwc_item, *bwc_item;             // per split item: {target, first slot, end slot, slot} (conic_symbolic.h)
    const int4 *fb_cmb;                          // per phase-B item: slot ranges of its entry and of its pivot
    int npart;                                   // partial-sum slots per seed in global memory (all programs)
    int npf, nps;                                // the most slots of one level: factorisation, substitutions
};

struct IpmOpts {
    double feastol, abstol, reltol;   // ECOS defaults 1e-8
    double delta;                     // static regularisation each seed starts from (tiny: 1e-12)
    double delta_max;                 // ... and the ceiling it may be escalated to when a factorisation loses its inertia
    double delta_esc;                 // escalation factor
    double rho_min;                   // a rejected pivot (sgn*d <= delta/2) is replaced by sgn*max(delta, rho_min)
    double bad_abs;                   // a rejected pivot larger than this (or NaN) counts as lost inertia
    int maxit, nref, equil;   // equil: Ruiz iterations (0 = off)
    int threads;              // CTA size: 512 or 1024
    int nref_aff;             // refinement steps for the predictor (affine) direction
    double reftol;
    double mu_tight;          // below this complementarity (gap / cone degree) the refinement tolerance is 1e-13 whatever reftol says
    int warm;                 // 1: seeds whose IpmData.warm flag is set start from their stored warm point (see k_ipm_solve)
    double mu_warm;           // complementarity level (gap / cone degree, equilibrated units) at which the warm point is taken
};

struct IpmData {  // group-blocked device arrays, all for B seeds
    int B, G, R;   // R: lanes per sparse row (power of two, G*R <= 32)
    int g0;        // first seed group of this launch (a launch may cover a chunk of the groups; CTA i works on group g0 + i)
    // problem data
    double *Av, *Gv, *c, *b, *h;  // equilibrated in place by the solver
    // iterates
    double *x, *y, *z, *s;
    double *eqD, *eqA, *eqG;     // Ruiz equilibration factors (columns, equality rows, cone rows)
    double *xb, *yb, *zb, *sb;   // best iterate so far (restored when the run ends without reaching the tolerances)
    double *xw, *yw, *zw, *sw;   // warm point of every seed, in the caller's units: the first iterate of the LAST solve whose
                                 // complementarity was below IpmOpts.mu_warm -- interior and roughly centred, so the next,
                                 // slightly different program of the same seed (the next SCP iteration) can start from it
    int *warm;                   // [B] 1: the warm point of this seed is usable
    // work
    double *rx, *ry, *rz, *lam, *wm, *socw, *soceta;
    double *dx, *dy, *dz, *ds, *dsa, *dza, *tm, *gm, *r1, *r2, *e1, *e2, *rhs, *Y, *Ls, *Lrow, *invD;
    double *part;   // partial sums of split targets (IpmProgram.npart slots per seed), unless psmem
    double *pcnt;   // storage of the split targets' finished-item counters (unsigned, zero between uses), unless psmem
    int vsmem;   // 1: the substitution vector of kkt_ldl_solve lives in shared memory (nk*G doubles fit)
    int psmem;   // 1: the partial sums and counters of a level live in shared memory too (vsmem, and they fit)
    // per-seed outputs
    double *pobj, *dobj, *res;   // res: [3][B] pres, dres, gap
    int *status, *iters;
    const int *skip;   // nullable [B]: seeds marked non-zero are not solved (their outputs are left untouched)
    int debug_kkt;     // test hook (scpb_debug_kkt_solve_dev): assemble + factor with the caller's wm, solve rhs in place, return
    int lvl_prof;      // 1: also record per-level cycles behind prof[12..]
    int sn;            // 1: supernodal factorisation / sweeps (conic_sn.cuh); 0: scalar level-scheduled programs
    long long *prof;   // [8] cycle counters of CTA 0: equilibrate, init, residuals, scaling+assemble, factor, solves, line search+update, total
    double *trace;     // diagnostic (SCPB_IPM_TRACE=<seed>): per-iteration rows of 10 doubles for seed trace_seed, or nullptr
    int trace_seed;
};

enum { IPM_OPTIMAL = 0, IPM_MAXIT = 1, IPM_NUMERICAL = 2, IPM_ALMOST = 3, IPM_PINF = 4, IPM_DINF = 5 };

#define IPM_MAXG 8
#define IPM_NT_MAX 1024

#ifdef CONIC_IPM_IMPL   // the kernel itself is compiled in conic_api.cu only
// ---------------------------------------------------------------------------------------------
struct Ctx {
    int G, sg, slot, nslots, tid, nwarps;
    // row-type work (sparse dot products): R lanes cooperate on one row for the G seeds of the group;
    // lane layout inside a warp: tid = (item*R + rr)*G + sg, reduced with xor-shuffles over rr
    int R, rr, isl, nisl;               // current per-level values, see set_lanes()
    const int *s_lvl;                   // level pointers (nodes per level) staged in shared memory
    int o_fal, o_faR, o_fbl;                // balanced factorisation program: phase A item pointers / lanes, phase B pointers
    int o_fwl, o_bwl, o_fwR, o_bwR, o_vs;   // balanced substitution programs (item pointers, lanes per level) and
                                            // the substitution vector: int offsets into the dynamic shared window
    int Rmax;
    int *flag;                          // shared scratch word for CTA-uniform decisions
    long long *lprof;                   // thread 0 of CTA 0: per-level cycles [factor | forward | backward][nlevels]
    int sn;                             // supernodal mode
    const struct SnArgs *s_sn;          // supernodal mode: argument block of the panel kernels, in shared memory
    const struct HyArgs *s_hy;          // hybrid mode: argument block of the top-panel phases, in shared memory
    size_t ysize;                       // doubles per seed of the Y array
    const int *s_done;                  // shared: per-seed "finished" flags (finished seeds skip the per-seed panel work)
    double *s_delta;                    // shared: per-seed static regularisation
    int *s_bad;                         // shared: per-seed "inertia lost" flag raised by the factorisation
    const double *s_mu;                 // shared: per-seed mu (complementarity gap / deg) of the current iterate
    double *red;   // shared: [10][IPM_NT_MAX/32][IPM_MAXG]
    double *out;   // shared: [10][IPM_MAXG]
};

// This CTA's group arrays (group-blocked, already offset to the group) and the CTA-uniform scalars of the solve, in
// shared memory, filled by thread 0 once per launch.  As 64-bit bases in every thread's registers they do not fit the 64
// registers of a 1024-thread CTA: they end up in a per-thread stack frame (312 KB of local memory per CTA) that the
// loops reload mostly from L2, and what the body keeps live across the level programs' calls is taken from their
// registers.  A base read from here where it is used costs one shared load, and a barrier ends its life (the barrier
// orders shared memory, so the load is issued again after it).
struct IpmGroup {
    double *Av, *Gv, *cc, *bb, *hh;   // equilibrated problem data
    double *x, *y, *z, *s, *eqD, *eqA, *eqG, *xb, *yb, *zb, *sb;
    double *rx, *ry, *rz, *lam, *wm, *socw, *soceta;
    double *dx, *dy, *dz, *ds, *dsa, *dza, *tm, *gm, *r1, *r2, *e1, *rhs, *Y, *Ls, *invD;
    double *vs;                       // shared-memory substitution vector (nullptr: the sweeps work in global memory)
    double reftol;                    // iterative refinement stops once |residual|_inf <= reftol*(1+|rhs|_inf) while the
    double mu_tight;                  // seed's mu is above mu_tight, and at min(reftol, 1e-13) below it
};
__shared__ IpmGroup ipm_ar;
// A base read from shared memory is a generic pointer to the compiler: without this it would issue generic loads and
// stores, and take every store through such a pointer as one that may change the shared blocks
template <class T>
__device__ __forceinline__ T *glb(T *p) { __builtin_assume(__isGlobal(p)); return p; }

// per-seed reduction of up to K values; op 0 = sum, 1 = min, 2 = max. Result in c.out[k*MAXG + sg].
template <int K>
__device__ __forceinline__ void seed_reduce(const Ctx &c, double (&v)[K], int op)
{
    const int lane = c.tid & 31, warp = c.tid >> 5;
    const int G = c.G;
#pragma unroll
    for (int k = 0; k < K; k++) {
        double a = v[k];
        for (int o = 16; o >= G; o >>= 1) {
            const double t = __shfl_xor_sync(0xffffffffu, a, o);
            a = (op == 0) ? a + t : ((op == 1) ? fmin(a, t) : fmax(a, t));
        }
        v[k] = a;
    }
    __syncthreads();  // protect red/out from the previous use
    if (lane < G) {
#pragma unroll
        for (int k = 0; k < K; k++) c.red[(k * (IPM_NT_MAX / 32) + warp) * IPM_MAXG + lane] = v[k];
    }
    __syncthreads();
    if (c.tid < G) {
#pragma unroll
        for (int k = 0; k < K; k++) {
            double a = c.red[(k * (IPM_NT_MAX / 32)) * IPM_MAXG + c.tid];
            for (int w = 1; w < c.nwarps; w++) {
                const double t = c.red[(k * (IPM_NT_MAX / 32) + w) * IPM_MAXG + c.tid];
                a = (op == 0) ? a + t : ((op == 1) ? fmin(a, t) : fmax(a, t));
            }
            c.out[k * IPM_MAXG + c.tid] = a;
        }
    }
    __syncthreads();
}

#define GI(e) ((size_t)(e) * G + sg)

// cycle counters of the solve (written to IpmData.prof by thread 0 of CTA 0).  Only thread 0 keeps them, in shared
// memory: as per-thread registers they were live across every call of the level programs and took registers from them.
//   [0..7] phases (k_ipm_solve, PROF), [8] forward substitutions, [9] backward ones, [10] substitutions,
//   [11] factorisations, [12] repeated factorisations, [13] last phase stamp, [14] start, [15] substitution stamp
__shared__ long long ipm_s_prof[16];
#define IPM_STAMP(k) { if (threadIdx.x == 0) ipm_s_prof[k] = clock64(); }

__device__ __forceinline__ void set_lanes(Ctx &c, int R)
{
    const int sh = 31 - __clz(R);   // R is a power of two: shifts instead of integer division
    c.R = R; c.rr = c.slot & (R - 1); c.isl = c.slot >> sh; c.nisl = c.nslots >> sh;
}

// sum over the R lanes that share a row (offsets G, 2G, .. (R/2)G inside the warp)
__device__ __forceinline__ double lanes_sum(const Ctx &c, double a)
{
    for (int o = c.G; o < c.G * c.R; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    return a;
}


// ---- cone operators (one thread per LP row / per SOC cone, per seed) ----
// out = W^-2 * in
__device__ void apply_winv2(const IpmProgram &P, const Ctx &c, const double *wm, const double *socw,
                            const double *soceta, const double *in, double *out)
{
    const int G = c.G, sg = c.sg;
    for (int r = c.slot; r < P.l; r += c.nslots) out[GI(r)] = wm[GI(r)] * in[GI(r)];
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k], wo = o - P.l;
        const double ie2 = 1.0 / soceta[GI(k)];  // soceta holds eta^2
        double vd = socw[GI(wo)] * in[GI(o)];
        for (int i = 1; i < q; i++) vd -= socw[GI(wo + i)] * in[GI(o + i)];
        // (2 v v' - J) in, v = (w0, -w1)
        out[GI(o)] = ie2 * (2.0 * socw[GI(wo)] * vd - in[GI(o)]);
        for (int i = 1; i < q; i++) out[GI(o + i)] = ie2 * (-2.0 * socw[GI(wo + i)] * vd + in[GI(o + i)]);
    }
}
// out = W^2 * in
__device__ void apply_w2(const IpmProgram &P, const Ctx &c, const double *wm, const double *socw,
                         const double *soceta, const double *in, double *out)
{
    const int G = c.G, sg = c.sg;
    for (int r = c.slot; r < P.l; r += c.nslots) out[GI(r)] = in[GI(r)] / wm[GI(r)];
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k], wo = o - P.l;
        const double e2 = soceta[GI(k)];
        double wd = 0.0;
        for (int i = 0; i < q; i++) wd += socw[GI(wo + i)] * in[GI(o + i)];
        out[GI(o)] = e2 * (2.0 * socw[GI(wo)] * wd - in[GI(o)]);
        for (int i = 1; i < q; i++) out[GI(o + i)] = e2 * (2.0 * socw[GI(wo + i)] * wd + in[GI(o + i)]);
    }
}

// ---- LDL' : assemble, factor, solve ----
__device__ __forceinline__ void kkt_assemble(const IpmProgram &P, const Ctx &c, const IpmData &D, const double *Av, const double *Gv,
                             const double *wmx, double *Y, double delta)
{
    const int G = c.G, sg = c.sg;
    const int ntgt = P.nnzL + P.nk;
    (void)delta;
    const double dl = c.s_delta[sg];
    for (int t = c.slot; t < ntgt; t += c.nslots) {
        double acc = dl * (double)P.as_sign[t];
        const int src = P.as_src[t];
        if (src >= 0) acc += Av[GI(src)];
        for (int k = P.as_ptr[t]; k < P.as_ptr[t + 1]; k++)
            acc = fma(Gv[GI(P.as_a[k])] * Gv[GI(P.as_b[k])], wmx[GI(P.as_c[k])], acc);
        if (D.sn) Y[(size_t)sg * c.ysize + P.sn_pos[t]] = acc;   // supernodal mode: straight into this seed's dense panels
        else Y[GI(t)] = acc;
    }
    __syncthreads();
}

// ---- numeric LDL' : balanced, level-scheduled gather program (conic_symbolic.h, "balanced factorisation program") ----
// Phase A of a level: an item subtracts at most R*IPM_FPF products Y[a]*Ls[b] from one target; a lane owns at most
// IPM_FPF of them, so all its op indices and then all its gathers are in flight together.  An item of a target whose op
// list was split only stores its partial sum in its slot (numbered per level, conic_symbolic.h: combine_in_phase_b);
// the slots of a level live in shared memory (the window of the substitution vector, which is free while the
// factorisation runs) or, when they do not fit, in global memory.  Every read of Y goes to L2 (ld.cg).  Phase B
// finishes the level's columns behind the level's barrier: each item subtracts the slots of its entry and of its
// column's pivot in slot order as it reads them (the same bits in every item of the column, and the same bits as
// summing them in any other place in that order), regularises its own copy of the pivot; the diagonal item stores 1/d,
// the others write the combined entry back to Y for the later levels, scale it and store it twice (column order for the
// backward sweep, row order for the forward sweep).  Combine-only items (flag 4, the hybrid program's bridge level) just
// write their combined target back.  No fence, no atomic: the level's barrier orders the slots.
// The program data of the next phase (item descriptors, op indices) is requested one phase early.
// Separate (noinline) function with its arguments in shared memory: see ipm_fa.
#define IPM_FPF CONIC_FACTOR_PF
// Substitutions: an item of a split target stores its partial sum in its slot and counts itself in; the last item of
// the target to finish subtracts all slots from the target in slot order (and resets the counter), so the sum does not
// depend on the order in which the items ran.  Returns true in the thread that has to do that.  Slots and counters are
// the level's, in shared memory (or global memory when they do not fit): the block-scope fence and atomic are all the
// ordering the CTA-local hand-over needs.
__device__ __forceinline__ bool ipm_split_done(double *part, unsigned *cnt, int4 e, double v, int G, int sg)
{
    part[e.w * G + sg] = v;
    __threadfence_block();
    const bool last = atomicAdd(&cnt[e.y * G + sg], 1u) == (unsigned)(e.z - e.y - 1);
    if (last) { __threadfence_block(); cnt[e.y * G + sg] = 0u; }
    return last;
}
// acc minus the slots [k0, k1) in slot order
__device__ __forceinline__ double ipm_split_sum(const double *part, int k0, int k1, double acc, int G, int sg)
{
    for (int k = k0; k < k1; k++) acc -= part[k * G + sg];
    return acc;
}
struct FactorArgs {   // CTA-uniform: one block per launch in shared memory (ipm_fa)
    const int4 *fa_item, *fb_item;
    const int2 *ft_op;
    const int4 *fb_cmb;             // per phase-B item: slot ranges of its entry and of its pivot
    double *Y, *Ls, *Lrow, *invD;   // group-blocked, already offset to this CTA's group
    double *part;                   // partial sums of the level's split targets (shared or global memory)
    int o_fal, o_faR, o_fbl;        // offsets (ints) into the dynamic shared memory window
    int nl, nnzLd, G, nslots;
    long long *lprof;               // per-level cycle counters of CTA 0 (written by its thread 0) or nullptr
};
extern __shared__ int ipm_smem[];
// per-seed regularisation state of the factorisation, file-scope shared so that the noinline level programs reach it
__shared__ double ipm_s_delta[IPM_MAXG];   // static regularisation of each seed of the group
__shared__ int ipm_s_bad[IPM_MAXG];        // "inertia lost" flags raised by the factorisation
__shared__ double ipm_s_reg[2];            // rho_min, bad_abs
// The factorisation's arguments live in shared memory (filled once per launch), not in registers.  A subroutine called
// inside the solver's loops gets less than the 64 registers of a 1024-thread CTA (the body keeps some of its values in
// registers across the call); a by-value block plus the phase-A pipeline did not fit, and what does not fit is spilled
// to local memory inside the pass loops.  Loads from the block after a barrier are reissued (the barrier orders shared
// memory), so the phase-B pointers and the profile state take no register across phase A.  The group size G is a
// compile-time constant (one inlined copy per G behind the one call site, kkt_factor_levels) and all indices are 32-bit
// element offsets into this group's arrays, so the index arithmetic needs no 64-bit or multiply temporaries.
__shared__ FactorArgs ipm_fa;
__shared__ long long ipm_lvl_t;            // thread 0 of CTA 0: cycle counter at the end of the previous level

template <int G>
__device__ __forceinline__ void kkt_factor_levels_g()
{
    const FactorArgs &a = ipm_fa;
    __builtin_assume(__isGlobal(a.fa_item)); __builtin_assume(__isGlobal(a.fb_item)); __builtin_assume(__isGlobal(a.ft_op));
    __builtin_assume(__isGlobal(a.Y)); __builtin_assume(__isGlobal(a.Ls)); __builtin_assume(__isGlobal(a.Lrow));
    __builtin_assume(__isGlobal(a.invD));
    const int sg = threadIdx.x & (G - 1), slot = threadIdx.x / G, nslots = a.nslots;
    const int *fal = ipm_smem + a.o_fal, *faR = ipm_smem + a.o_faR, *fbl = ipm_smem + a.o_fbl;
    // three-stage software pipeline over the passes of phase A: the item descriptor of pass p+2 and the op indices of
    // pass p+1 are requested while the gathers of pass p are in flight, so a pass costs one memory latency
    int t_tgt;                 // current pass: target, or partial-sum slot | 1 << 30 for a split target, or -1
    int2 t_op[IPM_FPF];        // current pass: op indices of this lane (x < 0: none)
    int i_tgt, i_k0, i_k1;     // next pass: item descriptor (k0 already offset to this lane)
#define IPM_FA_ITEM(LV, OFF)                                                              \
    {                                                                                     \
        const int R_ = faR[LV], sh_ = 31 - __clz(R_);                                     \
        const int w_ = fal[LV] + (OFF) + (slot >> sh_);                                   \
        i_tgt = -1; i_k0 = 0; i_k1 = 0;                                                   \
        if ((OFF) < fal[(LV) + 1] - fal[LV] && w_ < fal[(LV) + 1]) {                      \
            const int4 it_ = a.fa_item[w_];                                               \
            i_tgt = it_.w ? ((it_.w - 1) | (1 << 30)) : it_.x;                              \
            i_k0 = it_.y + (slot & (R_ - 1)); i_k1 = it_.z;                               \
        }                                                                                 \
    }
#define IPM_FA_OPS(TGT, OP, R_)                                                           \
    {                                                                                     \
        TGT = i_tgt;                                                                      \
        _Pragma("unroll") for (int j = 0; j < IPM_FPF; j++) {                             \
            const int k_ = i_k0 + j * (R_);                                               \
            OP[j] = (i_tgt >= 0 && k_ < i_k1) ? a.ft_op[k_] : make_int2(-1, 0);           \
        }                                                                                 \
    }
    IPM_FA_ITEM(0, 0)
    IPM_FA_OPS(t_tgt, t_op, faR[0])
    IPM_FA_ITEM(0, (nslots >> (31 - __clz(faR[0]))))
    if (threadIdx.x == 0 && a.lprof) ipm_lvl_t = clock64();
    for (int lv = 0; lv < a.nl; lv++) {
        // ---- phase A ----
        const int R = faR[lv], nisl = nslots >> (31 - __clz(R));
        const int nA = fal[lv + 1] - fal[lv];
        for (int off = 0; off < nA; off += nisl) {
            double ya_[IPM_FPF], la_[IPM_FPF];
#pragma unroll
            for (int j = 0; j < IPM_FPF; j++) {
                const bool on_ = t_op[j].x >= 0;
                ya_[j] = on_ ? __ldcg(&a.Y[t_op[j].x * G + sg]) : 0.0;
                la_[j] = on_ ? a.Lrow[t_op[j].y * G + sg] : 0.0;   // row order: consecutive within an item
            }
            int n_tgt; int2 n_op[IPM_FPF];
            IPM_FA_OPS(n_tgt, n_op, R)                       // pass p+1 (descriptor requested one pass ago)
            IPM_FA_ITEM(lv, off + 2 * nisl)                  // pass p+2
            double part_ = 0.0;
#pragma unroll
            for (int j = 0; j < IPM_FPF; j++) part_ = fma(ya_[j], la_[j], part_);
            for (int o_ = G; o_ < G * R; o_ <<= 1) part_ += __shfl_xor_sync(0xffffffffu, part_, o_);
            if (t_tgt >= 0 && (slot & (R - 1)) == 0) {
                if (t_tgt >> 30) a.part[(t_tgt & 0x3fffffff) * G + sg] = part_;   // phase B combines it
                else { double *p_ = &a.Y[t_tgt * G + sg]; *p_ = __ldcg(p_) - part_; }
            }
            t_tgt = n_tgt;
#pragma unroll
            for (int j = 0; j < IPM_FPF; j++) t_op[j] = n_op[j];
        }
        // first phase-B item of this lane and its slot ranges, and the descriptor of the next level's first pass: in
        // flight across the barrier
        const int b0 = fbl[lv], b1 = fbl[lv + 1];
        int4 sc = make_int4(-1, 0, 0, 0), sr = make_int4(0, 0, 0, 0);
        if (b0 + slot < b1) { sc = a.fb_item[b0 + slot]; sr = a.fb_cmb[b0 + slot]; }
        if (lv + 1 < a.nl) IPM_FA_ITEM(lv + 1, 0)
        __syncthreads();
        // ---- phase B: one latency per pass (the next item is requested while the current loads are in flight) ----
        for (int w = b0 + slot; w < b1; w += nslots) {
            const double sgn = (sc.w & 1) ? 1.0 : -1.0;
            const bool isd = (sc.w & 2) != 0;
            double e = __ldcg(&a.Y[sc.x * G + sg]);
            double d = isd ? 0.0 : __ldcg(&a.Y[(a.nnzLd + sc.y) * G + sg]);
            const int4 cur = sc, cr = sr;
            if (w + nslots < b1) { sc = a.fb_item[w + nslots]; sr = a.fb_cmb[w + nslots]; }
            e = ipm_split_sum(a.part, cr.x, cr.y, e, G, sg);
            if (isd) d = e;
            else {
                d = ipm_split_sum(a.part, cr.z, cr.w, d, G, sg);
                if (cr.y > cr.x) a.Y[cur.x * G + sg] = e;   // a later level reads it as an operand
                if (cur.w & 4) continue;                // combine-only item
            }
            const double dl_ = ipm_s_delta[sg];
            if (!(sgn * d > 0.5 * dl_)) {   // dynamic regularisation keeps the expected inertia
                if (isd && !(fabs(d) <= ipm_s_reg[1])) ipm_s_bad[sg] = 1;   // not a small pivot: cancellation destroyed it
                d = sgn * fmax(dl_, ipm_s_reg[0]);
            }
            const double inv = 1.0 / d;
            if (isd) a.invD[cur.y * G + sg] = inv;
            else {
                const double lv_ = e * inv;
                a.Ls[cur.x * G + sg] = lv_;
                a.Lrow[cur.z * G + sg] = lv_;
            }
        }
        if (lv + 1 < a.nl) {   // op indices of the next level's first pass, descriptor of its second pass
            const int Rn = faR[lv + 1];
            IPM_FA_OPS(t_tgt, t_op, Rn)
            IPM_FA_ITEM(lv + 1, (nslots >> (31 - __clz(Rn))))
        }
        __syncthreads();
        if (threadIdx.x == 0 && a.lprof) { const long long tn = clock64(); a.lprof[lv] += tn - ipm_lvl_t; ipm_lvl_t = tn; }
    }
#undef IPM_FA_ITEM
#undef IPM_FA_OPS
}
__device__ __noinline__ void kkt_factor_levels()
{
    switch (ipm_fa.G) {
        case 1: kkt_factor_levels_g<1>(); break;
        case 2: kkt_factor_levels_g<2>(); break;
        case 4: kkt_factor_levels_g<4>(); break;
        default: kkt_factor_levels_g<8>(); break;
    }
}

// supernodal numeric factorisation: one thread (small leaves) or one lane group (8, 16 or 32 lanes, by panel height)
// per (supernode, seed) item, one barrier per supernodal level; panels live in registers (conic_sn.cuh).  The
// descriptor of a unit's next item is requested before the current item is worked on.
// Like the scalar programs these are separate (noinline) functions whose arguments come from shared memory: passing the
// solver's context or the kernel parameters by reference would force them into local memory for the whole kernel.
struct SnArgs {
    SnProgram sn;
    double *Y, *invD, *vs;          // this group's panels (one seed after the other), 1/D (group-blocked), shared vector
    const int *s_done;              // shared: finished seeds are skipped
    const double *s_delta;          // shared: per-seed static regularisation
    int *s_bad;                     // shared: per-seed "inertia lost" flags
    double rho_min, bad_abs;
    size_t ysize;
    int G, tid, nwarps, nls;        // nls: scalar level count (stride of the profile arrays)
    long long *lprof;
};

template <int GS, class F>
__device__ __forceinline__ void sn_for_items(const SnArgs &a, int lv, int cls, F &&f)
{
    const int i0 = a.sn.cls_ptr[5 * lv + cls], nit = (a.sn.cls_ptr[5 * lv + cls + 1] - i0) * a.G;
    const int gsh = 31 - __clz(a.G);
    int unit, nunits;
    if (GS == 1) { unit = a.tid; nunits = a.nwarps * 32; }
    else { constexpr int GPW = 32 / (GS == 1 ? 32 : GS); unit = (a.tid >> 5) * GPW + ((a.tid & 31) / (GS == 1 ? 32 : GS)); nunits = a.nwarps * GPW; }
    int it = unit;
    int4 d0 = make_int4(0, 0, 0, 0), d1 = d0;
    if (it < nit) { const int q = 2 * (i0 + (it >> gsh)); d0 = a.sn.desc[q]; d1 = a.sn.desc[q + 1]; }
    while (it < nit) {
        const int sgi = it & (a.G - 1);
        const int4 c0 = d0, c1 = d1;
        const int nx = it + nunits;
        if (nx < nit) { const int q = 2 * (i0 + (nx >> gsh)); d0 = a.sn.desc[q]; d1 = a.sn.desc[q + 1]; }
        if (!a.s_done[sgi]) f(c0, c1, sgi);    // lane groups: uniform within the group
        it = nx;
    }
}

__device__ __noinline__ void kkt_factor_sn(const SnArgs *ap, int tid)
{
    SnArgs a = *ap;       // from shared memory (filled once per launch): nothing of the caller's goes to the stack
    a.tid = tid;
    if (tid != 0) a.lprof = nullptr;
    const int G = a.G;
    long long tl_ = a.lprof ? clock64() : 0;
    for (int lv = 0; lv < a.sn.nlevels; lv++) {
        sn_for_items<1>(a, lv, 0, [&](const int4 d0, const int4 d1, int sgi) {
            const double dl = a.s_delta[sgi];
            sn1_factor_panel(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, a.invD, G, sgi, 0.5 * dl, fmax(dl, a.rho_min), a.bad_abs, &a.s_bad[sgi]); });
        sn_for_items<8>(a, lv, 1, [&](const int4 d0, const int4 d1, int sgi) {
            const double dl = a.s_delta[sgi];
            sn_factor_panel<8>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, a.invD, G, sgi, 0.5 * dl, fmax(dl, a.rho_min), a.bad_abs, &a.s_bad[sgi]); });
        sn_for_items<16>(a, lv, 2, [&](const int4 d0, const int4 d1, int sgi) {
            const double dl = a.s_delta[sgi];
            sn_factor_panel<16>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, a.invD, G, sgi, 0.5 * dl, fmax(dl, a.rho_min), a.bad_abs, &a.s_bad[sgi]); });
        sn_for_items<32>(a, lv, 3, [&](const int4 d0, const int4 d1, int sgi) {
            const double dl = a.s_delta[sgi];
            sn_factor_panel<32>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, a.invD, G, sgi, 0.5 * dl, fmax(dl, a.rho_min), a.bad_abs, &a.s_bad[sgi]); });
        __syncthreads();
        if (a.lprof) { const long long tn = clock64(); a.lprof[lv] += tn - tl_; tl_ = tn; }
    }
}

// supernodal substitutions on the shared-memory vector: DIR > 0 forward (levels ascending), DIR < 0 backward
template <int DIR>
__device__ __noinline__ void kkt_sweep_sn(const SnArgs *ap, int tid)
{
    SnArgs a = *ap;
    a.tid = tid;
    if (tid != 0) a.lprof = nullptr;
    const int G = a.G;
    double *vs = a.vs;
    long long tlp_ = a.lprof ? clock64() : 0;
    for (int st = 0; st < a.sn.nlevels; st++) {
        const int lv = DIR > 0 ? st : a.sn.nlevels - 1 - st;
        if (DIR > 0) {
            sn_for_items<1>(a, lv, 0, [&](const int4 d0, const int4 d1, int sgi) { sn1_forward_panel(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
            sn_for_items<8>(a, lv, 1, [&](const int4 d0, const int4 d1, int sgi) { sn_forward_panel<8>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
            sn_for_items<16>(a, lv, 2, [&](const int4 d0, const int4 d1, int sgi) { sn_forward_panel<16>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
            sn_for_items<32>(a, lv, 3, [&](const int4 d0, const int4 d1, int sgi) { sn_forward_panel<32>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
        } else {
            sn_for_items<1>(a, lv, 0, [&](const int4 d0, const int4 d1, int sgi) { sn1_backward_panel(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
            sn_for_items<8>(a, lv, 1, [&](const int4 d0, const int4 d1, int sgi) { sn_backward_panel<8>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
            sn_for_items<16>(a, lv, 2, [&](const int4 d0, const int4 d1, int sgi) { sn_backward_panel<16>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
            sn_for_items<32>(a, lv, 3, [&](const int4 d0, const int4 d1, int sgi) { sn_backward_panel<32>(a.sn, d0, d1, a.Y + (size_t)sgi * a.ysize, vs, G, sgi); });
        }
        __syncthreads();
        if (a.lprof) { const long long tn = clock64(); a.lprof[(DIR > 0 ? 1 : 2) * a.nls + lv] += tn - tlp_; tlp_ = tn; }
    }
}

// (L D L') v = v for v = ipm_ar.rhs
__device__ __forceinline__ void kkt_ldl_solve_sn(const IpmProgram &P, Ctx &c)
{
    const int G = c.G, sg = c.sg;
    const IpmGroup &ar = ipm_ar;
    IPM_STAMP(15)
    for (int i = c.slot; i < P.nk; i += c.nslots) ar.vs[i * G + sg] = glb(ar.rhs)[GI(i)];
    __syncthreads();
    kkt_sweep_sn<1>(c.s_sn, c.tid);
    if (c.tid == 0) { const long long t1_ = clock64(); ipm_s_prof[8] += t1_ - ipm_s_prof[15]; ipm_s_prof[15] = t1_; }
    for (int i = c.slot; i < P.nk; i += c.nslots) ar.vs[i * G + sg] *= glb(ar.invD)[GI(i)];
    __syncthreads();
    kkt_sweep_sn<-1>(c.s_sn, c.tid);
    for (int i = c.slot; i < P.nk; i += c.nslots) glb(ar.rhs)[GI(i)] = ar.vs[i * G + sg];
    __syncthreads();
    if (c.tid == 0) { ipm_s_prof[9] += clock64() - ipm_s_prof[15]; ipm_s_prof[10] += 1; }
}

// ---- hybrid program: the top supernodes (conic_sn.cuh, hy_*), one warp per (supernode, seed) item, one barrier per
// top level.  Separate noinline functions whose arguments come from shared memory, like the supernodal ones.
struct HyArgs {
    HyProgram hy;
    double *Y, *Ls, *invD;          // group-blocked, offset to this CTA's group
    const int *s_done;              // shared: finished seeds are skipped
    const double *s_delta;          // shared: per-seed static regularisation
    int *s_bad;                     // shared: per-seed "inertia lost" flags
    double rho_min, bad_abs;
    int o_vs, nnzL, G, nwarps;
    long long *lprof;               // [3][ntl] cycle counters behind the scalar ones (CTA 0, thread 0) or nullptr
};

template <class F>
__device__ __forceinline__ void hy_for_items(const HyArgs &a, int tl, int tid, F &&f)
{
    const int i0 = a.hy.tl_ptr[tl], nit = (a.hy.tl_ptr[tl + 1] - i0) * a.G;
    const int gsh = 31 - __clz(a.G);
    int it = tid >> 5;
    int4 d0 = make_int4(0, 0, 0, 0), d1 = d0;
    if (it < nit) { const int q = 2 * (i0 + (it >> gsh)); d0 = a.hy.desc[q]; d1 = a.hy.desc[q + 1]; }
    while (it < nit) {
        const int sgi = it & (a.G - 1);
        const int4 c0 = d0, c1 = d1;
        const int nx = it + a.nwarps;
        if (nx < nit) { const int q = 2 * (i0 + (nx >> gsh)); d0 = a.hy.desc[q]; d1 = a.hy.desc[q + 1]; }
        if (!a.s_done[sgi]) f(c0, c1, sgi);    // warp-uniform
        it = nx;
    }
}

__device__ __noinline__ void kkt_factor_top(const HyArgs *ap, int tid)
{
    const HyArgs &a = *ap;   // read in place: a register copy of the whole block is spilled at 1024 threads
    long long *lp = (tid == 0) ? a.lprof : nullptr;
    long long tl_ = lp ? clock64() : 0;
    for (int tl = 0; tl < a.hy.ntl; tl++) {
        hy_for_items(a, tl, tid, [&](const int4 d0, const int4 d1, int sgi) {
            const double dl = a.s_delta[sgi];
            hy_factor_panel<32>(d0, d1, a.hy.upd_dst, a.Y, a.Ls, a.invD, a.nnzL, a.G, sgi, 0.5 * dl, fmax(dl, a.rho_min), a.bad_abs,
                                &a.s_bad[sgi]); });
        __syncthreads();
        if (lp) { const long long tn = clock64(); lp[tl] += tn - tl_; tl_ = tn; }
    }
}

template <int DIR>
__device__ __noinline__ void kkt_sweep_top(const HyArgs *ap, int tid)
{
    const HyArgs &a = *ap;
    double *vs = (double *)(ipm_smem + a.o_vs);
    long long *lp = (tid == 0 && a.lprof) ? a.lprof + (DIR > 0 ? 1 : 2) * a.hy.ntl : nullptr;
    long long tl_ = lp ? clock64() : 0;
    for (int st = 0; st < a.hy.ntl; st++) {
        const int tl = DIR > 0 ? st : a.hy.ntl - 1 - st;
        if (DIR > 0) hy_for_items(a, tl, tid, [&](const int4 d0, const int4 d1, int sgi) { hy_forward_panel<32>(d0, d1, a.hy.rows, a.Ls, vs, a.G, sgi); });
        else hy_for_items(a, tl, tid, [&](const int4 d0, const int4 d1, int sgi) { hy_backward_panel<32>(d0, d1, a.hy.rows, a.Ls, vs, a.G, sgi); });
        __syncthreads();
        if (lp) { const long long tn = clock64(); lp[tl] += tn - tl_; tl_ = tn; }
    }
}

// SN (compile time): the supernodal kernels are instantiated only in the kernel variant that uses them -- their mere
// presence as call sites costs the default (scalar) variant ~3 KB of spill traffic per thread (ptxas -v)
template <int SN>
__device__ __forceinline__ void kkt_factor(const Ctx &c)
{
    if constexpr (SN == 1) { kkt_factor_sn(c.s_sn, c.tid); return; }
    kkt_factor_levels();
    if constexpr (SN == 2) kkt_factor_top(c.s_hy, c.tid);
}

// ---- shared-memory, prefetching substitution ------------------------------------------------------------
// The vector lives in shared memory.  The host splits every L row (forward) / column (backward) into items of at most
// R*IPM_PF entries (conic_symbolic.h, "balanced substitution programs"), so a lane never owns more than IPM_PF
// entries of an item: right after a level's items are consumed the lane issues ALL global loads of the next level
// (indices + values, through an item descriptor fetched one level earlier) and only then waits at the barrier.
// Items of a split row store their partial sums in slots that the last of them subtracts in slot order
// (ipm_split_done); the slots and counters of a level live in shared memory after the vector (global memory when they
// do not fit).
// The sweep is a separate (noinline) function whose arguments live in shared memory (ipm_sw, like ipm_fa): its
// register allocation is separate from the solver body's, and no argument block occupies registers across the levels
// (a spilled prefetch is a synchronous load).
#define IPM_PF CONIC_SOLVE_PF
struct SweepArgs {
    const int4 *items;      // balanced items {node, start, end, split}
    const int *idxarr;      // entry -> vector index (column of the row entry / row of the column entry)
    const double *vals;     // group-blocked L values in the same entry order
    const int4 *cmb;        // split items: {row / column, first slot, end slot, slot}
    double *part;           // partial sums of the level's split rows / columns, and their counters
    unsigned *pcnt;
    int o_lvl, o_R, o_vs;   // offsets (ints) into the dynamic shared memory window
    int nl, lv0, G, nslots;
    long long *lprof;       // per-level cycle counters of CTA 0 (written by its thread 0) or nullptr
};
// forward and backward sweep arguments, CTA-uniform, filled once per launch (see ipm_fa)
__shared__ SweepArgs ipm_sw[2];

template <int DIR>
__device__ __noinline__ void solve_sweep()
{
    const SweepArgs &a = ipm_sw[DIR > 0 ? 0 : 1];
    __builtin_assume(__isGlobal(a.items)); __builtin_assume(__isGlobal(a.idxarr)); __builtin_assume(__isGlobal(a.vals));
    const int *lvl = ipm_smem + a.o_lvl, *Rl = ipm_smem + a.o_R;
    double *vs = (double *)(ipm_smem + a.o_vs);
    const int G = a.G, sg = threadIdx.x & (G - 1), slot = threadIdx.x >> (31 - __clz(G));
    const int nsteps = DIR > 0 ? a.nl - a.lv0 : a.lv0 + 1;
    if (nsteps <= 0) return;
    // item descriptor of this lane for the level after next; node (or partial-sum slot | 1 << 30), first entry, end
    int i_node, i_k0, i_k1, i_R;
    int q_node;                    // current item: node, or slot | 1 << 30 for a split row, or -1
    int q_idx[IPM_PF];
    double q_val[IPM_PF];
#define IPM_ITEM_LOAD(LV, OFF)                                                            \
    {                                                                                     \
        const int R_ = Rl[LV], sh_ = 31 - __clz(R_);                                      \
        const int w_ = lvl[LV] + (OFF) + (slot >> sh_);                                   \
        i_node = -1; i_R = R_; i_k0 = 0; i_k1 = 0;                                        \
        if (w_ < lvl[(LV) + 1]) {                                                         \
            const int4 it_ = a.items[w_];                                                 \
            i_node = it_.w ? ((it_.w - 1) | (1 << 30)) : it_.x;                             \
            i_k0 = it_.y + (slot & (R_ - 1)); i_k1 = it_.z;                               \
        }                                                                                 \
    }
#define IPM_VALS_LOAD()                                                                   \
    {                                                                                     \
        q_node = i_node;                                                                  \
        _Pragma("unroll") for (int j = 0; j < IPM_PF; j++) {                              \
            const int k_ = i_k0 + j * i_R;                                                \
            const bool on_ = i_node >= 0 && k_ < i_k1;                                    \
            q_idx[j] = on_ ? a.idxarr[k_] : 0;                                            \
            q_val[j] = on_ ? a.vals[(size_t)k_ * G + sg] : 0.0;                           \
        }                                                                                 \
    }
#define IPM_CONSUME(R)                                                                    \
    {                                                                                     \
        double part_ = 0.0;                                                               \
        _Pragma("unroll") for (int j = 0; j < IPM_PF; j++) part_ = fma(q_val[j], vs[q_idx[j] * G + sg], part_); \
        for (int o_ = G; o_ < G * (R); o_ <<= 1) part_ += __shfl_xor_sync(0xffffffffu, part_, o_); \
        if (q_node >= 0 && (slot & ((R) - 1)) == 0) {                                     \
            if (q_node >> 30) {                                                           \
                const int4 e_ = a.cmb[q_node & 0x3fffffff];                               \
                if (ipm_split_done(a.part, a.pcnt, e_, part_, G, sg))                     \
                    vs[e_.x * G + sg] = ipm_split_sum(a.part, e_.y, e_.z, vs[e_.x * G + sg], G, sg); \
            } else vs[q_node * G + sg] -= part_;                                          \
        }                                                                                 \
    }
    IPM_ITEM_LOAD(a.lv0, 0)
    IPM_VALS_LOAD()
    if (nsteps > 1) IPM_ITEM_LOAD(a.lv0 + DIR, 0) else i_node = -1;
    __syncthreads();
    if (threadIdx.x == 0 && a.lprof) ipm_lvl_t = clock64();
    for (int st = 0, lv = a.lv0; st < nsteps; st++, lv += DIR) {
        const int R = Rl[lv], nisl = a.nslots >> (31 - __clz(R));
        IPM_CONSUME(R)
        const int nit = lvl[lv + 1] - lvl[lv];
        if (nit > nisl) {   // wide levels: further passes (not prefetched); rare above the leaf levels
            const int sn = i_node, s0 = i_k0, s1 = i_k1, sR = i_R;
            for (int off = nisl; off < nit; off += nisl) {
                IPM_ITEM_LOAD(lv, off)
                IPM_VALS_LOAD()
                IPM_CONSUME(R)
            }
            i_node = sn; i_k0 = s0; i_k1 = s1; i_R = sR;
        }
        // prefetch: values of the next level (descriptor already here), descriptor of the level after it
        IPM_VALS_LOAD()
        if (st + 2 < nsteps) IPM_ITEM_LOAD(lv + 2 * DIR, 0) else i_node = -1;
        __syncthreads();
        if (threadIdx.x == 0 && a.lprof) { const long long tn = clock64(); a.lprof[lv] += tn - ipm_lvl_t; ipm_lvl_t = tn; }
    }
#undef IPM_ITEM_LOAD
#undef IPM_VALS_LOAD
#undef IPM_CONSUME
}

template <int SN>
__device__ __forceinline__ void kkt_ldl_solve_smem(const IpmProgram &P, Ctx &c)
{
    const int G = c.G, sg = c.sg;
    const IpmGroup &ar = ipm_ar;
    IPM_STAMP(15)
    for (int i = c.slot; i < P.nk; i += c.nslots) ar.vs[i * G + sg] = glb(ar.rhs)[GI(i)];
    // forward (level 0 rows are empty: leaves have no dependencies); the barrier inside the sweep publishes vs
    solve_sweep<1>();
    if (P.nlevels <= 1) __syncthreads();
    if constexpr (SN == 2) kkt_sweep_top<1>(c.s_hy, c.tid);   // after the bridge level: column-oriented top panels
    if (c.tid == 0) { const long long t1_ = clock64(); ipm_s_prof[8] += t1_ - ipm_s_prof[15]; ipm_s_prof[15] = t1_; }
    for (int i = c.slot; i < P.nk; i += c.nslots) ar.vs[i * G + sg] *= glb(ar.invD)[GI(i)];
    if constexpr (SN == 2) { __syncthreads(); kkt_sweep_top<-1>(c.s_hy, c.tid); }
    // backward (the top level holds roots only: empty columns)
    solve_sweep<-1>();
    if (P.nlevels <= 1) __syncthreads();
    for (int i = c.slot; i < P.nk; i += c.nslots) glb(ar.rhs)[GI(i)] = ar.vs[i * G + sg];
    __syncthreads();
    if (c.tid == 0) { ipm_s_prof[9] += clock64() - ipm_s_prof[15]; ipm_s_prof[10] += 1; }
}

// in-place solve of (L D L') v = rhs on the permuted vector v = ipm_ar.rhs
template <int SN>
__device__ __forceinline__ void kkt_ldl_solve(const IpmProgram &P, Ctx &c)
{
    if constexpr (SN == 1) { kkt_ldl_solve_sn(P, c); return; }
    if (SN == 2 || ipm_ar.vs) { kkt_ldl_solve_smem<SN>(P, c); return; }
    set_lanes(c, c.Rmax);
    const int G = c.G, sg = c.sg;
    const double *Ls = glb(ipm_ar.Ls);
    double *v = glb(ipm_ar.rhs);
    for (int lv = 0; lv < P.nlevels; lv++) {   // forward, rows of L
        const int wend = c.s_lvl[lv + 1];
        for (int w0 = c.s_lvl[lv]; w0 < wend; w0 += c.nisl) {
            const int w = w0 + c.isl;
            const bool on = w < wend;
            int4 item = make_int4(0, 0, 0, 0);
            double part = 0.0, vi = 0.0;
            if (on) {
                item = P.fw_item[w];
                if (c.rr == 0) vi = v[GI(item.x)];
                const int k1 = item.z;
                int k = item.y + c.rr;
                for (; k + c.R < k1; k += 2 * c.R) {
                    const int2 a = P.Lr_pc[k], b = P.Lr_pc[k + c.R];
                    const double l0 = Ls[GI(a.x)], v0 = v[GI(a.y)], l1 = Ls[GI(b.x)], v1 = v[GI(b.y)];
                    part = fma(l0, v0, part);
                    part = fma(l1, v1, part);
                }
                if (k < k1) { const int2 a = P.Lr_pc[k]; part = fma(Ls[GI(a.x)], v[GI(a.y)], part); }
            }
            part = lanes_sum(c, part);
            if (on && c.rr == 0) v[GI(item.x)] = vi - part;
        }
        __syncthreads();
    }
    for (int i = c.slot; i < P.nk; i += c.nslots) v[GI(i)] *= glb(ipm_ar.invD)[GI(i)];
    __syncthreads();
    for (int lv = P.nlevels - 1; lv >= 0; lv--) {   // backward, columns of L
        const int wend = c.s_lvl[lv + 1];
        for (int w0 = c.s_lvl[lv]; w0 < wend; w0 += c.nisl) {
            const int w = w0 + c.isl;
            const bool on = w < wend;
            int4 item = make_int4(0, 0, 0, 0);
            double part = 0.0, vj = 0.0;
            if (on) {
                item = P.bw_item[w];
                if (c.rr == 0) vj = v[GI(item.x)];
                const int k1 = item.z;
                int k = item.y + c.rr;
                for (; k + c.R < k1; k += 2 * c.R) {
                    const int r0 = P.L_ri[k], r1 = P.L_ri[k + c.R];
                    const double l0 = Ls[GI(k)], v0 = v[GI(r0)], l1 = Ls[GI(k + c.R)], v1 = v[GI(r1)];
                    part = fma(l0, v0, part);
                    part = fma(l1, v1, part);
                }
                if (k < k1) part = fma(Ls[GI(k)], v[GI(P.L_ri[k])], part);
            }
            part = lanes_sum(c, part);
            if (on && c.rr == 0) v[GI(item.x)] = vj - part;
        }
        __syncthreads();
    }
}

// ---- sparse products of the residuals and of kkt_solve ------------------------------------------------------------
// Row r of M x is one thread's sequential fma chain from 0.0 over the row's entries in order, and so is a column of a
// transposed product M'y (through the transposed pattern and its value map); composite expressions keep their order,
// e.g. (c + A'y) + G'z.  A thread issues the index loads, then the value and operand gathers, of up to IPM_PF entries of
// its row at once, and requests the extent of its next row while the current one is in flight.  The products are
// separate (noinline) functions whose arguments come from shared memory (ipm_mv, ipm_ar), like the level programs:
// inlined in the solver body, rows with several entries in flight do not fit the registers of a 1024-thread CTA and are
// spilled.  G is a compile-time constant (one inlined copy per group size behind each entry point).
struct SpmvArgs {   // CTA-uniform: one block per launch in shared memory
    const int *A_rp, *A_ci, *G_rp, *G_ci;
    const int *At_rp, *At_ri, *At_vi, *Gt_rp, *Gt_ri, *Gt_vi;
    const int *iperm;
    int n, p, m, G;
    const double *by, *bz;   // operands of the current kkt_solve, written by thread 0 when it starts
    double *dx, *dy, *dz;
};
__shared__ SpmvArgs ipm_mv;

// sum of Mv[vi(k)] * x[ci(k)] over k in [k0, k1) in k order; T: vi is the value map of a transposed pattern, else vi(k) = k
template <int G, bool T>
__device__ __forceinline__ double spmv_dot(const int *ci, const int *vi, const double *Mv, const double *x, int k0, int k1)
{
    const int sg = threadIdx.x & (G - 1);
    __builtin_assume(__isGlobal(ci)); __builtin_assume(__isGlobal(Mv)); __builtin_assume(__isGlobal(x));
    if (T) __builtin_assume(__isGlobal(vi));
    double acc = 0.0;
    for (int k = k0; k < k1; k += IPM_PF) {
        int xi[IPM_PF], mi[IPM_PF];
#pragma unroll
        for (int j = 0; j < IPM_PF; j++) {
            const bool on = k + j < k1;
            xi[j] = on ? ci[k + j] : 0;
            mi[j] = on ? (T ? vi[k + j] : k + j) : 0;
        }
        double mv[IPM_PF], xv[IPM_PF];
#pragma unroll
        for (int j = 0; j < IPM_PF; j++) {
            const bool on = k + j < k1;
            mv[j] = on ? Mv[mi[j] * G + sg] : 0.0;
            xv[j] = on ? x[xi[j] * G + sg] : 0.0;
        }
#pragma unroll
        for (int j = 0; j < IPM_PF; j++)
            if (k + j < k1) acc = fma(mv[j], xv[j], acc);   // skipped, not fma(0, 0, acc): that would turn -0 into +0
    }
    return acc;
}
// f(r, (M x)_r) for this thread's rows r = slot, slot + nslots, ... < nrows
template <int G, bool T, class F>
__device__ __forceinline__ void spmv_rows(const int *rp, const int *ci, const int *vi, const double *Mv, const double *x,
                                          int nrows, F &&f)
{
    __builtin_assume(__isGlobal(rp));
    const int nslots = blockDim.x / G;
    int r = threadIdx.x / G, k0 = 0, k1 = 0;
    if (r < nrows) { k0 = rp[r]; k1 = rp[r + 1]; }
    for (; r < nrows; r += nslots) {
        const int c0 = k0, c1 = k1;
        if (r + nslots < nrows) { k0 = rp[r + nslots]; k1 = rp[r + nslots + 1]; }
        f(r, spmv_dot<G, T>(ci, vi, Mv, x, c0, c1));
    }
}
// f(v, (M1' x1)_v, (M2' x2)_v) for this thread's columns v < ncols of two transposed products
template <int G, class F>
__device__ __forceinline__ void spmv_cols2(const int *rp1, const int *ri1, const int *vi1, const double *M1, const double *x1,
                                           const int *rp2, const int *ri2, const int *vi2, const double *M2, const double *x2,
                                           int ncols, F &&f)
{
    __builtin_assume(__isGlobal(rp1)); __builtin_assume(__isGlobal(rp2));
    const int nslots = blockDim.x / G;
    int v = threadIdx.x / G, k0 = 0, k1 = 0, l0 = 0, l1 = 0;
    if (v < ncols) { k0 = rp1[v]; k1 = rp1[v + 1]; l0 = rp2[v]; l1 = rp2[v + 1]; }
    for (; v < ncols; v += nslots) {
        const int c0 = k0, c1 = k1, d0 = l0, d1 = l1;
        if (v + nslots < ncols) { k0 = rp1[v + nslots]; k1 = rp1[v + nslots + 1]; l0 = rp2[v + nslots]; l1 = rp2[v + nslots + 1]; }
        const double a1 = spmv_dot<G, true>(ri1, vi1, M1, x1, c0, c1);
        f(v, a1, spmv_dot<G, true>(ri2, vi2, M2, x2, d0, d1));
    }
}
#define IPM_G_DISPATCH(F)                                                                 \
    switch (ipm_mv.G) {                                                                   \
        case 1: return F<1>();                                                            \
        case 2: return F<2>();                                                            \
        case 4: return F<4>();                                                            \
        default: return F<8>();                                                           \
    }

// residuals: rx = (c + A'y) + G'z, ry = Ax - b, rz = (Gx + s) - h
template <int G>
__device__ __forceinline__ void spmv_residuals_g()
{
    const SpmvArgs &a = ipm_mv;
    const IpmGroup &ar = ipm_ar;
    const int sg = threadIdx.x & (G - 1);
    spmv_cols2<G>(a.At_rp, a.At_ri, a.At_vi, glb(ar.Av), glb(ar.y), a.Gt_rp, a.Gt_ri, a.Gt_vi, glb(ar.Gv), glb(ar.z), a.n,
                  [&](int i, double ay, double gz) { glb(ar.rx)[i * G + sg] = glb(ar.cc)[i * G + sg] + ay + gz; });
    spmv_rows<G, false>(a.A_rp, a.A_ci, nullptr, glb(ar.Av), glb(ar.x), a.p,
                        [&](int i, double ax) { glb(ar.ry)[i * G + sg] = ax - glb(ar.bb)[i * G + sg]; });
    spmv_rows<G, false>(a.G_rp, a.G_ci, nullptr, glb(ar.Gv), glb(ar.x), a.m,
                        [&](int i, double gx) { glb(ar.rz)[i * G + sg] = gx + glb(ar.s)[i * G + sg] - glb(ar.hh)[i * G + sg]; });
}
__device__ __noinline__ void spmv_residuals() { IPM_G_DISPATCH(spmv_residuals_g) }

// right-hand side of the reduced system: r1 = r1 + G'tm, rhs = r1 (permuted), dx = 0
template <int G>
__device__ __forceinline__ void spmv_kkt_rhs_g()
{
    const SpmvArgs &a = ipm_mv;
    const IpmGroup &ar = ipm_ar;
    const int sg = threadIdx.x & (G - 1);
    spmv_rows<G, true>(a.Gt_rp, a.Gt_ri, a.Gt_vi, glb(ar.Gv), glb(ar.tm), a.n, [&](int v, double gt) {
        const double r = glb(ar.r1)[v * G + sg] + gt;
        glb(ar.r1)[v * G + sg] = r;
        glb(ar.rhs)[glb(a.iperm)[v] * G + sg] = r;
        glb(a.dx)[v * G + sg] = 0.0;
    });
}
__device__ __noinline__ void spmv_kkt_rhs() { IPM_G_DISPATCH(spmv_kkt_rhs_g) }

// gm = G dx, or G dx - bz
template <bool BZ, int G>
__device__ __forceinline__ void spmv_kkt_gdx_g()
{
    const SpmvArgs &a = ipm_mv;
    const IpmGroup &ar = ipm_ar;
    const int sg = threadIdx.x & (G - 1);
    spmv_rows<G, false>(a.G_rp, a.G_ci, nullptr, glb(ar.Gv), glb(a.dx), a.m,
                        [&](int r, double gx) { glb(ar.gm)[r * G + sg] = BZ ? gx - glb(a.bz)[r * G + sg] : gx; });
}
template <int G> __device__ __forceinline__ void spmv_kkt_gdx_g0() { spmv_kkt_gdx_g<false, G>(); }
template <int G> __device__ __forceinline__ void spmv_kkt_gdx_g1() { spmv_kkt_gdx_g<true, G>(); }
template <bool BZ>
__device__ __noinline__ void spmv_kkt_gdx()
{
    if constexpr (BZ) { IPM_G_DISPATCH(spmv_kkt_gdx_g1) } else { IPM_G_DISPATCH(spmv_kkt_gdx_g0) }
}

// residual of the reduced system into rhs (permuted): r1 - G'e1 - A'dy (e1 = W^-2 G dx) and by - A dx.  Returns this
// thread's |residual|_inf and |r1, by|_inf; a NaN entry counts as +inf (fmax would drop it)
template <int G>
__device__ __forceinline__ double2 spmv_kkt_refine_g()
{
    const SpmvArgs &a = ipm_mv;
    const IpmGroup &ar = ipm_ar;
    const int sg = threadIdx.x & (G - 1);
    double n0 = 0.0, n1 = 0.0;
    spmv_cols2<G>(a.Gt_rp, a.Gt_ri, a.Gt_vi, glb(ar.Gv), glb(ar.e1), a.At_rp, a.At_ri, a.At_vi, glb(ar.Av), glb(a.dy), a.n,
                  [&](int v, double ge, double ay) {
                      const double bx = glb(ar.r1)[v * G + sg];
                      const double r = bx - ge - ay;
                      glb(ar.rhs)[glb(a.iperm)[v] * G + sg] = r;
                      n0 = fmax(n0, r == r ? fabs(r) : CUDART_INF); n1 = fmax(n1, fabs(bx));
                  });
    spmv_rows<G, false>(a.A_rp, a.A_ci, nullptr, glb(ar.Av), glb(a.dx), a.p, [&](int r, double ax) {
        const double by = glb(a.by)[r * G + sg];
        const double rr = by - ax;
        glb(ar.rhs)[glb(a.iperm)[a.n + r] * G + sg] = rr;
        n0 = fmax(n0, rr == rr ? fabs(rr) : CUDART_INF); n1 = fmax(n1, fabs(by));
    });
    return make_double2(n0, n1);
}
__device__ __noinline__ double2 spmv_kkt_refine() { IPM_G_DISPATCH(spmv_kkt_refine_g) }
#undef IPM_G_DISPATCH

// Solve [0 A' G'; A 0 0; G 0 -W'W][dx;dy;dz] = [bx;by;bz] through the reduced system
//   (G' W^-2 G) dx + A' dy = bx + G' W^-2 bz ,  A dx = by ,  dz = W^-2 (G dx - bz)
// with nref steps of iterative refinement against the unregularised reduced operator.
// bx is r1, overwritten by bx + G' W^-2 bz; by and bz are kept.  Leaves G dx - bz in gm.
template <int SN>
__device__ __forceinline__ void kkt_solve(const IpmProgram &P, Ctx &c, const double *by, const double *bz, double *dx,
                                          double *dy, double *dz, int nref)
{
    const int G = c.G, sg = c.sg;
    const IpmGroup &ar = ipm_ar;
    const SpmvArgs &a = ipm_mv;
    if (c.tid == 0) { ipm_mv.by = by; ipm_mv.bz = bz; ipm_mv.dx = dx; ipm_mv.dy = dy; ipm_mv.dz = dz; }
    // tm = W^-2 bz ; r1 = bx + G' tm  (the barrier publishes the operands too)
    apply_winv2(P, c, glb(ar.wm), glb(ar.socw), glb(ar.soceta), bz, glb(ar.tm));
    __syncthreads();
    spmv_kkt_rhs();
    for (int r = c.slot; r < P.p; r += c.nslots) { glb(ar.rhs)[GI(P.iperm[P.n + r])] = glb(a.by)[GI(r)]; glb(a.dy)[GI(r)] = 0.0; }
    __syncthreads();
    int again = 1;   // 0: the refinement loop ended on its residual check
    for (int it = 0;; it++) {
        kkt_ldl_solve<SN>(P, c);
        for (int v = c.slot; v < P.n; v += c.nslots) glb(a.dx)[GI(v)] += glb(ar.rhs)[GI(P.iperm[v])];
        for (int r = c.slot; r < P.p; r += c.nslots) glb(a.dy)[GI(r)] += glb(ar.rhs)[GI(P.iperm[P.n + r])];
        __syncthreads();
        if (it >= nref) break;
        // residual of the reduced system: e1 = r1 - (G' W^-2 G dx + A' dy), e2 = by - A dx
        spmv_kkt_gdx<false>();
        __syncthreads();
        apply_winv2(P, c, glb(ar.wm), glb(ar.socw), glb(ar.soceta), glb(ar.gm), glb(ar.e1));  // e1: max(n,m)-sized scratch holding W^-2 G dx
        __syncthreads();
        // |residual|_inf, |rhs|_inf
        const double2 n_ = spmv_kkt_refine();
        double nrm[2] = {n_.x, n_.y};
        seed_reduce<2>(c, nrm, 2);   // ends with a barrier: rhs is complete as well
        if (c.tid == 0) {
            // the group refines again while one of its seeds asks for it.  Finished seeds (converged, failed, skipped by
            // the caller, padded lanes) have no vote: their directions are not used.  Nor has a seed whose residual is
            // not finite: refining cannot repair it, and its next residual check ends it as NUMERICAL.  Without these
            // exclusions a seed's bits depended on whether its group was padded or held a NaN seed.
            int again_ = 0;
            for (int q = 0; q < G; q++) {
                const double res = c.out[q], ref = c.out[IPM_MAXG + q];
                if (c.s_done[q] || !isfinite(res)) continue;
                // early iterations only need a direction; the last ones (small mu: the scaling matrix spans > 20 orders of
                // magnitude) need every digit, or the iterates stall a decade or two above the requested gap
                const double tol_ = (c.s_mu[q] > ar.mu_tight) ? ar.reftol : fmin(ar.reftol, 1e-13);
                if (!(res <= tol_ * (1.0 + ref))) again_ = 1;
            }
            *c.flag = again_;
        }
        __syncthreads();
        again = *c.flag;
        __syncthreads();
        if (!again) break;
    }
    // dz = W^-2 (G dx - bz).  After a residual check that ended the loop, gm already holds G dx of the final dx (the
    // subtraction follows the full row sum either way: the same bits)
    if (again) spmv_kkt_gdx<true>();
    else for (int r = c.slot; r < P.m; r += c.nslots) glb(ar.gm)[GI(r)] -= glb(a.bz)[GI(r)];
    __syncthreads();
    apply_winv2(P, c, glb(ar.wm), glb(ar.socw), glb(ar.soceta), glb(ar.gm), glb(a.dz));
    __syncthreads();
}

// smallest t with u + t e in K  (max over cones); thread-partial, to be max-reduced
__device__ double cone_shift_partial(const IpmProgram &P, const Ctx &c, const double *u)
{
    const int G = c.G, sg = c.sg;
    double t = -CUDART_INF;
    for (int r = c.slot; r < P.l; r += c.nslots) t = fmax(t, -u[GI(r)]);
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k];
        double nn = 0.0;
        for (int i = 1; i < q; i++) nn += u[GI(o + i)] * u[GI(o + i)];
        t = fmax(t, sqrt(nn) - u[GI(o)]);
    }
    return t;
}

// largest alpha with u + alpha*du in K (thread-partial min)
__device__ double cone_alpha_partial(const IpmProgram &P, const Ctx &c, const double *u, const double *du)
{
    const int G = c.G, sg = c.sg;
    double a = CUDART_INF;
    for (int r = c.slot; r < P.l; r += c.nslots) {
        const double d = du[GI(r)];
        if (d < 0.0) a = fmin(a, -u[GI(r)] / d);
    }
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k];
        const double l0 = u[GI(o)], v0 = du[GI(o)];
        double aa = v0 * v0, bb = l0 * v0, cc = l0 * l0;
        for (int i = 1; i < q; i++) {
            const double l1 = u[GI(o + i)], v1 = du[GI(o + i)];
            aa -= v1 * v1; bb -= l1 * v1; cc -= l1 * l1;
        }
        bb *= 2.0;
        if (fabs(aa) < 1e-300) { if (bb < 0.0) a = fmin(a, -cc / bb); continue; }
        const double disc = bb * bb - 4.0 * aa * cc;
        if (aa < 0.0) a = fmin(a, (-bb - sqrt(fmax(disc, 0.0))) / (2.0 * aa));
        else if (disc >= 0.0 && bb < 0.0) a = fmin(a, (-bb - sqrt(disc)) / (2.0 * aa));
    }
    return a;
}

// min over cones of the interior margin of u + alpha*du (LP: value; SOC: u0 - |u1|); thread-partial min
__device__ double cone_margin_partial(const IpmProgram &P, const Ctx &c, const double *u, const double *du,
                                      double alpha)
{
    const int G = c.G, sg = c.sg;
    double mg = CUDART_INF;
    for (int r = c.slot; r < P.l; r += c.nslots) mg = fmin(mg, u[GI(r)] + alpha * du[GI(r)]);
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k];
        double nn = 0.0;
        for (int i = 1; i < q; i++) {
            const double v = u[GI(o + i)] + alpha * du[GI(o + i)];
            nn += v * v;
        }
        mg = fmin(mg, u[GI(o)] + alpha * du[GI(o)] - sqrt(nn));
    }
    return mg;
}

// Nesterov-Todd scaling from (s, z): lam = W z, W^-2 data.  LP: wm = z/s; SOC: wbar, eta^2.
__device__ void nt_scaling(const IpmProgram &P, const Ctx &c, const double *s, const double *z, double *lam,
                           double *wm, double *socw, double *soceta)
{
    const int G = c.G, sg = c.sg;
    for (int r = c.slot; r < P.l; r += c.nslots) {
        const double sv = s[GI(r)], zv = z[GI(r)];
        wm[GI(r)] = zv / sv;
        lam[GI(r)] = sqrt(sv * zv);
    }
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k], wo = o - P.l, wb = P.soc_woff[k];
        // s'Js = (s0 - |s1|)(s0 + |s1|): same expression as the interior test of the line search, so a
        // point accepted there can never produce a negative determinant here
        double s1s1 = 0.0, z1z1 = 0.0, sz = s[GI(o)] * z[GI(o)];
        for (int i = 1; i < q; i++) {
            s1s1 += s[GI(o + i)] * s[GI(o + i)];
            z1z1 += z[GI(o + i)] * z[GI(o + i)];
            sz += s[GI(o + i)] * z[GI(o + i)];
        }
        const double ns1 = sqrt(s1s1), nz1 = sqrt(z1z1);
        const double ss = (s[GI(o)] - ns1) * (s[GI(o)] + ns1), zz = (z[GI(o)] - nz1) * (z[GI(o)] + nz1);
        const double sn = sqrt(ss), zn = sqrt(zz);
        const double gam = sqrt(0.5 * (1.0 + sz / (sn * zn)));
        const double ig = 1.0 / (2.0 * gam);
        const double e2 = sn / zn;  // eta^2
        const double eta = sqrt(e2);
        const double w0 = (s[GI(o)] / sn + z[GI(o)] / zn) * ig;
        socw[GI(wo)] = w0;
        double w1z = 0.0;
        for (int i = 1; i < q; i++) {
            const double w1 = (s[GI(o + i)] / sn - z[GI(o + i)] / zn) * ig;
            socw[GI(wo + i)] = w1;
            w1z += w1 * z[GI(o + i)];
        }
        soceta[GI(k)] = e2;
        // lam = W z = eta [w0 z0 + w1.z1 ; z0 w1 + z1 + w1 (w1.z1)/(1+w0)]
        lam[GI(o)] = eta * (w0 * z[GI(o)] + w1z);
        for (int i = 1; i < q; i++)
            lam[GI(o + i)] = eta * (z[GI(o)] * socw[GI(wo + i)] + z[GI(o + i)] + socw[GI(wo + i)] * w1z / (1.0 + w0));
        // dense W^-2 block for the KKT assembly: (2 v v' - J)/eta^2, v = (w0, -w1)
        for (int i = 0; i < q; i++)
            for (int j = 0; j < q; j++) {
                const double vi = (i == 0) ? w0 : -socw[GI(wo + i)], vj = (j == 0) ? w0 : -socw[GI(wo + j)];
                const double Jij = (i == j) ? ((i == 0) ? 1.0 : -1.0) : 0.0;
                wm[GI(wb + i * q + j)] = (2.0 * vi * vj - Jij) / e2;
            }
    }
}

__device__ void set_identity_scaling(const IpmProgram &P, const Ctx &c, double *wm, double *socw, double *soceta)
{
    const int G = c.G, sg = c.sg;
    for (int r = c.slot; r < P.l; r += c.nslots) wm[GI(r)] = 1.0;
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k], wo = o - P.l, wb = P.soc_woff[k];
        soceta[GI(k)] = 1.0;
        for (int i = 0; i < q; i++) socw[GI(wo + i)] = (i == 0) ? 1.0 : 0.0;
        for (int i = 0; i < q; i++)
            for (int j = 0; j < q; j++) wm[GI(wb + i * q + j)] = (i == j) ? 1.0 : 0.0;
    }
}

// tmp = -s + W( lam \ (sigma*mu*e - (W^-1 dsa) o (W dza)) )   (combined-direction right-hand side)
__device__ void combined_tmp(const IpmProgram &P, const Ctx &c, const double *s, const double *z, const double *lam,
                             const double *socw, const double *soceta, const double *dsa, const double *dza,
                             const double *sigmu /*shared per seed*/, double *tmp)
{
    const int G = c.G, sg = c.sg;
    const double sm = sigmu[sg];
    for (int r = c.slot; r < P.l; r += c.nslots)
        tmp[GI(r)] = -s[GI(r)] + (sm - dsa[GI(r)] * dza[GI(r)]) / z[GI(r)];
    for (int k = c.slot; k < P.nsoc; k += c.nslots) {
        const int o = P.soc_off[k], q = P.soc_dim[k], wo = o - P.l;
        const double eta = sqrt(soceta[GI(k)]), w0 = socw[GI(wo)];
        // a = W^-1 dsa, b = W dza  (computed on the fly, q small)
        double w1ds = 0.0, w1dz = 0.0;
        for (int i = 1; i < q; i++) { w1ds += socw[GI(wo + i)] * dsa[GI(o + i)]; w1dz += socw[GI(wo + i)] * dza[GI(o + i)]; }
        const double a0 = (w0 * dsa[GI(o)] - w1ds) / eta, b0 = eta * (w0 * dza[GI(o)] + w1dz);
        // Jordan product a o b = (a'b, a0 b1 + b0 a1)
        double ab = a0 * b0;
        for (int i = 1; i < q; i++) {
            const double w1 = socw[GI(wo + i)];
            const double a1 = (-dsa[GI(o)] * w1 + dsa[GI(o + i)] + w1 * w1ds / (1.0 + w0)) / eta;
            const double b1 = eta * (dza[GI(o)] * w1 + dza[GI(o + i)] + w1 * w1dz / (1.0 + w0));
            ab += a1 * b1;
        }
        // d = sigma*mu*e - a o b ; u = lam \ d ; tmp = -s + W u.   Two passes over the cone (q small).
        const double l0 = lam[GI(o)];
        double l1l1 = 0.0, l1d1 = 0.0;
        const double d0 = sm - ab;
        for (int i = 1; i < q; i++) {
            const double w1 = socw[GI(wo + i)];
            const double a1 = (-dsa[GI(o)] * w1 + dsa[GI(o + i)] + w1 * w1ds / (1.0 + w0)) / eta;
            const double b1 = eta * (dza[GI(o)] * w1 + dza[GI(o + i)] + w1 * w1dz / (1.0 + w0));
            const double d1 = -(a0 * b1 + b0 * a1);
            l1l1 += lam[GI(o + i)] * lam[GI(o + i)];
            l1d1 += lam[GI(o + i)] * d1;
        }
        const double det = l0 * l0 - l1l1;
        const double u0 = (l0 * d0 - l1d1) / det;
        double w1u = 0.0;
        for (int i = 1; i < q; i++) {
            const double w1 = socw[GI(wo + i)];
            const double a1 = (-dsa[GI(o)] * w1 + dsa[GI(o + i)] + w1 * w1ds / (1.0 + w0)) / eta;
            const double b1 = eta * (dza[GI(o)] * w1 + dza[GI(o + i)] + w1 * w1dz / (1.0 + w0));
            const double d1 = -(a0 * b1 + b0 * a1);
            const double u1 = (d1 - u0 * lam[GI(o + i)]) / l0;
            tmp[GI(o + i)] = u1;  // stash u1
            w1u += w1 * u1;
        }
        const double t0 = eta * (w0 * u0 + w1u);
        for (int i = 1; i < q; i++) {
            const double w1 = socw[GI(wo + i)], u1 = tmp[GI(o + i)];
            tmp[GI(o + i)] = -s[GI(o + i)] + eta * (u0 * w1 + u1 + w1 * w1u / (1.0 + w0));
        }
        tmp[GI(o)] = -s[GI(o)] + t0;
    }
}

// Ruiz equilibration of [A; G] in place (ECOS preprocesses its data the same way): rows and columns are
// repeatedly divided by the square root of their max-norm; all rows of one second-order cone share a
// factor (the cone must stay a cone).  b, h, c are scaled consistently; the solution is mapped back by
// x = D x^, y = Ea y^, z = Eg z^, s = s^ / Eg in the epilogue.
__device__ void equilibrate(const IpmProgram &P, const Ctx &c, double *Av, double *Gv, double *cc, double *bb,
                            double *hh, double *eqD, double *eqA, double *eqG, int iters)
{
    const int G = c.G, sg = c.sg;
    for (int i = c.slot; i < P.n; i += c.nslots) eqD[GI(i)] = 1.0;
    for (int i = c.slot; i < P.p; i += c.nslots) eqA[GI(i)] = 1.0;
    for (int i = c.slot; i < P.m; i += c.nslots) eqG[GI(i)] = 1.0;
    __syncthreads();
    for (int it = 0; it < iters; it++) {
        // rows
        for (int r = c.slot; r < P.p; r += c.nslots) {
            double mx = 0.0;
            for (int k = P.A_rp[r]; k < P.A_rp[r + 1]; k++) mx = fmax(mx, fabs(Av[GI(k)]));
            const double f = mx > 0.0 ? rsqrt(mx) : 1.0;
            for (int k = P.A_rp[r]; k < P.A_rp[r + 1]; k++) Av[GI(k)] *= f;
            eqA[GI(r)] *= f;
        }
        for (int r = c.slot; r < P.l; r += c.nslots) {
            double mx = 0.0;
            for (int k = P.G_rp[r]; k < P.G_rp[r + 1]; k++) mx = fmax(mx, fabs(Gv[GI(k)]));
            const double f = mx > 0.0 ? rsqrt(mx) : 1.0;
            for (int k = P.G_rp[r]; k < P.G_rp[r + 1]; k++) Gv[GI(k)] *= f;
            eqG[GI(r)] *= f;
        }
        for (int q = c.slot; q < P.nsoc; q += c.nslots) {
            const int o = P.soc_off[q], d = P.soc_dim[q];
            double mx = 0.0;
            for (int k = P.G_rp[o]; k < P.G_rp[o + d]; k++) mx = fmax(mx, fabs(Gv[GI(k)]));
            const double f = mx > 0.0 ? rsqrt(mx) : 1.0;
            for (int k = P.G_rp[o]; k < P.G_rp[o + d]; k++) Gv[GI(k)] *= f;
            for (int r = o; r < o + d; r++) eqG[GI(r)] *= f;
        }
        __syncthreads();
        // columns
        for (int v = c.slot; v < P.n; v += c.nslots) {
            double mx = 0.0;
            for (int k = P.At_rp[v]; k < P.At_rp[v + 1]; k++) mx = fmax(mx, fabs(Av[GI(P.At_vi[k])]));
            for (int k = P.Gt_rp[v]; k < P.Gt_rp[v + 1]; k++) mx = fmax(mx, fabs(Gv[GI(P.Gt_vi[k])]));
            const double f = mx > 0.0 ? rsqrt(mx) : 1.0;
            for (int k = P.At_rp[v]; k < P.At_rp[v + 1]; k++) Av[GI(P.At_vi[k])] *= f;
            for (int k = P.Gt_rp[v]; k < P.Gt_rp[v + 1]; k++) Gv[GI(P.Gt_vi[k])] *= f;
            eqD[GI(v)] *= f;
        }
        __syncthreads();
    }
    for (int i = c.slot; i < P.n; i += c.nslots) cc[GI(i)] *= eqD[GI(i)];
    for (int i = c.slot; i < P.p; i += c.nslots) bb[GI(i)] *= eqA[GI(i)];
    for (int i = c.slot; i < P.m; i += c.nslots) hh[GI(i)] *= eqG[GI(i)];
    __syncthreads();
}

// =============================================================================================
template <int NT, int SN>
__global__ void __launch_bounds__(NT) k_ipm_solve(const IpmProgram P, const IpmData D, const IpmOpts O)
{
    __shared__ double s_red[10 * (IPM_NT_MAX / 32) * IPM_MAXG];
    __shared__ double s_out[10 * IPM_MAXG];
    __shared__ double s_nb[IPM_MAXG], s_nh[IPM_MAXG], s_nc[IPM_MAXG];
    __shared__ double s_mu[IPM_MAXG], s_sigmu[IPM_MAXG], s_alpha[IPM_MAXG], s_scale[IPM_MAXG];
    __shared__ int s_flag;
    __shared__ int s_done[IPM_MAXG], s_status[IPM_MAXG], s_iters[IPM_MAXG], s_alldone, s_save[IPM_MAXG], s_stall[IPM_MAXG];
    __shared__ double s_best[IPM_MAXG], s_bp[IPM_MAXG], s_bd[IPM_MAXG], s_br[3 * IPM_MAXG];
    __shared__ double s_alpha_d[IPM_MAXG];
    __shared__ int s_warm[IPM_MAXG], s_wsaved[IPM_MAXG], s_wsave[IPM_MAXG], s_allwarm, s_redo;
    __shared__ int s_skip[IPM_MAXG];
    double *const s_delta = ipm_s_delta;
    int *const s_bad = ipm_s_bad;
    __shared__ SnArgs s_snargs;
    __shared__ HyArgs s_hyargs;

    int *s_lv = ipm_smem;   // [9][nlevels+1]: lvl_ptr | fa_lvl | fb_lvl | - | fa_R | fwp_lvl | bwp_lvl | fwp_R | bwp_R
    const int nl1 = P.nlevels + 1;
    for (int i = threadIdx.x; i <= P.nlevels; i += NT) {
        s_lv[i] = P.lvl_ptr[i]; s_lv[nl1 + i] = P.fa_lvl[i]; s_lv[2 * nl1 + i] = P.fb_lvl[i];
        s_lv[5 * nl1 + i] = P.fwp_lvl[i]; s_lv[6 * nl1 + i] = P.bwp_lvl[i];
    }
    for (int i = threadIdx.x; i < P.nlevels; i += NT) {
        s_lv[4 * nl1 + i] = P.fa_R[i]; s_lv[7 * nl1 + i] = P.fwp_R[i]; s_lv[8 * nl1 + i] = P.bwp_R[i];
    }
    Ctx c;
    c.s_lvl = s_lv;
    c.o_fal = nl1; c.o_fbl = 2 * nl1; c.o_faR = 4 * nl1;
    c.o_fwl = 5 * nl1; c.o_bwl = 6 * nl1; c.o_fwR = 7 * nl1; c.o_bwR = 8 * nl1;
    c.o_vs = (9 * (P.nlevels + 1) + 3) & ~3;
    c.G = D.G; c.tid = threadIdx.x; c.sg = c.tid % c.G; c.slot = c.tid / c.G; c.nslots = NT / c.G; c.nwarps = NT / 32;
    c.flag = &s_flag; c.s_mu = s_mu;
    c.Rmax = D.R;
    c.lprof = (blockIdx.x == 0 && threadIdx.x == 0 && D.prof && D.lvl_prof) ? D.prof + 12 : nullptr;
    if (c.lprof) for (int i = 0; i < 3 * (P.nlevels + (SN == 2 ? P.hy.ntl : 0)); i++) c.lprof[i] = 0;
    set_lanes(c, c.Rmax);
    __syncthreads();
    c.red = s_red; c.out = s_out;
    const int G = c.G, sg = c.sg;
    const size_t g = (size_t)blockIdx.x + D.g0;
    const int seed = (int)g * G + sg;
    const bool live = seed < D.B;  // padded seeds replicate work harmlessly (arrays are padded)
    (void)live;

    c.s_done = s_done; c.s_delta = s_delta; c.s_bad = s_bad;
    c.sn = D.sn; c.ysize = (size_t)P.ysize;
    c.s_sn = &s_snargs;
    c.s_hy = &s_hyargs;
    double *const vs = D.vsmem ? (double *)(s_lv + c.o_vs) : nullptr;
    unsigned *const pcnt_s = (unsigned *)(s_lv + c.o_vs + 2 * (P.nk > P.npf ? P.nk : P.npf) * G + 2 * P.nps * G);
    if (D.psmem) for (int i = c.tid; i < P.nps * G; i += NT) pcnt_s[i] = 0u;   // the barrier below publishes it
    if (threadIdx.x == 0) {   // the CTA-uniform argument blocks (published by the barrier below)
        ipm_s_reg[0] = O.rho_min; ipm_s_reg[1] = O.bad_abs;
#define GP(arr, E) ((arr) + g * (size_t)(E) * G)
        IpmGroup r;
        r.Av = GP(D.Av, P.nnzA); r.Gv = GP(D.Gv, P.nnzG); r.cc = GP(D.c, P.n); r.bb = GP(D.b, P.p); r.hh = GP(D.h, P.m);
        r.eqD = GP(D.eqD, P.n); r.eqA = GP(D.eqA, P.p); r.eqG = GP(D.eqG, P.m);
        r.x = GP(D.x, P.n); r.y = GP(D.y, P.p); r.z = GP(D.z, P.m); r.s = GP(D.s, P.m);
        r.xb = GP(D.xb, P.n); r.yb = GP(D.yb, P.p); r.zb = GP(D.zb, P.m); r.sb = GP(D.sb, P.m);
        r.rx = GP(D.rx, P.n); r.ry = GP(D.ry, P.p); r.rz = GP(D.rz, P.m); r.lam = GP(D.lam, P.m);
        r.wm = GP(D.wm, P.nwm); r.socw = GP(D.socw, P.m - P.l + 1); r.soceta = GP(D.soceta, P.nsoc + 1);
        r.dx = GP(D.dx, P.n); r.dy = GP(D.dy, P.p); r.dz = GP(D.dz, P.m); r.ds = GP(D.ds, P.m);
        r.dsa = GP(D.dsa, P.m); r.dza = GP(D.dza, P.m); r.tm = GP(D.tm, P.m); r.gm = GP(D.gm, P.m);
        r.r1 = GP(D.r1, P.n); r.r2 = GP(D.r2, P.p);
        r.e1 = GP(D.e1, (P.n > P.m ? P.n : P.m)); r.rhs = GP(D.rhs, P.nk);
        r.Y = GP(D.Y, P.ysize); r.Ls = GP(D.Ls, P.nnzL + 1); r.invD = GP(D.invD, P.nk);
        r.vs = vs; r.reftol = O.reftol; r.mu_tight = O.mu_tight;
        ipm_ar = r;
        SpmvArgs m;
        m.A_rp = P.A_rp; m.A_ci = P.A_ci; m.G_rp = P.G_rp; m.G_ci = P.G_ci;
        m.At_rp = P.At_rp; m.At_ri = P.At_ri; m.At_vi = P.At_vi; m.Gt_rp = P.Gt_rp; m.Gt_ri = P.Gt_ri; m.Gt_vi = P.Gt_vi;
        m.iperm = P.iperm; m.n = P.n; m.p = P.p; m.m = P.m; m.G = G;
        ipm_mv = m;
        if (SN == 2) {
            HyArgs a;
            a.hy = P.hy; a.Y = r.Y; a.Ls = r.Ls; a.invD = r.invD; a.s_done = s_done; a.s_delta = s_delta; a.s_bad = s_bad;
            a.rho_min = O.rho_min; a.bad_abs = O.bad_abs; a.o_vs = c.o_vs; a.nnzL = P.nnzL; a.G = D.G; a.nwarps = NT / 32;
            a.lprof = (blockIdx.x == 0 && D.prof && D.lvl_prof) ? D.prof + 12 + 3 * P.nlevels : nullptr;
            s_hyargs = a;
        }
        if (SN == 1) {
            SnArgs a;
            a.sn = P.sn; a.Y = r.Y; a.invD = r.invD; a.vs = vs; a.s_done = s_done; a.s_delta = s_delta; a.s_bad = s_bad;
            a.rho_min = O.rho_min; a.bad_abs = O.bad_abs; a.ysize = (size_t)P.ysize; a.G = D.G; a.tid = 0; a.nwarps = NT / 32;
            a.nls = P.nlevels; a.lprof = (blockIdx.x == 0 && D.prof && D.lvl_prof) ? D.prof + 12 : nullptr;
            s_snargs = a;
        }
        if (SN != 1) {
            // partial sums of the split targets of a level: in the dynamic window (level pointers | vector, or the
            // factorisation's slots | substitution slots | counters), or in global memory
            double *Lrow = GP(D.Lrow, P.nnzL + 1), *fpart, *spart;
            unsigned *pcnt;
            if (D.psmem) {
                fpart = (double *)(s_lv + c.o_vs);
                spart = (double *)(s_lv + c.o_vs + 2 * (P.nk > P.npf ? P.nk : P.npf) * G);
                pcnt = pcnt_s;
            } else {
                fpart = spart = GP(D.part, P.npart + 1);
                pcnt = (unsigned *)GP(D.pcnt, P.npart + 1);
            }
            FactorArgs a;
            a.fa_item = P.fa_item; a.fb_item = P.fb_item; a.ft_op = P.ft_op; a.fb_cmb = P.fb_cmb;
            a.Y = r.Y; a.Ls = r.Ls; a.Lrow = Lrow; a.invD = r.invD; a.part = fpart;
            a.o_fal = c.o_fal; a.o_faR = c.o_faR; a.o_fbl = c.o_fbl;
            a.nl = P.nlevels; a.nnzLd = P.nnzL; a.G = G; a.nslots = c.nslots;
            a.lprof = c.lprof;   // thread 0 of CTA 0 only (c.lprof is nullptr everywhere else)
            ipm_fa = a;
            SweepArgs w;
            w.nl = P.nlevels; w.G = G; w.nslots = c.nslots; w.o_vs = c.o_vs; w.part = spart; w.pcnt = pcnt;
            w.items = P.fwp_item; w.idxarr = P.Lr_col; w.vals = Lrow; w.o_lvl = c.o_fwl; w.o_R = c.o_fwR; w.lv0 = 1;
            w.cmb = P.fwc_item;
            w.lprof = c.lprof ? c.lprof + P.nlevels : nullptr;
            ipm_sw[0] = w;
            w.items = P.bwp_item; w.idxarr = P.L_ri; w.vals = r.Ls; w.o_lvl = c.o_bwl; w.o_R = c.o_bwR; w.lv0 = P.nlevels - 2;
            w.cmb = P.bwc_item;
            w.lprof = c.lprof ? c.lprof + 2 * P.nlevels : nullptr;
            ipm_sw[1] = w;
        }
#undef GP
    }
    const IpmGroup &ar = ipm_ar;

    if (threadIdx.x == 0) {
        for (int i = 0; i < 13; i++) ipm_s_prof[i] = 0;
        ipm_s_prof[13] = ipm_s_prof[14] = clock64();
    }
#define PROF(i) { if (threadIdx.x == 0) { const long long tn = clock64(); ipm_s_prof[i] += tn - ipm_s_prof[13]; ipm_s_prof[13] = tn; } }
    if (c.tid < G) {
        const int sd = (int)g * G + c.tid;
        // padded seeds and seeds the caller marked (SCP seeds that have already stopped) are not solved
        const int sk = (sd >= D.B) || (D.skip && D.skip[sd]);
        s_skip[c.tid] = sk; s_done[c.tid] = sk;
        s_status[c.tid] = IPM_MAXIT; s_iters[c.tid] = 0; s_best[c.tid] = CUDART_INF; s_save[c.tid] = 0; s_stall[c.tid] = 0;
        s_delta[c.tid] = O.delta; s_bad[c.tid] = 0;
        s_mu[c.tid] = CUDART_INF;
        s_warm[c.tid] = (!sk && O.warm && D.warm && D.warm[sd]) ? 1 : 0;
        s_wsaved[c.tid] = 0; s_wsave[c.tid] = 0;
    }
    __syncthreads();
    {
        int all = 1;
        for (int q = 0; q < G; q++) all &= s_skip[q];
        if (all) return;   // CTA-uniform: nothing to solve in this group
    }
    if (D.debug_kkt) {   // test hook: one KKT solve on the device with the caller's scaling and right-hand side
        kkt_assemble(P, c, D, glb(ar.Av), glb(ar.Gv), glb(ar.wm), glb(ar.Y), 0.0);
        kkt_factor<SN>(c);
        kkt_ldl_solve<SN>(P, c);
        if (c.tid < G && (int)g * G + c.tid < D.B) D.status[(int)g * G + c.tid] = s_bad[c.tid];
        return;
    }
    // (re)assemble and factor; a seed whose factorisation lost its inertia to cancellation (the scaling matrix spans
    // > 25 orders of magnitude in the last iterations) gets a larger static regularisation and the group factors again
#define IPM_FACTOR()                                                                               \
    for (int tr_ = 0;; tr_++) {                                                                    \
        if (c.tid < G) s_bad[c.tid] = 0;                                                           \
        kkt_assemble(P, c, D, glb(ar.Av), glb(ar.Gv), glb(ar.wm), glb(ar.Y), 0.0);                                                 \
        kkt_factor<SN>(c);                                                                         \
        if (c.tid == 0) {                                                                          \
            int again_ = 0;                                                                        \
            for (int q = 0; q < G; q++)                                                            \
                if (s_bad[q] && !s_done[q] && s_delta[q] < O.delta_max) {                          \
                    s_delta[q] = fmin(s_delta[q] * O.delta_esc, O.delta_max); again_ = 1;          \
                }                                                                                  \
            s_flag = again_;                                                                       \
        }                                                                                          \
        __syncthreads();                                                                           \
        const int again_ = s_flag;                                                                 \
        __syncthreads();                                                                           \
        if (!again_ || tr_ >= 4) break;                                                            \
        if (c.tid == 0) ipm_s_prof[12]++;                                                          \
    }
    if (O.equil > 0) equilibrate(P, c, glb(ar.Av), glb(ar.Gv), glb(ar.cc), glb(ar.bb), glb(ar.hh), glb(ar.eqD), glb(ar.eqA), glb(ar.eqG), O.equil);
    PROF(0)
    // ---- data norms ----
    {
        double v[3] = {0.0, 0.0, 0.0};
        for (int i = c.slot; i < P.p; i += c.nslots) v[0] += glb(ar.bb)[GI(i)] * glb(ar.bb)[GI(i)];
        for (int i = c.slot; i < P.m; i += c.nslots) v[1] += glb(ar.hh)[GI(i)] * glb(ar.hh)[GI(i)];
        for (int i = c.slot; i < P.n; i += c.nslots) v[2] += glb(ar.cc)[GI(i)] * glb(ar.cc)[GI(i)];
        seed_reduce<3>(c, v, 0);
        if (c.tid < G) {
            s_nb[c.tid] = fmax(1.0, sqrt(s_out[0 * IPM_MAXG + c.tid]));
            s_nh[c.tid] = fmax(1.0, sqrt(s_out[1 * IPM_MAXG + c.tid]));
            s_nc[c.tid] = fmax(1.0, sqrt(s_out[2 * IPM_MAXG + c.tid]));
        }
        __syncthreads();
    }
    // ---- warm start: a seed whose previous solve left a warm point starts from it (converted to this program's
    // equilibrated units: x/D, y/E_A, z/E_G, s*E_G; cone membership of s and z is unaffected, the scalings are positive and
    // uniform inside a second-order cone).  If that run does not end OPTIMAL / ALMOST_OPTIMAL / with a certificate, the
    // whole group is solved again from the cold starting point (restart_cold below).
    int tried_cold = 0;
restart_cold:
    if (c.tid == 0) {
        int all = 1;
        for (int q = 0; q < G; q++) all &= (s_warm[q] || s_skip[q]);
        s_allwarm = all;
    }
    __syncthreads();
    if (!s_allwarm) {
        // ---- starting point (CVXOPT conelp 7.1 / ECOS init): factor with W = I ----
        set_identity_scaling(P, c, glb(ar.wm), glb(ar.socw), glb(ar.soceta));
        __syncthreads();
        IPM_FACTOR()
        // solve 1: [0;b;h] -> x, s = h - G x
        for (int v = c.slot; v < P.n; v += c.nslots) glb(ar.r1)[GI(v)] = 0.0;
        __syncthreads();
        kkt_solve<SN>(P, c, glb(ar.bb), glb(ar.hh), glb(ar.x), glb(ar.dy), glb(ar.dz), O.nref);
        for (int r = c.slot; r < P.m; r += c.nslots) glb(ar.s)[GI(r)] = -glb(ar.dz)[GI(r)];
        __syncthreads();
        {
            double vv[1] = {cone_shift_partial(P, c, glb(ar.s))};
            double w2[1] = {0.0};
            for (int r = c.slot; r < P.m; r += c.nslots) w2[0] += glb(ar.s)[GI(r)] * glb(ar.s)[GI(r)];
            seed_reduce<1>(c, vv, 2);
            const double ts = s_out[sg];
            __syncthreads();
            seed_reduce<1>(c, w2, 0);
            const double ns = sqrt(s_out[sg]);
            if (ts >= -1e-8 * fmax(1.0, ns)) {
                const double sh = 1.0 + ts;
                for (int r = c.slot; r < P.l; r += c.nslots) glb(ar.s)[GI(r)] += sh;
                for (int k = c.slot; k < P.nsoc; k += c.nslots) glb(ar.s)[GI(P.soc_off[k])] += sh;
            }
            __syncthreads();
        }
        // solve 2: [-c;0;0] -> y, z
        for (int v = c.slot; v < P.n; v += c.nslots) glb(ar.r1)[GI(v)] = -glb(ar.cc)[GI(v)];
        for (int r = c.slot; r < P.p; r += c.nslots) glb(ar.r2)[GI(r)] = 0.0;
        for (int r = c.slot; r < P.m; r += c.nslots) glb(ar.rz)[GI(r)] = 0.0;
        __syncthreads();
        kkt_solve<SN>(P, c, glb(ar.r2), glb(ar.rz), glb(ar.dx), glb(ar.y), glb(ar.z), O.nref);
        {
            double vv[1] = {cone_shift_partial(P, c, glb(ar.z))};
            double w2[1] = {0.0};
            for (int r = c.slot; r < P.m; r += c.nslots) w2[0] += glb(ar.z)[GI(r)] * glb(ar.z)[GI(r)];
            seed_reduce<1>(c, vv, 2);
            const double tz = s_out[sg];
            __syncthreads();
            seed_reduce<1>(c, w2, 0);
            const double nz = sqrt(s_out[sg]);
            if (tz >= -1e-8 * fmax(1.0, nz)) {
                const double sh = 1.0 + tz;
                for (int r = c.slot; r < P.l; r += c.nslots) glb(ar.z)[GI(r)] += sh;
                for (int k = c.slot; k < P.nsoc; k += c.nslots) glb(ar.z)[GI(P.soc_off[k])] += sh;
            }
            __syncthreads();
        }


    }
    if (s_warm[sg]) {
        const bool eq = O.equil > 0;
        for (int i = c.slot; i < P.n; i += c.nslots) glb(ar.x)[GI(i)] = eq ? D.xw[g * (size_t)P.n * G + GI(i)] / glb(ar.eqD)[GI(i)] : D.xw[g * (size_t)P.n * G + GI(i)];
        for (int i = c.slot; i < P.p; i += c.nslots) glb(ar.y)[GI(i)] = eq ? D.yw[g * (size_t)P.p * G + GI(i)] / glb(ar.eqA)[GI(i)] : D.yw[g * (size_t)P.p * G + GI(i)];
        for (int i = c.slot; i < P.m; i += c.nslots) {
            const double e_ = eq ? glb(ar.eqG)[GI(i)] : 1.0;
            glb(ar.z)[GI(i)] = D.zw[g * (size_t)P.m * G + GI(i)] / e_;
            glb(ar.s)[GI(i)] = D.sw[g * (size_t)P.m * G + GI(i)] * e_;
        }
    }
    __syncthreads();
    PROF(1)
    const double deg = (double)(P.l + P.nsoc);
    for (int it = 0; it <= O.maxit; it++) {
        // ---- residuals + objective pieces ----
        // v[7..9]: |A'y + G'z|^2, |Ax|^2, |Gx + s|^2 for the infeasibility certificates (ECOS reports INFEASIBLE /
        // DUAL_INFEASIBLE the same way; src/solvers/scp.jl:470-473 and :975 branch on those statuses)
        // (rx, ry, rz are written by the thread that reads them back here: no barrier in between)
        spmv_residuals();
        double v[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int i = c.slot; i < P.n; i += c.nslots) {
            const double ci_ = glb(ar.cc)[GI(i)], r = glb(ar.rx)[GI(i)];
            v[0] += r * r;
            v[3] += ci_ * glb(ar.x)[GI(i)];
            v[7] += (r - ci_) * (r - ci_);
        }
        for (int i = c.slot; i < P.p; i += c.nslots) {
            const double bi_ = glb(ar.bb)[GI(i)], r = glb(ar.ry)[GI(i)];
            v[1] += r * r;
            v[4] += bi_ * glb(ar.y)[GI(i)];
            v[8] += (r + bi_) * (r + bi_);
        }
        for (int i = c.slot; i < P.m; i += c.nslots) {
            const double hi_ = glb(ar.hh)[GI(i)], r = glb(ar.rz)[GI(i)];
            v[2] += r * r;
            v[5] += hi_ * glb(ar.z)[GI(i)];
            v[6] += glb(ar.s)[GI(i)] * glb(ar.z)[GI(i)];
            v[9] += (r + hi_) * (r + hi_);
        }
        seed_reduce<10>(c, v, 0);
        if (c.tid < G) {
            const int q = c.tid;
            const double nrx = sqrt(s_out[0 * IPM_MAXG + q]), nry = sqrt(s_out[1 * IPM_MAXG + q]),
                         nrz = sqrt(s_out[2 * IPM_MAXG + q]);
            const double pcost = s_out[3 * IPM_MAXG + q], dcost = -s_out[4 * IPM_MAXG + q] - s_out[5 * IPM_MAXG + q];
            const double gap = s_out[6 * IPM_MAXG + q];
            const double pres = fmax(nry / s_nb[q], nrz / s_nh[q]), dres = nrx / s_nc[q];
            const double relgap = gap / fmax(fmax(fabs(pcost), fabs(dcost)), 1.0);
            s_mu[q] = gap / deg;
            s_save[q] = 0;
            s_wsave[q] = 0;
            // the warm point of the NEXT solve of this seed: the first iterate this close to the path's end.  A warm-started
            // run begins at about that level already: it only replaces the point by an iterate of ITS OWN path (it >= 1) that
            // is still inside [0.1, 1] mu_warm -- otherwise the stored point would creep towards the boundary from one SCP
            // iteration to the next -- and keeps the one it started from if no iterate qualifies
            if (!s_done[q] && !s_wsaved[q] && D.warm && isfinite(pres) && isfinite(dres) && gap >= 0.0 && gap / deg <= O.mu_warm &&
                (!s_warm[q] || (it >= 1 && gap / deg >= 0.1 * O.mu_warm))) {
                s_wsave[q] = 1; s_wsaved[q] = 1;
            }
            if (D.trace && (int)g * G + q == D.trace_seed && !s_done[q]) {   // it, pres, dres, gap, pcost, dcost, last steps, delta, sigma*mu
                double *tr_ = D.trace + 10 * (size_t)it;
                tr_[0] = it; tr_[1] = pres; tr_[2] = dres; tr_[3] = gap; tr_[4] = pcost; tr_[5] = dcost;
                tr_[6] = it ? s_alpha[q] : 0.0; tr_[7] = it ? s_alpha_d[q] : 0.0; tr_[8] = s_delta[q]; tr_[9] = it ? s_sigmu[q] : 0.0;
            }
            if (!s_done[q]) {
                s_iters[q] = it;
                const double acc = fmax(fmax(pres, dres), fmin(gap, relgap));
                if (isfinite(acc) && gap >= 0.0 && acc < s_best[q]) {
                    s_best[q] = acc; s_save[q] = 1; s_stall[q] = 0;
                    s_bp[q] = pcost; s_bd[q] = dcost; s_br[q] = pres; s_br[IPM_MAXG + q] = dres; s_br[2 * IPM_MAXG + q] = gap;
                } else s_stall[q]++;
                // certificates: (y, z) with A'y + G'z ~ 0 and b'y + h'z < 0 proves primal infeasibility; x with
                // Ax ~ 0, Gx + s ~ 0 and c'x < 0 proves dual infeasibility (an unbounded program)
                const double pinf = (dcost > 0.0) ? sqrt(s_out[7 * IPM_MAXG + q]) / dcost : CUDART_INF;
                const double dinf = (pcost < 0.0) ? sqrt(fmax(s_out[8 * IPM_MAXG + q], s_out[9 * IPM_MAXG + q])) / (-pcost) : CUDART_INF;
                if (!(isfinite(pres) && isfinite(dres) && isfinite(gap))) { s_done[q] = 1; s_status[q] = IPM_NUMERICAL; }
                else if (pres <= O.feastol && dres <= O.feastol && (gap <= O.abstol || relgap <= O.reltol)) {
                    s_done[q] = 1; s_status[q] = IPM_OPTIMAL;
                }
                // (a certificate at 1e-8 relative is a proof whatever optimality tolerance was asked for: tighter requests
                // would only let the diverging iterates run into the numerical floor first)
                else if (it >= 2 && pinf <= fmax(O.feastol, 1e-8)) { s_done[q] = 1; s_status[q] = IPM_PINF; s_save[q] = 1; }
                else if (it >= 2 && dinf <= fmax(O.feastol, 1e-8)) { s_done[q] = 1; s_status[q] = IPM_DINF; s_save[q] = 1; }
                else if (s_stall[q] >= 3 && s_best[q] <= 1e-6) { s_done[q] = 1; s_status[q] = IPM_NUMERICAL; }  // numerical floor
                else if (it == O.maxit) { s_done[q] = 1; s_status[q] = IPM_MAXIT; }
            }
        }
        __syncthreads();
        if (s_save[sg]) {
            for (int i = c.slot; i < P.n; i += c.nslots) glb(ar.xb)[GI(i)] = glb(ar.x)[GI(i)];
            for (int i = c.slot; i < P.p; i += c.nslots) glb(ar.yb)[GI(i)] = glb(ar.y)[GI(i)];
            for (int i = c.slot; i < P.m; i += c.nslots) { glb(ar.zb)[GI(i)] = glb(ar.z)[GI(i)]; glb(ar.sb)[GI(i)] = glb(ar.s)[GI(i)]; }
        }
        if (s_wsave[sg]) {   // in the caller's units (the next program is equilibrated differently)
            const bool eq = O.equil > 0;
            for (int i = c.slot; i < P.n; i += c.nslots) D.xw[g * (size_t)P.n * G + GI(i)] = eq ? glb(ar.x)[GI(i)] * glb(ar.eqD)[GI(i)] : glb(ar.x)[GI(i)];
            for (int i = c.slot; i < P.p; i += c.nslots) D.yw[g * (size_t)P.p * G + GI(i)] = eq ? glb(ar.y)[GI(i)] * glb(ar.eqA)[GI(i)] : glb(ar.y)[GI(i)];
            for (int i = c.slot; i < P.m; i += c.nslots) {
                const double e_ = eq ? glb(ar.eqG)[GI(i)] : 1.0;
                D.zw[g * (size_t)P.m * G + GI(i)] = glb(ar.z)[GI(i)] * e_;
                D.sw[g * (size_t)P.m * G + GI(i)] = glb(ar.s)[GI(i)] / e_;
            }
        }
        __syncthreads();
        if (c.tid == 0) {
            int all = 1;
            for (int q = 0; q < G; q++) all &= (s_done[q] || ((int)g * G + q >= D.B));
            s_alldone = all;
        }
        __syncthreads();
        if (s_alldone) break;
        PROF(2)

        // ---- scaling, KKT assembly, factorisation ----
        nt_scaling(P, c, glb(ar.s), glb(ar.z), glb(ar.lam), glb(ar.wm), glb(ar.socw), glb(ar.soceta));
        __syncthreads();
        PROF(3)
        IPM_FACTOR()
        PROF(4)
        if (c.tid == 0) ipm_s_prof[11]++;

        // ---- affine direction: bx=-rx, by=-ry, bz=-rz+s ; ds = -s - W^2 dz ----
        for (int i = c.slot; i < P.n; i += c.nslots) glb(ar.r1)[GI(i)] = -glb(ar.rx)[GI(i)];
        for (int i = c.slot; i < P.p; i += c.nslots) glb(ar.r2)[GI(i)] = -glb(ar.ry)[GI(i)];
        for (int i = c.slot; i < P.m; i += c.nslots) glb(ar.ds)[GI(i)] = -glb(ar.rz)[GI(i)] + glb(ar.s)[GI(i)];  // ds used as bz scratch
        __syncthreads();
        PROF(6)
        kkt_solve<SN>(P, c, glb(ar.r2), glb(ar.ds), glb(ar.dx), glb(ar.dy), glb(ar.dza), O.nref_aff);
        PROF(5)
        // ds = tmp - W^2 dz with tmp = -s; W^2 dz == G dx - bz is left in gm by kkt_solve (no W^2 W^-2
        // round trip: keeps G dx + ds = -rz to rounding even when the scaling is ill-conditioned)
        for (int i = c.slot; i < P.m; i += c.nslots) glb(ar.dsa)[GI(i)] = -glb(ar.s)[GI(i)] - glb(ar.gm)[GI(i)];
        __syncthreads();
        {   // separate primal / dual step lengths (the primal and dual residuals shrink independently); centring
            // parameter from the predicted complementarity, sigma = (mu_aff / mu)^3 (Mehrotra)
            double a[2] = {cone_alpha_partial(P, c, glb(ar.s), glb(ar.dsa)), cone_alpha_partial(P, c, glb(ar.z), glb(ar.dza))};
            seed_reduce<2>(c, a, 1);
            const double ap = fmin(1.0, s_out[sg]), ad = fmin(1.0, s_out[IPM_MAXG + sg]);
            double ma[1] = {0.0};
            for (int i = c.slot; i < P.m; i += c.nslots) ma[0] = fma(glb(ar.s)[GI(i)] + ap * glb(ar.dsa)[GI(i)], glb(ar.z)[GI(i)] + ad * glb(ar.dza)[GI(i)], ma[0]);
            seed_reduce<1>(c, ma, 0);
            if (c.tid < G) {
                double r = s_out[c.tid] / (deg * s_mu[c.tid]);
                r = fmin(1.0, fmax(0.0, r));
                if (!(r == r)) r = 1.0;
                const double sig = r * r * r;
                s_sigmu[c.tid] = sig * s_mu[c.tid];
                s_scale[c.tid] = 1.0 - sig;
            }
            __syncthreads();
        }
        // ---- combined direction ----
        combined_tmp(P, c, glb(ar.s), glb(ar.z), glb(ar.lam), glb(ar.socw), glb(ar.soceta), glb(ar.dsa), glb(ar.dza), s_sigmu, glb(ar.tm));
        __syncthreads();
        {
            const double sc = s_scale[sg];
            for (int i = c.slot; i < P.n; i += c.nslots) glb(ar.r1)[GI(i)] = -sc * glb(ar.rx)[GI(i)];
            for (int i = c.slot; i < P.p; i += c.nslots) glb(ar.r2)[GI(i)] = -sc * glb(ar.ry)[GI(i)];
            for (int i = c.slot; i < P.m; i += c.nslots) {
                const double t = glb(ar.tm)[GI(i)];
                glb(ar.dsa)[GI(i)] = t;                        // keep tmp
                glb(ar.ds)[GI(i)] = -sc * glb(ar.rz)[GI(i)] - t;       // bz
            }
        }
        __syncthreads();
        PROF(6)
        kkt_solve<SN>(P, c, glb(ar.r2), glb(ar.ds), glb(ar.dx), glb(ar.dy), glb(ar.dz), O.nref);
        PROF(5)
        for (int i = c.slot; i < P.m; i += c.nslots) glb(ar.ds)[GI(i)] = glb(ar.dsa)[GI(i)] - glb(ar.gm)[GI(i)];
        __syncthreads();
        {
            double a[2] = {cone_alpha_partial(P, c, glb(ar.s), glb(ar.ds)), cone_alpha_partial(P, c, glb(ar.z), glb(ar.dz))};
            seed_reduce<2>(c, a, 1);
            if (c.tid < G) {
                s_alpha[c.tid] = s_done[c.tid] ? 0.0 : fmin(1.0, 0.99 * s_out[c.tid]);                 // primal: x, s
                s_alpha_d[c.tid] = s_done[c.tid] ? 0.0 : fmin(1.0, 0.99 * s_out[IPM_MAXG + c.tid]);   // dual: y, z
            }
            __syncthreads();
        }
        // safeguard: make sure the new point is strictly interior (halve the step otherwise) so that the
        // next NT scaling is well defined
        for (int bt = 0; bt < 12; bt++) {
            double mg[2] = {cone_margin_partial(P, c, glb(ar.s), glb(ar.ds), s_alpha[sg]), cone_margin_partial(P, c, glb(ar.z), glb(ar.dz), s_alpha_d[sg])};
            seed_reduce<2>(c, mg, 1);
            if (c.tid == 0) s_alldone = 1;
            __syncthreads();
            if (c.tid < G) {
                if (s_alpha[c.tid] > 0.0 && !(s_out[c.tid] > 0.0)) { s_alpha[c.tid] *= 0.5; s_alldone = 0; }
                if (s_alpha_d[c.tid] > 0.0 && !(s_out[IPM_MAXG + c.tid] > 0.0)) { s_alpha_d[c.tid] *= 0.5; s_alldone = 0; }
            }
            __syncthreads();
            const int okall = s_alldone;
            __syncthreads();
            if (okall) break;
        }
        {
            const double ap = s_alpha[sg], ad = s_alpha_d[sg];
            if (ap > 0.0) {
                for (int i = c.slot; i < P.n; i += c.nslots) glb(ar.x)[GI(i)] += ap * glb(ar.dx)[GI(i)];
                for (int i = c.slot; i < P.m; i += c.nslots) glb(ar.s)[GI(i)] += ap * glb(ar.ds)[GI(i)];
            }
            if (ad > 0.0) {
                for (int i = c.slot; i < P.p; i += c.nslots) glb(ar.y)[GI(i)] += ad * glb(ar.dy)[GI(i)];
                for (int i = c.slot; i < P.m; i += c.nslots) glb(ar.z)[GI(i)] += ad * glb(ar.dz)[GI(i)];
            }
        }
        __syncthreads();
        PROF(6)
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && D.prof) {
        ipm_s_prof[7] = clock64() - ipm_s_prof[14];
        for (int i = 0; i < 11; i++) D.prof[i] = ipm_s_prof[i];
        D.prof[11] = ipm_s_prof[11] | (ipm_s_prof[12] << 32);
    }
#undef PROF
    // ---- a warm-started seed that did not reach the tolerances: the group starts again from the cold starting point ----
    __syncthreads();
    if (c.tid == 0) {
        int redo = 0;
        if (!tried_cold)
            for (int q = 0; q < G; q++)
                if (s_warm[q] && !s_skip[q] && s_status[q] != IPM_OPTIMAL && s_status[q] != IPM_PINF && s_status[q] != IPM_DINF &&
                    !(s_best[q] <= 10.0 * fmax(O.feastol, O.reltol)))
                    redo = 1;
        s_redo = redo;
    }
    __syncthreads();
    if (s_redo) {
        tried_cold = 1;
        if (c.tid < G) {
            const int q = c.tid;
            s_done[q] = s_skip[q]; s_status[q] = IPM_MAXIT; s_iters[q] = 0; s_best[q] = CUDART_INF; s_save[q] = 0; s_stall[q] = 0;
            s_delta[q] = O.delta; s_bad[q] = 0; s_warm[q] = 0; s_wsaved[q] = 0; s_wsave[q] = 0;
        }
        __syncthreads();
        goto restart_cold;
    }
    // ---- epilogue: the best iterate is the answer (ECOS reports its best point the same way) ----
    __syncthreads();
    // the numerical floor of the fp64 normal-equation factorisation sits within ~10x of ECOS' 1e-8 targets
    if (c.tid < G && s_status[c.tid] != IPM_OPTIMAL && s_status[c.tid] != IPM_PINF && s_status[c.tid] != IPM_DINF) {
        if (s_best[c.tid] <= 10.0 * fmax(O.feastol, O.reltol)) s_status[c.tid] = IPM_OPTIMAL;
        else if (s_best[c.tid] <= 5e-5) s_status[c.tid] = IPM_ALMOST;
    }
    __syncthreads();
    if (s_best[sg] < CUDART_INF) {
        for (int i = c.slot; i < P.n; i += c.nslots) glb(ar.x)[GI(i)] = glb(ar.xb)[GI(i)];
        for (int i = c.slot; i < P.p; i += c.nslots) glb(ar.y)[GI(i)] = glb(ar.yb)[GI(i)];
        for (int i = c.slot; i < P.m; i += c.nslots) { glb(ar.z)[GI(i)] = glb(ar.zb)[GI(i)]; glb(ar.s)[GI(i)] = glb(ar.sb)[GI(i)]; }
    }
    if (O.equil > 0) {  // back to the caller's units
        __syncthreads();
        for (int i = c.slot; i < P.n; i += c.nslots) glb(ar.x)[GI(i)] *= glb(ar.eqD)[GI(i)];
        for (int i = c.slot; i < P.p; i += c.nslots) glb(ar.y)[GI(i)] *= glb(ar.eqA)[GI(i)];
        for (int i = c.slot; i < P.m; i += c.nslots) { glb(ar.z)[GI(i)] *= glb(ar.eqG)[GI(i)]; glb(ar.s)[GI(i)] /= glb(ar.eqG)[GI(i)]; }
    }
    if (c.tid < G) {
        const int sd = (int)g * G + c.tid;
        if (sd < D.B && !s_skip[c.tid]) {
            D.status[sd] = s_status[c.tid]; D.iters[sd] = s_iters[c.tid];
            if (D.warm) D.warm[sd] = ((s_wsaved[c.tid] || s_warm[c.tid]) && (s_status[c.tid] == IPM_OPTIMAL || s_status[c.tid] == IPM_ALMOST)) ? 1 : 0;
            D.pobj[sd] = s_bp[c.tid]; D.dobj[sd] = s_bd[c.tid];
            D.res[sd] = s_br[c.tid]; D.res[D.B + sd] = s_br[IPM_MAXG + c.tid]; D.res[2 * D.B + sd] = s_br[2 * IPM_MAXG + c.tid];
        }
    }
}
#undef GI
#endif  // CONIC_IPM_IMPL
