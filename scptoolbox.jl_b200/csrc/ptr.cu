// ptr.cu -- native batched PTR loop (scpb_ptr_*): the device-resident replacement of the loop body of
// PTR.solve (src/solvers/ptr.jl:448-532) for a batch of independent seeds in lock step:
//   formulate  : k_linearize (s,C,D,G at the reference, scp.jl:744-794; scaled references for the trust
//                region, ptr.jl:575-577) + k_assemble ([Avals;Gvals;c;b;h] = W * src -- kernel K6, replaces
//                the per-iteration JuMP rebuild ptr.jl:470-478)
//   solve      : k_ipm_solve (conic_ipm.cuh)                       -- solve_subproblem!, scp.jl:942-950
//   discretize : k_discretize_foh on the new iterate (ptr.jl:380)  -- writes the DLTV straight into `src`
//   accept/stop: k_ptr_step -- solution_deviation (scp.jl:909-931) + check_stopping_criterion! (ptr.jl:908-932)
// Seeds that have stopped are frozen (their iterate is re-extracted unchanged) so a finished or failed
// seed never stalls the batch.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <functional>
#include <thread>
#include "handle.cuh"
#include "discretize.cuh"
#include "constraints.cuh"
#include "conic_symbolic.h"
#include "conic_ipm.cuh"

// pieces of conic_api.cu used here
struct scpb_cone_s;
int scpb_internal_cone_run(scpb_cone_s *c, const IpmOpts &o, const int *skip, cudaStream_t st, int g0, int ngc);
int scpb_internal_cone_reserve(scpb_cone_s *c, int B, int G, int lanes);
IpmData *scpb_internal_cone_data(scpb_cone_s *c);
const ConeSymbolic *scpb_internal_cone_sym(scpb_cone_s *c);
scpb_handle_s *scpb_internal_cone_handle(scpb_cone_s *c);
IpmOpts scpb_internal_make_opts(const scpb_cone_opts *o);
void scpb_internal_relax_refinement(IpmOpts &r);
int scpb_internal_pick_group(int B, int want, int sms);
int scpb_internal_discretize(scpb_handle_s *h, DiscArgs &a, double feas_tol, int *feas, int method, cudaStream_t st);

struct PtrDev {
    int B, G, N, nx, nu, np, ns;
    int nsrc, oC, oD, oG, ors, oxh, ouh, oph;
    const double *t_grid, *Sx, *cx, *Su, *cu, *Sp, *cp;
    double *src;
    ModelPar par;
    const double *eta = nullptr;   // SCvx / GuSTO: per-seed trust-region radius written to source oeta (scvx.jl:245)
    int oeta = 0;
    const double *lam = nullptr;   // GuSTO: per-seed soft-penalty weight lambda, written to source olam (gusto.jl:228)
    int olam = 0;
    const double *kappa = nullptr; // in-loop homotopy schedule: per-seed value of the pack's homotopy parameter
    int b0 = 0, nb = 0;            // chunk of seeds [b0, b0 + nb) of this launch (nb = 0: all B)
};

__device__ __forceinline__ size_t gaddr(int b, int G, long long E, long long e)
{
    return ((size_t)(b / G) * E + e) * G + (b % G);
}

// one thread per (seed, node): nonconvex constraint linearisation + scaled reference
template <class CP>
__global__ void k_linearize(const PtrDev d, const double *xd, const double *ud, const double *p)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)(d.nb > 0 ? d.nb : d.B) * d.N) return;
    const int b = d.b0 + (int)(i / d.N), k = (int)(i % d.N);
    if (b >= d.B) return;
    const double *x = xd + ((size_t)b * d.N + k) * d.nx, *u = ud + ((size_t)b * d.N + k) * d.nu, *pp = p + (size_t)b * d.np;
    const int G = d.G;
    const long long E = d.nsrc;
    if constexpr (CP::NS > 0) {
        constexpr int NS = CP::NS, NX = CP::NX, NU = CP::NU, NG = CP::NG;
        double s[NS], C[NS * NX], D[NS * NU], Gm[NS * NG];
        constr_eval<CP>(d.par, d.kappa ? d.kappa + b : nullptr, d.t_grid[k], d.N, k, x, u, pp, s, C, D, Gm);
        for (int r = 0; r < NS; r++) {
            double rs = s[r];
            for (int j = 0; j < NX; j++) { rs -= C[r * NX + j] * x[j]; d.src[gaddr(b, G, E, d.oC + ((long long)k * NS + r) * NX + j)] = C[r * NX + j]; }
            for (int j = 0; j < NU; j++) { rs -= D[r * NU + j] * u[j]; d.src[gaddr(b, G, E, d.oD + ((long long)k * NS + r) * NU + j)] = D[r * NU + j]; }
            for (int j = 0; j < NG; j++) { rs -= Gm[r * NG + j] * pp[CP::gcol(k, j)]; d.src[gaddr(b, G, E, d.oG + ((long long)k * NS + r) * NG + j)] = Gm[r * NG + j]; }
            d.src[gaddr(b, G, E, d.ors + (long long)k * NS + r)] = rs;
        }
    }
    for (int j = 0; j < d.nx; j++) d.src[gaddr(b, G, E, d.oxh + (long long)k * d.nx + j)] = (x[j] - d.cx[j]) / d.Sx[j];
    for (int j = 0; j < d.nu; j++) d.src[gaddr(b, G, E, d.ouh + (long long)k * d.nu + j)] = (u[j] - d.cu[j]) / d.Su[j];
    if (k == 0) {
        for (int j = 0; j < d.np; j++) d.src[gaddr(b, G, E, d.oph + j)] = (pp[j] - d.cp[j]) / d.Sp[j];
        d.src[gaddr(b, G, E, 0)] = 1.0;
        if (d.eta) d.src[gaddr(b, G, E, d.oeta)] = d.eta[b];
        if (d.lam) d.src[gaddr(b, G, E, d.olam)] = d.lam[b];
    }
}

struct AsmDev {
    int B, G, nsrc, nval, nnzA, nnzG, n, p, m;
    int b0 = 0, nbp = 0;   // chunk of whole seed groups [b0, b0 + nbp) of this launch (nbp = 0: all padded seeds)
    const int *W_rp, *W_ci;
    const double *W_v;
    const double *src;
    double *Av, *Gv, *c, *b, *h, *c0;
};

// K6: [Avals; Gvals; c; b; h; c0] = W * src, one thread per (value row, seed); seed is the fast index
__global__ void k_assemble(const AsmDev a)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int Bp = a.nbp > 0 ? a.nbp : ((a.B + a.G - 1) / a.G) * a.G;
    if (i >= (long long)a.nval * Bp) return;
    const int sd = a.b0 + (int)(i % Bp);
    long long e = i / Bp;
    const int G = a.G, gq = sd / G, sg = sd % G;
    const double *s = a.src + (size_t)gq * a.nsrc * G + sg;
    double acc = 0.0;
    for (int k = a.W_rp[e]; k < a.W_rp[e + 1]; k++) acc = fma(a.W_v[k], s[(size_t)a.W_ci[k] * G], acc);
    double *dst; long long E;
    if (e < a.nnzA) { dst = a.Av; E = a.nnzA; }
    else if ((e -= a.nnzA) < a.nnzG) { dst = a.Gv; E = a.nnzG; }
    else if ((e -= a.nnzG) < a.n) { dst = a.c; E = a.n; }
    else if ((e -= a.n) < a.p) { dst = a.b; E = a.p; }
    else if ((e -= a.p) < a.m) { dst = a.h; E = a.m; }
    else { if (sd < a.B) a.c0[sd] = acc; return; }
    dst[((size_t)gq * E + e) * G + sg] = acc;
}

struct StepDev {
    int B, G, N, nx, nu, np, n, vx, vu, vp, iter, q_exit;  // q_exit: 0 = Inf, 1, 2
    int b0 = 0, nb = 0;                                     // chunk of seeds [b0, b0 + nb) of this launch (nb = 0: all B)
    const int *cone_iters = nullptr;                        // streamed loop: interior-point iterations of the last solve ...
    unsigned long long *ipm_total = nullptr;                // ... summed over the live seeds into this device counter
    double eps_abs, eps_rel;
    const double *Sx, *cx, *Su, *cu, *Sp, *cp;
    const double *xsol;       // grouped solver x (scaled variables)
    const double *pobj, *c0;
    const int *cone_status;
    double *xd, *ud, *p;      // reference (accepted) trajectory, Julia layout
    double *xn, *un, *pn;     // new trajectory
    double *J_ref, *J_new, *dev, *imp;
    const int *feas_new;
    int *done, *status, *iters, *nactive;
    // in-loop homotopy schedule (scpb_ptr_set_homotopy; hom_n = 0: none), the device twin of the reference's callback
    // (rendezvous_3d/definition.jl:96-151, called at ptr.jl:496-506): per seed the grid index, the homotopy parameter,
    // the iteration of the last update, the effective iter_max and the update threshold beta
    int hom_n = 0, hist_cap = 0;
    double worsen_tol = 0.0;
    const double *hom_grid = nullptr, *hom_beta = nullptr;
    int *hom_idx = nullptr, *hom_last = nullptr, *hom_itmax = nullptr;
    double *hom_kappa = nullptr;
    int *hist_idx = nullptr;       // [B][hist_cap]: grid index each iteration's subproblem was built with ...
    double *hist_imp = nullptr;    // ... and its improv_rel
    int *ndone = nullptr;          // streamed loop with a schedule: seeds of this chunk that have finished
};

// extract the new iterate (physical units) for active seeds; frozen seeds re-emit their accepted iterate
__global__ void k_extract(const StepDev d)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)(d.nb > 0 ? d.nb : d.B) * d.N) return;
    const int b = d.b0 + (int)(i / d.N), k = (int)(i % d.N);
    if (b >= d.B) return;
    const bool frozen = d.done[b] != 0;
    const int G = d.G;
    for (int j = 0; j < d.nx; j++) {
        const size_t o = ((size_t)b * d.N + k) * d.nx + j;
        d.xn[o] = frozen ? d.xd[o] : d.Sx[j] * d.xsol[gaddr(b, G, d.n, d.vx + j + (long long)d.nx * k)] + d.cx[j];
    }
    for (int j = 0; j < d.nu; j++) {
        const size_t o = ((size_t)b * d.N + k) * d.nu + j;
        d.un[o] = frozen ? d.ud[o] : d.Su[j] * d.xsol[gaddr(b, G, d.n, d.vu + j + (long long)d.nu * k)] + d.cu[j];
    }
    if (k == 0) {
        for (int j = 0; j < d.np; j++) {
            const size_t o = (size_t)b * d.np + j;
            d.pn[o] = frozen ? d.p[o] : d.Sp[j] * d.xsol[gaddr(b, G, d.n, d.vp + j)] + d.cp[j];
        }
        if (!frozen) d.J_new[b] = d.pobj[b] + d.c0[b];
    }
}

__device__ __forceinline__ double qnorm_acc(double acc, double v, int q)
{
    v = fabs(v);
    return q == 0 ? fmax(acc, v) : (q == 1 ? acc + v : acc + v * v);
}

// The per-seed helpers below are shared by the step kernels of PTR (StepDev), SCvx (ScvxDev) and GuSTO (GustoDev):
// each reads the fields of the same name that all three descriptors carry.

// solution_deviation (scp.jl:909-931) of seed b's candidate (xn, and pn: its parameter block) from its reference (xd,
// p), in scaled units
template <class D>
__device__ __forceinline__ double solution_deviation(const D &d, int b, const double *pn)
{
    const int q = d.q_exit;
    double dp = 0.0;
    for (int j = 0; j < d.np; j++) dp = qnorm_acc(dp, (pn[j] - d.p[(size_t)b * d.np + j]) / d.Sp[j], q);
    if (q == 2) dp = sqrt(dp);
    double dx = 0.0;
    for (int k = 0; k < d.N; k++) {
        double a = 0.0;
        for (int j = 0; j < d.nx; j++) {
            const size_t o = ((size_t)b * d.N + k) * d.nx + j;
            a = qnorm_acc(a, (d.xn[o] - d.xd[o]) / d.Sx[j], q);
        }
        if (q == 2) a = sqrt(a);
        dx = fmax(dx, a);
    }
    return dp + dx;
}

// unsafe_solution (scp.jl:965-980): a seed whose subproblem is not (almost) optimal stops with status 2 + 16 * cone status
template <class D>
__device__ __forceinline__ bool unsafe_exit(const D &d, int b, int cs, int *ndone)
{
    if (cs == IPM_OPTIMAL || cs == IPM_ALMOST) return false;
    d.done[b] = 1; d.status[b] = 2 + 16 * cs; d.iters[b] = d.iter;
    if (ndone) atomicAdd(ndone, 1);
    return true;
}

// the candidate becomes seed b's reference, with cost J
template <class D>
__device__ __forceinline__ void accept_candidate(const D &d, int b, double J)
{
    for (int k = 0; k < d.N; k++) {
        for (int j = 0; j < d.nx; j++) { const size_t o = ((size_t)b * d.N + k) * d.nx + j; d.xd[o] = d.xn[o]; }
        for (int j = 0; j < d.nu; j++) { const size_t o = ((size_t)b * d.N + k) * d.nu + j; d.ud[o] = d.un[o]; }
    }
    for (int j = 0; j < d.np; j++) d.p[(size_t)b * d.np + j] = d.pn[(size_t)b * d.np + j];
    d.J_ref[b] = J;
}

// value of solver variable v (scaled) at the physical trajectory (x, u, p): only x, u, p blocks may appear
template <class D>
__device__ __forceinline__ double scaled_var(const D &d, const double *x, const double *u, const double *p, int v)
{
    if (v >= d.vx && v < d.vx + d.N * d.nx) { const int e = v - d.vx, i = e % d.nx; return (x[e] - d.cx[i]) / d.Sx[i]; }
    if (v >= d.vu && v < d.vu + d.N * d.nu) { const int e = v - d.vu, i = e % d.nu; return (u[e] - d.cu[i]) / d.Su[i]; }
    const int j = v - d.vp;
    return (p[j] - d.cp[j]) / d.Sp[j];
}

// one thread per seed: deviation, predicted improvement, stopping rule, acceptance (ptr.jl:908-932, 509)
__global__ void k_ptr_step(const StepDev d)
{
    const int q_ = blockIdx.x * blockDim.x + threadIdx.x;
    if (q_ >= (d.nb > 0 ? d.nb : d.B)) return;
    const int b = d.b0 + q_;
    if (b >= d.B) return;
    if (d.done[b]) return;
    if (d.ipm_total) atomicAdd(d.ipm_total, (unsigned long long)d.cone_iters[b]);
    const int cs = d.cone_status[b];
    if (d.hom_n > 0) d.hist_idx[(size_t)b * d.hist_cap + d.iter - 1] = d.hom_idx[b];
    if (unsafe_exit(d, b, cs, d.ndone)) return;   // before the callback (ptr.jl:488-491)
    const double deviation = solution_deviation(d, b, d.pn + (size_t)b * d.np);
    const double Jr = d.J_ref[b], Jn = d.J_new[b];
    const double imp = (Jr - Jn) / fabs(Jr);
    d.dev[b] = deviation; d.imp[b] = imp;
    const bool stop = d.iter > 1 && d.feas_new[b] && (fabs(imp) <= d.eps_rel || deviation <= d.eps_abs);
    // the schedule's update: the next grid value when improv_rel lies in [worsen_tol, beta] and the grid is not exhausted
    // (false for a NaN improv_rel, as at iteration 1); iter_max then grows by the iterations since the last update, and
    // a stop the stopping rule asked for in this iteration is cancelled (ptr.jl:496-506)
    bool acted = false;
    if (d.hom_n > 0) {
        d.hist_imp[(size_t)b * d.hist_cap + d.iter - 1] = imp;
        const int idx = d.hom_idx[b];
        acted = imp <= d.hom_beta[b] && imp >= d.worsen_tol && idx < d.hom_n - 1;
        if (acted) {
            d.hom_idx[b] = idx + 1;
            d.hom_kappa[b] = d.hom_grid[idx + 1];
            d.hom_itmax[b] += d.iter - d.hom_last[b];
            d.hom_last[b] = d.iter;
        }
    }
    accept_candidate(d, b, Jn);
    d.iters[b] = d.iter;
    if (stop && !acted) {
        d.done[b] = 1; d.status[b] = 0;
        if (d.ndone) atomicAdd(d.ndone, 1);
    } else if (d.hom_n > 0 && d.iter >= d.hom_itmax[b]) {   // the seed's own iter_max: status stays 1
        d.done[b] = 1;
        if (d.ndone) atomicAdd(d.ndone, 1);
    } else atomicAdd(d.nactive, 1);
}

// start of a solve with a schedule: every seed from grid[0], the configured iter_max and last_update = 1 (the
// reference's default when the reference solution carries no update yet); history cleared to -1 / NaN
__global__ void k_hom_init(const StepDev d, int iter_max, int nB)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nB) {
        d.hom_idx[i] = 0; d.hom_kappa[i] = d.hom_grid[0]; d.hom_last[i] = 1; d.hom_itmax[i] = iter_max;
    }
    if (i < (long long)nB * d.hist_cap) { d.hist_idx[i] = -1; d.hist_imp[i] = CUDART_NAN; }
}

// ----------------------------------------------------------------------------------------------
#ifndef SCPB_PTR_DEFAULT_CHUNKS
#define SCPB_PTR_DEFAULT_CHUNKS 0   // streamed PTR chains are opt-in (SCPB_PTR_CHUNKS=<n>): see scpb_ptr_solve
#endif

struct scpb_ptr_s {
    scpb_handle_s *h = nullptr;
    scpb_cone_s *cone = nullptr;
    int model_id = 0;            // dynamics pack and parameters captured at setup: a later scpb_model_set on the same
    ModelPar par{};              // handle (another problem sharing it) must not change what THIS problem solves
    int npar = 0;                // length of that block: scpb_ptr_set_par refuses a shorter one
    scpb_ptr_desc d{};
    std::vector<void *> dev;
    int *W_rp = nullptr, *W_ci = nullptr;
    double *W_v = nullptr;
    double *scale = nullptr, *tgrid = nullptr;
    // batch buffers
    int capB = 0, capG = 0;
    std::vector<void *> bb;
    double *src = nullptr, *xd = nullptr, *ud = nullptr, *p = nullptr, *xn = nullptr, *un = nullptr, *pn = nullptr;
    double *defect = nullptr, *J_ref = nullptr, *J_new = nullptr, *devi = nullptr, *imp = nullptr, *c0 = nullptr;
    int *feas = nullptr, *done = nullptr, *status = nullptr, *iters = nullptr, *nactive = nullptr;
    // SCvx (scpb_scvx_attach)
    bool scvx = false;
    scpb_scvx_desc sv{};
    int *Q_rp = nullptr, *Q_ci = nullptr;
    double *Q_v = nullptr, *Q_c = nullptr;
    double *src2 = nullptr, *eta = nullptr, *L_new = nullptr, *J_out = nullptr;
    int *accept = nullptr;
    // GuSTO (scpb_gusto_attach)
    bool gusto = false;
    scpb_gusto_desc gv{};
    double *Q_w = nullptr;
    double *lam = nullptr, *nodeq = nullptr;
    int *nodef = nullptr;
    // streamed PTR loop (scpb_ptr_solve): one stream per chunk of seed groups, device counter of interior-point iterations
    std::vector<cudaStream_t> chunk_streams;
    unsigned long long *d_ipm_total = nullptr;
    // in-loop homotopy schedule (scpb_ptr_set_homotopy): grid, threshold per seed, state and history of the last solve
    int hom_n = 0, hom_slot = -1, hom_cap = 0;   // hom_cap: history columns = the longest chain a seed can run
    double hom_wtol = 0.0;
    double *hom_grid = nullptr;
    std::vector<double> hom_grid_h;               // host copy of the device grid: an unchanged grid is not re-uploaded
    std::vector<double> hom_beta_h;               // scpb_ptr_set_homotopy_beta: one per seed of the next solves
    std::vector<void *> hb;                       // per-seed buffers below, sized for hom_capB seeds x hom_cap
    int hom_capB = 0, hom_bufcap = 0, last_B = 0, last_cap = 0;   // last_cap: history columns of the last solve (0: none)
    double *hom_beta = nullptr, *hom_kappa = nullptr, *hist_imp = nullptr;
    int *hom_idx = nullptr, *hom_last = nullptr, *hom_itmax = nullptr, *hist_idx = nullptr;
    int *d_chunk_done = nullptr, *h_chunk_done = nullptr;   // streamed loop: finished seeds per chunk (device, pinned copy)
    int chunk_cap = 0;
};

// the handle may have been pointed at another model pack since scpb_ptr_setup (several problems can share one handle):
// every solve re-selects the pack and parameters this problem was set up with
static void ptr_select_model(scpb_ptr_s *s)
{
    scpb_handle_s *h = s->h;
    h->model_id = s->model_id; h->par = s->par;
    h->nx = s->d.nx; h->nu = s->d.nu; h->np = s->d.np;
}

// events of the phase timers: destroyed on every exit path
struct EventList {
    std::vector<cudaEvent_t> ev;
    ~EventList() { for (cudaEvent_t e : ev) cudaEventDestroy(e); }
};

// singular-transition-matrix flag raised by k_discretize_foh during the loop: report it and clear it
static int ptr_check_disc_status(scpb_handle_s *h, const char *who)
{
    int hstat = 0;
    SCPB_CUDA(h, cudaMemcpy(&hstat, h->d_status, sizeof(int), cudaMemcpyDeviceToHost));
    if (hstat & 1) {
        cudaMemset(h->d_status, 0, sizeof(int));
        return set_err(h, SCPB_ERR_STATE, "%s: singular transition matrix during discretization", who);
    }
    return SCPB_OK;
}

template <class T>
static T *up(scpb_ptr_s *s, const T *src, size_t n)
{
    void *d = nullptr;
    if (cudaMalloc(&d, sizeof(T) * (n + 1)) != cudaSuccess) return nullptr;
    if (n) cudaMemcpy(d, src, sizeof(T) * n, cudaMemcpyHostToDevice);
    s->dev.push_back(d);
    return (T *)d;
}

// diagnostic (SCPB_IPM_STATS=1): distribution of the interior-point iteration counts of one solver launch over its live
// seeds -- the launch lasts as long as its slowest seed group
static void ipm_launch_stats(const std::vector<int> &hit, const std::vector<int> &hdone, int launch)
{
    static const bool on = getenv("SCPB_IPM_STATS") != nullptr;
    if (!on) return;
    std::vector<int> v;
    for (size_t b = 0; b < hit.size(); b++) if (!hdone[b]) v.push_back(hit[b]);
    if (v.empty()) return;
    std::sort(v.begin(), v.end());
    long long sum = 0;
    for (int x : v) sum += x;
    size_t am = 0;
    for (size_t b = 0; b < hit.size(); b++) if (!hdone[b] && (hdone[am] || hit[b] > hit[am])) am = b;
    fprintf(stderr, "[scpb] launch %d: live %zu  ipm iterations min %d  median %d  p90 %d  max %d  mean %.1f  argmax %zu\n", launch,
            v.size(), v.front(), v[v.size() / 2], v[(v.size() * 9) / 10], v.back(), (double)sum / v.size(), am);
}

static int ptr_reserve(scpb_ptr_s *s, int B, int G)
{
    scpb_handle_s *h = s->h;
    const int Bpad = ((B + G - 1) / G) * G;
    if (s->capB >= Bpad && s->capG == G) return SCPB_OK;
    // forget the old set before allocating the new one: a failed allocation must not leave stale pointers behind
    auto drop = [&]() {
        for (void *q : s->bb) if (q) cudaFree(q);
        s->bb.clear();
        s->capB = 0; s->capG = 0;
        s->src = s->xd = s->ud = s->p = s->xn = s->un = s->pn = nullptr;
        s->defect = s->J_ref = s->J_new = s->devi = s->imp = s->c0 = nullptr;
        s->feas = s->done = s->status = s->iters = s->nactive = nullptr;
        s->src2 = s->eta = s->L_new = s->J_out = nullptr; s->accept = nullptr;
        s->lam = s->nodeq = nullptr; s->nodef = nullptr;
    };
    drop();
    const scpb_ptr_desc &d = s->d;
    bool ok = true;
    auto al = [&](size_t bytes) { void *q = nullptr; if (cudaMalloc(&q, bytes + 64) != cudaSuccess) { ok = false; return (void *)nullptr; } s->bb.push_back(q); return q; };
    const size_t NB = (size_t)Bpad * d.N;
    s->src = (double *)al(sizeof(double) * (size_t)d.nsrc * Bpad);
    s->xd = (double *)al(sizeof(double) * NB * d.nx); s->xn = (double *)al(sizeof(double) * NB * d.nx);
    s->ud = (double *)al(sizeof(double) * NB * d.nu); s->un = (double *)al(sizeof(double) * NB * d.nu);
    s->p = (double *)al(sizeof(double) * (size_t)Bpad * d.np); s->pn = (double *)al(sizeof(double) * (size_t)Bpad * d.np);
    s->defect = (double *)al(sizeof(double) * NB * d.nx);
    s->J_ref = (double *)al(sizeof(double) * Bpad); s->J_new = (double *)al(sizeof(double) * Bpad);
    s->devi = (double *)al(sizeof(double) * Bpad); s->imp = (double *)al(sizeof(double) * Bpad);
    s->c0 = (double *)al(sizeof(double) * Bpad);
    s->feas = (int *)al(sizeof(int) * Bpad); s->done = (int *)al(sizeof(int) * Bpad);
    s->status = (int *)al(sizeof(int) * Bpad); s->iters = (int *)al(sizeof(int) * Bpad);
    s->nactive = (int *)al(sizeof(int));
    if (s->scvx || s->gusto) {
        s->src2 = (double *)al(sizeof(double) * (size_t)d.nsrc * Bpad);
        s->eta = (double *)al(sizeof(double) * Bpad); s->L_new = (double *)al(sizeof(double) * Bpad);
        s->J_out = (double *)al(sizeof(double) * Bpad); s->accept = (int *)al(sizeof(int) * Bpad);
    }
    if (s->gusto) {
        s->lam = (double *)al(sizeof(double) * Bpad);
        s->nodeq = (double *)al(sizeof(double) * 4 * NB); s->nodef = (int *)al(sizeof(int) * NB);
    }
    if (!ok) { cudaGetLastError(); drop(); return set_err(h, SCPB_ERR_CUDA, "ptr: device allocation failed (B=%d)", B); }
    s->capB = Bpad; s->capG = G;
    return SCPB_OK;
}

// the schedule's per-seed state and history for Bpad seeds
static int hom_reserve(scpb_ptr_s *s, int Bpad)
{
    if (s->hom_capB >= Bpad && s->hom_bufcap >= s->hom_cap) return SCPB_OK;
    for (void *q : s->hb) if (q) cudaFree(q);
    s->hb.clear();
    s->hom_capB = 0; s->hom_bufcap = 0;
    s->hom_beta = s->hom_kappa = s->hist_imp = nullptr;
    s->hom_idx = s->hom_last = s->hom_itmax = s->hist_idx = nullptr;
    bool ok = true;
    auto al = [&](size_t bytes) { void *q = nullptr; if (cudaMalloc(&q, bytes + 64) != cudaSuccess) { ok = false; return (void *)nullptr; } s->hb.push_back(q); return q; };
    const size_t H = (size_t)Bpad * s->hom_cap;
    s->hom_beta = (double *)al(sizeof(double) * Bpad); s->hom_kappa = (double *)al(sizeof(double) * Bpad);
    s->hom_idx = (int *)al(sizeof(int) * Bpad); s->hom_last = (int *)al(sizeof(int) * Bpad);
    s->hom_itmax = (int *)al(sizeof(int) * Bpad);
    s->hist_idx = (int *)al(sizeof(int) * H); s->hist_imp = (double *)al(sizeof(double) * H);
    if (!ok) {
        cudaGetLastError();
        for (void *q : s->hb) if (q) cudaFree(q);
        s->hb.clear();
        return set_err(s->h, SCPB_ERR_CUDA, "ptr: device allocation of the homotopy state failed (B=%d)", Bpad);
    }
    s->hom_capB = Bpad; s->hom_bufcap = s->hom_cap;
    return SCPB_OK;
}

static OutView grouped(double *src, int G, long long nsrc, long long off, long long blk)
{
    OutView v{};
    v.ptr = src + off * G; v.Gq = G; v.sGrp = nsrc * G; v.sB = 1; v.sK = blk * G; v.sE = G;
    return v;
}

static int run_discretize(scpb_ptr_s *s, int B, int G, const double *xd, const double *ud, const double *p,
                          double *srcbuf = nullptr, const int *skip = nullptr, cudaStream_t st = nullptr, int b0 = 0, int nb = 0)
{
    double *sb = srcbuf ? srcbuf : s->src;
    const scpb_ptr_desc &d = s->d;
    DiscArgs a{};
    a.B = B; a.N = d.N; a.Nsub = d.Nsub;
    a.t_grid = s->tgrid; a.xd = xd; a.ud = ud; a.p = p;
    a.iSx = s->scale + 2 * (size_t)(d.nx + d.nu + d.np);  // iSx stored after S and c blocks
    a.xsB = (long long)d.N * d.nx; a.xsK = d.nx; a.xsE = 1;
    a.usB = (long long)d.N * d.nu; a.usK = d.nu; a.usE = 1;
    a.psB = d.np; a.psE = 1;
    a.f_packed = 1;
    a.skip = skip;     // seeds that have stopped keep their DLTV blocks, defects and feasibility flag
    a.b0 = b0; a.nb = nb;
    const long long nx = d.nx, nu = d.nu;
    a.A = grouped(sb, G, d.nsrc, d.oA, nx * nx);
    a.Bm = grouped(sb, G, d.nsrc, d.oBm, nx * nu);
    a.Bp = grouped(sb, G, d.nsrc, d.oBp, nx * nu);
    a.F = grouped(sb, G, d.nsrc, d.oF, nx * d.nf);
    a.r = grouped(sb, G, d.nsrc, d.or_, nx);
    a.E = grouped(sb, G, d.nsrc, d.oE, nx * nx);
    OutView df{}; df.ptr = s->defect; df.Gq = 1; df.sGrp = (long long)(d.N - 1) * nx; df.sB = 0; df.sK = nx; df.sE = 1;
    a.defect = df;
    return scpb_internal_discretize(s->h, a, d.feas_tol, s->feas, d.method, st);
}


// ----------------------------------------------------------------------------------------------
// SCvx (src/solvers/scvx.jl): nonlinear augmented cost, ratio test, accept / reject, radius update
struct ScvxDev {
    int N, nx, nu, np, n_ic, n_tc, vx, vu, vp, q_exit, iter, iter_max, B;
    double lam, rho_0, rho_1, rho_2, beta_sh, beta_gr, eta_lb, eta_ub, eps_abs, eps_rel;
    const int *Q_rp, *Q_ci;
    const double *Q_v, *Q_c;
    const double *Sx, *cx, *Su, *cu, *Sp, *cp, *t_grid, *defect;
    ModelPar par;
    double *xd, *ud, *p, *xn, *un, *pn;
    double *J_ref, *J_new, *L_new, *J_out, *eta, *dev;
    const int *cone_status, *feas_new;
    int *done, *status, *iters, *nactive, *accept;
};

// the constraint packs k_scvx_cost has the penalty of (none, the starship's): scpb_scvx_attach refuses any other
template <class CP>
constexpr bool scvx_has_pack = CP::NS == 0 || std::is_same_v<CP, Constr<SCPB_MODEL_STARSHIP>>;

// one thread per seed: J = L + lambda (trapz_k(|defect_k|_1 + |max(s_k, 0)|_1) + |g_ic|_1 + |g_tc|_1)
// (solution_cost! / actual_cost_penalty!, scvx.jl:919-988) of the trajectory (x, u, p) whose defects are in d.defect
template <class CP>
__global__ void k_scvx_cost(const ScvxDev d, const double *xall, const double *uall, const double *pall, double *J, double *L)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    if (d.done[b]) return;
    const double *x = xall + (size_t)b * d.N * d.nx, *u = uall + (size_t)b * d.N * d.nu, *p = pall + (size_t)b * d.np;
    double q0 = 0.0, gsum = 0.0;
    for (int r = 0; r < 1 + d.n_ic + d.n_tc; r++) {
        double acc = d.Q_c[r];
        for (int k = d.Q_rp[r]; k < d.Q_rp[r + 1]; k++) acc = fma(d.Q_v[k], scaled_var(d, x, u, p, d.Q_ci[k]), acc);
        if (r == 0) q0 = acc; else gsum += fabs(acc);
    }
    double pen = 0.0, Pprev = 0.0;
    for (int k = 0; k < d.N; k++) {
        double Pk = 0.0;
        if (k < d.N - 1)
            for (int i = 0; i < d.nx; i++) Pk += fabs(d.defect[((size_t)b * (d.N - 1) + k) * d.nx + i]);
        if constexpr (CP::NS > 0) {
            constexpr int NS = CP::NS, NX = CP::NX, NU = CP::NU, NG = CP::NG;
            double s[NS], C[NS * NX], D[NS * NU], Gm[NS * NG];
            CP::eval(d.par, d.t_grid[k], d.N, k, x + (size_t)k * d.nx, u + (size_t)k * d.nu, p, s, C, D, Gm);
            for (int r = 0; r < NS; r++) Pk += fmax(s[r], 0.0);
        }
        Pk *= d.lam;
        if (k > 0) pen += (Pk + Pprev) * (0.5 * (d.t_grid[k] - d.t_grid[k - 1]));   // trapz, helper.jl:560-568
        Pprev = Pk;
    }
    L[b] = q0;
    J[b] = q0 + (pen + d.lam * gsum);
}

// one thread per seed: check_stopping_criterion! (scvx.jl:711-733), update_trust_region! / update_rule (:745-770,
// 1000-1045).  The candidate (xn, un, pn) becomes the reference when accepted; it is also what the loop returns when
// it stops or runs out of iterations (SCPSolution takes the last subproblem's solution, scp.jl:205-236).
__global__ void k_scvx_step(const ScvxDev d)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    d.accept[b] = 0;
    if (d.done[b]) return;
    if (unsafe_exit(d, b, d.cone_status[b], nullptr)) return;
    const double deviation = solution_deviation(d, b, d.pn + (size_t)b * d.np);
    d.dev[b] = deviation;
    const double Jr = d.J_ref[b], Jn = d.J_new[b], Ln = d.L_new[b];
    const double pre = Jr - Ln;                        // pre_improv = J_ref - L(sol)  (scvx.jl:724-726)
    const double pre_rel = pre / fabs(Jr);
    const bool stop = d.iter > 1 && d.feas_new[b] && (pre_rel <= d.eps_rel || deviation <= d.eps_abs);
    bool acc = true;
    double eta = d.eta[b];
    if (!stop) {
        const double rho = (Jr - Jn) / pre;
        if (rho < d.rho_0) { eta = fmax(d.eta_lb, eta / d.beta_sh); acc = false; }
        else if (d.rho_0 <= rho && rho < d.rho_1) eta = fmax(d.eta_lb, eta / d.beta_sh);
        else if (d.rho_1 <= rho && rho < d.rho_2) {}
        else eta = fmin(d.eta_ub, d.beta_gr * eta);
        d.eta[b] = eta;
    }
    const bool last = stop || d.iter >= d.iter_max;
    if (acc || last) accept_candidate(d, b, Jn);
    d.accept[b] = (acc && !last) ? 1 : 0;
    d.J_out[b] = Jn;
    d.iters[b] = d.iter;
    if (stop) { d.done[b] = 1; d.status[b] = 0; }
    else atomicAdd(d.nactive, 1);
}

// SCvx and GuSTO, accepted seeds: the candidate's DLTV blocks [lo, hi) (written by discretize! into src2) become the
// reference linearisation in src
__global__ void k_scvx_take_dltv(int B, int G, int nsrc, int lo, int hi, const int *accept, double *src, const double *src2)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long span = hi - lo;
    if (i >= span * B) return;
    const int b = (int)(i % B);
    if (!accept[b]) return;
    const long long e = lo + i / B;
    const size_t a = gaddr(b, G, nsrc, e);
    src[a] = src2[a];
}

// ----------------------------------------------------------------------------------------------
// GuSTO (src/solvers/gusto.jl, pen = :quad): nonconvex costs of the candidate, convexification error, update rule
struct GustoDev {
    int B, G, N, nx, nu, np, n, vx, vu, vp, q_exit, q_tr, iter, iter_max, iter_mu, nsq;
    double lam_init, lam_max, rho_0, rho_1, beta_sh, beta_gr, gamma_fail, eta_lb, eta_ub, mu, eps_abs, eps_rel;
    const int *Q_rp, *Q_ci;
    const double *Q_v, *Q_c, *Q_w;
    const double *Sx, *cx, *Su, *cu, *Sp, *cp, *t_grid;
    const double *xsol;
    ModelPar par;
    double *xd, *ud, *p, *xn, *un, *pn;
    double *J_ref, *L_aug, *J_out, *eta, *lam, *dev, *nodeq;
    int *nodef;
    const int *cone_status, *feas_new;
    int *done, *status, *iters, *nactive, *accept;
};

// one thread per (seed, node): the per-node terms of
//   * the convexification error of the dynamics (update_trust_region!, gusto.jl:1262-1283): |f(sol) - f_lin(sol)|_2 and
//     |f_lin(sol)|_2 with f_lin the linearisation about the reference node;
//   * the nonconvex state penalty of the candidate (state_penalty_cost, :nonconvex, gusto.jl:846-864):
//     lambda sum_i max(0, s_i)^2, and the hard feasibility flag of update_rule! (s_i > 1e-3, gusto.jl:1345-1360);
//   * the trust-region left-hand side |xh_k - xh_ref,k|_q (trust_region_cost, :nonconvex, gusto.jl:1167-1187).
template <class M, class CP>
__global__ void k_gusto_nodes(const GustoDev d)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)d.B * d.N) return;
    const int b = (int)(i / d.N), k = (int)(i % d.N);
    if (d.done[b]) return;
    constexpr int NX = M::NX, NU = M::NU, NF = M::NF;
    const double *xr = d.xd + ((size_t)b * d.N + k) * NX, *ur = d.ud + ((size_t)b * d.N + k) * NU, *pr = d.p + (size_t)b * d.np;
    const double *xs = d.xn + ((size_t)b * d.N + k) * NX, *us = d.un + ((size_t)b * d.N + k) * NU, *ps = d.pn + (size_t)b * d.np;
    const double t = d.t_grid[k];
    double f[NX], A[NX * NX], Bm[NX * NU], F[NX * at_least_1(NF)], fl[NX];
    M::eval(d.par, t, xr, ur, pr, f, A, Bm, F);
    for (int r = 0; r < NX; r++) {           // f_lin(sol) = f(ref) + A (xs - xr) + B (us - ur) + F (ps - pr)
        double a = f[r];
        for (int j = 0; j < NX; j++) a = fma(A[r + NX * j], xs[j] - xr[j], a);
        for (int j = 0; j < NU; j++) a = fma(Bm[r + NX * j], us[j] - ur[j], a);
        for (int j = 0; j < NF; j++) a = fma(F[r + NX * j], ps[M::fcol(j)] - pr[M::fcol(j)], a);
        fl[r] = a;
    }
    M::eval(d.par, t, xs, us, ps, f, A, Bm, F);
    double df = 0.0, dn = 0.0;
    for (int r = 0; r < NX; r++) { df += (f[r] - fl[r]) * (f[r] - fl[r]); dn += fl[r] * fl[r]; }
    double pen = 0.0;
    int viol = 0;
    if constexpr (CP::NS > 0) {
        constexpr int NS = CP::NS, NG = CP::NG;
        double s[NS], C[NS * NX], D[NS * NU], Gm[NS * NG];
        CP::eval(d.par, t, d.N, k, xs, us, ps, s, C, D, Gm);
        for (int r = 0; r < NS; r++) {
            const double m = fmax(s[r], 0.0);
            pen += m * m;
            if (s[r] > 1e-3) viol = 1;
        }
        pen *= d.lam[b];
    }
    double tr = 0.0;
    for (int j = 0; j < NX; j++) tr = qnorm_acc(tr, (xs[j] - d.cx[j]) / d.Sx[j] - (xr[j] - d.cx[j]) / d.Sx[j], d.q_tr);
    if (d.q_tr == 2) tr = sqrt(tr);
    double *o = d.nodeq + 4 * (size_t)i;
    o[0] = sqrt(df); o[1] = sqrt(dn); o[2] = pen; o[3] = tr;
    d.nodef[i] = viol;
}

// one thread per seed: SubproblemSolution(spbm) costs (gusto.jl:399-418), check_stopping_criterion! (:1203-1231),
// update_trust_region! (:1245-1293) and update_rule! (:1310-1427, with the mu-shrink of the next subproblem's eta, :268).
__global__ void k_gusto_step(const GustoDev d)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    d.accept[b] = 0;
    if (d.done[b]) return;
    if (unsafe_exit(d, b, d.cone_status[b], nullptr)) return;
    const double *x = d.xn + (size_t)b * d.N * d.nx, *u = d.un + (size_t)b * d.N * d.nu, *p = d.pn + (size_t)b * d.np;
    // original cost J of the candidate: affine row + weighted squares (original_cost, gusto.jl:680-707)
    double J = 0.0;
    for (int r = 0; r <= d.nsq; r++) {
        double acc = d.Q_c[r];
        for (int k = d.Q_rp[r]; k < d.Q_rp[r + 1]; k++) acc = fma(d.Q_v[k], scaled_var(d, x, u, p, d.Q_ci[k]), acc);
        J += r == 0 ? acc : d.Q_w[r - 1] * acc * acc;
    }
    // soft trust-region cost as the subproblem measured it (J_tr = value(L_tr), gusto.jl:409); the row is L_tr / lambda
    double J_tr = d.Q_c[d.nsq + 1];
    for (int k = d.Q_rp[d.nsq + 1]; k < d.Q_rp[d.nsq + 2]; k++) J_tr = fma(d.Q_v[k], d.xsol[gaddr(b, d.G, d.n, d.Q_ci[k])], J_tr);
    // trapezoid sums of the node terms
    const double *nq = d.nodeq + 4 * (size_t)b * d.N;
    const int *nf = d.nodef + (size_t)b * d.N;
    double dyn_err = 0.0, dyn_nrm = 0.0, J_st = 0.0, trmax = -1e300;
    int viol = 0;
    double dpn = 0.0;
    for (int j = 0; j < d.np; j++) dpn = qnorm_acc(dpn, (p[j] - d.cp[j]) / d.Sp[j] - (d.p[(size_t)b * d.np + j] - d.cp[j]) / d.Sp[j], d.q_tr);
    if (d.q_tr == 2) dpn = sqrt(dpn);
    for (int k = 0; k < d.N; k++) {
        if (k > 0) {
            const double w = 0.5 * (d.t_grid[k] - d.t_grid[k - 1]);
            dyn_err += (nq[4 * k] + nq[4 * (k - 1)]) * w;
            dyn_nrm += (nq[4 * k + 1] + nq[4 * (k - 1) + 1]) * w;
            J_st += (nq[4 * k + 2] + nq[4 * (k - 1) + 2]) * w;
        }
        trmax = fmax(trmax, nq[4 * k + 3]);
        viol |= nf[k];
    }
    const double eta = d.eta[b], lam = d.lam[b];
    J_tr *= lam;
    const double J_aug = J + J_st + J_tr, L_aug = d.L_aug[b];
    const double deviation = solution_deviation(d, b, p);
    d.dev[b] = deviation;
    const double Jr = d.J_ref[b];
    const double dJ = fabs(Jr - J_aug) / fabs(Jr);
    const bool infeas = lam > d.lam_max;
    const bool stop = d.iter > 1 && ((d.feas_new[b] && (dJ <= d.eps_rel || deviation <= d.eps_abs)) || infeas);
    bool acc = false;
    if (!stop) {
        const double cost_err = fabs(J_aug - L_aug), cost_nrm = fabs(L_aug);
        const double rho = (cost_err + dyn_err) / (cost_nrm + dyn_nrm);
        const bool trust_viol = (trmax + dpn - eta) > 1e-3;
        double n_eta = eta, n_lam = lam;
        if (trust_viol) n_lam = d.gamma_fail * lam;
        else if (rho < d.rho_1) {
            if (rho < d.rho_0) n_eta = fmin(d.eta_ub, d.beta_gr * eta);
            n_lam = viol ? d.gamma_fail * lam : d.lam_init;
            acc = true;
        } else n_eta = fmax(d.eta_lb, eta / d.beta_sh);
        const double kappa = d.iter < d.iter_mu ? 1.0 : pow(d.mu, (double)(1 + d.iter - d.iter_mu));
        if (kappa < 1.0) n_eta *= kappa;
        d.eta[b] = n_eta; d.lam[b] = n_lam;
    }
    const bool last = stop || d.iter >= d.iter_max;
    if (acc || last) accept_candidate(d, b, J_aug);   // also what the loop returns when it ends (scp.jl:205-236)
    d.accept[b] = (acc && !last) ? 1 : 0;
    d.J_out[b] = J_aug;            // SCPSolution.cost = last_sol.J_aug (scp.jl:236)
    d.iters[b] = d.iter;
    if (stop) { d.done[b] = 1; d.status[b] = 0; }
    else atomicAdd(d.nactive, 1);
}

__global__ void k_fill(double *v, double a, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = a;
}

// nonconvex-constraint linearisation with the pack of the problem's model (none: only the scaled references)
static void launch_linearize(scpb_ptr_s *s, const PtrDev &pd, int nbn, cudaStream_t st)
{
    with_constr(s->model_id, s->d.ns > 0,
                [&](auto cp) { k_linearize<decltype(cp)><<<nbn, 128, 0, st>>>(pd, s->xd, s->ud, s->p); });
}

// scpb_debug_constraints: the pack's s, C, D, G at every (seed, node), one thread each
template <class CP>
__global__ void k_debug_constr(const ModelPar par, int B, int N, const double *t_grid, const double *xd, const double *ud,
                               const double *p, int np, double *s, double *C, double *D, double *G)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * N) return;
    const int b = (int)(i / N), k = (int)(i % N);
    constexpr int NS = CP::NS, NX = CP::NX, NU = CP::NU, NG = CP::NG;
    constr_eval<CP>(par, nullptr, t_grid[k], N, k, xd + (size_t)i * NX, ud + (size_t)i * NU, p + (size_t)b * np,
                    s + (size_t)i * NS, C + (size_t)i * NS * NX, D + (size_t)i * NS * NU, G + (size_t)i * NS * NG);
}

template <class CP>
static int debug_constr_t(scpb_handle_s *h, int B, int N, int ns, int ng, const double *t_grid, const double *xd,
                          const double *ud, const double *p, double *s, double *C, double *D, double *G)
{
    constexpr int NS = CP::NS, NX = CP::NX, NU = CP::NU, NG = CP::NG;
    if (ns != NS || ng != NG || h->nx != NX || h->nu != NU)
        return set_err(h, SCPB_ERR_ARG, "debug_constraints: the pack has ns=%d, ng=%d, nx=%d, nu=%d", NS, NG, NX, NU);
    const size_t BN = (size_t)B * N;
    const size_t n_in[4] = {(size_t)N, BN * NX, BN * NU, (size_t)B * h->np};
    const size_t n_out[4] = {BN * NS, BN * NS * NX, BN * NS * NU, BN * NS * NG};
    const double *hin[4] = {t_grid, xd, ud, p};
    double *hout[4] = {s, C, D, G};
    double *din[4] = {}, *dout[4] = {};
    int rc = SCPB_OK;
    for (int j = 0; j < 4 && rc == SCPB_OK; j++) {
        if (cudaMalloc(&din[j], sizeof(double) * (n_in[j] + 1)) != cudaSuccess ||
            cudaMalloc(&dout[j], sizeof(double) * (n_out[j] + 1)) != cudaSuccess ||
            cudaMemcpyAsync(din[j], hin[j], sizeof(double) * n_in[j], cudaMemcpyHostToDevice, h->stream) != cudaSuccess)
            rc = set_err(h, SCPB_ERR_CUDA, "debug_constraints: device allocation or copy failed");
    }
    if (rc == SCPB_OK) {
        k_debug_constr<CP><<<(unsigned)((BN + 127) / 128), 128, 0, h->stream>>>(h->par, B, N, din[0], din[1], din[2], din[3],
                                                                                 h->np, dout[0], dout[1], dout[2], dout[3]);
        h->launches++;
        for (int j = 0; j < 4 && rc == SCPB_OK; j++)
            if (cudaMemcpyAsync(hout[j], dout[j], sizeof(double) * n_out[j], cudaMemcpyDeviceToHost, h->stream) != cudaSuccess)
                rc = set_err(h, SCPB_ERR_CUDA, "debug_constraints: %s", cudaGetErrorString(cudaGetLastError()));
        if (cudaStreamSynchronize(h->stream) != cudaSuccess && rc == SCPB_OK)
            rc = set_err(h, SCPB_ERR_CUDA, "debug_constraints: %s", cudaGetErrorString(cudaGetLastError()));
    }
    for (int j = 0; j < 4; j++) { if (din[j]) cudaFree(din[j]); if (dout[j]) cudaFree(dout[j]); }
    return rc;
}

// GuSTO's node terms with the problem's model and pack; SCPB_ERR_UNSUPPORTED for the rendezvous and the oscillator,
// whose deadband packs GuSTO lacks
static int launch_gusto_nodes(scpb_ptr_s *s, const GustoDev &gd, cudaStream_t st)
{
    const int nbn = (int)(((long long)gd.B * gd.N + 63) / 64);
    int rc = SCPB_ERR_UNSUPPORTED;
    with_model(s->model_id, [&](auto m) {
        using M = decltype(m);
        constexpr int id = ModelId<M>::value;
        if constexpr (id != SCPB_MODEL_RENDEZVOUS2D && id != SCPB_MODEL_OSCILLATOR) {
            if (s->d.ns > 0) k_gusto_nodes<M, PackOf<id>><<<nbn, 64, 0, st>>>(gd);
            else k_gusto_nodes<M, Constr<0>><<<nbn, 64, 0, st>>>(gd);
            rc = SCPB_OK;
        }
    });
    return rc;
}

// ----------------------------------------------------------------------------------------------
// One solve of PTR, SCvx or GuSTO: the state that solve_begin sets up, the loop body each algorithm parameterises, and
// the outputs solve_end returns.
struct Solve {
    scpb_ptr_s *s;
    scpb_handle_s *h;
    cudaStream_t st;
    int B, G;
    IpmData *D;
    IpmOpts o;
    PtrDev pd{};
    AsmDev ad{};
    StepDev sd{};
    // the algorithm: cone options of iteration it, where discretize! writes the candidate's DLTV (nullptr: src), the
    // candidate's cost (run in the discretize phase; may be empty) and the step that accepts, rejects and stops
    std::function<IpmOpts(int)> opts_at;
    double *cand_src = nullptr;
    std::function<int()> candidate;
    std::function<int(int it, cudaStream_t st, int nb)> step;
    // phase timers (the reference's keys: discretize / formulate / solve / overhead, scp.jl:177-178,990-995): phase id
    // of the interval that ENDS at event i
    EventList evl;
    std::vector<int> phase;
    int total_it = 0, n_chunks = 0;
    long long ipm_iters = 0;
    std::vector<int> init_status;   // sources of the resets' uploads, kept until the solve ends
    std::vector<double> nanv;
    void mark(int ph, cudaStream_t on)
    {
        cudaEvent_t e;
        cudaEventCreate(&e); cudaEventRecord(e, on);
        evl.ev.push_back(e); phase.push_back(ph);
    }
};

// what every solve does before its loop: check the batch, select the model, pick the seed group size G, reserve the
// buffers, upload the guesses, reset the per-seed state and describe it to the kernels
static int solve_begin(Solve &v, scpb_ptr_s *s, int B, const double *xd0, const double *ud0, const double *p0,
                       const scpb_cone_opts *opts, const char *who)
{
    scpb_handle_s *h = s->h;
    if (B <= 0 || !xd0 || !ud0 || !p0) return set_err(h, SCPB_ERR_ARG, "%s: bad arguments", who);
    SCPB_CUDA(h, cudaSetDevice(h->device));
    ptr_select_model(s);
    SCPB_CUDA(h, cudaMemsetAsync(h->d_status, 0, sizeof(int), h->stream));
    const scpb_ptr_desc &d = s->d;
    const int G = scpb_internal_pick_group(B, opts ? opts->group : 0, h->sms);
    int rc = scpb_internal_cone_reserve(s->cone, B, G, opts ? opts->lanes : 0);
    if (rc) return rc;
    if ((rc = ptr_reserve(s, B, G))) return rc;
    if (s->hom_n > 0) {   // PTR only: SCvx and GuSTO refuse a problem with a schedule
        if ((int)s->hom_beta_h.size() != B)
            return set_err(h, SCPB_ERR_STATE, "%s: the homotopy schedule has %d update thresholds for %d seeds "
                           "(scpb_ptr_set_homotopy_beta)", who, (int)s->hom_beta_h.size(), B);
        if ((rc = hom_reserve(s, s->capB))) return rc;
    }
    IpmData *D = scpb_internal_cone_data(s->cone);
    const ConeSymbolic *S = scpb_internal_cone_sym(s->cone);
    v.s = s; v.h = h; v.st = h->stream; v.B = B; v.G = G; v.D = D;
    v.o = scpb_internal_make_opts(opts);
    cudaStream_t st = h->stream;
    SCPB_CUDA(h, cudaMemcpyAsync(s->xd, xd0, sizeof(double) * B * d.N * d.nx, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(s->ud, ud0, sizeof(double) * B * d.N * d.nu, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(s->p, p0, sizeof(double) * B * d.np, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemsetAsync(s->src, 0, sizeof(double) * (size_t)d.nsrc * s->capB, st));
    if (s->src2) SCPB_CUDA(h, cudaMemsetAsync(s->src2, 0, sizeof(double) * (size_t)d.nsrc * s->capB, st));
    SCPB_CUDA(h, cudaMemsetAsync(s->done, 0, sizeof(int) * s->capB, st));
    SCPB_CUDA(h, cudaMemsetAsync(s->iters, 0, sizeof(int) * s->capB, st));
    v.init_status.assign(s->capB, 1);
    SCPB_CUDA(h, cudaMemcpyAsync(s->status, v.init_status.data(), sizeof(int) * s->capB, cudaMemcpyHostToDevice, st));
    v.nanv.assign(s->capB, nan(""));
    SCPB_CUDA(h, cudaMemcpyAsync(s->devi, v.nanv.data(), sizeof(double) * s->capB, cudaMemcpyHostToDevice, st));
    if (s->J_out) SCPB_CUDA(h, cudaMemcpyAsync(s->J_out, v.nanv.data(), sizeof(double) * s->capB, cudaMemcpyHostToDevice, st));
    // PTR and GuSTO start from J_ref = NaN (the guess has no cost); SCvx overwrites it with the guess's cost
    SCPB_CUDA(h, cudaMemcpyAsync(s->J_ref, v.nanv.data(), sizeof(double) * s->capB, cudaMemcpyHostToDevice, st));

    const size_t nsc = (size_t)(d.nx + d.nu + d.np);
    const double *Sx = s->scale, *Su = Sx + d.nx, *Sp = Su + d.nu, *cx = s->scale + nsc, *cu = cx + d.nx, *cp = cu + d.nu;
    PtrDev &pd = v.pd;
    pd.B = B; pd.G = G; pd.N = d.N; pd.nx = d.nx; pd.nu = d.nu; pd.np = d.np; pd.ns = d.ns;
    pd.nsrc = d.nsrc; pd.oC = d.oC; pd.oD = d.oD; pd.oG = d.oG; pd.ors = d.ors; pd.oxh = d.oxh; pd.ouh = d.ouh; pd.oph = d.oph;
    pd.t_grid = s->tgrid; pd.Sx = Sx; pd.cx = cx; pd.Su = Su; pd.cu = cu; pd.Sp = Sp; pd.cp = cp;
    pd.src = s->src; pd.par = s->par;
    AsmDev &ad = v.ad;
    ad.B = B; ad.G = G; ad.nsrc = d.nsrc; ad.nval = d.nval; ad.nnzA = (int)S->A_ci.size(); ad.nnzG = (int)S->G_ci.size();
    ad.n = S->n; ad.p = S->p; ad.m = S->m; ad.W_rp = s->W_rp; ad.W_ci = s->W_ci; ad.W_v = s->W_v; ad.src = s->src;
    ad.Av = D->Av; ad.Gv = D->Gv; ad.c = D->c; ad.b = D->b; ad.h = D->h; ad.c0 = s->c0;
    StepDev &sd = v.sd;   // SCvx and GuSTO: k_extract only
    sd.B = B; sd.G = G; sd.N = d.N; sd.nx = d.nx; sd.nu = d.nu; sd.np = d.np; sd.n = S->n; sd.vx = d.vx; sd.vu = d.vu; sd.vp = d.vp;
    sd.q_exit = d.q_exit; sd.eps_abs = d.eps_abs; sd.eps_rel = d.eps_rel;
    sd.Sx = Sx; sd.cx = cx; sd.Su = Su; sd.cu = cu; sd.Sp = Sp; sd.cp = cp;
    sd.xsol = D->x; sd.pobj = D->pobj; sd.c0 = s->c0; sd.cone_status = D->status;
    sd.xd = s->xd; sd.ud = s->ud; sd.p = s->p; sd.xn = s->xn; sd.un = s->un; sd.pn = s->pn;
    sd.J_ref = s->J_ref; sd.J_new = s->J_new; sd.dev = s->devi; sd.imp = s->imp; sd.feas_new = s->feas;
    sd.done = s->done; sd.status = s->status; sd.iters = s->iters; sd.nactive = s->nactive;
    return SCPB_OK;
}

// one SCP iteration: linearize -> assemble -> cone solve -> extract -> discretize! the candidate -> step.  The whole
// batch on the handle's stream (cs = nullptr, nb = nbp = 0; timed, and hit / nact receive the interior-point iterations
// and the live seeds), or the chunk [b0, b0 + nbp) of whole seed groups with nb seeds of a streamed chain on cs.
static int ptr_iteration(Solve &v, int it, cudaStream_t cs, int b0, int nb, int nbp, bool timed, int *hit, int *nact)
{
    scpb_ptr_s *s = v.s;
    scpb_handle_s *h = v.h;
    const scpb_ptr_desc &d = s->d;
    cudaStream_t ls = cs ? cs : v.st;   // stream of the launches and copies
    const int nbl = nb > 0 ? nb : v.B, nbn = (int)(((long long)nbl * d.N + 127) / 128);
    auto mark = [&](int ph) { if (timed) v.mark(ph, ls); };
    v.pd.b0 = b0; v.pd.nb = nb;
    launch_linearize(s, v.pd, nbn, ls);
    v.ad.b0 = b0; v.ad.nbp = nbp;
    k_assemble<<<(unsigned)(((long long)d.nval * (nbp > 0 ? nbp : s->capB) + 255) / 256), 256, 0, ls>>>(v.ad);
    h->launches += 2;
    mark(1);
    if (int r = scpb_internal_cone_run(s->cone, v.opts_at(it), s->done, cs, b0 / v.G, nbp / v.G)) return r;
    mark(2);
    if (hit) SCPB_CUDA(h, cudaMemcpyAsync(hit, v.D->iters, sizeof(int) * v.B, cudaMemcpyDeviceToHost, ls));
    v.sd.iter = it; v.sd.b0 = b0; v.sd.nb = nb;
    k_extract<<<nbn, 128, 0, ls>>>(v.sd);
    h->launches++;
    mark(3);
    if (int r = run_discretize(s, v.B, v.G, s->xn, s->un, s->pn, v.cand_src, s->done, cs, b0, nb)) return r;
    if (v.candidate)
        if (int r = v.candidate()) return r;
    mark(0);
    if (nact) SCPB_CUDA(h, cudaMemsetAsync(s->nactive, 0, sizeof(int), ls));
    if (int r = v.step(it, ls, nbl)) return r;
    if (nact) SCPB_CUDA(h, cudaMemcpyAsync(nact, s->nactive, sizeof(int), cudaMemcpyDeviceToHost, ls));
    mark(3);
    return SCPB_OK;
}

// the lock-step loop: every iteration runs on the whole batch and ends when no seed is live
static int lockstep_loop(Solve &v, int it_bound)
{
    scpb_handle_s *h = v.h;
    const int B = v.B;
    int nact = B;
    std::vector<int> hit(B), hdone(B, 0);   // hdone: seeds that were already finished when the solver was launched (skipped)
    for (int it = 1; it <= it_bound; it++) {
        if (int r = ptr_iteration(v, it, nullptr, 0, 0, 0, true, hit.data(), &nact)) return r;
        SCPB_CUDA(h, cudaStreamSynchronize(v.st));
        for (int b = 0; b < B; b++) if (!hdone[b]) v.ipm_iters += hit[b];   // skipped seeds keep a stale count in D->iters
        ipm_launch_stats(hit, hdone, v.total_it + 1);
        SCPB_CUDA(h, cudaMemcpyAsync(hdone.data(), v.s->done, sizeof(int) * B, cudaMemcpyDeviceToHost, v.st));
        SCPB_CUDA(h, cudaStreamSynchronize(v.st));
        v.total_it++;
        if (nact == 0) break;
    }
    return SCPB_OK;
}

// SCvx and GuSTO: the DLTV blocks of the accepted candidates become the reference linearisation
static void take_dltv(const Solve &v)
{
    const scpb_ptr_desc &d = v.s->d;
    const long long span = (long long)(d.oC - d.oA) * v.B;
    k_scvx_take_dltv<<<(unsigned)((span + 255) / 256), 256, 0, v.st>>>(v.B, v.G, d.nsrc, d.oA, d.oC, v.s->accept, v.s->src,
                                                                       v.s->src2);
}

// what every solve returns: the trajectories, status, iterations, cost (from Jd), deviation and feasibility, the
// per-seed extras {host, device}, and ntiming (8, or 10 with the initial discretize!) entries of timing
static int solve_end(Solve &v, double *xd, double *ud, double *p, int32_t *status, int32_t *iters, double *J,
                     const double *Jd, double *deviation, int32_t *feas,
                     std::initializer_list<std::pair<double *, const double *>> extras, double *timing, int ntiming,
                     const char *who)
{
    scpb_ptr_s *s = v.s;
    scpb_handle_s *h = v.h;
    const scpb_ptr_desc &d = s->d;
    cudaStream_t st = v.st;
    const int B = v.B;
    SCPB_CUDA(h, cudaGetLastError());
    if (xd) SCPB_CUDA(h, cudaMemcpyAsync(xd, s->xd, sizeof(double) * B * d.N * d.nx, cudaMemcpyDeviceToHost, st));
    if (ud) SCPB_CUDA(h, cudaMemcpyAsync(ud, s->ud, sizeof(double) * B * d.N * d.nu, cudaMemcpyDeviceToHost, st));
    if (p) SCPB_CUDA(h, cudaMemcpyAsync(p, s->p, sizeof(double) * B * d.np, cudaMemcpyDeviceToHost, st));
    if (status) SCPB_CUDA(h, cudaMemcpyAsync(status, s->status, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    if (iters) SCPB_CUDA(h, cudaMemcpyAsync(iters, s->iters, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    if (J) SCPB_CUDA(h, cudaMemcpyAsync(J, Jd, sizeof(double) * B, cudaMemcpyDeviceToHost, st));
    if (deviation) SCPB_CUDA(h, cudaMemcpyAsync(deviation, s->devi, sizeof(double) * B, cudaMemcpyDeviceToHost, st));
    if (feas) SCPB_CUDA(h, cudaMemcpyAsync(feas, s->feas, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    for (const auto &e : extras)
        if (e.first) SCPB_CUDA(h, cudaMemcpyAsync(e.first, e.second, sizeof(double) * B, cudaMemcpyDeviceToHost, st));
    SCPB_CUDA(h, cudaStreamSynchronize(st));
    const std::vector<cudaEvent_t> &ev = v.evl.ev;
    double acc[4] = {0, 0, 0, 0};
    for (size_t i = 1; i < ev.size(); i++) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev[i - 1], ev[i]);
        if (v.phase[i] >= 0) acc[v.phase[i]] += ms * 1e-3;
    }
    float tot_ms = 0.f;
    cudaEventElapsedTime(&tot_ms, ev.front(), ev.back());
    if (timing) {
        timing[0] = acc[0]; timing[1] = acc[1]; timing[2] = acc[2]; timing[3] = acc[3];
        timing[4] = tot_ms * 1e-3; timing[5] = (double)v.total_it; timing[6] = (double)v.ipm_iters;
        timing[7] = (double)v.n_chunks;
        if (ntiming > 8) {
            float k1_ms = 0.f;   // the initial full-batch discretize! (K1 timed alone, before the chains fork)
            cudaEventElapsedTime(&k1_ms, ev[0], ev[1]);
            timing[8] = k1_ms * 1e-3; timing[9] = 0.0;
        }
    }
    return ptr_check_disc_status(h, who);
}

extern "C" {

int32_t scpb_ptr_setup(scpb_handle h, scpb_cone cone, const scpb_ptr_desc *desc, const int32_t *W_rowptr,
                       const int32_t *W_colind, const double *W_vals, const double *scale, const double *t_grid,
                       scpb_ptr *out)
{
    if (!h || !cone || !desc || !W_rowptr || !scale || !t_grid || !out) return SCPB_ERR_ARG;
    *out = nullptr;
    if (scpb_internal_cone_handle(cone) != h) return set_err(h, SCPB_ERR_ARG, "ptr_setup: cone belongs to another handle");
    if (desc->nx != h->nx || desc->nu != h->nu || desc->np != h->np)
        return set_err(h, SCPB_ERR_STATE, "ptr_setup: dimensions differ from the selected model pack");
    const ConeSymbolic *S = scpb_internal_cone_sym(cone);
    if (desc->nval != (int)(S->A_ci.size() + S->G_ci.size()) + S->n + S->p + S->m + 1)
        return set_err(h, SCPB_ERR_ARG, "ptr_setup: nval does not match the cone program (%d)", desc->nval);
    if (desc->ns > 0) {
        int pns = 0, png = 0;
        with_constr(h->model_id, true, [&](auto cp) {
            using CP = decltype(cp);
            if constexpr (CP::NS > 0) { pns = CP::NS; png = CP::NG; }
        });
        if (pns != desc->ns || png != desc->ng)
            return set_err(h, SCPB_ERR_UNSUPPORTED, "ptr_setup: no constraint pack for model %d with ns=%d, ng=%d", h->model_id,
                           desc->ns, desc->ng);
        if (h->model_id == SCPB_MODEL_FREEFLYER && desc->np != 1 + Constr<SCPB_MODEL_FREEFLYER>::NISS * desc->N)
            return set_err(h, SCPB_ERR_ARG, "ptr_setup: the free-flyer pack expects np = 1 + 6 N");
        if (h->model_id == SCPB_MODEL_OSCILLATOR && desc->np != desc->N)
            return set_err(h, SCPB_ERR_ARG, "ptr_setup: the oscillator pack expects np = N (one parameter per node)");
    }
    int nf = -1;   // the DLTV's F block holds the pack's active columns only
    with_model(h->model_id, [&](auto m) { nf = decltype(m)::NF; });
    if (desc->nf != nf)
        return set_err(h, SCPB_ERR_ARG, "ptr_setup: model %d has %d active F columns, the descriptor %d", h->model_id, nf,
                       desc->nf);
    if (desc->method != SCPB_FOH && desc->method != SCPB_IMPULSE)
        return set_err(h, SCPB_ERR_ARG, "ptr_setup: unknown discretization method %d", desc->method);
    // refused here rather than at the first discretize! of a solve: only the rendezvous pack has impulse semantics
    if (desc->method == SCPB_IMPULSE && h->model_id != SCPB_MODEL_RENDEZVOUS2D)
        return set_err(h, SCPB_ERR_UNSUPPORTED, "ptr_setup: model %d has no impulse semantics (IMPULSE discretization)",
                       h->model_id);
    SCPB_CUDA(h, cudaSetDevice(h->device));
    scpb_ptr_s *s = new (std::nothrow) scpb_ptr_s();
    if (!s) return SCPB_ERR_CUDA;
    s->h = h; s->cone = cone; s->d = *desc;
    s->model_id = h->model_id; s->par = h->par; s->npar = h->npar;
    const int nnzW = W_rowptr[desc->nval];
    s->W_rp = up(s, W_rowptr, (size_t)desc->nval + 1);
    s->W_ci = up(s, W_colind, (size_t)nnzW);
    s->W_v = up(s, W_vals, (size_t)nnzW);
    const size_t nsc = (size_t)(desc->nx + desc->nu + desc->np);
    s->scale = up(s, scale, 2 * nsc + desc->nx);
    s->tgrid = up(s, t_grid, (size_t)desc->N);
    for (void *q : s->dev)
        if (!q) { scpb_ptr_free(s); return set_err(h, SCPB_ERR_CUDA, "ptr_setup: device allocation failed"); }
    *out = s;
    return SCPB_OK;
}

int32_t scpb_debug_constraints(scpb_handle h, int32_t B, int32_t N, int32_t ns, int32_t ng, const double *t_grid,
                               const double *xd, const double *ud, const double *p, double *s, double *C, double *D,
                               double *G)
{
    if (!h) return SCPB_ERR_ARG;
    if (B <= 0 || N <= 0 || !t_grid || !xd || !ud || !p || !s || !C || !D || !G)
        return set_err(h, SCPB_ERR_ARG, "debug_constraints: bad arguments");
    SCPB_CUDA(h, cudaSetDevice(h->device));
    int rc = SCPB_OK;
    with_constr(h->model_id, true, [&](auto cp) {
        using CP = decltype(cp);
        if constexpr (CP::NS > 0) rc = debug_constr_t<CP>(h, B, N, ns, ng, t_grid, xd, ud, p, s, C, D, G);
        else rc = set_err(h, SCPB_ERR_UNSUPPORTED, "debug_constraints: model %d has no constraint pack", h->model_id);
    });
    return rc;
}

int32_t scpb_ptr_set_par(scpb_ptr s, const double *par, int32_t npar)
{
    if (!s) return SCPB_ERR_ARG;
    if (!par || npar < 1 || npar > SCPB_MAX_PAR)
        return set_err(s->h, SCPB_ERR_ARG, "ptr_set_par: npar = %d outside 1..%d", npar, SCPB_MAX_PAR);
    // a shorter block would zero the trailing entries, e.g. the constraint pack's parameters after the dynamics ones
    if (npar < s->npar)
        return set_err(s->h, SCPB_ERR_ARG, "ptr_set_par: npar = %d is shorter than the %d entries given at setup", npar,
                       s->npar);
    // the kernels of a solve receive the block by value at launch, so an earlier solve that is still queued on the
    // stream keeps the parameters it was launched with
    ModelPar q{};
    for (int i = 0; i < npar; i++) q.v[i] = par[i];
    s->par = q;
    return SCPB_OK;
}

int32_t scpb_ptr_set_homotopy(scpb_ptr s, int32_t par_index, int32_t n_grid, const double *grid, double worsen_tol)
{
    if (!s) return SCPB_ERR_ARG;
    scpb_handle_s *h = s->h;
    if (n_grid == 0) { s->hom_n = 0; s->hom_cap = 0; s->hom_slot = -1; s->hom_grid_h.clear(); return SCPB_OK; }
    if (n_grid < 0 || !grid) return set_err(h, SCPB_ERR_ARG, "ptr_set_homotopy: n_grid = %d with grid %p", n_grid, grid);
    if (s->scvx || s->gusto) return set_err(h, SCPB_ERR_UNSUPPORTED, "ptr_set_homotopy: schedules are implemented for PTR only");
    int slot = -1;   // parameter slot of the pack's homotopy parameter (HomSlot, csrc/constraints.cuh), -1: none
    with_constr(s->model_id, s->d.ns > 0, [&](auto cp) { slot = HomSlot<decltype(cp)>::value; });
    if (slot < 0 || (par_index >= 0 && slot != par_index))
        return set_err(h, SCPB_ERR_UNSUPPORTED, "ptr_set_homotopy: the constraint pack of model %d does not read a homotopy "
                       "parameter at par[%d]", s->model_id, par_index);
    for (int i = 0; i < n_grid; i++)
        if (!std::isfinite(grid[i])) return set_err(h, SCPB_ERR_ARG, "ptr_set_homotopy: grid[%d] is not finite", i);
    if (std::isnan(worsen_tol)) return set_err(h, SCPB_ERR_ARG, "ptr_set_homotopy: worsen_tol is NaN");
    s->hom_slot = slot; s->hom_wtol = worsen_tol;
    s->hom_cap = s->d.iter_max + (n_grid - 1) * std::max(s->d.iter_max - 1, 0);
    if (s->hom_n == n_grid && std::equal(grid, grid + n_grid, s->hom_grid_h.begin())) return SCPB_OK;   // same grid
    SCPB_CUDA(h, cudaSetDevice(h->device));
    // the grid may still be read by a solve queued on the stream
    SCPB_CUDA(h, cudaStreamSynchronize(h->stream));
    if (s->hom_grid) cudaFree(s->hom_grid);
    s->hom_grid = nullptr; s->hom_n = 0; s->hom_cap = 0; s->hom_grid_h.clear();
    SCPB_CUDA(h, cudaMalloc((void **)&s->hom_grid, sizeof(double) * n_grid));
    SCPB_CUDA(h, cudaMemcpy(s->hom_grid, grid, sizeof(double) * n_grid, cudaMemcpyHostToDevice));
    s->hom_grid_h.assign(grid, grid + n_grid);
    s->hom_n = n_grid;
    s->hom_cap = s->d.iter_max + (n_grid - 1) * std::max(s->d.iter_max - 1, 0);
    return SCPB_OK;
}

int32_t scpb_ptr_set_homotopy_beta(scpb_ptr s, int32_t B, const double *beta)
{
    if (!s) return SCPB_ERR_ARG;
    if (B <= 0 || !beta) return set_err(s->h, SCPB_ERR_ARG, "ptr_set_homotopy_beta: bad arguments (B = %d)", B);
    for (int b = 0; b < B; b++)
        if (std::isnan(beta[b])) return set_err(s->h, SCPB_ERR_ARG, "ptr_set_homotopy_beta: beta[%d] is NaN", b);
    s->hom_beta_h.assign(beta, beta + B);
    return SCPB_OK;
}

int32_t scpb_ptr_homotopy_result(scpb_ptr s, int32_t B, int32_t *hom_index, int32_t *iter_max_eff, int32_t cap,
                                 int32_t *hist_index, double *hist_improv)
{
    if (!s) return SCPB_ERR_ARG;
    scpb_handle_s *h = s->h;
    if (s->last_cap == 0) return set_err(h, SCPB_ERR_STATE, "ptr_homotopy_result: the last solve had no schedule");
    if (B != s->last_B) return set_err(h, SCPB_ERR_ARG, "ptr_homotopy_result: the last solve had %d seeds, not %d", s->last_B, B);
    if (cap < 0 || ((hist_index || hist_improv) && cap == 0))
        return set_err(h, SCPB_ERR_ARG, "ptr_homotopy_result: cap = %d", cap);
    SCPB_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    if (hom_index) SCPB_CUDA(h, cudaMemcpyAsync(hom_index, s->hom_idx, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    if (iter_max_eff) SCPB_CUDA(h, cudaMemcpyAsync(iter_max_eff, s->hom_itmax, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    const int w = std::min(cap, s->last_cap);
    if (hist_index)
        SCPB_CUDA(h, cudaMemcpy2DAsync(hist_index, sizeof(int) * cap, s->hist_idx, sizeof(int) * s->last_cap, sizeof(int) * w,
                                       B, cudaMemcpyDeviceToHost, st));
    if (hist_improv)
        SCPB_CUDA(h, cudaMemcpy2DAsync(hist_improv, sizeof(double) * cap, s->hist_imp, sizeof(double) * s->last_cap,
                                       sizeof(double) * w, B, cudaMemcpyDeviceToHost, st));
    SCPB_CUDA(h, cudaStreamSynchronize(st));
    for (int b = 0; b < B; b++)
        for (int j = w; j < cap; j++) {
            if (hist_index) hist_index[(size_t)b * cap + j] = -1;
            if (hist_improv) hist_improv[(size_t)b * cap + j] = nan("");
        }
    return SCPB_OK;
}

int32_t scpb_ptr_free(scpb_ptr s)
{
    if (!s) return SCPB_ERR_ARG;
    cudaSetDevice(s->h->device);
    cudaStreamSynchronize(s->h->stream);
    for (void *q : s->dev) if (q) cudaFree(q);
    for (void *q : s->bb) if (q) cudaFree(q);
    for (cudaStream_t q : s->chunk_streams) if (q) cudaStreamDestroy(q);
    if (s->d_ipm_total) cudaFree(s->d_ipm_total);
    for (void *q : s->hb) if (q) cudaFree(q);
    if (s->hom_grid) cudaFree(s->hom_grid);
    if (s->d_chunk_done) cudaFree(s->d_chunk_done);
    if (s->h_chunk_done) cudaFreeHost(s->h_chunk_done);
    delete s;
    return SCPB_OK;
}

int32_t scpb_ptr_solve(scpb_ptr s, int32_t B, const double *xd0, const double *ud0, const double *p0,
                       const scpb_cone_opts *opts, double *xd, double *ud, double *p, int32_t *status,
                       int32_t *iters, double *J, double *deviation, int32_t *feas, double *timing)
{
    if (!s) return SCPB_ERR_ARG;
    Solve v;
    int rc = solve_begin(v, s, B, xd0, ud0, p0, opts, "ptr_solve");
    if (rc) return rc;
    scpb_handle_s *h = s->h;
    const scpb_ptr_desc &d = s->d;
    cudaStream_t st = v.st;
    const int G = v.G, Bpad = s->capB;
    IpmData *D = v.D;
    StepDev &sd = v.sd;
    if (D->warm) SCPB_CUDA(h, cudaMemsetAsync(D->warm, 0, sizeof(int) * s->capB, st));   // warm points of an earlier batch are not this batch's
    const bool hom = s->hom_n > 0;
    // a seed with a schedule can run iter_max + (n_grid - 1)(iter_max - 1) iterations (every update extends its
    // iter_max by the iterations since the previous one)
    const int it_bound = hom ? s->hom_cap : d.iter_max;
    s->last_B = B; s->last_cap = hom ? s->hom_cap : 0;
    if (hom) {
        v.pd.kappa = s->hom_kappa;
        sd.hom_n = s->hom_n; sd.hist_cap = s->hom_cap; sd.worsen_tol = s->hom_wtol;
        sd.hom_grid = s->hom_grid; sd.hom_beta = s->hom_beta;
        sd.hom_idx = s->hom_idx; sd.hom_last = s->hom_last; sd.hom_itmax = s->hom_itmax; sd.hom_kappa = s->hom_kappa;
        sd.hist_idx = s->hist_idx; sd.hist_imp = s->hist_imp;
        SCPB_CUDA(h, cudaMemcpyAsync(s->hom_beta, s->hom_beta_h.data(), sizeof(double) * B, cudaMemcpyHostToDevice, st));
        const long long n_init = (long long)B * s->hom_cap;
        k_hom_init<<<(unsigned)((n_init + 127) / 128), 128, 0, st>>>(sd, d.iter_max, B);
        h->launches++;
    }
    // interior-point warm start across PTR iterations: from iteration warm_from on, every seed starts the interior-point
    // method from the warm point its previous solve stored (the subproblems of consecutive PTR iterations differ little).
    // Built and correct, but not faster on the bench workload (the median iteration count of the later subproblems drops
    // from 37 to 28-33, the slowest seed of a launch needs more) -- opt-in with SCPB_WARM=1 (SCPB_NO_WARM=1 turns it off)
    const bool no_warm = getenv("SCPB_WARM") == nullptr || getenv("SCPB_NO_WARM") != nullptr;
    int warm_from = 5;   // SCPB_WARM_FROM
    if (const char *e = getenv("SCPB_WARM_FROM")) warm_from = atoi(e);
    IpmOpts o = v.o;
    scpb_internal_relax_refinement(o);
    v.opts_at = [=](int it) { IpmOpts ow = o; ow.warm = (it >= warm_from && !no_warm) ? 1 : 0; return ow; };
    v.step = [&](int, cudaStream_t ls, int nb) -> int {
        k_ptr_step<<<(nb + 127) / 128, 128, 0, ls>>>(sd);
        h->launches++;
        return SCPB_OK;
    };

    v.mark(-1, st);
    if ((rc = run_discretize(s, B, G, s->xd, s->ud, s->p))) return rc;   // generate_initial_guess -> discretize!
    v.mark(0, st);
    // ---- streamed chains: seeds are independent, so the batch is cut into chunks of whole seed groups and every
    // chunk runs ITS OWN sequence of iter_max PTR iterations on its own stream, with no host synchronisation in between: a
    // finished seed turns its share of every later kernel into a no-op (skip masks), a finished chunk costs a few empty
    // launches.  In lock-step every solver launch lasts as long as the slowest of ALL seeds (measured on the bench:
    // median 37, max 73 interior-point iterations in the later subproblems); streamed, a chunk only waits for its own seeds
    // and the batch takes max-over-chunks of the sums instead of the sum of the maxima.  SCPB_PTR_CHUNKS=<n> sets the
    // number of chunks; 0 or 1 (the default, SCPB_PTR_DEFAULT_CHUNKS = 0) runs the lock-step loop, which also serves the
    // SCPB_IPM_STATS diagnostic.
    int max_chunks = SCPB_PTR_DEFAULT_CHUNKS;
    if (const char *e = getenv("SCPB_PTR_CHUNKS")) max_chunks = atoi(e);
    const int ng_all = (B + G - 1) / G;
    if (max_chunks > 1 && ng_all >= 2 && !getenv("SCPB_IPM_STATS")) {
        const int cg = (ng_all + max_chunks - 1) / max_chunks;   // seed groups per chunk
        const int n_chunks = v.n_chunks = (ng_all + cg - 1) / cg;
        while ((int)s->chunk_streams.size() < n_chunks) {
            cudaStream_t q = nullptr;
            SCPB_CUDA(h, cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));
            s->chunk_streams.push_back(q);
        }
        if (!s->d_ipm_total) SCPB_CUDA(h, cudaMalloc((void **)&s->d_ipm_total, sizeof(unsigned long long)));
        SCPB_CUDA(h, cudaMemsetAsync(s->d_ipm_total, 0, sizeof(unsigned long long), st));
        sd.cone_iters = D->iters; sd.ipm_total = s->d_ipm_total;
        EventList sync_ev;   // fork / join events (no timing)
        auto sync_event = [&]() { cudaEvent_t e; cudaEventCreateWithFlags(&e, cudaEventDisableTiming); sync_ev.ev.push_back(e); return e; };
        cudaEvent_t e_fork = sync_event();
        SCPB_CUDA(h, cudaEventRecord(e_fork, st));
        for (int c = 0; c < n_chunks; c++) SCPB_CUDA(h, cudaStreamWaitEvent(s->chunk_streams[c], e_fork, 0));
        v.mark(-1, s->chunk_streams[0]);   // chunk 0 carries the phase timers: its own chain is one of the n_chunks concurrent critical paths
        // iteration `it` of chunk c's chain
        auto enqueue = [&](int c, int it) {
            const int b0 = c * cg * G;
            const int nbp = std::min(cg * G, Bpad - b0), nb = std::min(nbp, B - b0);
            sd.ndone = hom ? s->d_chunk_done + c : nullptr;
            return ptr_iteration(v, it, s->chunk_streams[c], b0, nb, nbp, c == 0, nullptr, nullptr);
        };
        auto chunk_seeds = [&](int c) { const int b0 = c * cg * G; return std::min(std::min(cg * G, Bpad - b0), B - b0); };
        if (!hom) {
            for (int it = 1; it <= it_bound; it++)
                for (int c = 0; c < n_chunks; c++)
                    if (chunk_seeds(c) > 0 && (rc = enqueue(c, it))) return rc;
        } else {
            // A schedule lets a seed run up to it_bound iterations, but most chains end far earlier.  Every chain keeps at
            // most LAG iterations queued: before iteration j it waits (without blocking the other chains) for the event
            // of iteration j - LAG and reads its chunk's count of finished seeds, copied to pinned memory after every
            // k_ptr_step.  The count only grows, so a stale value can only delay a chain's end by LAG empty iterations.
            constexpr int LAG = 3;
            if (s->chunk_cap < n_chunks) {
                if (s->d_chunk_done) cudaFree(s->d_chunk_done);
                if (s->h_chunk_done) cudaFreeHost(s->h_chunk_done);
                s->d_chunk_done = nullptr; s->h_chunk_done = nullptr; s->chunk_cap = 0;
                SCPB_CUDA(h, cudaMalloc((void **)&s->d_chunk_done, sizeof(int) * n_chunks));
                SCPB_CUDA(h, cudaMallocHost((void **)&s->h_chunk_done, sizeof(int) * n_chunks));
                s->chunk_cap = n_chunks;
            }
            SCPB_CUDA(h, cudaMemsetAsync(s->d_chunk_done, 0, sizeof(int) * n_chunks, st));
            for (int c = 0; c < n_chunks; c++) s->h_chunk_done[c] = 0;
            SCPB_CUDA(h, cudaEventRecord(e_fork, st));   // the chains also wait for the cleared counters
            for (int c = 0; c < n_chunks; c++) SCPB_CUDA(h, cudaStreamWaitEvent(s->chunk_streams[c], e_fork, 0));
            std::vector<cudaEvent_t> ring((size_t)n_chunks * LAG);
            for (cudaEvent_t &e : ring) e = sync_event();
            std::vector<int> next(n_chunks, 1), fin(n_chunks, 0);
            int live = 0;
            for (int c = 0; c < n_chunks; c++) { if (chunk_seeds(c) > 0) live++; else fin[c] = 1; }
            volatile int *seen = s->h_chunk_done;
            while (live > 0) {
                bool moved = false;
                for (int c = 0; c < n_chunks; c++) {
                    if (fin[c]) continue;
                    const int j = next[c];
                    cudaEvent_t &e = ring[(size_t)c * LAG + j % LAG];   // recorded after iteration j - LAG
                    if (j > it_bound) { fin[c] = 1; live--; continue; }
                    if (j > LAG) {
                        const cudaError_t q = cudaEventQuery(e);
                        if (q == cudaErrorNotReady) continue;
                        SCPB_CUDA(h, q);
                        if (seen[c] >= chunk_seeds(c)) { fin[c] = 1; live--; continue; }
                    }
                    if ((rc = enqueue(c, j))) return rc;
                    cudaStream_t cs = s->chunk_streams[c];
                    SCPB_CUDA(h, cudaMemcpyAsync(s->h_chunk_done + c, s->d_chunk_done + c, sizeof(int), cudaMemcpyDeviceToHost, cs));
                    SCPB_CUDA(h, cudaEventRecord(e, cs));
                    next[c] = j + 1;
                    moved = true;
                }
                if (!moved) std::this_thread::yield();
            }
        }
        for (int c = 0; c < n_chunks; c++) {   // join
            cudaEvent_t e = sync_event();
            SCPB_CUDA(h, cudaEventRecord(e, s->chunk_streams[c]));
            SCPB_CUDA(h, cudaStreamWaitEvent(st, e, 0));
        }
        v.mark(-1, st);
        unsigned long long tot_ipm = 0;
        SCPB_CUDA(h, cudaMemcpyAsync(&tot_ipm, s->d_ipm_total, sizeof tot_ipm, cudaMemcpyDeviceToHost, st));
        std::vector<int> hiters(B);
        SCPB_CUDA(h, cudaMemcpyAsync(hiters.data(), s->iters, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
        SCPB_CUDA(h, cudaStreamSynchronize(st));
        v.ipm_iters = (long long)tot_ipm;
        for (int b = 0; b < B; b++) v.total_it = std::max(v.total_it, hiters[b]);   // the longest chain
    } else if ((rc = lockstep_loop(v, it_bound))) {
        return rc;
    }
    return solve_end(v, xd, ud, p, status, iters, J, s->J_ref, deviation, feas, {}, timing, 10, "ptr_solve");
}

int32_t scpb_scvx_attach(scpb_ptr s, const scpb_scvx_desc *desc, const int32_t *Q_rowptr, const int32_t *Q_colind,
                         const double *Q_vals, const double *Q_const)
{
    if (!s) return SCPB_ERR_ARG;
    scpb_handle_s *h = s->h;
    if (!desc || !Q_rowptr || !Q_colind || !Q_vals || !Q_const) return set_err(h, SCPB_ERR_ARG, "scvx_attach: null pointer");
    const scpb_ptr_desc &d = s->d;
    if (s->hom_n > 0) return set_err(h, SCPB_ERR_UNSUPPORTED, "scvx_attach: the problem has an in-loop homotopy schedule (PTR only)");
    if (d.method != SCPB_FOH) return set_err(h, SCPB_ERR_UNSUPPORTED, "scvx_attach: SCvx runs with FOH discretization only");
    bool pack_ok = false;
    with_constr(s->model_id, d.ns > 0, [&](auto cp) { pack_ok = scvx_has_pack<decltype(cp)>; });
    if (!pack_ok)
        return set_err(h, SCPB_ERR_UNSUPPORTED, "scvx_attach: SCvx has no penalty for the constraint pack of model %d",
                       s->model_id);
    if (desc->oeta <= 0 || desc->oeta >= d.nsrc || desc->n_ic < 0 || desc->n_tc < 0)
        return set_err(h, SCPB_ERR_ARG, "scvx_attach: bad descriptor (oeta=%d)", desc->oeta);
    const int nq = 1 + desc->n_ic + desc->n_tc, nnz = Q_rowptr[nq];
    for (int k = 0; k < nnz; k++) {
        const int v = Q_colind[k];
        const bool ok = (v >= d.vx && v < d.vx + d.N * d.nx) || (v >= d.vu && v < d.vu + d.N * d.nu) ||
                        (v >= d.vp && v < d.vp + d.np);
        if (!ok) return set_err(h, SCPB_ERR_ARG, "scvx_attach: Q references solver variable %d outside x, u, p", v);
    }
    SCPB_CUDA(h, cudaSetDevice(h->device));
    s->sv = *desc;
    s->Q_rp = up(s, Q_rowptr, (size_t)nq + 1);
    s->Q_ci = up(s, Q_colind, (size_t)nnz);
    s->Q_v = up(s, Q_vals, (size_t)nnz);
    s->Q_c = up(s, Q_const, (size_t)nq);
    if (!s->Q_rp || !s->Q_ci || !s->Q_v || !s->Q_c) return set_err(h, SCPB_ERR_CUDA, "scvx_attach: device allocation failed");
    s->scvx = true;
    s->capB = 0;   // batch buffers are re-reserved with the SCvx extras
    return SCPB_OK;
}

int32_t scpb_scvx_solve(scpb_ptr s, int32_t B, const double *xd0, const double *ud0, const double *p0,
                        const scpb_cone_opts *opts, double *xd, double *ud, double *p, int32_t *status,
                        int32_t *iters, double *J, double *deviation, int32_t *feas, double *eta, double *timing)
{
    if (!s) return SCPB_ERR_ARG;
    if (!s->scvx) return set_err(s->h, SCPB_ERR_STATE, "scvx_solve: call scpb_scvx_attach first");
    Solve v;
    int rc = solve_begin(v, s, B, xd0, ud0, p0, opts, "scvx_solve");
    if (rc) return rc;
    scpb_handle_s *h = s->h;
    const scpb_ptr_desc &d = s->d;
    const scpb_scvx_desc &sv = s->sv;
    cudaStream_t st = v.st;
    k_fill<<<(s->capB + 127) / 128, 128, 0, st>>>(s->eta, sv.eta_init, s->capB);
    h->launches++;
    v.pd.eta = s->eta; v.pd.oeta = sv.oeta;
    const StepDev &sd = v.sd;
    ScvxDev cv{};
    cv.B = B; cv.N = d.N; cv.nx = d.nx; cv.nu = d.nu; cv.np = d.np; cv.n_ic = sv.n_ic; cv.n_tc = sv.n_tc;
    cv.vx = d.vx; cv.vu = d.vu; cv.vp = d.vp; cv.q_exit = d.q_exit; cv.iter_max = d.iter_max;
    cv.lam = sv.lam; cv.rho_0 = sv.rho_0; cv.rho_1 = sv.rho_1; cv.rho_2 = sv.rho_2; cv.beta_sh = sv.beta_sh; cv.beta_gr = sv.beta_gr;
    cv.eta_lb = sv.eta_lb; cv.eta_ub = sv.eta_ub; cv.eps_abs = d.eps_abs; cv.eps_rel = d.eps_rel;
    cv.Q_rp = s->Q_rp; cv.Q_ci = s->Q_ci; cv.Q_v = s->Q_v; cv.Q_c = s->Q_c;
    cv.Sx = sd.Sx; cv.cx = sd.cx; cv.Su = sd.Su; cv.cu = sd.cu; cv.Sp = sd.Sp; cv.cp = sd.cp; cv.t_grid = s->tgrid;
    cv.defect = s->defect; cv.par = s->par;
    cv.xd = s->xd; cv.ud = s->ud; cv.p = s->p; cv.xn = s->xn; cv.un = s->un; cv.pn = s->pn;
    cv.J_ref = s->J_ref; cv.J_new = s->J_new; cv.L_new = s->L_new; cv.J_out = s->J_out; cv.eta = s->eta; cv.dev = s->devi;
    cv.cone_status = v.D->status; cv.feas_new = s->feas;
    cv.done = s->done; cv.status = s->status; cv.iters = s->iters; cv.nactive = s->nactive; cv.accept = s->accept;
    // a pack without a penalty is refused, not run with its rows of J left unwritten (scpb_scvx_attach refuses it first)
    auto cost = [&](const double *X, const double *U, const double *P, double *Jd, double *Ld) -> int {
        bool launched = false;
        with_constr(s->model_id, d.ns > 0, [&](auto cp) {
            using CP = decltype(cp);
            if constexpr (scvx_has_pack<CP>) {
                k_scvx_cost<CP><<<(B + 63) / 64, 64, 0, st>>>(cv, X, U, P, Jd, Ld);
                h->launches++;
                launched = true;
            }
        });
        if (!launched)
            return set_err(h, SCPB_ERR_UNSUPPORTED, "scvx_solve: SCvx has no penalty for the constraint pack of model %d",
                           s->model_id);
        return SCPB_OK;
    };
    v.opts_at = [&](int) { return v.o; };
    v.cand_src = s->src2;
    v.candidate = [&]() { return cost(s->xn, s->un, s->pn, s->J_new, s->L_new); };
    v.step = [&](int it, cudaStream_t, int) -> int {
        cv.iter = it;
        k_scvx_step<<<(B + 127) / 128, 128, 0, st>>>(cv);
        take_dltv(v);
        h->launches += 2;
        return SCPB_OK;
    };

    v.mark(-1, st);
    // generate_initial_guess: SubproblemSolution(x, u, p, 0, pbm) = discretize! + nonlinear cost (scvx.jl:560-568, 392-394)
    if ((rc = run_discretize(s, B, v.G, s->xd, s->ud, s->p))) return rc;
    if ((rc = cost(s->xd, s->ud, s->p, s->J_ref, s->L_new))) return rc;
    v.mark(0, st);
    if ((rc = lockstep_loop(v, d.iter_max))) return rc;
    return solve_end(v, xd, ud, p, status, iters, J, s->J_out, deviation, feas, {{eta, s->eta}}, timing, 8, "scvx_solve");
}

int32_t scpb_gusto_attach(scpb_ptr s, const scpb_gusto_desc *desc, const int32_t *Q_rowptr, const int32_t *Q_colind,
                          const double *Q_vals, const double *Q_const, const double *Q_weight)
{
    if (!s) return SCPB_ERR_ARG;
    scpb_handle_s *h = s->h;
    if (!desc || !Q_rowptr || !Q_colind || !Q_vals || !Q_const || (desc->nsq > 0 && !Q_weight))
        return set_err(h, SCPB_ERR_ARG, "gusto_attach: null pointer");
    const scpb_ptr_desc &d = s->d;
    if (s->hom_n > 0) return set_err(h, SCPB_ERR_UNSUPPORTED, "gusto_attach: the problem has an in-loop homotopy schedule (PTR only)");
    if (d.method != SCPB_FOH) return set_err(h, SCPB_ERR_UNSUPPORTED, "gusto_attach: GuSTO runs with FOH discretization only");
    if (desc->oeta <= 0 || desc->oeta >= d.nsrc || desc->olam <= 0 || desc->olam >= d.nsrc || desc->olam == desc->oeta ||
        desc->nsq < 0 || desc->q_tr < 0 || desc->q_tr > 2)
        return set_err(h, SCPB_ERR_ARG, "gusto_attach: bad descriptor (oeta=%d, olam=%d, nsq=%d, q_tr=%d)", desc->oeta, desc->olam,
                       desc->nsq, desc->q_tr);
    if (s->scvx) return set_err(h, SCPB_ERR_STATE, "gusto_attach: the problem already carries the SCvx extras");
    const ConeSymbolic *S = scpb_internal_cone_sym(s->cone);
    const int nq = desc->nsq + 2, nnz = Q_rowptr[nq], nphys = Q_rowptr[desc->nsq + 1];
    for (int k = 0; k < nnz; k++) {
        const int v = Q_colind[k];
        const bool phys = (v >= d.vx && v < d.vx + d.N * d.nx) || (v >= d.vu && v < d.vu + d.N * d.nu) ||
                          (v >= d.vp && v < d.vp + d.np);
        if (k < nphys ? !phys : (v < 0 || v >= S->n))
            return set_err(h, SCPB_ERR_ARG, "gusto_attach: Q references solver variable %d outside its block", v);
    }
    SCPB_CUDA(h, cudaSetDevice(h->device));
    s->gv = *desc;
    s->Q_rp = up(s, Q_rowptr, (size_t)nq + 1);
    s->Q_ci = up(s, Q_colind, (size_t)nnz);
    s->Q_v = up(s, Q_vals, (size_t)nnz);
    s->Q_c = up(s, Q_const, (size_t)nq);
    s->Q_w = up(s, Q_weight, (size_t)desc->nsq);
    if (!s->Q_rp || !s->Q_ci || !s->Q_v || !s->Q_c || !s->Q_w) return set_err(h, SCPB_ERR_CUDA, "gusto_attach: device allocation failed");
    s->gusto = true;
    s->capB = 0;   // batch buffers are re-reserved with the GuSTO extras
    return SCPB_OK;
}

int32_t scpb_gusto_solve(scpb_ptr s, int32_t B, const double *xd0, const double *ud0, const double *p0,
                         const scpb_cone_opts *opts, double *xd, double *ud, double *p, int32_t *status,
                         int32_t *iters, double *J, double *deviation, int32_t *feas, double *eta, double *lam,
                         double *timing)
{
    if (!s) return SCPB_ERR_ARG;
    if (!s->gusto) return set_err(s->h, SCPB_ERR_STATE, "gusto_solve: call scpb_gusto_attach first");
    Solve v;
    int rc = solve_begin(v, s, B, xd0, ud0, p0, opts, "gusto_solve");
    if (rc) return rc;
    scpb_handle_s *h = s->h;
    const scpb_ptr_desc &d = s->d;
    const scpb_gusto_desc &g = s->gv;
    cudaStream_t st = v.st;
    k_fill<<<(s->capB + 127) / 128, 128, 0, st>>>(s->eta, g.eta_init, s->capB);
    k_fill<<<(s->capB + 127) / 128, 128, 0, st>>>(s->lam, g.lam_init, s->capB);
    h->launches += 2;
    v.pd.eta = s->eta; v.pd.oeta = g.oeta; v.pd.lam = s->lam; v.pd.olam = g.olam;
    const StepDev &sd = v.sd;   // its J_new = pobj + c0 is the subproblem's L_aug
    GustoDev gd{};
    gd.B = B; gd.G = v.G; gd.N = d.N; gd.nx = d.nx; gd.nu = d.nu; gd.np = d.np; gd.n = sd.n; gd.vx = d.vx; gd.vu = d.vu; gd.vp = d.vp;
    gd.q_exit = d.q_exit; gd.q_tr = g.q_tr; gd.iter_max = d.iter_max; gd.iter_mu = g.iter_mu; gd.nsq = g.nsq;
    gd.lam_init = g.lam_init; gd.lam_max = g.lam_max; gd.rho_0 = g.rho_0; gd.rho_1 = g.rho_1; gd.beta_sh = g.beta_sh;
    gd.beta_gr = g.beta_gr; gd.gamma_fail = g.gamma_fail; gd.eta_lb = g.eta_lb; gd.eta_ub = g.eta_ub; gd.mu = g.mu;
    gd.eps_abs = d.eps_abs; gd.eps_rel = d.eps_rel;
    gd.Q_rp = s->Q_rp; gd.Q_ci = s->Q_ci; gd.Q_v = s->Q_v; gd.Q_c = s->Q_c; gd.Q_w = s->Q_w;
    gd.Sx = sd.Sx; gd.cx = sd.cx; gd.Su = sd.Su; gd.cu = sd.cu; gd.Sp = sd.Sp; gd.cp = sd.cp; gd.t_grid = s->tgrid;
    gd.xsol = v.D->x; gd.par = s->par;
    gd.xd = s->xd; gd.ud = s->ud; gd.p = s->p; gd.xn = s->xn; gd.un = s->un; gd.pn = s->pn;
    gd.J_ref = s->J_ref; gd.L_aug = s->J_new; gd.J_out = s->J_out; gd.eta = s->eta; gd.lam = s->lam; gd.dev = s->devi;
    gd.nodeq = s->nodeq; gd.nodef = s->nodef;
    gd.cone_status = v.D->status; gd.feas_new = s->feas;
    gd.done = s->done; gd.status = s->status; gd.iters = s->iters; gd.nactive = s->nactive; gd.accept = s->accept;
    v.opts_at = [&](int) { return v.o; };
    v.cand_src = s->src2;
    v.step = [&](int it, cudaStream_t, int) -> int {
        gd.iter = it;
        if (launch_gusto_nodes(s, gd, st))
            return set_err(h, SCPB_ERR_UNSUPPORTED, "gusto_solve: no device pack for model %d", s->model_id);
        k_gusto_step<<<(B + 63) / 64, 64, 0, st>>>(gd);
        take_dltv(v);
        h->launches += 3;
        return SCPB_OK;
    };

    v.mark(-1, st);
    if ((rc = run_discretize(s, B, v.G, s->xd, s->ud, s->p))) return rc;   // generate_initial_guess -> discretize! (gusto.jl:517-526)
    v.mark(0, st);
    if ((rc = lockstep_loop(v, d.iter_max))) return rc;
    return solve_end(v, xd, ud, p, status, iters, J, s->J_out, deviation, feas, {{eta, s->eta}, {lam, s->lam}}, timing, 8,
                     "gusto_solve");
}

}  // extern "C"
