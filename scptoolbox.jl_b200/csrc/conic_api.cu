// conic_api.cu -- C ABI of the batched cone solver (scpb_cone_*), host orchestration.
#include <cstdlib>
#include "handle.cuh"
#include "conic_symbolic.h"
#define CONIC_IPM_IMPL
#include "conic_ipm.cuh"

#ifndef SCPB_HYBRID_DEFAULT_CUT
#define SCPB_HYBRID_DEFAULT_CUT 0   // hybrid program off unless SCPB_HYBRID=<cut> is set (see scpb_cone_setup)
#endif

struct scpb_cone_s {
    scpb_handle_s *h = nullptr;
    ConeSymbolic S;
    IpmProgram P{};
    IpmProgram P_hy{};    // hybrid program (scalar arrays replaced, top supernodes in .hy); valid when hy_ok
    bool hy_ok = false;
    int hy_used = 0;      // cut of the hybrid program the last launch ran (0: it ran another variant)
    std::vector<void *> dev_ints;
    // data buffers (grow-only), sized for (ngroups*G) seeds
    int capB = 0, capG = 0, lanes = 0;
    bool sn_ok = false;   // every supernodal panel fits the warp scratch
    std::vector<double *> bufs;
    IpmData D{};
    double *stage = nullptr;  // seed-major staging on device
    size_t stage_cap = 0;
    int *d_status = nullptr, *d_iters = nullptr, *d_warm = nullptr;
    double *d_scal = nullptr;  // pobj, dobj, res[3]
    long long *d_prof = nullptr;
    double *d_trace = nullptr;   // SCPB_IPM_TRACE diagnostic
    int trace_rows = 0;
};

static const int *upload_ints(scpb_cone_s *c, const std::vector<int> &v)
{
    void *d = nullptr;
    size_t bytes = sizeof(int) * (v.size() + 1);
    if (cudaMalloc(&d, bytes) != cudaSuccess) return nullptr;
    if (!v.empty()) cudaMemcpy(d, v.data(), sizeof(int) * v.size(), cudaMemcpyHostToDevice);
    c->dev_ints.push_back(d);
    return (const int *)d;
}

// seed-major [B][E] <-> group-blocked [(B/G)][E][G]; padded seeds replicate seed B-1
__global__ void k_to_grouped(const double *src, double *dst, int E, int B, int G, int Bpad)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)E * Bpad) return;
    const int sd = (int)(i % Bpad), e = (int)(i / Bpad);
    const int ssrc = sd < B ? sd : B - 1;
    dst[((size_t)(sd / G) * E + e) * G + (sd % G)] = src[(size_t)ssrc * E + e];
}
__global__ void k_from_grouped(const double *src, double *dst, int E, int B, int G)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)E * B) return;
    const int sd = (int)(i % B), e = (int)(i / B);
    dst[(size_t)sd * E + e] = src[((size_t)(sd / G) * E + e) * G + (sd % G)];
}

int scpb_internal_pick_group(int B, int want, int sms)
{
    if (want > 0) {
        int g = 1;
        while (g < want && g < IPM_MAXG) g <<= 1;
        return g;
    }
    int g = 1;
    while ((B + g - 1) / g > sms && g < IPM_MAXG) g <<= 1;   // one persistent CTA per SM
    return g;
}

static int cone_reserve(scpb_cone_s *c, int B, int G)
{
    scpb_handle_s *h = c->h;
    const int ng = (B + G - 1) / G, Bpad = ng * G;
    c->D.R = std::max(1, std::min(c->lanes > 0 ? c->lanes : 8, 32 / G));
    if (c->capB >= Bpad && c->capG == G) { c->D.B = B; c->D.G = G; return SCPB_OK; }
    // release the old set and forget it BEFORE allocating: if an allocation below fails, the problem is left with
    // capacity zero and null pointers (the next call re-reserves) instead of stale pointers to freed memory
    for (double *p : c->bufs) if (p) cudaFree(p);
    c->bufs.clear();
    if (c->d_status) cudaFree(c->d_status);
    if (c->d_iters) cudaFree(c->d_iters);
    if (c->d_scal) cudaFree(c->d_scal);
    if (c->d_warm) cudaFree(c->d_warm);
    c->d_status = nullptr; c->d_iters = nullptr; c->d_scal = nullptr; c->d_warm = nullptr;
    c->capB = 0; c->capG = 0;
    {
        IpmData z{};
        z.R = c->D.R; z.prof = c->D.prof;
        c->D = z;
    }
    const ConeSymbolic &S = c->S;
    auto al = [&](size_t E) -> double * {
        double *p = nullptr;
        if (cudaMalloc((void **)&p, sizeof(double) * (E + 1) * Bpad) != cudaSuccess) p = nullptr;
        c->bufs.push_back(p);
        return p;
    };
    IpmData &D = c->D;
    const size_t n = S.n, p = S.p, m = S.m, nk = S.nk, nm = std::max(S.n, S.m);
    double *Av = al(S.A_ci.size()), *Gv = al(S.G_ci.size()), *cc = al(n), *bb = al(p), *hh = al(m);
    D.Av = Av; D.Gv = Gv; D.c = cc; D.b = bb; D.h = hh;
    D.x = al(n); D.y = al(p); D.z = al(m); D.s = al(m);
    D.xb = al(n); D.yb = al(p); D.zb = al(m); D.sb = al(m);
    D.xw = al(n); D.yw = al(p); D.zw = al(m); D.sw = al(m);
    D.eqD = al(n); D.eqA = al(p); D.eqG = al(m);
    D.rx = al(n); D.ry = al(p); D.rz = al(m); D.lam = al(m); D.wm = al(S.nwm); D.socw = al(m - S.l + 1);
    D.soceta = al(S.nsoc + 1);
    D.dx = al(n); D.dy = al(p); D.dz = al(m); D.ds = al(m); D.dsa = al(m); D.dza = al(m); D.tm = al(m); D.gm = al(m);
    D.r1 = al(n); D.r2 = al(p); D.e1 = al(nm); D.e2 = al(p); D.rhs = al(nk);
    D.part = al(S.npart); D.pcnt = al(S.npart);
    D.Y = al(std::max<size_t>((size_t)S.nnzL + nk, (size_t)S.sn_panel_size)); D.Ls = al(S.nnzL + 1); D.Lrow = al(S.nnzL + 1); D.invD = al(nk);
    bool ok = true;
    for (double *q : c->bufs) ok = ok && q != nullptr;
    ok = ok && cudaMalloc((void **)&c->d_status, sizeof(int) * Bpad) == cudaSuccess &&
         cudaMalloc((void **)&c->d_iters, sizeof(int) * Bpad) == cudaSuccess &&
         cudaMalloc((void **)&c->d_scal, sizeof(double) * 5 * Bpad) == cudaSuccess &&
         cudaMalloc((void **)&c->d_warm, sizeof(int) * Bpad) == cudaSuccess &&
         cudaMemsetAsync(c->d_warm, 0, sizeof(int) * Bpad, h->stream) == cudaSuccess &&
         // split-target counters start at zero; on the handle's stream, which the solver launches (and the chunk
         // streams of ptr.cu) are ordered after
         cudaMemsetAsync(D.pcnt, 0, sizeof(double) * ((size_t)S.npart + 1) * Bpad, h->stream) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        for (double *q : c->bufs) if (q) cudaFree(q);
        c->bufs.clear();
        if (c->d_status) cudaFree(c->d_status);
        if (c->d_iters) cudaFree(c->d_iters);
        if (c->d_scal) cudaFree(c->d_scal);
        if (c->d_warm) cudaFree(c->d_warm);
        c->d_status = nullptr; c->d_iters = nullptr; c->d_scal = nullptr; c->d_warm = nullptr;
        IpmData z{};
        z.R = c->D.R; z.prof = c->D.prof;
        c->D = z;
        return set_err(h, SCPB_ERR_CUDA, "cone solver: device allocation failed (B=%d)", B);
    }
    D.status = c->d_status; D.iters = c->d_iters; D.warm = c->d_warm;
    D.pobj = c->d_scal; D.dobj = c->d_scal + Bpad; D.res = c->d_scal + 2 * (size_t)Bpad;
    if (!c->d_prof && cudaMalloc((void **)&c->d_prof, sizeof(long long) * (12 + 3 * (size_t)c->S.nlevels)) != cudaSuccess) c->d_prof = nullptr;
    D.prof = c->d_prof;
    c->capB = Bpad; c->capG = G;
    D.B = B; D.G = G;
    return SCPB_OK;
}

// run the solver on the data currently in the grouped buffers (device-resident entry, internal API)
// `st` (nullptr: the handle's stream) and the chunk [g0, g0 + ngc) of seed groups (ngc = 0: all groups) let the caller run
// independent chunks of a batch on different streams (ptr.cu)
int scpb_internal_cone_run(scpb_cone_s *c, const IpmOpts &o, const int *skip, cudaStream_t st, int g0, int ngc)
{
    c->D.skip = skip;
    scpb_handle_s *h = c->h;
    if (!st) st = h->stream;
    const int ng_all = (c->D.B + c->D.G - 1) / c->D.G;
    const int ng = ngc > 0 ? (g0 + ngc <= ng_all ? ngc : ng_all - g0) : ng_all;
    if (ng <= 0) return SCPB_OK;
    c->D.g0 = ngc > 0 ? g0 : 0;
    // dynamic shared memory: level pointers (+ the substitution vector when nk*G doubles fit next to the
    // ~20 KB of static shared memory; H100 allows 227 KB per CTA)
    size_t smem = sizeof(int) * ((9 * (size_t)(c->S.nlevels + 1) + 3) & ~(size_t)3);
    const size_t vbytes = sizeof(double) * (size_t)c->S.nk * c->D.G;
    c->D.vsmem = (smem + vbytes <= 200 * 1024 && !getenv("SCPB_NO_VSMEM")) ? 1 : 0;   // env: force the global-memory sweep (tests)
    if (c->D.vsmem) smem += vbytes;
    // supernodal factorisation / substitutions (csrc/conic_sn.cuh), SCPB_SUPERNODAL=1: every panel must fit a lane
    // group and the substitution vector must live in shared memory.  Correct on the device (tests/test_conic_gpu.py)
    // but slower than the scalar level-scheduled programs on the bench KKT, so the scalar programs stay the default.
    {
        const char *e = getenv("SCPB_SUPERNODAL");
        c->D.sn = (c->sn_ok && c->D.vsmem && e && e[0] == '1') ? 1 : 0;
    }
    // hybrid program (built at setup, SCPB_HYBRID): scalar programs below the cut, in-place panels above; needs the
    // shared-memory substitution vector like the supernodal variant
    const bool hy = c->hy_ok && c->D.vsmem && !c->D.sn;
    const IpmProgram &Pl = hy ? c->P_hy : c->P;
    // partial sums of the split targets of one level: the factorisation's slots share the window of the substitution
    // vector (it is free while the factorisation runs), the substitutions' slots and counters follow it; global memory
    // when that does not fit or the vector itself is not in shared memory
    {
        const size_t G = (size_t)c->D.G;
        const size_t win = sizeof(double) * std::max<size_t>((size_t)c->S.nk, (size_t)Pl.npf) * G;
        const size_t sbytes = (sizeof(double) + sizeof(unsigned)) * (size_t)Pl.nps * G;
        c->D.psmem = (c->D.vsmem && !c->D.sn && smem - vbytes + win + sbytes <= 200 * 1024 &&
                      !getenv("SCPB_GLOBAL_SLOTS")) ? 1 : 0;   // env: force the global slots (tests)
        if (c->D.psmem) smem += win - vbytes + sbytes;
    }
    c->hy_used = hy ? c->S.hy_cut : 0;
    c->D.lvl_prof = (c->d_prof && getenv("SCPB_LEVEL_PROFILE")) ? 1 : 0;   // diagnostic: per-level cycle counters of CTA 0
    if (hy && c->S.hy_nlevels + c->S.hy_ntl > c->S.nlevels) c->D.lvl_prof = 0;   // the counters are sized by the scalar levels
    c->D.trace = nullptr;
    if (const char *e = getenv("SCPB_IPM_TRACE")) {   // diagnostic: per-iteration residual trace of one seed (last launch)
        const int rows = o.maxit + 2;
        if (c->trace_rows < rows) {
            if (c->d_trace) cudaFree(c->d_trace);
            c->d_trace = nullptr; c->trace_rows = 0;
            if (cudaMalloc((void **)&c->d_trace, sizeof(double) * 10 * (size_t)rows) == cudaSuccess) c->trace_rows = rows;
        }
        if (c->d_trace) {
            cudaMemsetAsync(c->d_trace, 0, sizeof(double) * 10 * (size_t)c->trace_rows, st);
            c->D.trace = c->d_trace; c->D.trace_seed = atoi(e);
        }
    }
#define SCPB_LAUNCH_IPM(NT_, SN_)                                                                                        \
    {                                                                                                                    \
        SCPB_CUDA(h, cudaFuncSetAttribute(k_ipm_solve<NT_, SN_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_ipm_solve<NT_, SN_><<<ng, NT_, smem, st>>>(Pl, c->D, o);                                                       \
    }
    if (o.threads >= 1024) { if (c->D.sn) SCPB_LAUNCH_IPM(1024, 1) else if (hy) SCPB_LAUNCH_IPM(1024, 2) else SCPB_LAUNCH_IPM(1024, 0) }
    else { if (c->D.sn) SCPB_LAUNCH_IPM(512, 1) else if (hy) SCPB_LAUNCH_IPM(512, 2) else SCPB_LAUNCH_IPM(512, 0) }
#undef SCPB_LAUNCH_IPM
    h->launches++;
    SCPB_CUDA(h, cudaGetLastError());
    return SCPB_OK;
}

IpmOpts scpb_internal_make_opts(const scpb_cone_opts *o)
{
    IpmOpts r;
    r.feastol = (o && o->feastol > 0) ? o->feastol : 1e-8;
    r.abstol = (o && o->abstol > 0) ? o->abstol : 1e-8;
    r.reltol = (o && o->reltol > 0) ? o->reltol : 1e-8;
    r.delta = (o && o->delta > 0) ? o->delta : 1e-12;
    r.delta_max = (o && o->delta_dyn > 0) ? o->delta_dyn : 1e-6;
    if (r.delta_max < r.delta) r.delta_max = r.delta;
    r.delta_esc = 1e3;
    r.rho_min = 1e-9;
    r.bad_abs = 1e-6;
    r.maxit = (o && o->maxit > 0) ? o->maxit : 100;
    r.nref = (o && o->nref >= 0) ? o->nref : 3;
    r.equil = (o && o->equil >= 0) ? o->equil : 5;
    r.threads = (o && o->threads > 0) ? o->threads : 1024;
    r.nref_aff = 0;
    r.warm = 0;              // set per launch by the SCP loops (ptr.cu) from their second iteration on
    r.mu_warm = 1e-2;
    if (const char *e = getenv("SCPB_WARM_MU")) { const double v = atof(e); if (v > 0) r.mu_warm = v; }   // experiments
    // iterative refinement stops at |residual| <= reftol (1 + |rhs|).  1e-13 is the library default (cone solves, SCvx,
    // GuSTO); the PTR loop relaxes it while an iterate is far from the end of the path (scpb_internal_relax_refinement)
    r.reftol = 1e-13;
    r.mu_tight = 0.0;
    if (const char *e = getenv("SCPB_REFTOL")) { const double v = atof(e); if (v > 0) r.reftol = v; }   // experiments
    return r;
}

// PTR loop: early interior-point iterations only need a direction, so refinement stops two digits below the requested
// feasibility (inside [1e-13, 1e-11]) while gap/deg > 1e-6 and at 1e-13 below that -- on the bench seeds 2.06 instead of
// 2.19 LDL' solves per interior-point iteration with the same iteration counts.  With 1e-11 all the way one of the
// N = 31 starship test programs stalled at a relative gap of 1e-6, hence the switch.
void scpb_internal_relax_refinement(IpmOpts &r)
{
    if (getenv("SCPB_REFTOL")) return;
    r.reftol = fmin(1e-11, fmax(1e-13, 1e-2 * r.feastol));
    r.mu_tight = 1e-6;
    if (const char *e = getenv("SCPB_MU_TIGHT")) { const double v = atof(e); if (v >= 0) r.mu_tight = v; }   // experiments
}

int scpb_internal_cone_reserve(scpb_cone_s *c, int B, int G, int lanes) { c->lanes = lanes; return cone_reserve(c, B, G); }
IpmData *scpb_internal_cone_data(scpb_cone_s *c) { return &c->D; }
const ConeSymbolic *scpb_internal_cone_sym(scpb_cone_s *c) { return &c->S; }
scpb_handle_s *scpb_internal_cone_handle(scpb_cone_s *c) { return c->h; }

extern "C" {

int32_t scpb_cone_setup(scpb_handle h, int32_t n, int32_t p, int32_t m, const int32_t *A_rowptr,
                        const int32_t *A_colind, const int32_t *G_rowptr, const int32_t *G_colind, int32_t l,
                        int32_t nsoc, const int32_t *soc_dims, const int32_t *perm, scpb_cone *out)
{
    if (!h || !out) return SCPB_ERR_ARG;
    *out = nullptr;
    if (n <= 0 || p < 0 || m < 0 || !A_rowptr || !G_rowptr || l < 0 || nsoc < 0 || (nsoc > 0 && !soc_dims))
        return set_err(h, SCPB_ERR_ARG, "cone_setup: bad arguments");
    SCPB_CUDA(h, cudaSetDevice(h->device));
    scpb_cone_s *c = new (std::nothrow) scpb_cone_s();
    if (!c) return set_err(h, SCPB_ERR_CUDA, "out of host memory");
    c->h = h;
    static const int zero = 0;
    if (!cone_symbolic_build(c->S, n, p, m, A_rowptr, A_colind ? A_colind : &zero, G_rowptr,
                             G_colind ? G_colind : &zero, l, nsoc, soc_dims, perm)) {
        int rc = set_err(h, SCPB_ERR_ARG, "cone_setup: %s", c->S.err.c_str());
        delete c;
        return rc;
    }
    const ConeSymbolic &S = c->S;
    IpmProgram &P = c->P;
    P.n = n; P.p = p; P.m = m; P.l = l; P.nsoc = nsoc; P.nk = S.nk; P.nnzL = S.nnzL; P.nlevels = S.nlevels;
    P.nwm = S.nwm; P.nnzA = (int)S.A_ci.size(); P.nnzG = (int)S.G_ci.size();
#define UP(f) P.f = upload_ints(c, S.f)
    UP(soc_dim); UP(soc_off); UP(soc_woff); UP(A_rp); UP(A_ci); UP(G_rp); UP(G_ci);
    UP(At_rp); UP(At_ri); UP(At_vi); UP(Gt_rp); UP(Gt_ri); UP(Gt_vi); UP(iperm);
    UP(L_cp); UP(L_ri); UP(Lr_rp); UP(Lr_pos); UP(Lr_col); UP(lvl_ptr); UP(lvl_nodes);
    UP(as_ptr); UP(as_a); UP(as_b); UP(as_c); UP(as_src); UP(as_sign);
#undef UP
    P.fw_item = (const int4 *)upload_ints(c, S.fw_item); P.bw_item = (const int4 *)upload_ints(c, S.bw_item);
    P.fa_item = (const int4 *)upload_ints(c, S.fa_item); P.fb_item = (const int4 *)upload_ints(c, S.fb_item);
    P.ysize = (int)std::max<long long>((long long)S.nnzL + S.nk, S.sn_panel_size);
    P.sn.first = upload_ints(c, S.sn_first); P.sn.width = upload_ints(c, S.sn_width); P.sn.nrows = upload_ints(c, S.sn_nrows);
    P.sn.rows_ptr = upload_ints(c, S.sn_rows_ptr); P.sn.rows = upload_ints(c, S.sn_rows);
    P.sn.lvl_ptr = upload_ints(c, S.sn_lvl_ptr); P.sn.lvl_nodes = upload_ints(c, S.sn_lvl_nodes);
    P.sn.upd_xy = upload_ints(c, S.sn_upd_xy); P.sn.sign = upload_ints(c, S.sn_sign);
    P.sn.panel_off = upload_ints(c, S.sn_panel_off); P.sn.upd_ptr = upload_ints(c, S.sn_upd_ptr);
    P.sn.upd_dst = upload_ints(c, S.sn_upd_dst); P.sn.nlevels = S.sn_nlevels;
    P.sn_pos = upload_ints(c, S.sn_pos_of_target);
    P.sn.cls_ptr = upload_ints(c, S.sn_cls_ptr);
    {
        std::vector<int> desc(8 * S.sn_first.size() + 8, 0);   // in level order: item i of lvl_nodes
        for (size_t i = 0; i < S.sn_lvl_nodes.size(); i++) {
            const int q = S.sn_lvl_nodes[i];
            desc[8 * i] = S.sn_first[q]; desc[8 * i + 1] = S.sn_width[q]; desc[8 * i + 2] = S.sn_nrows[q];
            desc[8 * i + 3] = S.sn_panel_off[q]; desc[8 * i + 4] = S.sn_rows_ptr[q]; desc[8 * i + 5] = S.sn_upd_ptr[q];
        }
        P.sn.desc = (const int4 *)upload_ints(c, desc);
    }
    c->sn_ok = S.sn_fits;
    P.fa_lvl = upload_ints(c, S.fa_lvl); P.fa_R = upload_ints(c, S.fa_R); P.fb_lvl = upload_ints(c, S.fb_lvl);
    P.fwp_item = (const int4 *)upload_ints(c, S.fwp_item); P.bwp_item = (const int4 *)upload_ints(c, S.bwp_item);
    P.fwp_lvl = upload_ints(c, S.fwp_lvl); P.bwp_lvl = upload_ints(c, S.bwp_lvl);
    P.fwp_R = upload_ints(c, S.fwp_R); P.bwp_R = upload_ints(c, S.bwp_R);
    P.Lr_pc = (const int2 *)upload_ints(c, S.Lr_pc); P.ft_op = (const int2 *)upload_ints(c, S.ft_op);
    P.fwc_item = (const int4 *)upload_ints(c, S.fwc_item);
    P.bwc_item = (const int4 *)upload_ints(c, S.bwc_item);
    P.fb_cmb = (const int4 *)upload_ints(c, S.fb_cmb);
    P.npf = S.fslots; P.nps = S.sslots;
    // hybrid program: SCPB_HYBRID=<cut> (supernodal level at which the in-place panels take over; 0 = off)
    {
        const char *e = getenv("SCPB_HYBRID");
        const int cut = e ? atoi(e) : SCPB_HYBRID_DEFAULT_CUT;
        if (cut > 0 && cone_symbolic_build_hybrid(c->S, cut)) {
            IpmProgram &H = c->P_hy;
            H = P;
            H.nlevels = S.hy_nlevels;
            H.fa_item = (const int4 *)upload_ints(c, S.hy_fa_item); H.fb_item = (const int4 *)upload_ints(c, S.hy_fb_item);
            H.fa_lvl = upload_ints(c, S.hy_fa_lvl); H.fa_R = upload_ints(c, S.hy_fa_R); H.fb_lvl = upload_ints(c, S.hy_fb_lvl);
            H.ft_op = (const int2 *)upload_ints(c, S.hy_ft_op);
            H.fwp_item = (const int4 *)upload_ints(c, S.hy_fwp_item); H.bwp_item = (const int4 *)upload_ints(c, S.hy_bwp_item);
            H.fwp_lvl = upload_ints(c, S.hy_fwp_lvl); H.bwp_lvl = upload_ints(c, S.hy_bwp_lvl);
            H.fwp_R = upload_ints(c, S.hy_fwp_R); H.bwp_R = upload_ints(c, S.hy_bwp_R);
            H.fwc_item = (const int4 *)upload_ints(c, S.hy_fwc_item);
            H.bwc_item = (const int4 *)upload_ints(c, S.hy_bwc_item);
            H.fb_cmb = (const int4 *)upload_ints(c, S.hy_fb_cmb);
            H.npf = S.hy_fslots; H.nps = S.hy_sslots;
            H.hy.desc = (const int4 *)upload_ints(c, S.hy_desc); H.hy.tl_ptr = upload_ints(c, S.hy_tl_ptr);
            H.hy.upd_dst = upload_ints(c, S.hy_upd_dst); H.hy.rows = P.sn.rows; H.hy.ntl = S.hy_ntl;
            c->hy_ok = true;
        }
    }
    P.npart = S.npart;   // the hybrid program's slots are counted in S.npart too
    c->P_hy.npart = S.npart;
    for (void *d : c->dev_ints)
        if (!d) {
            scpb_cone_free(c);
            return set_err(h, SCPB_ERR_CUDA, "cone_setup: device allocation failed");
        }
    *out = c;
    return SCPB_OK;
}

int32_t scpb_cone_info(scpb_cone c, int64_t *info)
{
    if (!c || !info) return SCPB_ERR_ARG;
    info[0] = c->S.nk; info[1] = c->S.nnzL; info[2] = c->S.nlevels; info[3] = c->S.factor_ops;
    info[4] = (int64_t)c->S.as_a.size(); info[5] = c->S.nwm; info[6] = c->capG; info[7] = c->capB;
    info[20] = c->hy_used; info[21] = c->hy_ok ? c->S.hy_nlevels : 0; info[22] = c->hy_ok ? c->S.hy_ntl : 0; info[23] = c->hy_ok ? c->S.hy_cut : 0;
    if (c->d_prof) {   // info[8..15]: cycle counters of the last launch (CTA 0)
        long long hp[12];
        if (cudaMemcpy(hp, c->d_prof, sizeof hp, cudaMemcpyDeviceToHost) == cudaSuccess)
            for (int i = 0; i < 12; i++) info[8 + i] = hp[i];
    }
    return SCPB_OK;
}

int32_t scpb_debug_level_profile(scpb_cone c, int64_t *out, int32_t cap)
{
    if (!c || !out) return SCPB_ERR_ARG;
    const int nl = c->S.nlevels;
    if (cap < 3 * nl || !c->d_prof) return SCPB_ERR_ARG;
    std::vector<long long> hp(3 * (size_t)nl);
    if (cudaMemcpy(hp.data(), c->d_prof + 12, sizeof(long long) * hp.size(), cudaMemcpyDeviceToHost) != cudaSuccess)
        return SCPB_ERR_CUDA;
    for (size_t i = 0; i < hp.size(); i++) out[i] = hp[i];
    return SCPB_OK;
}

int32_t scpb_debug_ipm_trace(scpb_cone c, double *out, int32_t cap_rows)
{
    if (!c || !out || cap_rows <= 0) return SCPB_ERR_ARG;
    if (!c->d_trace) return SCPB_ERR_STATE;
    const int rows = cap_rows < c->trace_rows ? cap_rows : c->trace_rows;
    cudaStreamSynchronize(c->h->stream);
    if (cudaMemcpy(out, c->d_trace, sizeof(double) * 10 * (size_t)rows, cudaMemcpyDeviceToHost) != cudaSuccess) return SCPB_ERR_CUDA;
    return rows;
}

/* test hook: one assemble + factor + solve of the reduced KKT system ON THE DEVICE (the code path of k_ipm_solve,
 * supernodal or scalar by SCPB_SUPERNODAL) for B seeds; rhs / sol in natural node order [B][n+p]; wm[B][nwm] is W^-2
 * (LP rows: one weight; SOC: dense q x q blocks); bad[B] = 1 when the factorisation flagged lost inertia. */
int32_t scpb_debug_kkt_solve_dev(scpb_cone c, int32_t B, const double *Avals, const double *Gvals, const double *wm,
                                 double delta, const double *rhs, double *sol, int32_t *bad)
{
    if (!c || B <= 0 || !wm || !rhs || !sol) return SCPB_ERR_ARG;
    scpb_handle_s *h = c->h;
    SCPB_CUDA(h, cudaSetDevice(h->device));
    const int G = scpb_internal_pick_group(B, 0, h->sms);
    int rc = cone_reserve(c, B, G);
    if (rc) return rc;
    const ConeSymbolic &S = c->S;
    const int Bpad = c->capB, nk = S.nk;
    const size_t maxE = std::max<size_t>({S.A_ci.size(), S.G_ci.size(), (size_t)S.nwm, (size_t)nk, 1});
    if (c->stage_cap < maxE * B) {
        if (c->stage) cudaFree(c->stage);
        c->stage = nullptr; c->stage_cap = 0;
        SCPB_CUDA(h, cudaMalloc((void **)&c->stage, sizeof(double) * maxE * B));
        c->stage_cap = maxE * B;
    }
    cudaStream_t st = h->stream;
    auto put = [&](const double *src, double *dst, size_t E) -> int {
        if (E == 0) return SCPB_OK;
        if (!src) { SCPB_CUDA(h, cudaMemsetAsync(dst, 0, sizeof(double) * E * Bpad, st)); return SCPB_OK; }
        SCPB_CUDA(h, cudaMemcpyAsync(c->stage, src, sizeof(double) * E * B, cudaMemcpyHostToDevice, st));
        const long long tot = (long long)E * Bpad;
        k_to_grouped<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(c->stage, dst, (int)E, B, G, Bpad);
        SCPB_CUDA(h, cudaStreamSynchronize(st));   // the staging buffer is reused by the next array
        return SCPB_OK;
    };
    std::vector<double> rp((size_t)B * nk);
    for (int b = 0; b < B; b++)
        for (int i = 0; i < nk; i++) rp[(size_t)b * nk + S.iperm[i]] = rhs[(size_t)b * nk + i];
    if ((rc = put(Avals, c->D.Av, S.A_ci.size())) || (rc = put(Gvals, c->D.Gv, S.G_ci.size())) ||
        (rc = put(wm, c->D.wm, (size_t)S.nwm)) || (rc = put(rp.data(), c->D.rhs, (size_t)nk)))
        return rc;
    scpb_cone_opts oo{};
    oo.delta = delta;
    IpmOpts o = scpb_internal_make_opts(&oo);
    c->D.debug_kkt = 1;
    rc = scpb_internal_cone_run(c, o, nullptr, nullptr, 0, 0);
    c->D.debug_kkt = 0;
    if (rc) return rc;
    k_from_grouped<<<(unsigned)(((long long)nk * B + 255) / 256), 256, 0, st>>>(c->D.rhs, c->stage, nk, B, G);
    SCPB_CUDA(h, cudaMemcpyAsync(rp.data(), c->stage, sizeof(double) * nk * B, cudaMemcpyDeviceToHost, st));
    std::vector<int> hb(B, 0);
    SCPB_CUDA(h, cudaMemcpyAsync(hb.data(), c->D.status, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    SCPB_CUDA(h, cudaStreamSynchronize(st));
    for (int b = 0; b < B; b++) {
        for (int i = 0; i < nk; i++) sol[(size_t)b * nk + i] = rp[(size_t)b * nk + S.iperm[i]];
        if (bad) bad[b] = hb[b];
    }
    return SCPB_OK;
}

int32_t scpb_cone_free(scpb_cone c)
{
    if (!c) return SCPB_ERR_ARG;
    cudaSetDevice(c->h->device);
    cudaStreamSynchronize(c->h->stream);
    for (void *d : c->dev_ints)
        if (d) cudaFree(d);
    for (double *p : c->bufs)
        if (p) cudaFree(p);
    if (c->stage) cudaFree(c->stage);
    if (c->d_status) cudaFree(c->d_status);
    if (c->d_iters) cudaFree(c->d_iters);
    if (c->d_warm) cudaFree(c->d_warm);
    if (c->d_scal) cudaFree(c->d_scal);
    if (c->d_prof) cudaFree(c->d_prof);
    if (c->d_trace) cudaFree(c->d_trace);
    delete c;
    return SCPB_OK;
}

int32_t scpb_cone_solve(scpb_cone c, int32_t B, const double *Avals, const double *Gvals, const double *cvec,
                        const double *bvec, const double *hvec, const scpb_cone_opts *opts, double *x, double *y,
                        double *z, double *s, double *pobj, double *dobj, int32_t *status, int32_t *iters,
                        double *seconds)
{
    if (!c) return SCPB_ERR_ARG;
    scpb_handle_s *h = c->h;
    if (B <= 0 || !cvec || (c->S.p > 0 && !bvec) || (c->S.m > 0 && !hvec)) return set_err(h, SCPB_ERR_ARG, "cone_solve: bad arguments");
    SCPB_CUDA(h, cudaSetDevice(h->device));
    const int G = scpb_internal_pick_group(B, opts ? opts->group : 0, h->sms);
    c->lanes = opts ? opts->lanes : 0;
    int rc = cone_reserve(c, B, G);
    if (rc) return rc;
    const ConeSymbolic &S = c->S;
    const int Bpad = c->capB;
    const size_t maxE = std::max<size_t>({S.A_ci.size(), S.G_ci.size(), (size_t)S.n, (size_t)S.m, (size_t)S.p, 1});
    if (c->stage_cap < maxE * B) {
        if (c->stage) cudaFree(c->stage);
        c->stage = nullptr; c->stage_cap = 0;
        SCPB_CUDA(h, cudaMalloc((void **)&c->stage, sizeof(double) * maxE * B));
        c->stage_cap = maxE * B;
    }
    cudaStream_t st = h->stream;
    auto put = [&](const double *src, const double *dstc, size_t E) -> int {
        if (E == 0) return SCPB_OK;
        double *dst = const_cast<double *>(dstc);
        if (!src) { SCPB_CUDA(h, cudaMemsetAsync(dst, 0, sizeof(double) * E * Bpad, st)); return SCPB_OK; }
        SCPB_CUDA(h, cudaMemcpyAsync(c->stage, src, sizeof(double) * E * B, cudaMemcpyHostToDevice, st));
        const long long tot = (long long)E * Bpad;
        k_to_grouped<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(c->stage, dst, (int)E, B, G, Bpad);
        h->launches++;
        return SCPB_OK;
    };
    if ((rc = put(Avals, c->D.Av, S.A_ci.size())) || (rc = put(Gvals, c->D.Gv, S.G_ci.size())) ||
        (rc = put(cvec, c->D.c, S.n)) || (rc = put(bvec, c->D.b, S.p)) || (rc = put(hvec, c->D.h, S.m)))
        return rc;
    IpmOpts o = scpb_internal_make_opts(opts);
    SCPB_CUDA(h, cudaEventRecord(h->ev0, st));
    rc = scpb_internal_cone_run(c, o, nullptr, nullptr, 0, 0);
    if (rc) return rc;
    SCPB_CUDA(h, cudaEventRecord(h->ev1, st));
    auto get = [&](double *dst, const double *src, size_t E) -> int {
        if (!dst || E == 0) return SCPB_OK;
        const long long tot = (long long)E * B;
        k_from_grouped<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(src, c->stage, (int)E, B, G);
        h->launches++;
        SCPB_CUDA(h, cudaMemcpyAsync(dst, c->stage, sizeof(double) * E * B, cudaMemcpyDeviceToHost, st));
        return SCPB_OK;
    };
    if ((rc = get(x, c->D.x, S.n)) || (rc = get(y, c->D.y, S.p)) || (rc = get(z, c->D.z, S.m)) ||
        (rc = get(s, c->D.s, S.m)))
        return rc;
    if (pobj) SCPB_CUDA(h, cudaMemcpyAsync(pobj, c->D.pobj, sizeof(double) * B, cudaMemcpyDeviceToHost, st));
    if (dobj) SCPB_CUDA(h, cudaMemcpyAsync(dobj, c->D.dobj, sizeof(double) * B, cudaMemcpyDeviceToHost, st));
    if (status) SCPB_CUDA(h, cudaMemcpyAsync(status, c->D.status, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    if (iters) SCPB_CUDA(h, cudaMemcpyAsync(iters, c->D.iters, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    SCPB_CUDA(h, cudaStreamSynchronize(st));
    if (seconds) {
        float ms = 0.f;
        SCPB_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
        *seconds = ms * 1e-3;
    }
    return SCPB_OK;
}

}  // extern "C"
