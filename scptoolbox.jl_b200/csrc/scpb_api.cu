// scpb_api.cu -- C ABI entry points (include/scpb.h): lifetime, model selection, discretize.
#include <cstdlib>
#include "handle.cuh"
#include "discretize.cuh"
#include "propagate.cuh"

#ifndef SCPB_K1_DEFAULT_MB
#define SCPB_K1_DEFAULT_MB 2   // resident K1 blocks per SM the register allocation targets (SCPB_K1_MB overrides: 2, 3, 4);
                               // 2 has the least spill code (sm_90a, starship pack: 44 bytes, against 0.6 and 0.8 KB at 3 and 4)
                               // and K1 is a small share of a PTR step
#endif

static int check_model(scpb_handle_s *h)
{
    if (!h) return SCPB_ERR_ARG;
    if (h->model_id == 0) return set_err(h, SCPB_ERR_STATE, "no model set (call scpb_model_set first)");
    return SCPB_OK;
}

template <class M>
static int launch_disc(scpb_handle_s *h, DiscArgs &a, int method, cudaStream_t st)
{
    constexpr int QSZ = (M::NU + M::NF + 1) * M::NX;
    const int wpb = 4;
    const long long warps = (long long)(a.nb > 0 ? a.nb : a.B) * (a.N - 1);
    const int blocks = (int)((warps + wpb - 1) / wpb);
    const size_t smem = sizeof(double) * QSZ * wpb;
    if (method == SCPB_IMPULSE) {
        if constexpr (M::IMPULSE) k_discretize_foh<M, 1><<<blocks, wpb * 32, smem, st>>>(a);
        else return set_err(h, SCPB_ERR_UNSUPPORTED, "model %d has no impulse semantics (IMPULSE discretization)", h->model_id);
    } else {
        static const int mb = [] { const char *e = getenv("SCPB_K1_MB"); return e ? atoi(e) : SCPB_K1_DEFAULT_MB; }();
        if (mb == 3) k_discretize_foh<M, 0, 3><<<blocks, wpb * 32, smem, st>>>(a);
        else if (mb == 4) k_discretize_foh<M, 0, 4><<<blocks, wpb * 32, smem, st>>>(a);
        else k_discretize_foh<M, 0, 2><<<blocks, wpb * 32, smem, st>>>(a);
    }
    h->launches++;
    return SCPB_OK;
}

// Launch K1 (+ the feasibility reduction when feas != nullptr). All pointers are device pointers.
// `st`: stream to launch on (nullptr: the handle's); a.b0 / a.nb select a chunk of seeds (ptr.cu runs the SCP chains of
// different seed chunks on different streams)
int scpb_internal_discretize(scpb_handle_s *h, DiscArgs &a, double feas_tol, int *feas, int method, cudaStream_t st)
{
    if (!st) st = h->stream;
    int rc = check_model(h);
    if (rc) return rc;
    if (method != SCPB_FOH && method != SCPB_IMPULSE) return set_err(h, SCPB_ERR_ARG, "unknown discretization method %d", method);
    if (a.B <= 0 || a.N < 2 || a.Nsub < 2) return set_err(h, SCPB_ERR_ARG, "bad sizes B=%d N=%d Nsub=%d", a.B, a.N, a.Nsub);
    a.par = h->par;
    a.np = h->np;
    a.status = h->d_status;
    double *dn = (double *)h->scratch(0, sizeof(double) * (size_t)a.B * (a.N - 1));
    if (!dn) return set_err(h, SCPB_ERR_CUDA, "scratch allocation failed");
    a.dnorm = dn;
    if (!with_model(h->model_id, [&](auto m) { rc = launch_disc<decltype(m)>(h, a, method, st); }))
        return set_err(h, SCPB_ERR_MODEL, "unknown model id %d", h->model_id);
    if (rc) return rc;
    if (feas) {
        const int cnt = a.nb > 0 ? a.nb : a.B;
        k_feas_reduce<<<(cnt + 127) / 128, 128, 0, st>>>(dn, a.B, a.N - 1, feas_tol, feas, a.skip, a.b0, a.nb);
        h->launches++;
    }
    SCPB_CUDA(h, cudaGetLastError());
    return SCPB_OK;
}

static void julia_views(DiscArgs &a, int nx, int nu, int np, double *A, double *Bm, double *Bp, double *F,
                        double *r, double *E, double *defect)
{
    const long long M = a.N - 1;
    auto jl = [&](double *ptr, long long sz) { OutView v{}; v.ptr = ptr; v.sB = 0; v.sK = sz; v.sE = 1; v.sGrp = M * sz; v.Gq = 1; return v; };
    a.A = jl(A, (long long)nx * nx);
    a.Bm = jl(Bm, (long long)nx * nu);
    a.Bp = jl(Bp, (long long)nx * nu);
    a.F = jl(F, (long long)nx * np);
    a.r = jl(r, nx);
    a.E = jl(E, (long long)nx * nx);
    a.defect = jl(defect, nx);
    a.f_packed = 0;
    a.xsB = (long long)a.N * nx; a.xsK = nx; a.xsE = 1;
    a.usB = (long long)a.N * nu; a.usK = nu; a.usE = 1;
    a.psB = np; a.psE = 1;
}

extern "C" {

int32_t scpb_version(void) { return 103; }

int32_t scpb_create(int32_t device, scpb_handle *out)
{
    if (!out) return SCPB_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SCPB_ERR_CUDA;
    if (device < 0 || device >= ndev) return SCPB_ERR_ARG;
    if (cudaSetDevice(device) != cudaSuccess) return SCPB_ERR_CUDA;
    scpb_handle_s *h = new (std::nothrow) scpb_handle_s();
    if (!h) return SCPB_ERR_CUDA;
    h->device = device;
    if (cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
        cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess ||
        cudaMalloc((void **)&h->d_status, sizeof(int)) != cudaSuccess ||
        cudaMemset(h->d_status, 0, sizeof(int)) != cudaSuccess) {
        delete h;
        return SCPB_ERR_CUDA;
    }
    *out = h;
    return SCPB_OK;
}

int32_t scpb_destroy(scpb_handle h)
{
    if (!h) return SCPB_ERR_ARG;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    for (auto &b : h->pool)
        if (b.ptr) cudaFree(b.ptr);
    if (h->d_status) cudaFree(h->d_status);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return SCPB_OK;
}

int32_t scpb_last_error(scpb_handle h, char *buf, size_t len)
{
    if (!h || !buf || len == 0) return SCPB_ERR_ARG;
    strncpy(buf, h->err, len - 1);
    buf[len - 1] = 0;
    return SCPB_OK;
}

int64_t scpb_launch_count(scpb_handle h) { return h ? h->launches : -1; }

void *scpb_stream(scpb_handle h) { return h ? (void *)h->stream : nullptr; }

int32_t scpb_sync(scpb_handle h)
{
    if (!h) return SCPB_ERR_ARG;
    SCPB_CUDA(h, cudaStreamSynchronize(h->stream));
    return SCPB_OK;
}

int32_t scpb_model_set(scpb_handle h, int32_t model_id, const double *par, int32_t npar, int32_t nx,
                       int32_t nu, int32_t np)
{
    if (!h) return SCPB_ERR_ARG;
    if (npar < 0 || npar > SCPB_MAX_PAR || (npar > 0 && !par)) return set_err(h, SCPB_ERR_ARG, "bad parameter block");
    int enx = 0, enu = 0, enp_min = 0;   // np >= the leading parameters the dynamics pack reads
    if (!with_model(model_id, [&](auto m) { enx = decltype(m)::NX; enu = decltype(m)::NU; enp_min = decltype(m)::NPD; }))
        return set_err(h, SCPB_ERR_MODEL, "unknown model id %d", model_id);
    if (nx != enx || nu != enu || np < enp_min)
        return set_err(h, SCPB_ERR_MODEL, "model %d expects nx=%d nu=%d np>=%d, got %d %d %d", model_id, enx, enu,
                       enp_min, nx, nu, np);
    h->model_id = model_id;
    h->nx = nx; h->nu = nu; h->np = np;
    memset(&h->par, 0, sizeof h->par);
    for (int i = 0; i < npar; i++) h->par.v[i] = par[i];
    h->npar = npar;
    return SCPB_OK;
}

int32_t scpb_discretize_dev(scpb_handle h, int32_t method, int32_t B, int32_t N, int32_t Nsub,
                            const double *t_grid, const double *xd, const double *ud, const double *p,
                            const double *iSx_diag, double feas_tol, double *A, double *Bm, double *Bp,
                            double *F, double *r, double *E, double *defect, int32_t *feas)
{
    int rc = check_model(h);
    if (rc) return rc;
    if (!t_grid || !xd || !ud || !p || !iSx_diag) return set_err(h, SCPB_ERR_ARG, "null input pointer");
    SCPB_CUDA(h, cudaSetDevice(h->device));
    DiscArgs a{};
    a.B = B; a.N = N; a.Nsub = Nsub;
    a.t_grid = t_grid; a.xd = xd; a.ud = ud; a.p = p; a.iSx = iSx_diag;
    julia_views(a, h->nx, h->nu, h->np, A, Bm, Bp, F, r, E, defect);
    return scpb_internal_discretize(h, a, feas_tol, feas, method, nullptr);
}

int32_t scpb_discretize(scpb_handle h, int32_t method, int32_t B, int32_t N, int32_t Nsub,
                        const double *t_grid, const double *xd, const double *ud, const double *p,
                        const double *iSx_diag, double feas_tol, double *A, double *Bm, double *Bp, double *F,
                        double *r, double *E, double *defect, int32_t *feas, double *seconds)
{
    int rc = check_model(h);
    if (rc) return rc;
    if (method != SCPB_FOH && method != SCPB_IMPULSE) return set_err(h, SCPB_ERR_ARG, "unknown discretization method %d", method);
    if (!t_grid || !xd || !ud || !p || !iSx_diag) return set_err(h, SCPB_ERR_ARG, "null input pointer");
    if (B <= 0 || N < 2 || Nsub < 2) return set_err(h, SCPB_ERR_ARG, "bad sizes B=%d N=%d Nsub=%d", B, N, Nsub);
    SCPB_CUDA(h, cudaSetDevice(h->device));
    const size_t nx = h->nx, nu = h->nu, np = h->np, M = N - 1, nb = B;
    const size_t s_t = N, s_x = nb * N * nx, s_u = nb * N * nu, s_p = nb * np, s_s = nx;
    const size_t s_A = nb * M * nx * nx, s_B = nb * M * nx * nu, s_F = nb * M * nx * np, s_r = nb * M * nx;
    const size_t in_d = s_t + s_x + s_u + s_p + s_s;
    const size_t out_d = 2 * s_A + 2 * s_B + s_F + 2 * s_r;
    double *din = (double *)h->scratch(1, sizeof(double) * in_d);
    double *dout = (double *)h->scratch(2, sizeof(double) * out_d);
    int *dfeas = (int *)h->scratch(3, sizeof(int) * nb);
    if (!din || !dout || !dfeas) return set_err(h, SCPB_ERR_CUDA, "device allocation failed");
    double *d_t = din, *d_x = d_t + s_t, *d_u = d_x + s_x, *d_p = d_u + s_u, *d_s = d_p + s_p;
    double *d_A = dout, *d_E = d_A + s_A, *d_Bm = d_E + s_A, *d_Bp = d_Bm + s_B, *d_F = d_Bp + s_B,
           *d_r = d_F + s_F, *d_df = d_r + s_r;
    cudaStream_t st = h->stream;
    SCPB_CUDA(h, cudaMemsetAsync(h->d_status, 0, sizeof(int), st));   // a stale flag of an earlier call is not this call's error
    SCPB_CUDA(h, cudaMemcpyAsync(d_t, t_grid, sizeof(double) * s_t, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(d_x, xd, sizeof(double) * s_x, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(d_u, ud, sizeof(double) * s_u, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(d_p, p, sizeof(double) * s_p, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(d_s, iSx_diag, sizeof(double) * s_s, cudaMemcpyHostToDevice, st));
    // inactive columns of the dense F stay zero (F has np columns, only the time-dilation ones are written; a model with
    // a fixed final time has none, and F stays all zeros)
    SCPB_CUDA(h, cudaMemsetAsync(d_F, 0, sizeof(double) * s_F, st));
    DiscArgs a{};
    a.B = B; a.N = N; a.Nsub = Nsub;
    a.t_grid = d_t; a.xd = d_x; a.ud = d_u; a.p = d_p; a.iSx = d_s;
    julia_views(a, h->nx, h->nu, h->np, d_A, d_Bm, d_Bp, d_F, d_r, d_E, d_df);
    SCPB_CUDA(h, cudaEventRecord(h->ev0, st));
    rc = scpb_internal_discretize(h, a, feas_tol, dfeas, method, nullptr);
    if (rc) return rc;
    SCPB_CUDA(h, cudaEventRecord(h->ev1, st));
    if (A) SCPB_CUDA(h, cudaMemcpyAsync(A, d_A, sizeof(double) * s_A, cudaMemcpyDeviceToHost, st));
    if (E) SCPB_CUDA(h, cudaMemcpyAsync(E, d_E, sizeof(double) * s_A, cudaMemcpyDeviceToHost, st));
    if (Bm) SCPB_CUDA(h, cudaMemcpyAsync(Bm, d_Bm, sizeof(double) * s_B, cudaMemcpyDeviceToHost, st));
    if (Bp) SCPB_CUDA(h, cudaMemcpyAsync(Bp, d_Bp, sizeof(double) * s_B, cudaMemcpyDeviceToHost, st));
    if (F) SCPB_CUDA(h, cudaMemcpyAsync(F, d_F, sizeof(double) * s_F, cudaMemcpyDeviceToHost, st));
    if (r) SCPB_CUDA(h, cudaMemcpyAsync(r, d_r, sizeof(double) * s_r, cudaMemcpyDeviceToHost, st));
    if (defect) SCPB_CUDA(h, cudaMemcpyAsync(defect, d_df, sizeof(double) * s_r, cudaMemcpyDeviceToHost, st));
    if (feas) SCPB_CUDA(h, cudaMemcpyAsync(feas, dfeas, sizeof(int) * nb, cudaMemcpyDeviceToHost, st));
    int hstat = 0;
    SCPB_CUDA(h, cudaMemcpyAsync(&hstat, h->d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    SCPB_CUDA(h, cudaStreamSynchronize(st));
    if (seconds) {
        float ms = 0.f;
        SCPB_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
        *seconds = ms * 1e-3;
    }
    if (hstat & 1) {
        cudaMemsetAsync(h->d_status, 0, sizeof(int), st);
        return set_err(h, SCPB_ERR_STATE, "singular transition matrix during discretization");
    }
    return SCPB_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// fp64 FMA peak of this device, measured: the denominator of K1's roofline (bench.py, "roofline_k1").
// 16 independent FMA chains per thread keep the fp64 pipe full; the result is stored so nothing is optimised away.
__global__ void k_fp64_peak(double *out, int iters, double a, double b)
{
    double v[16];
#pragma unroll
    for (int j = 0; j < 16; j++) v[j] = (double)(threadIdx.x + j) * 1e-3;
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int j = 0; j < 16; j++) v[j] = fma(v[j], a, b);
    }
    double sacc = 0.0;
#pragma unroll
    for (int j = 0; j < 16; j++) sacc += v[j];
    out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = sacc;
}

extern "C" int32_t scpb_debug_fp64_peak(scpb_handle h, double *tflops)
{
    if (!h || !tflops) return SCPB_ERR_ARG;
    SCPB_CUDA(h, cudaSetDevice(h->device));
    cudaDeviceProp pr;
    SCPB_CUDA(h, cudaGetDeviceProperties(&pr, h->device));
    const int blocks = pr.multiProcessorCount * 8, threads = 256, iters = 1 << 14;
    double *buf = (double *)h->scratch(4, sizeof(double) * (size_t)blocks * threads);
    if (!buf) return set_err(h, SCPB_ERR_CUDA, "scratch allocation failed");
    cudaStream_t st = h->stream;
    double best = 0.0;
    for (int rep = 0; rep < 4; rep++) {
        SCPB_CUDA(h, cudaEventRecord(h->ev0, st));
        k_fp64_peak<<<blocks, threads, 0, st>>>(buf, iters, 0.999999, 1e-6);
        h->launches++;
        SCPB_CUDA(h, cudaEventRecord(h->ev1, st));
        SCPB_CUDA(h, cudaStreamSynchronize(st));
        float ms = 0.f;
        SCPB_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
        const double tf = 2.0 * 16.0 * (double)iters * blocks * threads / (ms * 1e-3) / 1e12;
        if (rep > 0 && tf > best) best = tf;
    }
    *tflops = best;
    return SCPB_OK;
}

// ---------------------------------------------------------------------------------------------
// scpb_propagate: final continuous-time trajectory (discretization.jl:515-562, FOH branch)
template <class M>
static int launch_prop(scpb_handle_s *h, const PropArgs &a, int method, int subres)
{
    if (method == SCPB_IMPULSE) {
        if constexpr (M::IMPULSE) {
            const long long items = (long long)a.B * (a.N - 1);
            k_propagate_impulse<M><<<(unsigned)((items + 63) / 64), 64, 0, h->stream>>>(a, subres);
        } else {
            return set_err(h, SCPB_ERR_UNSUPPORTED, "model %d has no impulse semantics (IMPULSE propagation)", h->model_id);
        }
    } else {
        k_propagate_foh<M><<<(a.B + 31) / 32, 32, 0, h->stream>>>(a);
    }
    h->launches++;
    return SCPB_OK;
}

int32_t scpb_propagate(scpb_handle h, int32_t method, int32_t B, int32_t N, int32_t res, const double *t_grid,
                       const double *xd, const double *ud, const double *p, double *xc, double *seconds)
{
    int rc = check_model(h);
    if (rc) return rc;
    if (method != SCPB_FOH && method != SCPB_IMPULSE) return set_err(h, SCPB_ERR_ARG, "unknown discretization method %d", method);
    if (!t_grid || !xd || !ud || !p || !xc) return set_err(h, SCPB_ERR_ARG, "null pointer");
    if (B <= 0 || N < 2 || res < 2) return set_err(h, SCPB_ERR_ARG, "bad sizes B=%d N=%d res=%d", B, N, res);
    SCPB_CUDA(h, cudaSetDevice(h->device));
    const size_t nx = h->nx, nu = h->nu, np = h->np, nb = B;
    // IMPULSE: 1 + (N-1)*ceil(res/(N-1)) columns per seed (discretization.jl:541-556), FOH: res columns
    const int subres = (res + (N - 1) - 1) / (N - 1);
    const size_t ncol = (method == SCPB_IMPULSE) ? 1 + (size_t)(N - 1) * subres : (size_t)res;
    if (method == SCPB_IMPULSE && subres < 2) return set_err(h, SCPB_ERR_ARG, "IMPULSE propagation needs res >= 2 (N-1)");
    const size_t s_t = N, s_x = nb * N * nx, s_u = nb * N * nu, s_p = nb * np, s_c = nb * ncol * nx;
    double *din = (double *)h->scratch(1, sizeof(double) * (s_t + s_x + s_u + s_p));
    double *dout = (double *)h->scratch(2, sizeof(double) * s_c);
    if (!din || !dout) return set_err(h, SCPB_ERR_CUDA, "device allocation failed");
    double *d_t = din, *d_x = d_t + s_t, *d_u = d_x + s_x, *d_p = d_u + s_u;
    cudaStream_t st = h->stream;
    SCPB_CUDA(h, cudaMemcpyAsync(d_t, t_grid, sizeof(double) * s_t, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(d_x, xd, sizeof(double) * s_x, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(d_u, ud, sizeof(double) * s_u, cudaMemcpyHostToDevice, st));
    SCPB_CUDA(h, cudaMemcpyAsync(d_p, p, sizeof(double) * s_p, cudaMemcpyHostToDevice, st));
    PropArgs a{};
    a.B = B; a.N = N; a.res = res; a.t_grid = d_t; a.xd = d_x; a.ud = d_u; a.p = d_p; a.np = (int)np; a.xc = dout;
    a.par = h->par;
    cudaEvent_t e0 = h->ev0, e1 = h->ev1;   // the handle's own pair: nothing to leak on an error path
    SCPB_CUDA(h, cudaEventRecord(e0, st));
    if (!with_model(h->model_id, [&](auto m) { rc = launch_prop<decltype(m)>(h, a, method, subres); }))
        return set_err(h, SCPB_ERR_MODEL, "unknown model id %d", h->model_id);
    if (rc) return rc;
    SCPB_CUDA(h, cudaEventRecord(e1, st));
    SCPB_CUDA(h, cudaGetLastError());
    SCPB_CUDA(h, cudaMemcpyAsync(xc, dout, sizeof(double) * s_c, cudaMemcpyDeviceToHost, st));
    SCPB_CUDA(h, cudaStreamSynchronize(st));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    if (seconds) *seconds = 1e-3 * ms;
    return SCPB_OK;
}
