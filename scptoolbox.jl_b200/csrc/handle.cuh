// handle.cuh -- library-owned state behind the opaque scpb_handle (include/scpb.h).
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "models.cuh"

struct DevBuf {
    void *ptr = nullptr;
    size_t cap = 0;
};

struct scpb_handle_s {
    int device = 0;
    int sms = 0;               // streaming multiprocessors of `device` (132 on an H100 SXM)
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int model_id = 0, nx = 0, nu = 0, np = 0;
    ModelPar par{};
    int npar = 0;              // entries of par the caller gave (scpb_model_set); the rest are zero
    long long launches = 0;
    char err[512] = {0};
    int *d_status = nullptr;
    std::vector<DevBuf> pool;  // grow-only scratch buffers, indexed by slot

    void *scratch(int slot, size_t bytes)
    {
        if ((int)pool.size() <= slot) pool.resize(slot + 1);
        DevBuf &b = pool[slot];
        if (b.cap < bytes) {
            if (b.ptr) cudaFree(b.ptr);
            b.ptr = nullptr;
            b.cap = 0;
            if (cudaMalloc(&b.ptr, bytes) != cudaSuccess) return nullptr;
            b.cap = bytes;
        }
        return b.ptr;
    }
};

inline int set_err(scpb_handle_s *h, int code, const char *fmt, ...)
{
    if (h) {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(h->err, sizeof h->err, fmt, ap);
        va_end(ap);
    }
    return code;
}

#define SCPB_CUDA(h, call)                                                                       \
    do {                                                                                         \
        cudaError_t e_ = (call);                                                                 \
        if (e_ != cudaSuccess)                                                                   \
            return set_err((h), SCPB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                           __FILE__, __LINE__);                                                  \
    } while (0)
