// ctx.h -- host-side context shared by the translation units of libtombo_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <memory>
#include <functional>
#include <string>
#include <vector>
#include "../../include/tombo_b200.h"

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    // grow-only device buffer
    cudaError_t reserve(size_t bytes)
    {
        if (bytes <= cap) return cudaSuccess;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            want = bytes;
            e = cudaMalloc(&p, want);
        }
        if (e == cudaSuccess) cap = want;
        return e;
    }
    bool owned = true;   // false: alias of another context's buffer (pipeline lanes)
    void release()
    {
        if (p && owned) cudaFree(p);
        p = nullptr; cap = 0;
    }
    template <class T> T *as() { return (T *)p; }
};

struct tb2_ctx {
    int device = 0;
    int sm_count = 132;            // H100 SXM; set from the device in tb2_ctx_create
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
    cudaEvent_t ev_h0 = nullptr, ev_h1 = nullptr;   // TB2_TRACE: upload bracket
    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;   // tb2_timer_start / _stop
    std::string err;
    int64_t launches = 0;
    double last_ms_total = 0, last_ms_dp = 0, last_dp_launches = 0, last_dp_reads = 0;
    std::shared_ptr<void> batch;   // BatchHolder (pipeline.cu)
    std::shared_ptr<void> region;  // RegionState (region_stats.cu)
    long long resident_llr_sites = 0;   // tb2_batch_alt_llr: sites / reads of the resident LLRs
    int resident_llr_reads = 0;
    // tb2_resquiggle_batch pipelines large batches over two lanes (child contexts with
    // their own stream and pools): H2D of chunk k+1 overlaps the kernels of chunk k
    std::vector<tb2_ctx *> lanes;
    bool async_mode = false;       // upload / download do not synchronise
    int read_index_base = 0;       // first read of the chunk within the caller's batch
    std::function<int()> after_first_launch;   // pipelined path: enqueue the next chunk's upload
    // model tables
    DevBuf model_means, model_sds, alt_means;
    int kmer_width = 0, central_pos = 0, alt_kmer_width = 0;
    // generic scratch pool (named slots), grow-only
    // slots: 0-11 mirror calls, 12-49 batch arrays (pipeline.cu), 50-69 llr.cu,
    // 70-79 per-warp scratch pools, 80-109 region_stats.cu, 110-124 group_stats.cu
    std::vector<DevBuf> pool = std::vector<DevBuf>(128);
    // pinned host staging for small results
    void *pinned = nullptr;
    size_t pinned_cap = 0;
};

#define TB2_CUDA_TRY(ctx, expr)                                                        \
    do {                                                                               \
        cudaError_t _e = (expr);                                                       \
        if (_e != cudaSuccess) {                                                       \
            char _b[512];                                                              \
            snprintf(_b, sizeof(_b), "%s:%d: %s -> %s", __FILE__, __LINE__, #expr,     \
                     cudaGetErrorString(_e));                                          \
            (ctx)->err = _b;                                                           \
            cudaGetLastError();                                                        \
            return TB2_ERR_CUDA;                                                       \
        }                                                                              \
    } while (0)

#define TB2_CHECK_LAUNCH(ctx)                                                          \
    do {                                                                               \
        (ctx)->launches++;                                                             \
        TB2_CUDA_TRY(ctx, cudaGetLastError());                                         \
    } while (0)

static inline int tb2_use(tb2_ctx *ctx)
{
    if (!ctx) return TB2_ERR_INVALID_ARG;
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); return TB2_ERR_CUDA; }
    return TB2_OK;
}
