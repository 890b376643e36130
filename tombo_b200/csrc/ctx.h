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

// grow-only device buffer; frees what it owns when destroyed
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
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
    // count elements of T from the host, enqueued on s.  The 8 spare bytes keep an empty
    // upload on a valid pointer; an empty upload copies nothing, so host may then be null.
    template <class T> cudaError_t upload(const T *host, size_t count, cudaStream_t s)
    {
        cudaError_t e = reserve(count * sizeof(T) + 8);
        if (e != cudaSuccess || count == 0) return e;
        return cudaMemcpyAsync(p, host, count * sizeof(T), cudaMemcpyHostToDevice, s);
    }
    bool owned = true;   // false: alias of another context's buffer (pipeline lanes)
    void release()
    {
        if (p && owned) cudaFree(p);
        p = nullptr; cap = 0;
    }
    template <class T> T *as() const { return (T *)p; }
};

// device state of each module, defined (and created, see tb2_state) in its own file
struct BatchHolder;      // resident batch (pipeline.cu)
struct BatchBuffers;     // arrays of one batch view: the single-read mirrors' own set (pipeline.cu)
struct LaunchScratch;    // per-launch scratch of tb2_launch_align / tb2_launch_resolve (kernels.h)
struct DpMirrorState;    // dp_kernels.cu
struct LlrState;         // llr.cu
struct RegionState;      // region_stats.cu
struct GroupState;       // group_stats.cu
struct DebugState;       // debug.cu
struct KdeState;         // model_est.cu

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
    std::shared_ptr<BatchHolder> batch;
    std::shared_ptr<BatchBuffers> one_read;
    std::shared_ptr<LaunchScratch> launch_scratch;
    std::shared_ptr<DpMirrorState> dp;
    std::shared_ptr<LlrState> llr;
    std::shared_ptr<RegionState> region;
    std::shared_ptr<GroupState> group;
    std::shared_ptr<DebugState> debug;
    std::shared_ptr<KdeState> kde;
    // tb2_resquiggle_batch pipelines large batches over two lanes (child contexts with
    // their own stream and buffers): H2D of chunk k+1 overlaps the kernels of chunk k
    std::vector<tb2_ctx *> lanes;
    bool async_mode = false;       // upload / download do not synchronise
    int read_index_base = 0;       // first read of the chunk within the caller's batch
    std::function<int()> after_first_launch;   // pipelined path: enqueue the next chunk's upload
    // model tables
    DevBuf model_means, model_sds, alt_means;
    int kmer_width = 0, central_pos = 0, alt_kmer_width = 0;
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

// a module's state on the context, created on first use.  Called where T is complete: the
// shared_ptr keeps T's deleter, so tb2_ctx_destroy frees it without knowing the type.
template <class T> T &tb2_state(std::shared_ptr<T> &state)
{
    if (!state) state = std::make_shared<T>();
    return *state;
}

// tb2_last_timing after a call that recorded ev0 before its first kernel: out[0] = device ms
// from ev0 to now (the upload before and the download after excluded); with split_at,
// out[1] = ms from ev0 to that event (the first part of the call's kernels); the rest 0
static inline int tb2_record_kernel_time(tb2_ctx *ctx, cudaEvent_t split_at = nullptr)
{
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev1));
    float ms = 0, first = 0;
    TB2_CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    if (split_at) TB2_CUDA_TRY(ctx, cudaEventElapsedTime(&first, ctx->ev0, split_at));
    ctx->last_ms_total = ms;
    ctx->last_ms_dp = first;
    ctx->last_dp_launches = ctx->last_dp_reads = 0;
    return TB2_OK;
}

static inline int tb2_use(tb2_ctx *ctx)
{
    if (!ctx) return TB2_ERR_INVALID_ARG;
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); return TB2_ERR_CUDA; }
    return TB2_OK;
}
