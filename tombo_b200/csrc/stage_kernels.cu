// stage_kernels.cu -- launch wrappers of the stage kernels (device code: stage_kernels.cuh)
#include "stage_kernels.cuh"
#include "kernels.h"

// ===========================================================================
// launch wrappers
// ===========================================================================
static inline int grid1d(int n, int bs) { return (n + bs - 1) / bs; }

int tb2_launch_prep(tb2_ctx *ctx, const BatchView &b, const void *raw_dev, int raw_dtype,
                    int is_rna, long long, long long)
{
    if (raw_dtype == 0)
        k_prep<double><<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(
            b, (const double *)raw_dev, is_rna, ctx->model_means.as<double>(),
            ctx->model_sds.as<double>());
    else
        k_prep<short><<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(
            b, (const short *)raw_dev, is_rna, ctx->model_means.as<double>(),
            ctx->model_sds.as<double>());
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_start_attempt(tb2_ctx *ctx, const BatchView &b, int attempt)
{
    k_start_attempt<<<grid1d(b.n_reads, 256), 256, 0, ctx->stream>>>(b, attempt);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_begin_call(tb2_ctx *ctx, const BatchView &b, const tb2_params &p,
                          const StagePolicy &pol)
{
    k_begin_call<<<grid1d(b.n_reads, 256), 256, 0, ctx->stream>>>(b, p, pol);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_end_call(tb2_ctx *ctx, const BatchView &b, int max_iters)
{
    k_end_call<<<grid1d(b.n_reads, 256), 256, 0, ctx->stream>>>(b, max_iters);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_count_active(tb2_ctx *ctx, const BatchView &b, int *dev_counter)
{
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(dev_counter, 0, 2 * sizeof(int), ctx->stream));
    k_count_active<<<grid1d(b.n_reads, 256), 256, 0, ctx->stream>>>(b, dev_counter);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_normalize(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol, int first_call)
{
    k_normalize<<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(b, pol, first_call);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_cpts(tb2_ctx *ctx, const BatchView &b, const tb2_params &p, int on_raw)
{
    // bit sets of the greedy pass: 4 + (min_obs_per_base - 1) words per 32 candidates, in
    // shared memory when the longest read of the batch fits in 48 KB (else the read's scratch)
    if (!p.use_t_test_seg) {
        k_cumsum<<<(b.n_reads + CS_WARPS - 1) / CS_WARPS, CS_WARPS * 32, 0, ctx->stream>>>(b, on_raw);
        TB2_CHECK_LAUNCH(ctx);
    }
    const long long nw = (b.max_raw + 32) / 32;
    long long words = (4 + std::max(0, (int)p.min_obs_per_base - 1)) * nw;
    if (words * 4 > 48 * 1024) words = 0;   // the default dynamic shared-memory limit
    k_cpts<<<b.n_reads, ST_THREADS, (size_t)words * 4, ctx->stream>>>(b, p, on_raw, (int)words);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_rna_scale(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol)
{
    k_rna_scale<<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(b, pol);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_event_means(tb2_ctx *ctx, const BatchView &b)
{
    k_event_means<<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(b);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_stalls(tb2_ctx *ctx, const BatchView &b)
{
    k_stalls<<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(b);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_resolve(tb2_ctx *ctx, const BatchView &b, const tb2_params &p,
                       const StagePolicy &pol, size_t cap)
{
    const int warps_per_block = 4;
    int grid = ctx->sm_count * 8;
    const int max_useful = (b.n_reads + warps_per_block - 1) / warps_per_block;
    if (grid > max_useful) grid = max_useful > 0 ? max_useful : 1;
    const size_t slots = (size_t)grid * warps_per_block;
    LaunchScratch &ls = tb2_state(ctx->launch_scratch);
    TB2_CUDA_TRY(ctx, ls.raw_dp.reserve(slots * cap * sizeof(double)));
    TB2_CUDA_TRY(ctx, ls.resolve_cnt.reserve(16));
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(ls.resolve_cnt.p, 0, 16, ctx->stream));
    // overflow arena for windows beyond the per-warp slab: a window is at most
    // (2 * MAX_DEL_FIX_WINDOW + few) bases x its samples; sized from the longest read,
    // 64 MB .. 2 GB
    const unsigned long long big_cap = std::min<unsigned long long>(
        (2ULL << 30) / 8, std::max<unsigned long long>((64ULL << 20) / 8, 24ULL * 64ULL * (unsigned long long)std::max(1, b.max_raw)));
    TB2_CUDA_TRY(ctx, ls.raw_big.reserve((size_t)big_cap * sizeof(double)));
    k_resolve<<<grid, warps_per_block * 32, 0, ctx->stream>>>(
        b, p, pol, ls.raw_dp.as<double>(), cap, ls.resolve_cnt.as<int>(), ls.raw_big.as<double>(),
        big_cap, (unsigned long long *)(ls.resolve_cnt.as<int>() + 2));
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_base_means(tb2_ctx *ctx, const BatchView &b)
{
    k_base_means<<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(b);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_theil_sen(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol, int first_call)
{
    const size_t smem = sizeof(TsSmem);
    TB2_CUDA_TRY(ctx, cudaFuncSetAttribute(k_theil_sen, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem));
    k_theil_sen<<<b.n_reads, ST_THREADS, smem, ctx->stream>>>(b, pol, first_call);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

int tb2_launch_finalize(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol, int first_call,
                        double *norm_mean_out, double *norm_signal_out)
{
    k_finalize<<<b.n_reads, ST_THREADS, 0, ctx->stream>>>(b, pol, first_call, norm_mean_out,
                                                          norm_signal_out);
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

extern "C" int tb2_debug_counters(tb2_ctx *ctx, unsigned long long *out8, int reset)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!out8) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    TB2_CUDA_TRY(ctx, cudaMemcpyFromSymbol(out8, g_tb2_counters, 64));
    if (reset) {
        unsigned long long z[8] = {0};
        TB2_CUDA_TRY(ctx, cudaMemcpyToSymbol(g_tb2_counters, z, 64));
    }
    return TB2_OK;
}
