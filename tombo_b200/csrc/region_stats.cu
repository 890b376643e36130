// region_stats.cu -- SURVEY.md 8(f)-1 and 8(f)-2 on the device.
//
// 8(f)-1  per-position aggregation of per-read statistics: collate_reg_stats
//         tombo_stats.py:4124-4178, apply_per_read_thresh :4084-4122,
//         calc_damp_fraction :2537-2552.  The reference sorts all (position, stat) pairs
//         of a region and splits them per position.  Positions are integers inside one
//         region block (10 kb by default, :4591-4595), so the sort is a counting sort:
//         three dense int32 counters per position (coverage, valid coverage, stats >=
//         threshold) filled with atomics straight from the per-read LLR kernel's output,
//         then an ordered compaction of the covered positions.  Counters are plain sums,
//         so reads of one region sharded over several GPUs reduce by adding the counter
//         arrays (tb2_region_counts_get / _set; NCCL or any all-reduce on the host side).
// 8(f)-2  de novo / sample-compare per-read tests: compute_de_novo_read_stats
//         :3771-3873, compute_sample_compare_read_stats :3675-3769,
//         calc_window_fishers_method :2252-2271: z -> two-sided normal p ->
//         windowed Fisher (chi2.sf with even degrees of freedom has the closed form
//         exp(-y) * sum_{i<k} y^i / i!, y = -sum log p).
#include "batch.h"
#include "kernels.h"
#include "fisher.cuh"
#include <cmath>
#include <vector>

namespace {
// per-call scratch of the entry points below; nothing reads it after a call returns
// F_MEAN .. F_START: the reads of tb2_de_novo_read_stats_batch (tb2_stage_reads; F_RM holds
// mean_off there)
enum { R_STAT = 0, R_POS, R_OUT_POS, R_OUT_F, R_OUT_D, R_OUT_C, R_OUT_V, R_N,
       F_MEAN, F_RM, F_SEQ, F_SOFF, F_START, F_RS, F_OFF, F_OUT, F_LOGP, F_POS, RS_COUNT };
}  // namespace

struct RegionState {
    // the open region and its counters: 3 * len ints, then the out-of-region count
    long long start = 0, len = 0;
    bool open = false;
    DevBuf cnt;
    DevBuf scratch[RS_COUNT];
};

namespace {
// stat_type 0: alternative-model LLRs (|stat| >= thresh is "valid" when no lower
// threshold is given, apply_per_read_thresh :4099-4105); 1: everything else
__global__ void k_region_accumulate(long long n, const double *stats, const long long *pos,
                                    long long reg_start, long long reg_len, double thresh,
                                    double lower, int stat_type, int *cnt, unsigned long long *dropped)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double s = stats[i];
    if (isnan(s)) return;                               // collate_reg_stats :4130-4133
    const long long p = pos[i] - reg_start;
    if (p < 0 || p >= reg_len) { atomicAdd(dropped, 1ULL); return; }
    atomicAdd(cnt + p, 1);                              // reg_cov
    bool valid = true;
    if (!isnan(lower)) valid = (s <= lower) || (s >= thresh);          // :4090-4098
    else if (stat_type == 0) valid = fabs(s) >= thresh;               // :4099-4105
    if (!valid) return;
    atomicAdd(cnt + reg_len + p, 1);                    // valid_cov
    if (s >= thresh) atomicAdd(cnt + 2 * reg_len + p, 1);
}

// ordered compaction of covered positions; one block (regions are ~1e4 positions)
__global__ void __launch_bounds__(1024)
k_region_finalize(const int *cnt, long long reg_start, long long reg_len, double unmod, double mod,
                  long long cap, long long *pos_out, double *frac_out, double *damp_out,
                  long long *cov_out, long long *valid_out, long long *n_out)
{
    __shared__ int warp_tot[32];
    __shared__ long long base_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) base_s = 0;
    __syncthreads();
    for (long long c0 = 0; c0 < reg_len; c0 += 1024) {
        const long long p = c0 + tid;
        const int cov = p < reg_len ? cnt[p] : 0;
        const int has = cov > 0;
        int inc = has;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, inc, off);
            if (lane >= off) inc += o;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        int before = 0, total = 0;
        for (int q = 0; q < 32; ++q) { if (q < warp) before += warp_tot[q]; total += warp_tot[q]; }
        const long long o = base_s + before + inc - has;
        if (has && o < cap) {
            const int valid = cnt[reg_len + p], ge = cnt[2 * reg_len + p];
            // np.greater_equal(...).sum() / base_stats.shape[0], NaN on empty (:4114-4118)
            const double frac = valid > 0 ? (double)ge / (double)valid : NAN;
            pos_out[o] = reg_start + p;
            frac_out[o] = frac;
            cov_out[o] = cov;
            valid_out[o] = valid;
            // calc_damp_fraction :2546-2550: np.round = round half to even = rint
            damp_out[o] = isnan(unmod) ? NAN
                                       : (rint(frac * (double)valid) + unmod) / ((double)valid + (unmod + mod));
        }
        __syncthreads();
        if (tid == 0) base_s += total;
        __syncthreads();
    }
    if (tid == 0) *n_out = base_s;
}

}  // namespace

// ---------------------------------------------------------------------------
// C ABI: 8(f)-1
// ---------------------------------------------------------------------------
extern "C" int tb2_region_stats_begin(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (reg_len < 1 || reg_len > (1LL << 28)) return TB2_ERR_INVALID_ARG;
    RegionState &rs = tb2_state(ctx->region);
    TB2_CUDA_TRY(ctx, rs.cnt.reserve((size_t)reg_len * 3 * 4 + 16));
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(rs.cnt.p, 0, (size_t)reg_len * 3 * 4 + 16, ctx->stream));
    rs.start = reg_start; rs.len = reg_len; rs.open = true;
    return TB2_OK;
}

// device arrays in, counters updated; the 8 bytes after the counters count out-of-region stats
int tb2_region_accumulate_dev(tb2_ctx *ctx, long long n, const double *stats_dev,
                              const long long *pos_dev, double thresh, double lower, int stat_type)
{
    RegionState &rs = tb2_state(ctx->region);
    if (!rs.open) { ctx->err = "tb2_region_stats_begin has not been called"; return TB2_ERR_INVALID_ARG; }
    if (n <= 0) return TB2_OK;
    int *cnt = rs.cnt.as<int>();
    k_region_accumulate<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
        n, stats_dev, pos_dev, rs.start, rs.len, thresh, lower, stat_type, cnt,
        (unsigned long long *)(cnt + 3 * rs.len + ((3 * rs.len) & 1)));
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

extern "C" int tb2_region_stats_add(tb2_ctx *ctx, int64_t n, const double *stats, const int64_t *pos,
                                    double single_read_thresh, double lower_thresh, int stat_type)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!stats || !pos)) || isnan(single_read_thresh)) return TB2_ERR_INVALID_ARG;
    if (n == 0) return TB2_OK;
    auto &P = tb2_state(ctx->region).scratch;
    TB2_CUDA_TRY(ctx, P[R_STAT].upload(stats, (size_t)n, ctx->stream));
    TB2_CUDA_TRY(ctx, P[R_POS].upload(pos, (size_t)n, ctx->stream));
    rc = tb2_region_accumulate_dev(ctx, n, P[R_STAT].as<double>(), P[R_POS].as<long long>(),
                                   single_read_thresh, lower_thresh, stat_type);
    if (rc) return rc;
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));   // the host buffers may go away
    return TB2_OK;
}

extern "C" int tb2_region_counts_get(tb2_ctx *ctx, int32_t *counts)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    RegionState &rs = tb2_state(ctx->region);
    if (!rs.open || !counts) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(counts, rs.cnt.p, (size_t)rs.len * 3 * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return TB2_OK;
}

extern "C" int tb2_region_counts_set(tb2_ctx *ctx, const int32_t *counts)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    RegionState &rs = tb2_state(ctx->region);
    if (!rs.open || !counts) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(rs.cnt.p, counts, (size_t)rs.len * 3 * 4, cudaMemcpyHostToDevice, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return TB2_OK;
}

extern "C" int tb2_region_stats_finalize(tb2_ctx *ctx, double unmod_count, double mod_count,
                                         int64_t cap, int64_t *pos_out, double *frac_out,
                                         double *damp_frac_out, int64_t *cov_out,
                                         int64_t *valid_cov_out, int64_t *n_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    RegionState &rs = tb2_state(ctx->region);
    if (!rs.open || cap < 0 || !n_out || (cap > 0 && (!pos_out || !frac_out || !damp_frac_out || !cov_out || !valid_cov_out)))
        return TB2_ERR_INVALID_ARG;
    auto &P = rs.scratch;
    cudaStream_t s = ctx->stream;
    const size_t c = (size_t)std::min<long long>(cap, rs.len);
    TB2_CUDA_TRY(ctx, P[R_OUT_POS].reserve(c * 8 + 8));
    TB2_CUDA_TRY(ctx, P[R_OUT_F].reserve(c * 8 + 8));
    TB2_CUDA_TRY(ctx, P[R_OUT_D].reserve(c * 8 + 8));
    TB2_CUDA_TRY(ctx, P[R_OUT_C].reserve(c * 8 + 8));
    TB2_CUDA_TRY(ctx, P[R_OUT_V].reserve(c * 8 + 8));
    TB2_CUDA_TRY(ctx, P[R_N].reserve(8));
    k_region_finalize<<<1, 1024, 0, s>>>(rs.cnt.as<int>(), rs.start, rs.len, unmod_count, mod_count,
                                         (long long)c, P[R_OUT_POS].as<long long>(), P[R_OUT_F].as<double>(),
                                         P[R_OUT_D].as<double>(), P[R_OUT_C].as<long long>(),
                                         P[R_OUT_V].as<long long>(), P[R_N].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    long long n = 0;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(&n, P[R_N].p, 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    *n_out = n;
    const size_t m = (size_t)std::min<long long>(n, (long long)c);
    if (m) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, P[R_OUT_POS].p, m * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(frac_out, P[R_OUT_F].p, m * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(damp_frac_out, P[R_OUT_D].p, m * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cov_out, P[R_OUT_C].p, m * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(valid_cov_out, P[R_OUT_V].p, m * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    }
    return n > (long long)c ? TB2_ERR_CAPACITY : TB2_OK;
}

// ---------------------------------------------------------------------------
// C ABI: 8(f)-2
// ---------------------------------------------------------------------------
static int fisher_common(tb2_ctx *ctx, FisherArgs &a, int n_segs, long long total, bool kmer,
                         double *pvals_out, int64_t *pos_out)
{
    auto &P = tb2_state(ctx->region).scratch;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, P[F_OUT].reserve((size_t)total * 8 + 8));
    TB2_CUDA_TRY(ctx, P[F_LOGP].reserve((size_t)total * 8 + 8));
    a.out = P[F_OUT].as<double>();
    a.logp = P[F_LOGP].as<double>();
    a.smallest = 1e-50;                                  // SMALLEST_PVAL _default_parameters.py:158
    if (kmer) {
        TB2_CUDA_TRY(ctx, P[F_POS].reserve((size_t)total * 8 + 8));
        a.pos_out = P[F_POS].as<long long>();
        k_fisher<true><<<n_segs, 256, 0, s>>>(a);
    } else {
        a.pos_out = nullptr;
        k_fisher<false><<<n_segs, 256, 0, s>>>(a);
    }
    TB2_CHECK_LAUNCH(ctx);
    if (total > 0) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pvals_out, P[F_OUT].p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
        if (kmer && pos_out)
            TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, P[F_POS].p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
    }
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

extern "C" int tb2_window_fisher_pvals(tb2_ctx *ctx, int64_t n_segs, const double *means,
                                       const double *ref_means, const double *ref_sds,
                                       const int64_t *seg_off, int64_t fm_offset, int final_clamp,
                                       double *pvals_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n_segs < 0 || fm_offset < 0 || fm_offset > 64 || !seg_off) return TB2_ERR_INVALID_ARG;
    if (n_segs == 0) return TB2_OK;
    const long long total = seg_off[n_segs];
    const bool is_p = !ref_means && !ref_sds;           // p-values in, Fisher window only
    if (total < 0 || seg_off[0] != 0 || (total > 0 && (!means || !pvals_out)) || (!ref_means != !ref_sds))
        return TB2_ERR_INVALID_ARG;
    auto &P = tb2_state(ctx->region).scratch;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, P[F_MEAN].upload(means, (size_t)total, s));
    // p-values in: k_fisher reads no reference levels
    TB2_CUDA_TRY(ctx, P[F_RM].upload(ref_means, is_p ? 0 : (size_t)total, s));
    TB2_CUDA_TRY(ctx, P[F_RS].upload(ref_sds, is_p ? 0 : (size_t)total, s));
    TB2_CUDA_TRY(ctx, P[F_OFF].upload(seg_off, (size_t)n_segs + 1, s));
    FisherArgs a;
    memset(&a, 0, sizeof(a));
    a.means = P[F_MEAN].as<double>(); a.rm = P[F_RM].as<double>(); a.rs = P[F_RS].as<double>();
    a.off = P[F_OFF].as<long long>();
    a.lag = (int)fm_offset; a.final_clamp = final_clamp ? 1 : 0; a.input_is_p = is_p ? 1 : 0;
    return fisher_common(ctx, a, (int)n_segs, total, false, pvals_out, nullptr);
}

extern "C" int tb2_de_novo_read_stats_batch(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                                            const int64_t *mean_off, const uint8_t *seq,
                                            const int64_t *seq_off, const int64_t *read_start,
                                            int64_t fm_offset, double *pvals_out, int64_t *pos_out,
                                            int64_t *stat_off)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (fm_offset < 0 || fm_offset > 64 || !stat_off) return TB2_ERR_INVALID_ARG;
    if (ctx->kmer_width <= 0) { ctx->err = "tb2_set_model has not been called"; return TB2_ERR_INVALID_ARG; }
    auto &P = tb2_state(ctx->region).scratch;
    FisherArgs a;
    memset(&a, 0, sizeof(a));
    if ((rc = tb2_stage_reads(ctx, n_reads, norm_mean, mean_off, seq, seq_off, read_start, P + F_MEAN, a)))
        return rc;
    stat_off[0] = 0;
    if (n_reads == 0) return TB2_OK;
    const int n = (int)n_reads, K = ctx->kmer_width;
    // len(r_seq) < kmer_width raises in the reference (:3846-3848): no stats for that read
    for (int r = 0; r < n; ++r)
        stat_off[r + 1] = stat_off[r] + std::max<long long>(0, mean_off[r + 1] - mean_off[r] - (K - 1));
    const long long total = stat_off[n];
    if (total > 0 && (!norm_mean || !seq || !pvals_out || !pos_out)) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, P[F_OFF].upload(stat_off, (size_t)n + 1, ctx->stream));
    a.off = P[F_OFF].as<long long>();
    a.kmeans = ctx->model_means.as<double>(); a.ksds = ctx->model_sds.as<double>();
    a.K = K; a.cpos = ctx->central_pos;
    a.lag = (int)fm_offset; a.final_clamp = 1;
    return fisher_common(ctx, a, n, total, true, pvals_out, pos_out);
}
