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
//         exp(-y) * sum_{i<k} y^i / i!, y = -sum log p).  The de novo test runs in k_de_novo
//         over host-computed per-read descriptors (region clip, strand); sample-compare
//         runs k_fisher on host-staged genome-ordered segments, then compacts each read's
//         non-NaN entries.  Both leave their statistics in RegionState for
//         tb2_region_stats_add_tests.
#include "batch.h"
#include "kernels.h"
#include "common.cuh"
#include "fisher.cuh"
#include <cmath>
#include <cstring>
#include <vector>

namespace {
// per-call scratch of the entry points below; nothing reads it after a call returns
// F_MEAN .. F_START: the reads of tb2_de_novo_read_stats_batch (tb2_stage_reads; F_RM holds
// mean_off there)
// D_RD .. D_CNT: per-read descriptors, statuses and survivor counts of the region tests
enum { R_STAT = 0, R_POS, R_OUT_POS, R_OUT_F, R_OUT_D, R_OUT_C, R_OUT_V, R_N,
       F_MEAN, F_RM, F_SEQ, F_SOFF, F_START, F_RS, F_OFF, F_OUT, F_LOGP, F_POS,
       D_RD, D_STATUS, D_CNT, D_SOFF, RS_COUNT };
}  // namespace

struct RegionState {
    // the open region and its counters: 3 * len ints, then the out-of-region count
    long long start = 0, len = 0;
    bool open = false;
    DevBuf cnt;
    DevBuf scratch[RS_COUNT];
    // statistics and positions of the last de novo / sample-compare region call, for
    // tb2_region_stats_add_tests; tests_n < 0: no such call yet
    DevBuf tests_stat, tests_pos;
    long long tests_n = -1;
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
    const int tid = threadIdx.x;
    long long base = 0;
    for (long long c0 = 0; c0 < reg_len; c0 += 1024) {
        const long long p = c0 + tid;
        const int cov = p < reg_len ? cnt[p] : 0;
        const int has = cov > 0;
        int total;
        const long long o = base + tb2_block_excl_scan<1024>(has, warp_tot, total);
        base += total;
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
    }
    if (tid == 0) *n_out = base;
}


// one read of k_de_novo, decided on the host (region clip, strand, zero-width slice)
struct DeNovoRead {
    long long out0;     // first output entry (stat_off[r])
    long long gstart;   // genome position of output 0
    int clip5;          // bases clipped off the read's 5' end
    int n_kmers;        // k-mers of the clipped bases (looked up, so checked)
    int n_out;          // outputs: n_kmers, or 0 (zero-width slice, window longer than the read)
    int strand;         // 0: output i is read-centric k-mer i; 1: k-mer n_out - 1 - i
    int status;         // status decided on the host
    int pad_;
};

struct DeNovoArgs {
    FisherArgs f;       // the reads (norm_mean, mean_off, seq, seq_off), model, window, outputs
    const DeNovoRead *rd;
    int *status_out;
    const int *rsq_status;   // resident batch: resquiggle status[r * rsq_stride]; null otherwise
    int rsq_stride;
    int check;          // report non-ACGT codes and k-mers absent from the model
};

// compute_de_novo_read_stats :3843-3871 for one read per block.  K-mer q of the clipped
// read-centric bases pairs with its central mean; '-' reads emit k-mers in reverse
// (get_seq_kmers(..., rev_strand) and r_means[::-1]), so outputs are in genome order.
__global__ void __launch_bounds__(256) k_de_novo(DeNovoArgs a)
{
    const int r = blockIdx.x, tid = threadIdx.x;
    const DeNovoRead d = a.rd[r];
    const int K = a.f.K;
    const unsigned char *bases = a.f.seq + a.f.seq_off[r] + a.f.cpos + d.clip5;
    int st = d.status;
    if (a.rsq_status && a.rsq_status[(size_t)r * a.rsq_stride] != TB2_OK) {
        st = a.rsq_status[(size_t)r * a.rsq_stride];
    } else if (a.check && (st == TB2_OK || st == TB2_ERR_FISHER_TOO_SHORT)) {
        // get_exp_levels_from_seq precedes the window check (:3843, :3865)
        int bad = 0;
        for (int i = tid; i < d.n_kmers; i += 256) {
            int code = 0;
            for (int j = 0; j < K; ++j) {
                const int c = bases[i + j];
                bad |= c > 3;
                code = code * 4 + (c & 3);
            }
            bad |= isnan(a.f.kmeans[code]);
        }
        if (__syncthreads_or(bad)) st = TB2_ERR_INVALID_SEQ;
    }
    if (a.status_out && tid == 0) a.status_out[r] = st;
    const int n = d.n_out;
    if (n <= 0) return;
    double *out = a.f.out + d.out0, *logp = a.f.logp + d.out0;
    long long *pos = a.f.pos_out + d.out0;
    if (st != TB2_OK) {                   // NaN statistics never reach the region counters
        for (int i = tid; i < n; i += 256) { out[i] = NAN; pos[i] = d.gstart + i; }
        return;
    }
    const double *means = a.f.norm_mean + a.f.mean_off[r] + a.f.cpos + d.clip5;
    const int lag = a.f.lag;
    for (int i = tid; i < n; i += 256) {
        const int q = d.strand ? n - 1 - i : i;
        int code = 0;
        for (int j = 0; j < K; ++j) code = code * 4 + (bases[q + j] & 3);
        const double rm = a.f.kmeans[code], rs = a.f.ksds[code];
        pos[i] = d.gstart + i;
        const double p = two_sided_p(means[q], rm, rs);
        if (lag == 0) out[i] = a.f.final_clamp ? np_maximum(p, a.f.smallest) : p;
        else logp[i] = log(np_maximum(p, a.f.smallest));      // :2261-2263
    }
    if (lag == 0) return;
    __syncthreads();
    fisher_window(logp, out, n, lag, a.f.final_clamp, a.f.smallest, tid);
}

// one read of the sample-compare test: its genome-ordered segment in the staged arrays
struct CompareRead {
    long long seg0;     // first entry of the segment (means, control levels, k_fisher output)
    long long gstart;   // genome position of entry 0
    int n;              // segment length
    int skip;           // strand -1: no statistics, status 0
};

// compute_sample_compare_read_stats :3755-3767 after k_fisher: the read's status, then its
// non-NaN entries in order.  FILL = false counts them (and writes the status); FILL = true
// writes them at stat_off[r].
template <bool FILL>
__global__ void __launch_bounds__(256)
k_compare_compact(const CompareRead *rd, const double *m, const double *rm, const double *rs,
                  const double *fout, int lag, int *cnt, int *status, const long long *stat_off,
                  double *stat_out, long long *pos_out)
{
    __shared__ int warp_tot[8];
    const int r = blockIdx.x, tid = threadIdx.x;
    const CompareRead d = rd[r];
    if (!FILL) {
        int st = TB2_OK;
        if (!d.skip) {
            int valid = 0;
            for (int i = tid; i < d.n; i += 256)
                valid |= !isnan(fabs(m[d.seg0 + i] - rm[d.seg0 + i]) / rs[d.seg0 + i]);   // :3736-3740
            if (!__syncthreads_or(valid)) st = TB2_ERR_NO_VALID_Z;
            else if (lag > 0 && d.n < 2 * lag + 1) st = TB2_ERR_FISHER_TOO_SHORT;
        }
        if (tid == 0) status[r] = st;
        if (d.skip || st != TB2_OK) { if (tid == 0) cnt[r] = 0; return; }
    } else if (d.skip || status[r] != TB2_OK) {
        return;
    }
    if (FILL) { stat_out += stat_off[r]; pos_out += stat_off[r]; }
    int base = 0;
    for (int c0 = 0; c0 < d.n; c0 += 256) {
        const int i = c0 + tid;
        const double v = i < d.n ? fout[d.seg0 + i] : NAN;
        const int keep = !isnan(v);
        int total;
        const int o = base + tb2_block_excl_scan<256>(keep, warp_tot, total);
        base += total;
        if (FILL && keep) {
            stat_out[o] = v;
            pos_out[o] = d.gstart + i;
        }
        __syncthreads();
    }
    if (!FILL && tid == 0) cnt[r] = base;
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
static int fisher_common(tb2_ctx *ctx, FisherArgs &a, int n_segs, long long total,
                         double *pvals_out)
{
    auto &P = tb2_state(ctx->region).scratch;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, P[F_OUT].reserve((size_t)total * 8 + 8));
    TB2_CUDA_TRY(ctx, P[F_LOGP].reserve((size_t)total * 8 + 8));
    a.out = P[F_OUT].as<double>();
    a.logp = P[F_LOGP].as<double>();
    a.smallest = 1e-50;                                  // SMALLEST_PVAL _default_parameters.py:158
    a.pos_out = nullptr;
    k_fisher<false><<<n_segs, 256, 0, s>>>(a);
    TB2_CHECK_LAUNCH(ctx);
    if (total > 0)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pvals_out, P[F_OUT].p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
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
    return fisher_common(ctx, a, (int)n_segs, total, pvals_out);
}

namespace {
// the window, model and read layout of a k_de_novo launch; the reads' arrays are set by the
// caller (tb2_stage_reads or the resident batch)
void de_novo_args(tb2_ctx *ctx, int64_t fm_offset, DeNovoArgs &a)
{
    a.f.kmeans = ctx->model_means.as<double>(); a.f.ksds = ctx->model_sds.as<double>();
    a.f.K = ctx->kmer_width; a.f.cpos = ctx->central_pos;
    a.f.lag = (int)fm_offset; a.f.final_clamp = 1;
    a.f.smallest = 1e-50;                                // SMALLEST_PVAL _default_parameters.py:158
}

// k_de_novo over n reads with descriptors rd (total outputs) into `stat` / `pos`; copies the
// statistics out where pvals_out is given and the statuses where read_status is
int run_de_novo(tb2_ctx *ctx, DeNovoArgs &a, const std::vector<DeNovoRead> &rd, long long total,
                DevBuf &stat, DevBuf &pos, double *pvals_out, int64_t *pos_out, int32_t *read_status)
{
    auto &P = tb2_state(ctx->region).scratch;
    cudaStream_t s = ctx->stream;
    const int n = (int)rd.size();
    TB2_CUDA_TRY(ctx, P[D_RD].upload(rd.data(), rd.size(), s));
    TB2_CUDA_TRY(ctx, P[D_STATUS].reserve((size_t)n * 4 + 8));
    TB2_CUDA_TRY(ctx, P[F_LOGP].reserve((size_t)total * 8 + 8));
    TB2_CUDA_TRY(ctx, stat.reserve((size_t)total * 8 + 8));
    TB2_CUDA_TRY(ctx, pos.reserve((size_t)total * 8 + 8));
    a.rd = P[D_RD].as<DeNovoRead>();
    a.status_out = P[D_STATUS].as<int>();
    a.f.logp = P[F_LOGP].as<double>();
    a.f.out = stat.as<double>();
    a.f.pos_out = pos.as<long long>();
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, s));     // kernel time: tb2_last_timing
    k_de_novo<<<n, 256, 0, s>>>(a);
    TB2_CHECK_LAUNCH(ctx);
    int rc = tb2_record_kernel_time(ctx);
    if (rc) return rc;
    if (total > 0 && pvals_out)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pvals_out, stat.p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
    if (total > 0 && pos_out)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, pos.p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
    if (read_status)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(read_status, P[D_STATUS].p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

int region_args_ok(tb2_ctx *ctx, int64_t n_reads, const int8_t *strand, int64_t fm_offset,
                   int64_t reg_start, int64_t reg_end)
{
    if (n_reads < 0 || n_reads > INT_MAX || (n_reads > 0 && !strand) || fm_offset < 0 ||
        fm_offset > 64 || reg_end <= reg_start) {
        ctx->err = "invalid read count, strand array, fm_offset or region";
        return TB2_ERR_INVALID_ARG;
    }
    for (int64_t r = 0; r < n_reads; ++r)
        if (strand[r] < -1 || strand[r] > 1) { ctx->err = "strand outside {-1, 0, 1}"; return TB2_ERR_INVALID_ARG; }
    return TB2_OK;
}

// compute_de_novo_read_stats' clip (:3813-3853) for read r of nb bases starting at `start`:
// its descriptor and number of outputs.  The clip keeps the reference's slicing: a clip longer
// than the read empties it, and r_means[begin:-0] is empty (end lag 0).
DeNovoRead de_novo_read(long long start, long long nb, int strand, int K, int cpos, int fm,
                        long long reg_start, long long reg_end)
{
    DeNovoRead d;
    memset(&d, 0, sizeof(d));
    d.strand = strand;
    if (strand < 0) return d;                            // skipped read: no statistics
    const int dn = K - cpos - 1;
    const int begin_lag = strand == 0 ? cpos : dn, end_lag = strand == 0 ? dn : cpos;
    const long long lo = begin_lag + fm, hi = end_lag + fm;
    const long long low_over = std::max(0LL, reg_start - (start + lo));
    const long long high_over = std::max(0LL, (start + nb - hi) - reg_end);
    const long long clip5 = strand == 0 ? low_over : high_over, clip3 = strand == 0 ? high_over : low_over;
    const long long len = std::max(0LL, nb - clip5 - clip3);
    if (len < K) { d.status = TB2_ERR_NO_INFO_IN_REGION; return d; }
    const long long read_start = low_over ? reg_start - lo : start;
    d.clip5 = (int)clip5;
    d.n_kmers = (int)(len - K + 1);
    d.gstart = read_start + begin_lag;
    d.n_out = end_lag ? d.n_kmers : 0;
    if (fm > 0 && d.n_out < 2 * fm + 1) { d.status = TB2_ERR_FISHER_TOO_SHORT; d.n_out = 0; }
    return d;
}

// descriptors of n reads and their output offsets (stat_off, n + 1, filled)
long long de_novo_reads(tb2_ctx *ctx, int n, const long long *base_off, const int64_t *read_start,
                        const int8_t *strand, int64_t fm_offset, int64_t reg_start, int64_t reg_end,
                        std::vector<DeNovoRead> &rd, int64_t *stat_off)
{
    rd.resize(n);
    long long total = 0;
    for (int r = 0; r < n; ++r) {
        rd[r] = de_novo_read(read_start[r], base_off[r + 1] - base_off[r], strand[r], ctx->kmer_width,
                             ctx->central_pos, (int)fm_offset, reg_start, reg_end);
        rd[r].out0 = total;
        if (stat_off) stat_off[r] = total;
        total += rd[r].n_out;
    }
    if (stat_off) stat_off[n] = total;
    return total;
}

int model_ok(tb2_ctx *ctx)
{
    if (ctx->kmer_width > 0) return TB2_OK;
    ctx->err = "tb2_set_model has not been called";
    return TB2_ERR_INVALID_ARG;
}
}  // namespace

extern "C" int tb2_de_novo_read_stats_batch(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                                            const int64_t *mean_off, const uint8_t *seq,
                                            const int64_t *seq_off, const int64_t *read_start,
                                            int64_t fm_offset, double *pvals_out, int64_t *pos_out,
                                            int64_t *stat_off)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (fm_offset < 0 || fm_offset > 64 || !stat_off) return TB2_ERR_INVALID_ARG;
    if ((rc = model_ok(ctx))) return rc;
    auto &P = tb2_state(ctx->region).scratch;
    DeNovoArgs a;
    memset(&a, 0, sizeof(a));
    if ((rc = tb2_stage_reads(ctx, n_reads, norm_mean, mean_off, seq, seq_off, read_start, P + F_MEAN, a.f)))
        return rc;
    stat_off[0] = 0;
    if (n_reads == 0) return TB2_OK;
    const int n = (int)n_reads, K = ctx->kmer_width;
    // whole '+' reads: every k-mer, no clip; len(r_seq) < kmer_width raises in the reference
    // (:3846-3848): no stats for that read
    std::vector<DeNovoRead> rd(n);
    for (int r = 0; r < n; ++r) {
        const long long m = std::max<long long>(0, mean_off[r + 1] - mean_off[r] - (K - 1));
        memset(&rd[r], 0, sizeof(DeNovoRead));
        rd[r].out0 = stat_off[r];
        rd[r].gstart = read_start[r] + ctx->central_pos;
        rd[r].n_kmers = rd[r].n_out = (int)m;
        stat_off[r + 1] = stat_off[r] + m;
    }
    const long long total = stat_off[n];
    if (total > 0 && (!norm_mean || !seq || !pvals_out || !pos_out)) return TB2_ERR_INVALID_ARG;
    de_novo_args(ctx, fm_offset, a);
    return run_de_novo(ctx, a, rd, total, P[F_OUT], P[F_POS], pvals_out, pos_out, nullptr);
}

extern "C" int tb2_de_novo_region_stats(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                                        const int64_t *mean_off, const uint8_t *seq,
                                        const int64_t *seq_off, const int64_t *read_start,
                                        const int8_t *strand, int64_t fm_offset, int64_t reg_start,
                                        int64_t reg_end, double *pvals_out, int64_t *pos_out,
                                        int64_t *stat_off, int32_t *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!stat_off) return TB2_ERR_INVALID_ARG;
    if ((rc = model_ok(ctx)) || (rc = region_args_ok(ctx, n_reads, strand, fm_offset, reg_start, reg_end)))
        return rc;
    RegionState &R = tb2_state(ctx->region);
    DeNovoArgs a;
    memset(&a, 0, sizeof(a));
    if ((rc = tb2_stage_reads(ctx, n_reads, norm_mean, mean_off, seq, seq_off, read_start, R.scratch + F_MEAN, a.f)))
        return rc;
    const int n = (int)n_reads;
    std::vector<DeNovoRead> rd;
    const long long total = de_novo_reads(ctx, n, (const long long *)mean_off, read_start, strand,
                                          fm_offset, reg_start, reg_end, rd, stat_off);
    if (total > 0 && (!pvals_out || !pos_out)) return TB2_ERR_INVALID_ARG;
    R.tests_n = 0;
    if (n == 0) return TB2_OK;
    de_novo_args(ctx, fm_offset, a);
    a.check = 1;
    if ((rc = run_de_novo(ctx, a, rd, total, R.tests_stat, R.tests_pos, pvals_out, pos_out, read_status)))
        return rc;
    R.tests_n = total;
    return TB2_OK;
}

extern "C" int tb2_batch_de_novo_region(tb2_ctx *ctx, const int64_t *read_start, const int8_t *strand,
                                        int64_t fm_offset, int64_t reg_start, int64_t reg_end,
                                        double *pvals_out, int64_t *pos_out, int64_t *stat_off,
                                        int32_t *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!read_start || !strand) return TB2_ERR_INVALID_ARG;
    if ((rc = model_ok(ctx))) return rc;
    BatchResultView v;
    if ((rc = tb2_batch_result_view(ctx, &v))) return rc;
    if ((rc = region_args_ok(ctx, v.n_reads, strand, fm_offset, reg_start, reg_end))) return rc;
    RegionState &R = tb2_state(ctx->region);
    const int n = v.n_reads;
    std::vector<DeNovoRead> rd;
    std::vector<int64_t> off(stat_off ? 0 : n + 1);
    const long long total = de_novo_reads(ctx, n, v.host_base_off, read_start, strand, fm_offset,
                                          reg_start, reg_end, rd, stat_off ? stat_off : off.data());
    R.tests_n = 0;
    if (n == 0) return TB2_OK;
    DeNovoArgs a;
    memset(&a, 0, sizeof(a));
    a.f.norm_mean = v.norm_mean; a.f.mean_off = v.base_off; a.f.seq = v.seq; a.f.seq_off = v.seq_off;
    a.rsq_status = v.status; a.rsq_stride = v.stride;
    de_novo_args(ctx, fm_offset, a);
    a.check = 1;
    if ((rc = run_de_novo(ctx, a, rd, total, R.tests_stat, R.tests_pos, pvals_out, pos_out, read_status)))
        return rc;
    R.tests_n = total;
    return TB2_OK;
}

extern "C" int tb2_sample_compare_region_stats(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                                               const int64_t *mean_off, const int64_t *read_start,
                                               const int8_t *strand, const double *ctrl_means,
                                               const double *ctrl_sds, int64_t fm_offset,
                                               int64_t reg_start, int64_t reg_end, double *pvals_out,
                                               int64_t *pos_out, int64_t *stat_off, int32_t *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!stat_off || !ctrl_means || !ctrl_sds || !mean_off || (n_reads > 0 && !read_start))
        return TB2_ERR_INVALID_ARG;
    if ((rc = region_args_ok(ctx, n_reads, strand, fm_offset, reg_start, reg_end))) return rc;
    const int n = (int)n_reads;
    if (mean_off[0] < 0) return TB2_ERR_INVALID_ARG;
    for (int r = 0; r < n; ++r) {
        const long long nb = mean_off[r + 1] - mean_off[r];
        if (nb < 0 || nb > INT_MAX) return TB2_ERR_INVALID_ARG;
    }
    if (mean_off[n] > mean_off[0] && !norm_mean) return TB2_ERR_INVALID_ARG;
    RegionState &R = tb2_state(ctx->region);
    auto &P = R.scratch;
    cudaStream_t s = ctx->stream;
    // host staging (:3713-3740): clip by fm_offset, flip '-' reads to genome order, and slice
    // the control levels over [reg_start - fm, reg_end + fm) to each read's positions
    const long long fm = fm_offset;
    std::vector<CompareRead> rd(n);
    std::vector<long long> seg_off(n + 1, 0);
    std::vector<double> m, cm, cs;
    for (int r = 0; r < n; ++r) {
        CompareRead &d = rd[r];
        memset(&d, 0, sizeof(d));
        d.seg0 = seg_off[r];
        d.skip = strand[r] < 0;
        const long long nb = mean_off[r + 1] - mean_off[r];
        if (!d.skip) {
            const long long start = read_start[r];
            const long long low_over = std::max(0LL, reg_start - (start + fm));
            const long long high_over = std::max(0LL, (start + nb - fm) - reg_end);
            const long long clip5 = strand[r] == 0 ? low_over : high_over;
            const long long clip3 = strand[r] == 0 ? high_over : low_over;
            const long long len = std::max(0LL, nb - clip5 - clip3);
            d.gstart = low_over ? reg_start - fm : start;
            d.n = (int)len;
            const double *rm = norm_mean + mean_off[r] + clip5;
            const long long c0 = d.gstart - reg_start + fm;
            for (long long i = 0; i < len; ++i) {
                m.push_back(strand[r] == 0 ? rm[i] : rm[len - 1 - i]);
                cm.push_back(ctrl_means[c0 + i]);
                cs.push_back(ctrl_sds[c0 + i]);
            }
        }
        seg_off[r + 1] = seg_off[r] + d.n;
    }
    const long long staged = seg_off[n];
    TB2_CUDA_TRY(ctx, P[F_MEAN].upload(m.data(), m.size(), s));
    TB2_CUDA_TRY(ctx, P[F_RM].upload(cm.data(), cm.size(), s));
    TB2_CUDA_TRY(ctx, P[F_RS].upload(cs.data(), cs.size(), s));
    TB2_CUDA_TRY(ctx, P[F_OFF].upload(seg_off.data(), seg_off.size(), s));
    TB2_CUDA_TRY(ctx, P[D_RD].upload(rd.data(), rd.size(), s));
    TB2_CUDA_TRY(ctx, P[D_STATUS].reserve((size_t)n * 4 + 8));
    TB2_CUDA_TRY(ctx, P[D_CNT].reserve((size_t)n * 4 + 8));
    TB2_CUDA_TRY(ctx, P[D_SOFF].reserve((size_t)(n + 1) * 8));
    TB2_CUDA_TRY(ctx, P[F_OUT].reserve((size_t)staged * 8 + 8));
    TB2_CUDA_TRY(ctx, P[F_LOGP].reserve((size_t)staged * 8 + 8));
    TB2_CUDA_TRY(ctx, R.tests_stat.reserve((size_t)staged * 8 + 8));
    TB2_CUDA_TRY(ctx, R.tests_pos.reserve((size_t)staged * 8 + 8));
    R.tests_n = 0;
    stat_off[0] = 0;
    if (n == 0) return TB2_OK;
    FisherArgs a;
    memset(&a, 0, sizeof(a));
    a.means = P[F_MEAN].as<double>(); a.rm = P[F_RM].as<double>(); a.rs = P[F_RS].as<double>();
    a.off = P[F_OFF].as<long long>();
    a.lag = (int)fm; a.final_clamp = 0; a.input_is_p = 0;
    a.out = P[F_OUT].as<double>(); a.logp = P[F_LOGP].as<double>();
    a.smallest = 1e-50;                                  // SMALLEST_PVAL _default_parameters.py:158
    const CompareRead *drd = P[D_RD].as<CompareRead>();
    int *cnt = P[D_CNT].as<int>(), *st = P[D_STATUS].as<int>();
    long long *soff = P[D_SOFF].as<long long>();
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, s));     // kernel time: tb2_last_timing
    k_fisher<false><<<n, 256, 0, s>>>(a);
    TB2_CHECK_LAUNCH(ctx);
    k_compare_compact<false><<<n, 256, 0, s>>>(drd, a.means, a.rm, a.rs, a.out, a.lag, cnt, st,
                                               nullptr, nullptr, nullptr);
    TB2_CHECK_LAUNCH(ctx);
    k_scan_offsets<<<1, 1024, 0, s>>>(cnt, soff, n);
    TB2_CHECK_LAUNCH(ctx);
    k_compare_compact<true><<<n, 256, 0, s>>>(drd, a.means, a.rm, a.rs, a.out, a.lag, nullptr, st,
                                              soff, R.tests_stat.as<double>(), R.tests_pos.as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(stat_off, soff, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, s));
    if (read_status)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(read_status, st, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    const long long total = stat_off[n];
    if (total > 0) {
        if (!pvals_out || !pos_out) return TB2_ERR_INVALID_ARG;
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pvals_out, R.tests_stat.p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, R.tests_pos.p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    }
    R.tests_n = total;
    return TB2_OK;
}

// the statistics of the last region call feed the open region's counters on the device
extern "C" int tb2_region_stats_add_tests(tb2_ctx *ctx, double single_read_thresh, double lower_thresh)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    RegionState &R = tb2_state(ctx->region);
    if (R.tests_n < 0 || isnan(single_read_thresh)) {
        ctx->err = "no de novo or sample-compare region call, or a NaN threshold";
        return TB2_ERR_INVALID_ARG;
    }
    return tb2_region_accumulate_dev(ctx, R.tests_n, R.tests_stat.as<double>(),
                                     R.tests_pos.as<long long>(), single_read_thresh, lower_thresh, 1);
}
