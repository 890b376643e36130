// browser_tracks.cu -- the read-derived genome browser tracks of `tombo text_output
// browser_files` on the device.
//
//   tb2_coverage_runs     every (chromosome, strand) group's read coverage as runs of equal
//                         value (TomboReads.iter_coverage_regions, tombo_helper.py:1394-1453)
//   tb2_slot_sums_begin / _add / _means
//                         per-position means of an Events slot over the reads of one
//                         (chromosome, strand), accumulated across calls in read order
//                         (get_mean_slot_genome_centric, tombo_helper.py:1661-1676)
//
// The coverage comes from the project's one coverage builder (coverage.h); the runs are a flag
// per entry, the same in-place scan, and a scatter of (start, coverage) per run head.
//
// The slot sums keep the reference's summation order exactly: numpy's slice-add visits the
// reads in index order, so each position's sum is a sequential fp64 sum of its values in read
// order, from +0.0.  One add call lays its values out in read-major order, sorts them by
// position with the stable LSD radix sort of radix_sort.cuh (skipping the digits a single bin
// holds), and gives one thread to each touched position: it loads the stored running sum and
// adds that position's values one by one.  Running sums and counts stay on the device between
// calls, so the caller never holds a whole chromosome's Events.  DESIGN.md §3.
#include "ctx.h"
#include "coverage.h"
#include "browser_tracks.cuh"
#include <algorithm>
#include <climits>
#include <vector>

namespace {
enum { R_FLAG = 0, R_BASE, R_START, R_COV, R_OFF, R_COUNT };
enum { S_SUMS = 0, S_CNT, S_OFF, S_START, S_REV, S_VALS, S_KEY0, S_KEY1, S_VAL0, S_VAL1, S_THIST, S_TOFF,
       S_HIST, S_MEAN, S_COUNT };
}

struct BrowserTracksState {
    DevBuf cov[COV_BUFS];          // coverage workspace (coverage.h)
    DevBuf runs[R_COUNT];
    DevBuf slot[S_COUNT];
    long long chrm_len = -1;       // open accumulation's length; -1 none
    bool failed = false;           // an add failed since begin
};

namespace {

unsigned grid_of(long long n, int nt) { return (unsigned)std::max<long long>(1, (n + nt - 1) / nt); }

}  // namespace

extern "C" int tb2_coverage_runs(tb2_ctx *ctx, int64_t n_groups, const int64_t *grp_off, const int64_t *start,
                                 const int64_t *end, int64_t *run_off, int64_t *run_start, int64_t *run_cov)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n_groups < 0 || !run_off || (n_groups > 0 && !grp_off)) return TB2_ERR_INVALID_ARG;
    if (n_groups == 0) { run_off[0] = 0; return TB2_OK; }
    if (grp_off[0] != 0) { ctx->err = "coverage runs: group offsets must start at 0"; return TB2_ERR_INVALID_ARG; }
    for (int64_t g = 0; g < n_groups; ++g)
        if (grp_off[g + 1] < grp_off[g]) { ctx->err = "coverage runs: decreasing group offsets"; return TB2_ERR_INVALID_ARG; }
    const int64_t n = grp_off[n_groups];
    if (n > INT_MAX) { ctx->err = "coverage runs: more than 2^31 - 1 reads"; return TB2_ERR_INVALID_ARG; }
    if (n == 0) {
        std::fill(run_off, run_off + n_groups + 1, 0);
        return TB2_OK;
    }
    if (!start || !end || !run_start || !run_cov) return TB2_ERR_INVALID_ARG;
    BrowserTracksState &S = tb2_state(ctx->browser_tracks);
    DevBuf *R = S.runs;
    cudaStream_t q = ctx->stream;
    // runs are at most 2 n + n_groups: the extra 1 per group bounds the reserve up front
    TB2_RESERVE(ctx, "coverage runs", R[R_START], (size_t)(2 * n + n_groups) * 8);
    TB2_RESERVE(ctx, "coverage runs", R[R_COV], (size_t)(2 * n + n_groups) * 8);
    TB2_RESERVE(ctx, "coverage runs", R[R_OFF], (size_t)(n_groups + 1) * 8);
    std::vector<long long> base;
    if ((rc = tb2_coverage_build(ctx, "coverage runs", S.cov, n_groups, grp_off, start, end, base))) return rc;
    const long long len = base[(size_t)n_groups];
    TB2_RESERVE(ctx, "coverage runs", R[R_FLAG], (size_t)len * 4);
    TB2_CUDA_TRY(ctx, R[R_BASE].upload(base.data(), base.size(), q));
    const int *cov = S.cov[COV_DIFF].as<int>();
    int *flag = R[R_FLAG].as<int>();
    const long long *d_base = R[R_BASE].as<long long>();
    k_bt_run_flags<<<grid_of(len, 256), 256, 0, q>>>(cov, len, flag);
    TB2_CHECK_LAUNCH(ctx);
    k_bt_run_ends<<<grid_of(n_groups, 256), 256, 0, q>>>(d_base, n_groups, flag);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_coverage_scan(ctx, "coverage runs", S.cov, flag, len))) return rc;
    k_bt_run_scatter<<<grid_of(len, 256), 256, 0, q>>>(cov, flag, len, d_base, n_groups, R[R_START].as<long long>(),
                                                       R[R_COV].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    k_bt_run_off<<<grid_of(n_groups + 1, 256), 256, 0, q>>>(flag, d_base, n_groups, R[R_OFF].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(run_off, R[R_OFF].p, (size_t)(n_groups + 1) * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    const size_t m = (size_t)run_off[n_groups];
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(run_start, R[R_START].p, m * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(run_cov, R[R_COV].p, m * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}

extern "C" int tb2_slot_sums_begin(tb2_ctx *ctx, int64_t chrm_len)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    BrowserTracksState &S = tb2_state(ctx->browser_tracks);
    S.chrm_len = -1;
    S.failed = false;
    if (chrm_len < 0 || chrm_len > (1LL << 40)) {
        ctx->err = "slot sums: chromosome length outside [0, 2^40]";
        return TB2_ERR_INVALID_ARG;
    }
    DevBuf *B = S.slot;
    cudaStream_t q = ctx->stream;
    TB2_RESERVE(ctx, "slot sums", B[S_SUMS], (size_t)chrm_len * 8 + 8);
    TB2_RESERVE(ctx, "slot sums", B[S_CNT], (size_t)chrm_len * 4 + 8);
    // all-zero bytes: +0.0 sums and zero counts
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(B[S_SUMS].p, 0, (size_t)chrm_len * 8, q));
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(B[S_CNT].p, 0, (size_t)chrm_len * 4, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    S.chrm_len = chrm_len;
    return TB2_OK;
}

namespace {

// the body of tb2_slot_sums_add; any failure here invalidates the accumulation
int slot_add(tb2_ctx *ctx, BrowserTracksState &S, int64_t n_reads, const int64_t *start, const int64_t *val_off,
             const double *vals, const uint8_t *reverse)
{
    if (S.chrm_len < 0 || S.failed) {
        ctx->err = "slot sums: tb2_slot_sums_begin has not been called, or an add failed since";
        return TB2_ERR_INVALID_ARG;
    }
    if (n_reads < 0 || (n_reads > 0 && (!start || !val_off || !reverse))) return TB2_ERR_INVALID_ARG;
    if (n_reads == 0) return TB2_OK;
    long long kmin = LLONG_MAX, kmax = -1;
    for (int64_t r = 0; r < n_reads; ++r) {
        const long long nv = val_off[r + 1] - val_off[r];
        if (nv < 0) { ctx->err = "slot sums: decreasing value offsets"; return TB2_ERR_INVALID_ARG; }
        if (start[r] < 0 || start[r] > S.chrm_len - nv) {
            ctx->err = "slot sums: a read's values run outside [0, chrm_len)";
            return TB2_ERR_INVALID_ARG;
        }
        if (nv > 0) {
            kmin = std::min<long long>(kmin, start[r]);
            kmax = std::max<long long>(kmax, start[r] + nv - 1);
        }
    }
    const long long total = val_off[n_reads] - val_off[0];
    if (total == 0) return TB2_OK;
    if (total > INT_MAX) { ctx->err = "slot sums: more than 2^31 - 1 values in one add"; return TB2_ERR_INVALID_ARG; }
    if (!vals) return TB2_ERR_INVALID_ARG;
    DevBuf *B = S.slot;
    cudaStream_t q = ctx->stream;
    const long long n_tiles = (total + RADIX_TILE - 1) / RADIX_TILE;
    std::vector<long long> off((size_t)n_reads + 1);
    for (int64_t r = 0; r <= n_reads; ++r) off[(size_t)r] = val_off[r] - val_off[0];
    TB2_RESERVE(ctx, "slot sums", B[S_KEY0], (size_t)total * 8);
    TB2_RESERVE(ctx, "slot sums", B[S_KEY1], (size_t)total * 8);
    TB2_RESERVE(ctx, "slot sums", B[S_VAL0], (size_t)total * 8);
    TB2_RESERVE(ctx, "slot sums", B[S_VAL1], (size_t)total * 8);
    TB2_RESERVE(ctx, "slot sums", B[S_THIST], (size_t)256 * n_tiles * 4);
    TB2_RESERVE(ctx, "slot sums", B[S_TOFF], (size_t)256 * n_tiles * 8);
    TB2_RESERVE(ctx, "slot sums", B[S_HIST], (size_t)BT_DIGITS * 256 * 8 + 8);
    TB2_CUDA_TRY(ctx, B[S_OFF].upload(off.data(), off.size(), q));
    TB2_CUDA_TRY(ctx, B[S_START].upload(start, (size_t)n_reads, q));
    TB2_CUDA_TRY(ctx, B[S_REV].upload(reverse, (size_t)n_reads, q));
    TB2_CUDA_TRY(ctx, B[S_VALS].upload(vals + val_off[0], (size_t)total, q));
    unsigned long long *gh = B[S_HIST].as<unsigned long long>();
    int *overflow = (int *)(gh + BT_DIGITS * 256);
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));          // kernel time: tb2_last_timing
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(gh, 0, (size_t)BT_DIGITS * 256 * 8 + 8, q));
    const unsigned egrid = (unsigned)std::min<long long>(grid_of(total, 256), 8LL * ctx->sm_count);
    k_bt_entries<<<egrid, 256, 0, q>>>(B[S_VALS].as<double>(), B[S_OFF].as<long long>(), B[S_START].as<long long>(),
                                       B[S_REV].as<unsigned char>(), n_reads, total, kmin,
                                       B[S_KEY0].as<unsigned long long>(), B[S_VAL0].as<double>(), gh);
    TB2_CHECK_LAUNCH(ctx);
    std::vector<unsigned long long> h((size_t)BT_DIGITS * 256);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(h.data(), gh, h.size() * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    // a digit that one bin holds keeps the order and is skipped
    int cur = 0;
    for (int d = 0; d < BT_DIGITS && (kmax - kmin) >> (8 * d); ++d) {
        const unsigned long long *ph = h.data() + (size_t)d * 256;
        if (std::any_of(ph, ph + 256, [&](unsigned long long c) { return c == (unsigned long long)total; })) continue;
        unsigned long long *kin = B[S_KEY0 + cur].as<unsigned long long>(), *kout = B[S_KEY1 - cur].as<unsigned long long>();
        double *vin = B[S_VAL0 + cur].as<double>(), *vout = B[S_VAL1 - cur].as<double>();
        k_radix_tile_hist<<<(unsigned)n_tiles, RADIX_NT, 0, q>>>(kin, vin, total, 8 * d, B[S_THIST].as<unsigned int>(),
                                                                n_tiles);
        TB2_CHECK_LAUNCH(ctx);
        k_radix_tile_scan<<<256, RADIX_NT, 0, q>>>(B[S_THIST].as<unsigned int>(), n_tiles, gh + (size_t)d * 256,
                                                   B[S_TOFF].as<unsigned long long>());
        TB2_CHECK_LAUNCH(ctx);
        k_radix_scatter_pass<<<(unsigned)n_tiles, RADIX_NT, 0, q>>>(kin, vin, kout, vout, total, 8 * d,
                                                                    B[S_TOFF].as<unsigned long long>(), n_tiles);
        TB2_CHECK_LAUNCH(ctx);
        cur ^= 1;
    }
    k_bt_accumulate<<<grid_of(total, 256), 256, 0, q>>>(B[S_KEY0 + cur].as<unsigned long long>(),
                                                        B[S_VAL0 + cur].as<double>(), total, kmin,
                                                        B[S_SUMS].as<double>(), B[S_CNT].as<int>(), overflow);
    TB2_CHECK_LAUNCH(ctx);
    int rc = tb2_record_kernel_time(ctx);
    if (rc) return rc;
    int ovf = 0;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(&ovf, overflow, 4, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    if (ovf) { ctx->err = "slot sums: coverage above 2^31 - 1 at a position"; return TB2_ERR_INVALID_ARG; }
    return TB2_OK;
}

}  // namespace

extern "C" int tb2_slot_sums_add(tb2_ctx *ctx, int64_t n_reads, const int64_t *start, const int64_t *val_off,
                                 const double *vals, const uint8_t *reverse)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    BrowserTracksState &S = tb2_state(ctx->browser_tracks);
    rc = slot_add(ctx, S, n_reads, start, val_off, vals, reverse);
    if (rc) S.failed = true;
    return rc;
}

extern "C" int tb2_slot_sums_means(tb2_ctx *ctx, double *out_mean)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    BrowserTracksState &S = tb2_state(ctx->browser_tracks);
    if (S.chrm_len < 0) { ctx->err = "slot sums: tb2_slot_sums_begin has not been called"; return TB2_ERR_INVALID_ARG; }
    if (S.failed) { ctx->err = "slot sums: an add failed since tb2_slot_sums_begin"; return TB2_ERR_INVALID_ARG; }
    const long long n = S.chrm_len;
    if (n == 0) return TB2_OK;
    if (!out_mean) return TB2_ERR_INVALID_ARG;
    DevBuf *B = S.slot;
    cudaStream_t q = ctx->stream;
    TB2_RESERVE(ctx, "slot sums", B[S_MEAN], (size_t)n * 8);
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));
    k_bt_means<<<grid_of(n, 256), 256, 0, q>>>(B[S_SUMS].as<double>(), B[S_CNT].as<int>(), n, B[S_MEAN].as<double>());
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(out_mean, B[S_MEAN].p, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}
