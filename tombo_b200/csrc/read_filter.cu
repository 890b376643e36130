// read_filter.cu -- the read filters of the resquiggle index on the device.
//
//   tb2_dwell_percentiles   np.percentile of each read's per-base dwells (the `stuck` filter,
//                           _filter_reads.py:61-69)
//   tb2_batch_read_filters  the reversible filters of _io_and_map_read (resquiggle.py:1437-1453)
//                           on the resident batch after tb2_batch_compute
//   tb2_read_mid_coverage   the per-(chromosome, strand) coverage of `level_coverage` and each
//                           read's mid-read value (_filter_reads.py:112-126)
//   tb2_coverage_build      that coverage, the one builder of the project (coverage.h); also
//                           behind tb2_coverage_runs (browser_tracks.cu)
//
// The percentiles take the two order statistics of numpy's linear interpolation from
// tb2_block_select2 (select.cuh), one 256-thread block per read, reading the lengths from global
// memory on every pass: reads of any length, nothing sorted or copied.  The coverage is a
// difference array and one device-wide prefix sum built on tb2_block_excl_scan.  Each group's
// differences sum to zero, so one scan over the concatenated groups is every group's scan.
#include "ctx.h"
#include "batch.h"
#include "read_filter.cuh"
#include "coverage.h"
#include <algorithm>
#include <climits>
#include <vector>

namespace {
enum { B_LENS = 0, B_OFF, B_PCTL, B_THR, B_OUT, B_CODE, B_START, B_END, B_DIFF, B_TSUM, B_TOFF, B_MID, B_COUNT };
}

struct ReadFilterState {
    DevBuf buf[B_COUNT];
};

namespace {

bool pctl_ok(int n_pctl, const double *pctl)
{
    if (n_pctl < 1 || !pctl) return false;
    for (int j = 0; j < n_pctl; ++j)
        if (!(pctl[j] >= 0.0 && pctl[j] <= 100.0)) return false;
    return true;
}

unsigned grid_of(long long n, int nt) { return (unsigned)std::max<long long>(1, (n + nt - 1) / nt); }

}  // namespace

static_assert(B_END == B_START + COV_END && B_DIFF == B_START + COV_DIFF && B_TSUM == B_START + COV_TSUM &&
              B_TOFF == B_START + COV_TOFF, "coverage workspace order");

int tb2_coverage_build(tb2_ctx *ctx, const char *what, DevBuf *ws, int64_t n_groups, const int64_t *grp_off,
                       const int64_t *start, const int64_t *end, std::vector<long long> &base)
{
    const int64_t n = grp_off[n_groups];
    // absolute positions in the concatenated coverage arrays
    std::vector<long long> as((size_t)n), ae((size_t)n);
    base.assign((size_t)n_groups + 1, 0);
    long long len = 0;
    for (int64_t g = 0; g < n_groups; ++g) {
        long long mx = 0;
        for (int64_t i = grp_off[g]; i < grp_off[g + 1]; ++i) {
            if (start[i] < 0 || end[i] <= start[i]) {
                ctx->err = std::string(what) + ": every read needs 0 <= start < end";
                return TB2_ERR_INVALID_ARG;
            }
            mx = std::max<long long>(mx, end[i]);
        }
        for (int64_t i = grp_off[g]; i < grp_off[g + 1]; ++i) { as[i] = len + start[i]; ae[i] = len + end[i]; }
        len += grp_off[g + 1] > grp_off[g] ? mx + 1 : 0;
        if (len > (1LL << 40)) { ctx->err = std::string(what) + ": coverage arrays too long"; return TB2_ERR_INVALID_ARG; }
        base[(size_t)g + 1] = len;
    }
    const long long n_tiles = (len + RF_TILE - 1) / RF_TILE;
    cudaStream_t q = ctx->stream;
    TB2_RESERVE(ctx, what, ws[COV_DIFF], (size_t)len * 4);
    TB2_RESERVE(ctx, what, ws[COV_TSUM], (size_t)n_tiles * 8);
    TB2_RESERVE(ctx, what, ws[COV_TOFF], (size_t)(n_tiles + 1) * 8);
    TB2_CUDA_TRY(ctx, ws[COV_START].upload(as.data(), (size_t)n, q));
    TB2_CUDA_TRY(ctx, ws[COV_END].upload(ae.data(), (size_t)n, q));
    int *cov = ws[COV_DIFF].as<int>();
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(cov, 0, (size_t)len * 4, q));
    k_rf_cov_diff<<<grid_of(n, 256), 256, 0, q>>>(ws[COV_START].as<long long>(), ws[COV_END].as<long long>(), n, cov);
    TB2_CHECK_LAUNCH(ctx);
    return tb2_coverage_scan(ctx, what, ws, cov, len);
}

int tb2_coverage_scan(tb2_ctx *ctx, const char *what, DevBuf *ws, int *x, long long len)
{
    const long long n_tiles = (len + RF_TILE - 1) / RF_TILE;
    cudaStream_t q = ctx->stream;
    TB2_RESERVE(ctx, what, ws[COV_TSUM], (size_t)n_tiles * 8);
    TB2_RESERVE(ctx, what, ws[COV_TOFF], (size_t)(n_tiles + 1) * 8);
    k_rf_tile_sum<<<(unsigned)n_tiles, RF_NT, 0, q>>>(x, len, ws[COV_TSUM].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    k_scan_offsets<long long><<<1, 1024, 0, q>>>(ws[COV_TSUM].as<long long>(), ws[COV_TOFF].as<long long>(), n_tiles);
    TB2_CHECK_LAUNCH(ctx);
    k_rf_tile_scan<<<(unsigned)n_tiles, RF_NT, 0, q>>>(x, len, ws[COV_TOFF].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

extern "C" int tb2_dwell_percentiles(tb2_ctx *ctx, int64_t n_reads, const int64_t *lens,
                                     const int64_t *len_off, int n_pctl, const double *pctl,
                                     double *out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n_reads < 0 || n_reads > INT_MAX || !pctl_ok(n_pctl, pctl) || (n_reads > 0 && (!len_off || !lens || !out)))
        return TB2_ERR_INVALID_ARG;
    if (n_reads == 0) return TB2_OK;
    if (len_off[0] < 0) { ctx->err = "read filters: negative length offset"; return TB2_ERR_INVALID_ARG; }
    for (int64_t r = 0; r < n_reads; ++r)
        if (len_off[r + 1] <= len_off[r] || len_off[r + 1] - len_off[r] > INT_MAX) {
            ctx->err = "read filters: every read needs 1 to 2^31 - 1 lengths, in increasing offsets";
            return TB2_ERR_INVALID_ARG;
        }
    ReadFilterState &S = tb2_state(ctx->read_filter);
    DevBuf *B = S.buf;
    cudaStream_t q = ctx->stream;
    const int64_t total = len_off[n_reads] - len_off[0];
    TB2_RESERVE(ctx, "read filters", B[B_LENS], (size_t)total * 8 + 8);
    TB2_RESERVE(ctx, "read filters", B[B_OFF], (size_t)(n_reads + 1) * 8);
    TB2_RESERVE(ctx, "read filters", B[B_PCTL], (size_t)n_pctl * 8);
    TB2_RESERVE(ctx, "read filters", B[B_OUT], (size_t)n_reads * n_pctl * 8);
    TB2_CUDA_TRY(ctx, B[B_LENS].upload(lens + len_off[0], (size_t)total, q));
    TB2_CUDA_TRY(ctx, B[B_OFF].upload(len_off, (size_t)n_reads + 1, q));
    TB2_CUDA_TRY(ctx, B[B_PCTL].upload(pctl, (size_t)n_pctl, q));
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));          // kernel time: tb2_last_timing
    k_rf_dwell_pctl<<<(unsigned)n_reads, TB2_SEL_THREADS, 0, q>>>(
        B[B_LENS].as<long long>(), B[B_OFF].as<long long>(), n_pctl, B[B_PCTL].as<double>(),
        B[B_OUT].as<double>());
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(out, B[B_OUT].p, (size_t)n_reads * n_pctl * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}

extern "C" int tb2_batch_read_filters(tb2_ctx *ctx, double sig_match_thresh, int n_pctl,
                                      const double *pctl, const double *thresh, int8_t *code,
                                      double *pctl_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!code || n_pctl < 0 || (n_pctl > 0 && (!pctl_ok(n_pctl, pctl) || !thresh)))
        return TB2_ERR_INVALID_ARG;
    BatchResultView v;
    if ((rc = tb2_batch_result_view(ctx, &v))) return rc;
    ReadFilterState &S = tb2_state(ctx->read_filter);
    DevBuf *B = S.buf;
    cudaStream_t q = ctx->stream;
    const int n = v.n_reads;
    TB2_RESERVE(ctx, "read filters", B[B_PCTL], (size_t)n_pctl * 8 + 8);
    TB2_RESERVE(ctx, "read filters", B[B_THR], (size_t)n_pctl * 8 + 8);
    TB2_RESERVE(ctx, "read filters", B[B_CODE], (size_t)n + 8);
    if (pctl_out) TB2_RESERVE(ctx, "read filters", B[B_OUT], (size_t)n * n_pctl * 8 + 8);
    TB2_CUDA_TRY(ctx, B[B_PCTL].upload(pctl, (size_t)n_pctl, q));
    TB2_CUDA_TRY(ctx, B[B_THR].upload(thresh, (size_t)n_pctl, q));
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));
    k_rf_batch<<<(unsigned)n, TB2_SEL_THREADS, 0, q>>>(
        v.segs, v.base_off, v.status, v.stride, v.score, sig_match_thresh, n_pctl,
        B[B_PCTL].as<double>(), B[B_THR].as<double>(), B[B_CODE].as<signed char>(),
        pctl_out ? B[B_OUT].as<double>() : nullptr);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(code, B[B_CODE].p, (size_t)n, cudaMemcpyDeviceToHost, q));
    if (pctl_out && n_pctl > 0)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pctl_out, B[B_OUT].p, (size_t)n * n_pctl * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}

extern "C" int tb2_read_mid_coverage(tb2_ctx *ctx, int64_t n_groups, const int64_t *grp_off,
                                     const int64_t *start, const int64_t *end, int64_t *mid_cov)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n_groups < 0 || (n_groups > 0 && !grp_off)) return TB2_ERR_INVALID_ARG;
    if (n_groups == 0) return TB2_OK;
    if (grp_off[0] != 0) { ctx->err = "read filters: group offsets must start at 0"; return TB2_ERR_INVALID_ARG; }
    for (int64_t g = 0; g < n_groups; ++g)
        if (grp_off[g + 1] < grp_off[g]) { ctx->err = "read filters: decreasing group offsets"; return TB2_ERR_INVALID_ARG; }
    const int64_t n = grp_off[n_groups];
    if (n > INT_MAX) { ctx->err = "read filters: more than 2^31 - 1 reads"; return TB2_ERR_INVALID_ARG; }
    if (n == 0) return TB2_OK;
    if (!start || !end || !mid_cov) return TB2_ERR_INVALID_ARG;
    ReadFilterState &S = tb2_state(ctx->read_filter);
    DevBuf *B = S.buf;
    cudaStream_t q = ctx->stream;
    TB2_RESERVE(ctx, "read filters", B[B_MID], (size_t)n * 8);
    std::vector<long long> base;
    if ((rc = tb2_coverage_build(ctx, "read filters", B + B_START, n_groups, grp_off, start, end, base))) return rc;
    int *cov = B[B_DIFF].as<int>();
    long long *ds = B[B_START].as<long long>(), *de = B[B_END].as<long long>();
    k_rf_mid<<<grid_of(n, 256), 256, 0, q>>>(ds, de, n, cov, B[B_MID].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(mid_cov, B[B_MID].p, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}
