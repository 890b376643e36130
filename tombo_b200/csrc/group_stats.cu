// group_stats.cu -- level_sample_compare and control-sample reference levels on the device.
//
//   tb2_group_reg_stats   compute_group_reg_stats tombo_stats.py:4335-4393 with
//                         compute_ks_tests / compute_u_tests / compute_t_tests :4236-4324,
//                         calc_window_fishers_method / calc_window_means :2252-2287
//   tb2_reads_ref_levels  get_reads_ref :3627-3673 (+ compute_posterior_samp_dists
//                         :3572-3625)
//
// One region per call.  Reads arrive as ragged genome-ordered level arrays (levels, off,
// start).  Steps (DESIGN.md §3 "Level tests"):
//   1. k_count: non-NaN levels per position (samp_cov / ctrl_cov), atomics.
//   2. k_compact (one block): positions inside coverage runs that are at least
//      min_run long, ascending; CSR offsets of their values; run (segment) offsets.
//   3. k_scatter: each kept level goes to its position's CSR slot with its read ordinal.
//   4. k_group_pos / k_ref_pos: one block per position; values sorted in shared memory
//      (bitonic, in place), or in place in the global CSR when the position's coverage
//      exceeds the shared buffer -- same code, exact either way.
//   5. windows over each run: k_fisher (fisher.cuh) for p-values, k_window_mean for the
//      *_stat_test variants; k_ref_final for the posterior and the sd == 0 mask.
#include "batch.h"
#include "level_gather.cuh"
#include "fisher.cuh"
#include "special.cuh"
#include <cmath>

namespace {
// per-call scratch of tb2_group_reg_stats / tb2_reads_ref_levels; nothing reads it after a
// call returns
// (the gather's slots, then the control sample's arrays and the results)
enum { G_LV_C = G_GATHER_COUNT, G_OFF_C, G_ST_C, G_RES, G_PRI_M, G_PRI_S, G_REF, G_COUNT };
}  // namespace
struct GroupState { DevBuf scratch[G_COUNT]; };

namespace {

constexpr int G_SH = 5632;         // doubles of shared memory per position (group tests)

// ---------------------------------------------------------------------------
// per-position statistics
// ---------------------------------------------------------------------------
__device__ __forceinline__ int upper_bound(const double *a, int n, double x)
{
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] <= x) lo = mid + 1; else hi = mid; }
    return lo;
}

__device__ __forceinline__ int lower_bound(const double *a, int n, double x)
{
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
    return lo;
}

// ndtr (scipy.special) as norm.cdf evaluates it
__device__ __forceinline__ double ndtr(double a)
{
    const double x = a * 0.70710678118654752440, z = fabs(x);
    if (z < 0.70710678118654752440) return 0.5 + 0.5 * erf(x);
    const double y = 0.5 * erfc(z);
    return x > 0 ? 1.0 - y : y;
}

__global__ void __launch_bounds__(BT)
k_group_pos(const long long *offs, const long long *offc, long long tot_s, double *vals, int test,
            int return_stat, double *stat)
{
    __shared__ double sh[G_SH];
    __shared__ double red_d[BT / 32];
    __shared__ long long red_l[BT / 32];
    const int o = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ns = (int)(offs[o + 1] - offs[o]), nc = (int)(offc[o + 1] - offc[o]);
    double *s = vals + offs[o], *c = vals + tot_s + offc[o];
    if (ns + nc <= G_SH) {
        for (int i = tid; i < ns; i += BT) sh[i] = s[i];
        for (int i = tid; i < nc; i += BT) sh[ns + i] = c[i];
        s = sh; c = sh + ns;
        __syncthreads();
    }
    block_sort<double, double>(s, nullptr, ns);
    block_sort<double, double>(c, nullptr, nc);
    double res = NAN;
    if (test == 0) {
        // KS :4236-4255: d = max |searchsorted(s, all, 'right')/n_s - searchsorted(c, ..)/n_c|
        double d = 0.0;
        for (int i = tid; i < ns + nc; i += BT) {
            const double x = i < ns ? s[i] : c[i - ns];
            const double e = fabs((double)upper_bound(s, ns, x) / (double)ns -
                                  (double)upper_bound(c, nc, x) / (double)nc);
            d = e > d ? e : d;
        }
        for (int w = 16; w > 0; w >>= 1) { const double u = __shfl_xor_sync(0xffffffffu, d, w); d = u > d ? u : d; }
        if (lane == 0) red_d[warp] = d;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < BT / 32; ++w) d = red_d[w] > d ? red_d[w] : d;
            if (return_stat) res = 1.0 - d;
            else {
                const double en = sqrt((double)((long long)ns * nc) / (double)(ns + nc));
                res = tb2_kolmogorov_sf((en + 0.12 + 0.11 / en) * d);
            }
        }
    } else if (test == 1) {
        // U :4266-4291: rank sum - n_s(n_s+1)/2 = sum_i #{c < s_i} (stable rule: sample first)
        long long cnt = 0;
        for (int i = tid; i < ns; i += BT) cnt += lower_bound(c, nc, s[i]);
        for (int w = 16; w > 0; w >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, w);
        if (lane == 0) red_l[warp] = cnt;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < BT / 32; ++w) cnt += red_l[w];
            const long long half = (long long)ns * (ns + 1) / 2, tot = (long long)ns * nc;
            const double u1 = (double)(cnt + half) - (double)half;
            const double u2 = (double)tot - u1;
            const double u = u2 < u1 ? u2 : u1;
            const double mu = (double)tot / 2.0;
            if (return_stat) res = (u - mu) / mu;
            else {
                const double rhou = sqrt(tb2_div12((unsigned __int128)tot * (unsigned __int128)(tot + 1)));
                res = ndtr((u - mu) / rhou) * 2.0;
            }
        }
    } else if (tid == 0) {
        // t :4302-4324 on the sorted values
        double sm, ssd, cm, csd;
        mean_std(s, ns, sm, ssd);
        mean_std(c, nc, cm, csd);
        if (return_stat) {
            const double den = sqrt(((ssd * ssd) + (csd * csd)) / 2.0);
            res = den > 0.0 ? -fabs(sm - cm) / den : NAN;    // the reference raises here
        } else if (ns + nc > 2) {
            const double sp = sqrt((((double)(ns - 1) * (ssd * ssd)) + (double)(nc - 1) * (csd * csd)) /
                                   (double)(ns + nc - 2));
            if (sp > 0.0) {
                const double t = -fabs(sm - cm) / (sp * sqrt((1.0 / (double)ns) + (1.0 / (double)nc)));
                res = tb2_t_two_sided_p((double)(ns + nc - 2), t);
            }
        }
    }
    if (tid == 0) stat[o] = res;
}

// calc_window_means :2273-2287: np.mean over 2 lag + 1 values (pairwise sum / width)
__global__ void __launch_bounds__(256)
k_window_mean(const double *in, const long long *seg, int lag, double *out)
{
    const long long o = seg[blockIdx.x];
    const int n = (int)(seg[blockIdx.x + 1] - o), width = 2 * lag + 1;
    for (int i = threadIdx.x; i < n; i += 256)
        out[o + i] = (i >= lag && i < n - lag) ? tb2_pairwise_sum(in + o + i - lag, width) / (double)width : NAN;
}

// uncovered -> NaN; compute_posterior_samp_dists :3589-3594; sd == 0 -> NaN (:3668-3671)
__global__ void k_ref_final(const int *map, const int *cov, long long n, const double *pm,
                            const double *ps, double w0, double w1, double *means, double *sds,
                            long long *cov_out)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    double m = map[p] >= 0 ? means[p] : NAN, s = map[p] >= 0 ? sds[p] : NAN;
    const double c = (double)cov[p];
    if (pm) {
        m = ((w0 * pm[p]) + (c * m)) / (w0 + c);
        s = ((w1 * ps[p]) + (c * s)) / (w1 + c);
    }
    if (s == 0.0) { m = NAN; s = NAN; }
    means[p] = m; sds[p] = s; cov_out[p] = cov[p];
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
}  // namespace

extern "C" int tb2_group_reg_stats(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len,
                                   int64_t n_samp, const double *samp_levels, const int64_t *samp_off,
                                   const int64_t *samp_start, int64_t n_ctrl, const double *ctrl_levels,
                                   const int64_t *ctrl_off, const int64_t *ctrl_start, int test,
                                   int return_stat, int64_t min_test_reads, int64_t fm_offset, int64_t cap,
                                   int64_t *pos_out, double *stat_out, int64_t *cov_out,
                                   int64_t *ctrl_cov_out, int64_t *n_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (reg_len < 1 || reg_len > MAX_REG_LEN || test < 0 || test > 2 || min_test_reads < 1 ||
        min_test_reads > (1LL << 31) - 1 || fm_offset < 0 || fm_offset > MAX_REG_LEN || cap < 0 || !n_out ||
        (cap > 0 && (!pos_out || !stat_out || !cov_out || !ctrl_cov_out)))
        return TB2_ERR_INVALID_ARG;
    if ((rc = check_sample(n_samp, samp_levels, samp_off, samp_start))) return rc;
    if ((rc = check_sample(n_ctrl, ctrl_levels, ctrl_off, ctrl_start))) return rc;
    auto &P = tb2_state(ctx->group).scratch;
    cudaStream_t q = ctx->stream;
    Sample a, b;
    if ((rc = upload_sample(ctx, P, G_LV, n_samp, samp_levels, samp_off, samp_start, a))) return rc;
    if ((rc = upload_sample(ctx, P, G_LV_C, n_ctrl, ctrl_levels, ctrl_off, ctrl_start, b))) return rc;
    long long hdr[4];
    if ((rc = gather(ctx, P, reg_start, reg_len, a, &b, (int)min_test_reads, (int)(2 * fm_offset + 1), false, hdr)))
        return rc;
    const long long n = reg_len, n_pos = hdr[0], n_seg = hdr[1];
    *n_out = n_pos;
    if (n_pos == 0) return tb2_record_kernel_time(ctx);
    long long *idx = P[G_IDX].as<long long>();
    const long long *offs = idx + 3 * n, *offc = offs + n + 1, *seg = offc + n + 1;
    TB2_CUDA_TRY(ctx, P[G_RES].reserve((size_t)n_pos * 3 * 8));
    double *stat = P[G_RES].as<double>(), *out = stat + n_pos, *logp = out + n_pos;
    k_group_pos<<<(unsigned)n_pos, BT, 0, q>>>(offs, offc, hdr[2], P[G_VAL].as<double>(), test,
                                               return_stat ? 1 : 0, stat);
    TB2_CHECK_LAUNCH(ctx);
    const double *res = stat;
    if (fm_offset > 0) {
        if (!return_stat) {
            FisherArgs fa;
            memset(&fa, 0, sizeof(fa));
            fa.means = stat; fa.off = seg; fa.lag = (int)fm_offset; fa.input_is_p = 1;
            fa.smallest = 1e-50;                              // SMALLEST_PVAL _default_parameters.py:158
            fa.logp = logp; fa.out = out;
            k_fisher<false><<<(unsigned)n_seg, 256, 0, q>>>(fa);
        } else {
            k_window_mean<<<(unsigned)n_seg, 256, 0, q>>>(stat, seg, (int)fm_offset, out);
        }
        TB2_CHECK_LAUNCH(ctx);
        res = out;
    }
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    const size_t m = (size_t)std::min<long long>(n_pos, cap);
    if (m) {
        // positions are relative to reg_start on the device
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, idx, m * 8, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cov_out, idx + n, m * 8, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(ctrl_cov_out, idx + 2 * n, m * 8, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(stat_out, res, m * 8, cudaMemcpyDeviceToHost, q));
    }
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    for (size_t i = 0; i < m; ++i) pos_out[i] += reg_start;
    return n_pos > cap ? TB2_ERR_CAPACITY : TB2_OK;
}

extern "C" int tb2_reads_ref_levels(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len, int64_t n_reads,
                                    const double *levels, const int64_t *off, const int64_t *start,
                                    int64_t min_test_reads, int est_mean, const double *prior_means,
                                    const double *prior_sds, double mean_prior_weight,
                                    double sd_prior_weight, double *means_out, double *sds_out,
                                    int64_t *cov_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (reg_len < 1 || reg_len > MAX_REG_LEN || min_test_reads < 1 || min_test_reads > (1LL << 31) - 1 ||
        !means_out || !sds_out || !cov_out || (!prior_means != !prior_sds))
        return TB2_ERR_INVALID_ARG;
    if ((rc = check_sample(n_reads, levels, off, start))) return rc;
    auto &P = tb2_state(ctx->group).scratch;
    cudaStream_t q = ctx->stream;
    Sample a;
    if ((rc = upload_sample(ctx, P, G_LV, n_reads, levels, off, start, a))) return rc;
    const long long n = reg_len;
    const double *pm = nullptr, *ps = nullptr;
    if (prior_means) {
        TB2_CUDA_TRY(ctx, P[G_PRI_M].upload(prior_means, (size_t)n, q));
        TB2_CUDA_TRY(ctx, P[G_PRI_S].upload(prior_sds, (size_t)n, q));
        pm = P[G_PRI_M].as<double>(); ps = P[G_PRI_S].as<double>();
    }
    long long hdr[4];
    if ((rc = gather(ctx, P, reg_start, reg_len, a, nullptr, (int)min_test_reads, 1, true, hdr))) return rc;
    const long long n_pos = hdr[0];
    long long *idx = P[G_IDX].as<long long>();
    TB2_CUDA_TRY(ctx, P[G_REF].reserve((size_t)n * 3 * 8));
    double *means = P[G_REF].as<double>(), *sds = means + n;
    long long *cov = (long long *)(sds + n);
    if (n_pos) {
        k_ref_pos<<<(unsigned)n_pos, BT, 0, q>>>(idx, idx + 3 * n, P[G_VAL].as<double>(), P[G_RD].as<int>(),
                                                 P[G_SQ].as<double>(), est_mean ? 1 : 0, means, sds);
        TB2_CHECK_LAUNCH(ctx);
    }
    const int *map = P[G_INT].as<int>() + 4 * n;
    k_ref_final<<<(unsigned)((n + 255) / 256), 256, 0, q>>>(map, P[G_INT].as<int>(), n, pm, ps, mean_prior_weight,
                                                           sd_prior_weight, means, sds, cov);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(means_out, means, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(sds_out, sds, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cov_out, cov, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}
