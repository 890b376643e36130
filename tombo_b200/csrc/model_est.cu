// model_est.cu -- per-k-mer Gaussian kernel densities for alternative-model estimation.
//
//   tb2_kernel_densities  est_kernel_density tombo_stats.py:1914-1939: for each set of
//                         levels, gaussian_kde(levels, bw / levels.std(ddof=1)).evaluate(x)
//
// Steps (DESIGN.md §3 "Kernel densities"):
//   1. k_kde_setup, one warp per set: np.std(ddof=1) in numpy's pairwise order (bit-exact),
//      factor = bw / std, and the kernel width c = sqrt(np.cov(levels, aweights=1/n)) * factor
//      with every sum pairwise (np.cov's dot goes through BLAS, so c alone is not bit-exact).
//      Sets where the reference raises get a NaN row.
//   2. k_kde, one CTA per (set, tile of 32 grid points): the set's whitened levels staged
//      through shared memory; warp w sums levels w, w + 8, ... for its lane's grid point with
//      scipy's per-term arithmetic (gaussian_kernel_estimate), then the 8 partial sums are
//      added in a fixed tree.
#include "kernels.h"
#include "common.cuh"
#include <climits>
#include <cmath>

namespace {
enum { K_LV = 0, K_OFF, K_X, K_SET, K_DENS, K_COUNT };

constexpr int KT = 256;                 // threads of k_kde
constexpr int KW = KT / 32;             // warps: level stripes per grid point
constexpr int TJ = 32;                  // grid points per CTA (one per lane)
constexpr int CH = 2048;                // whitened levels staged per pass (16 KB)
constexpr long long MAX_POINTS = 1LL << 20;
// |p - q| >= 40 -> a >= 1600, exp(-800) == 0 in glibc and in CUDA: the term is +0 exactly
constexpr double FAR = 40.0;

// per-set constants written by k_kde_setup
struct KdeSet {
    double w, inv, norm, pmin, pmax, c, factor;
    int ok;
};
}  // namespace
struct KdeState { DevBuf buf[K_COUNT]; };

namespace {

// one warp per set
__global__ void __launch_bounds__(128)
k_kde_setup(const double *lv, const long long *off, long long n_sets, double bw, double norm0,
            KdeSet *sets)
{
    const long long s = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (s >= n_sets) return;                    // whole warps
    const int lane = threadIdx.x & 31;
    const double *x = lv + off[s];
    const int n = (int)(off[s + 1] - off[s]);
    bool finite = true;
    double lo = INFINITY, hi = -INFINITY;
    for (int i = lane; i < n; i += 32) {
        finite = finite && isfinite(x[i]);
        lo = fmin(lo, x[i]); hi = fmax(hi, x[i]);
    }
    finite = __all_sync(TB2_FULL_MASK, finite) && n >= 2;
    for (int w = 16; w > 0; w >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(TB2_FULL_MASK, lo, w));
        hi = fmax(hi, __shfl_xor_sync(TB2_FULL_MASK, hi, w));
    }
    KdeSet k;
    k.w = k.inv = k.norm = k.pmin = k.pmax = k.c = k.factor = NAN;
    k.ok = 0;
    if (finite) {
        // norm_levels.std(ddof=1): _methods._var, pairwise sums, divided by n and n - 1
        const double mean = warp_pairwise_sum([x](int i) { return x[i]; }, n) / (double)n;
        const double var = warp_pairwise_sum([x, mean](int i) { const double d = x[i] - mean; return d * d; }, n) /
                           (double)(n - 1);
        const double sd = sqrt(var);
        const double factor = bw / sd;
        // np.cov(x, bias=False, aweights=ones(n) / n): average() with returned weight sum,
        // fact = w_sum - 1 * sum(w * w) / w_sum, c = dot(X, (X * w).T) * (1 / fact)
        const double w = 1.0 / (double)n;
        const double w_sum = warp_pairwise_sum([w](int) { return w; }, n);
        const double avg = warp_pairwise_sum([x, w](int i) { return x[i] * w; }, n) / w_sum;
        const double fact = w_sum - warp_pairwise_sum([w](int) { return w * w; }, n) / w_sum;
        const double dot = warp_pairwise_sum([x, w, avg](int i) { const double d = x[i] - avg; return d * (d * w); }, n);
        const double c = sqrt(dot * (1.0 / fact)) * factor;       // 1x1 Cholesky, then * factor
        // the reference raises on sd == 0 (divide by zero) and on overflow
        if (sd > 0.0 && isfinite(sd) && isfinite(factor) && fact > 0.0 && c > 0.0 && isfinite(c)) {
            // gaussian_kernel_estimate: solve_triangular by a 1x1 factor multiplies by 1 / c
            k.w = w; k.c = c; k.factor = factor; k.inv = 1.0 / c; k.norm = norm0 / c;
            k.pmin = lo * k.inv; k.pmax = hi * k.inv;       // x * inv is monotone in x
            k.ok = 1;
        }
    }
    if (lane == 0) sets[s] = k;
}

__global__ void __launch_bounds__(KT)
k_kde(const double *lv, const long long *off, const KdeSet *sets, const double *gx, int m, double *dens)
{
    __shared__ double sp[CH];
    __shared__ double part[KW][TJ];
    const long long s = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.y * TJ + lane;
    double *row = dens + s * (long long)m;
    const KdeSet k = sets[s];
    if (!k.ok) {
        if (warp == 0 && j < m) row[j] = NAN;
        return;
    }
    // points with |p - q| >= FAR for every level get +0, as in the reference; NaN
    // comparisons (a non-finite grid point) keep the point in and compute every term
    const double q = j < m ? gx[j] * k.inv : 0.0;
    const bool in = j < m && !(k.pmin - q >= FAR) && !(k.pmax - q <= -FAR);
    if (!__syncthreads_or(in)) {
        if (warp == 0 && j < m) row[j] = 0.0;
        return;
    }
    const double *x = lv + off[s];
    const long long n = off[s + 1] - off[s];
    double acc = 0.0;
    for (long long c0 = 0; c0 < n; c0 += CH) {
        const int len = (int)min((long long)CH, n - c0);
        __syncthreads();
        for (int i = threadIdx.x; i < len; i += KT) sp[i] = x[c0 + i] * k.inv;
        __syncthreads();
        if (in) {
#pragma unroll 4
            for (int i = warp; i < len; i += KW) {
                const double d = sp[i] - q;
                const double a = d * d;
                acc += k.w * (exp(-a / 2.0) * k.norm);
            }
        }
    }
    part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && j < m) {
        const double (*p)[TJ] = part;
        row[j] = in ? ((p[0][lane] + p[1][lane]) + (p[2][lane] + p[3][lane])) +
                          ((p[4][lane] + p[5][lane]) + (p[6][lane] + p[7][lane]))
                    : 0.0;
    }
}
static_assert(KW == 8, "k_kde's final tree adds 8 partial sums");

}  // namespace

extern "C" int tb2_kernel_densities(tb2_ctx *ctx, int64_t n_sets, const double *levels,
                                    const int64_t *off, int64_t n_points, const double *x,
                                    double bw, double *dens_out, double *cho_cov_out,
                                    double *factor_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n_sets < 0 || n_sets > INT_MAX || n_points < 1 || n_points > MAX_POINTS || !x ||
        !(bw > 0.0) || !std::isfinite(bw) || (n_sets > 0 && (!off || !dens_out || !cho_cov_out)))
        return TB2_ERR_INVALID_ARG;
    if (n_sets == 0) {
        ctx->last_ms_total = ctx->last_ms_dp = ctx->last_dp_launches = ctx->last_dp_reads = 0;
        return TB2_OK;
    }
    if (off[0] != 0) return TB2_ERR_INVALID_ARG;
    for (int64_t s = 0; s < n_sets; ++s)
        if (off[s + 1] < off[s] || off[s + 1] - off[s] > INT_MAX) return TB2_ERR_INVALID_ARG;
    const long long total = off[n_sets];
    if (total > 0 && !levels) return TB2_ERR_INVALID_ARG;
    auto &B = tb2_state(ctx->kde).buf;
    cudaStream_t q = ctx->stream;
    const int m = (int)n_points;
    TB2_CUDA_TRY(ctx, B[K_LV].upload(levels, (size_t)total, q));
    TB2_CUDA_TRY(ctx, B[K_OFF].upload(off, (size_t)n_sets + 1, q));
    TB2_CUDA_TRY(ctx, B[K_X].upload(x, (size_t)m, q));
    TB2_CUDA_TRY(ctx, B[K_SET].reserve((size_t)n_sets * sizeof(KdeSet)));
    TB2_CUDA_TRY(ctx, B[K_DENS].reserve((size_t)n_sets * m * 8));
    const double *lv = B[K_LV].as<double>();
    const long long *o = B[K_OFF].as<long long>();
    KdeSet *sets = B[K_SET].as<KdeSet>();
    double *dens = B[K_DENS].as<double>();
    // kernel time: tb2_last_timing out[0], the upload before and the download after excluded
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));
    // pow(2 pi, -d / 2) with d = 1 on the host, as gaussian_kernel_estimate evaluates it
    const double norm0 = std::pow(2.0 * M_PI, -0.5);
    k_kde_setup<<<(unsigned)((n_sets + 3) / 4), 128, 0, q>>>(lv, o, n_sets, bw, norm0, sets);
    TB2_CHECK_LAUNCH(ctx);
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev2, q));
    k_kde<<<dim3((unsigned)n_sets, (unsigned)((m + TJ - 1) / TJ)), KT, 0, q>>>(lv, o, sets, B[K_X].as<double>(), m,
                                                                             dens);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx, ctx->ev2))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(dens_out, dens, (size_t)n_sets * m * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpy2DAsync(cho_cov_out, 8, (const char *)sets + offsetof(KdeSet, c), sizeof(KdeSet),
                                        8, (size_t)n_sets, cudaMemcpyDeviceToHost, q));
    if (factor_out)
        TB2_CUDA_TRY(ctx, cudaMemcpy2DAsync(factor_out, 8, (const char *)sets + offsetof(KdeSet, factor),
                                            sizeof(KdeSet), 8, (size_t)n_sets, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}
