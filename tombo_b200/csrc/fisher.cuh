// fisher.cuh -- z -> two-sided normal p -> Fisher's method over a moving window
// (calc_window_fishers_method tombo_stats.py:2252-2271), shared by the per-read tests
// (region_stats.cu) and the per-position level tests (group_stats.cu).
#pragma once
#include <cmath>
#include "special.cuh"

namespace {
// One block per segment (a read, or a run of covered positions); `out` has the segment's
// length: NaN in the first / last `lag` entries and wherever an input is NaN.
__device__ __forceinline__ double two_sided_p(double m, double rm, double rs)
{
    const double z = fabs(m - rm) / rs;           // np.abs(r_means - ref) / sds  (:3865, :3739)
    return erfc(z * 0.70710678118654752440);      // stats.norm.cdf(-z) * 2.0
}

__device__ __forceinline__ double np_maximum(double a, double b)   // NaN propagates
{
    return (a != a) ? a : (a < b ? b : a);
}

struct FisherArgs {
    // explicit-level variant (k_fisher): flat means / ref levels, segment offsets
    const double *means, *rm, *rs;
    const long long *off;                     // segment offsets into out (and means)
    // reads staged by tb2_stage_reads for k_de_novo (region_stats.cu): read-centric means and
    // base codes; k_de_novo takes its per-read offsets from DeNovoRead descriptors instead
    const unsigned char *seq;
    const long long *seq_off, *mean_off, *read_start;
    const double *norm_mean, *kmeans, *ksds;
    int K, cpos;
    int lag, final_clamp, input_is_p;
    double smallest;
    double *logp, *out;
    long long *pos_out;
};

// Fisher's method over the window of 2 * lag + 1 log p-values around each entry of a segment
// of n entries (calc_window_fishers_method :2262-2269): the sequential sum, then
// chi2.sf(-2 sum, 2 width); NaN in the first / last `lag` entries and for a segment shorter
// than the window.  Each thread of the 256-thread block writes its own entries.
__device__ __forceinline__ void fisher_window(const double *logp, double *out, int n, int lag,
                                              int final_clamp, double smallest, int tid)
{
    const int width = 2 * lag + 1;
    for (int i = tid; i < n; i += 256) {
        double f = NAN;                                      // f_pvals[:] = NAN
        if (n >= width && i >= lag && i < n - lag) {
            double s = logp[i - lag];
            for (int j = 1; j < width; ++j) s += logp[i - lag + j];
            f = (s != s) ? s : tb2_chi2_sf_even(-s, width);  // chi2.sf(log_sums * -2, width * 2)
            if (final_clamp) f = np_maximum(f, smallest);    // :3870-3871 (de novo only)
        }
        out[i] = f;
    }
}

// explicit levels (or p-values) per segment.  The de novo test with k-mer levels from the
// model is k_de_novo (region_stats.cu), which shares the arithmetic above; only
// k_fisher<false> is instantiated, and it keeps its name and its machine code.
template <bool KMER>
__global__ void __launch_bounds__(256) k_fisher(FisherArgs a)
{
    static_assert(!KMER, "k-mer levels: k_de_novo");
    const int r = blockIdx.x, tid = threadIdx.x;
    const long long o = a.off[r];
    const int n = (int)(a.off[r + 1] - o);
    if (n <= 0) return;
    double *logp = a.logp + o, *out = a.out + o;
    const double *means = a.means + o;
    const int lag = a.lag;
    for (int i = tid; i < n; i += 256) {
        double rm, rs;
        if (!a.input_is_p) {
            rm = a.rm[o + i]; rs = a.rs[o + i];
        } else {
            rm = 0.0; rs = 1.0;
        }
        // input_is_p: `means` already holds p-values (calc_window_fishers_method mirror)
        const double p = a.input_is_p ? means[i] : two_sided_p(means[i], rm, rs);
        if (lag == 0) out[i] = a.final_clamp ? np_maximum(p, a.smallest) : p;
        else logp[i] = log(np_maximum(p, a.smallest));      // :2261-2263
    }
    if (lag == 0) return;
    __syncthreads();
    fisher_window(logp, out, n, lag, a.final_clamp, a.smallest, tid);
}
}  // namespace
