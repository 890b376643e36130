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
    // explicit-level variant (KMER == false): flat means / ref levels, segment offsets
    const double *means, *rm, *rs;
    const long long *off;                     // segment offsets into out (and means)
    // k-mer variant: whole '+' strand reads, levels looked up in the model tables
    const unsigned char *seq;
    const long long *seq_off, *mean_off, *read_start;
    const double *norm_mean, *kmeans, *ksds;
    int K, cpos;
    int lag, final_clamp, input_is_p;
    double smallest;
    double *logp, *out;
    long long *pos_out;
};

template <bool KMER>
__global__ void __launch_bounds__(256) k_fisher(FisherArgs a)
{
    const int r = blockIdx.x, tid = threadIdx.x;
    const long long o = a.off[r];
    const int n = (int)(a.off[r + 1] - o);
    if (n <= 0) return;
    double *logp = a.logp + o, *out = a.out + o;
    const unsigned char *bases = nullptr;
    const double *means;
    if (KMER) {
        bases = a.seq + a.seq_off[r] + a.cpos;              // stored (trimmed) read sequence
        means = a.norm_mean + a.mean_off[r] + a.cpos;       // r_means[gnm_begin_lag:-gnm_end_lag]
    } else {
        means = a.means + o;
    }
    const int lag = a.lag, width = 2 * lag + 1;
    for (int i = tid; i < n; i += 256) {
        double rm, rs;
        if (KMER) {
            int code = 0;
            for (int j = 0; j < a.K; ++j) code = code * 4 + (bases[i + j] & 3);
            rm = a.kmeans[code]; rs = a.ksds[code];
            a.pos_out[o + i] = a.read_start[r] + a.cpos + i;
        } else if (!a.input_is_p) {
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
    for (int i = tid; i < n; i += 256) {
        double f = NAN;                                      // f_pvals[:] = NAN
        if (n >= width && i >= lag && i < n - lag) {
            double s = logp[i - lag];
            for (int j = 1; j < width; ++j) s += logp[i - lag + j];
            f = (s != s) ? s : tb2_chi2_sf_even(-s, width);  // chi2.sf(log_sums * -2, width * 2)
            if (a.final_clamp) f = np_maximum(f, a.smallest);   // :3870-3871 (de novo only)
        }
        out[i] = f;
    }
}
}  // namespace
