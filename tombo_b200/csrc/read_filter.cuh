// read_filter.cuh -- device source of the read filters (read_filter.cu); also compiled for the
// host by tests/emul.  DESIGN.md §3 "Read filters".
#pragma once
#include "common.cuh"
#include "select.cuh"

constexpr int RF_NT = 1024;                  // threads of the coverage scan kernels
constexpr int RF_ITEMS = 4;                  // consecutive entries per thread
constexpr int RF_TILE = RF_NT * RF_ITEMS;    // entries per block of the scan

// np.percentile(x, pctl) of the n >= 1 values f(0 .. n-1), numpy 2.3.5 method='linear'
// (numpy/lib/_function_base_impl.py; DESIGN.md §3 gives the lines).  -fmad=false keeps every
// product and sum separately rounded, as numpy's are.
template <class F>
__device__ double rf_percentile(F f, int n, double pctl, SelectSmem &sm)
{
    const double q = pctl / 100.0;                  // percentile: true_divide(q, 100)
    const double v = (double)(n - 1) * q;           // 'linear' get_virtual_index: (n - 1) * q
    double prev = floor(v);                         // _get_indexes
    long long lo = (long long)prev, hi = lo + 1;
    if (v >= (double)(n - 1)) {                     // above bounds: both indexes -1 (the last)
        prev = -1.0;
        lo = hi = n - 1;
    }
    // (v < 0 cannot occur: q >= 0)
    const double g = v - prev;                      // _get_gamma, from the clipped index
    double a, b;
    tb2_block_select2(f, PredAll(), n, (int)lo, hi != lo, &a, &b, sm);
    const double d = b - a;                         // _lerp
    return g >= 0.5 ? b - d * (1.0 - g) : a + d * g;
}

struct RfLens {            // host lengths of one read
    const long long *p;
    __device__ double operator()(int i) const { return (double)p[i]; }
};
struct RfDwells {          // np.diff of one read's final segs
    const long long *s;
    __device__ double operator()(int i) const { return (double)(s[i + 1] - s[i]); }
};

// one block per read: out[r * n_pctl + j] = np.percentile(lens of read r, pctl[j])
__global__ void __launch_bounds__(TB2_SEL_THREADS)
k_rf_dwell_pctl(const long long *lens, const long long *off, int n_pctl, const double *pctl, double *out)
{
    __shared__ SelectSmem sm;
    const int r = blockIdx.x;
    const long long o = off[r];
    const int n = (int)(off[r + 1] - o);
    const RfLens f{lens + (o - off[0])};
    for (int j = 0; j < n_pctl; ++j) {
        const double v = rf_percentile(f, n, pctl[j], sm);
        if (threadIdx.x == 0) out[(long long)r * n_pctl + j] = v;
        __syncthreads();
    }
}

// one block per read of the resident batch: the reversible filters of _io_and_map_read
// (resquiggle.py:1437-1453).  code: -1 failed read, 1 signal matching, 2 observations per
// base, 0 kept.  The percentiles are consulted only for a read that passes the signal
// matching test (the reference's elif), but computed for every successful read when pout
// asks for them.
__global__ void __launch_bounds__(TB2_SEL_THREADS)
k_rf_batch(const long long *segs, const long long *base_off, const int *status, int stride,
           const double *score, double sig_thresh, int n_pctl, const double *pctl,
           const double *thresh, signed char *code, double *pout)
{
    __shared__ SelectSmem sm;
    const int r = blockIdx.x;
    const long long b0 = base_off[r];
    const int nb = (int)(base_off[r + 1] - b0);
    // a resquiggled read has at least one base; a read without is reported as failed
    if (status[(long long)r * stride] != 0 || nb < 1) {
        if (threadIdx.x == 0) {
            code[r] = -1;
            if (pout)
                for (int j = 0; j < n_pctl; ++j) pout[(long long)r * n_pctl + j] = __longlong_as_double(0x7ff8000000000000LL);
        }
        return;
    }
    const bool poor_match = score[r] > sig_thresh;
    bool stuck = false;
    if (!poor_match || pout) {
        const RfDwells f{segs + b0 + r};          // read r's segs start at seg_off = base_off + r
        for (int j = 0; j < n_pctl; ++j) {
            const double v = rf_percentile(f, nb, pctl[j], sm);
            stuck = stuck || v > thresh[j];
            if (pout && threadIdx.x == 0) pout[(long long)r * n_pctl + j] = v;
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) code[r] = poor_match ? 1 : (stuck ? 2 : 0);
}

// the difference array of every group's coverage: +1 at start, -1 at end (absolute indexes
// into the groups' concatenated arrays, each one entry longer than its max(end))
__global__ void k_rf_cov_diff(const long long *s, const long long *e, long long n, int *diff)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    atomicAdd(diff + s[i], 1);
    atomicAdd(diff + e[i], -1);
}

// device-wide inclusive prefix sum of x in place, in three launches: the sum of each tile
// (k_rf_tile_sum), the offsets of the tiles (k_scan_offsets, common.cuh), each tile's scan
// from its offset (k_rf_tile_scan)
__global__ void __launch_bounds__(RF_NT) k_rf_tile_sum(const int *x, long long n, long long *tile_sum)
{
    __shared__ long long warp_tot[RF_NT / 32];
    const long long i0 = (long long)blockIdx.x * RF_TILE + (long long)threadIdx.x * RF_ITEMS;
    long long s = 0;
    for (int k = 0; k < RF_ITEMS; ++k)
        if (i0 + k < n) s += x[i0 + k];
    long long total;
    tb2_block_excl_scan<RF_NT>(s, warp_tot, total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(RF_NT) k_rf_tile_scan(int *x, long long n, const long long *tile_off)
{
    __shared__ long long warp_tot[RF_NT / 32];
    const long long i0 = (long long)blockIdx.x * RF_TILE + (long long)threadIdx.x * RF_ITEMS;
    int v[RF_ITEMS];
    long long s = 0;
    for (int k = 0; k < RF_ITEMS; ++k) {
        v[k] = i0 + k < n ? x[i0 + k] : 0;
        s += v[k];
    }
    long long total;
    long long run = tile_off[blockIdx.x] + tb2_block_excl_scan<RF_NT>(s, warp_tot, total);
    for (int k = 0; k < RF_ITEMS; ++k) {
        run += v[k];
        if (i0 + k < n) x[i0 + k] = (int)run;
    }
}

// cov[start + (end - start) // 2] of every read (_filter_reads.py:125-126)
__global__ void k_rf_mid(const long long *s, const long long *e, long long n, const int *cov, long long *out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = cov[s[i] + (e[i] - s[i]) / 2];
}
