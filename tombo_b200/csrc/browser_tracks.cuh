// browser_tracks.cuh -- device source of the genome browser tracks (browser_tracks.cu); also
// compiled for the host by tests/emul.  DESIGN.md §3 "Genome browser tracks".
#pragma once
#include <climits>
#include "common.cuh"
#include "radix_sort.cuh"

constexpr int BT_DIGITS = 5;        // key digits of the slot sums: positions below 2^40

// ---------------------------------------------------------------------------
// coverage runs
// ---------------------------------------------------------------------------
// flag[i] = 1 where the coverage changes from the entry before (the first entry too); each
// group's own first entry and extra entry are set by k_bt_run_ends
__global__ void k_bt_run_flags(const int *cov, long long len, int *flag)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < len) flag[i] = i == 0 || cov[i] != cov[i - 1];
}

// group g (entries base[g] .. base[g + 1]) starts a run at its first entry; its last entry is
// the difference array's extra one, past max(end), and starts none
__global__ void k_bt_run_ends(const long long *base, long long n_groups, int *flag)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups || base[g + 1] == base[g]) return;
    flag[base[g]] = 1;
    flag[base[g + 1] - 1] = 0;
}

// with incl the inclusive scan of the flags: run incl[i] - 1 starts at entry i.  Its group is
// the last one whose base is <= i (empty groups share their successor's base and come first).
__global__ void k_bt_run_scatter(const int *cov, const int *incl, long long len, const long long *base,
                                 long long n_groups, long long *run_start, long long *run_cov)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= len) return;
    const int r = incl[i];
    if (r == (i ? incl[i - 1] : 0)) return;
    long long lo = 0, hi = n_groups;
    while (hi - lo > 1) {
        const long long mid = (lo + hi) >> 1;
        if (base[mid] <= i) lo = mid; else hi = mid;
    }
    run_start[r - 1] = i - base[lo];
    run_cov[r - 1] = cov[i];
}

// run_off[g] = runs before group g; run_off[n_groups] = all runs
__global__ void k_bt_run_off(const int *incl, const long long *base, long long n_groups, long long *run_off)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g <= n_groups) run_off[g] = base[g] > 0 ? incl[base[g] - 1] : 0;
}

// ---------------------------------------------------------------------------
// slot sums
// ---------------------------------------------------------------------------
// (key, value) of every value of one add call, in read-major order: value j of read r (offsets
// rebased to 0) goes to position start[r] + j, or start[r] + n_r - 1 - j when rev[r] (the
// reference's values[::-1] on the - strand); key = position - kmin.  ghist[d * 256 + v] counts
// digit d of the keys, so the sort knows which digits a single bin holds.
__global__ void __launch_bounds__(256)
k_bt_entries(const double *vals, const long long *off, const long long *start, const unsigned char *rev,
             long long n_reads, long long total, long long kmin, unsigned long long *key, double *val,
             unsigned long long *ghist)
{
    __shared__ unsigned int h[BT_DIGITS * 256];
    for (int i = threadIdx.x; i < BT_DIGITS * 256; i += blockDim.x) h[i] = 0;
    __syncthreads();
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < total;
         j += (long long)gridDim.x * blockDim.x) {
        long long lo = 0, hi = n_reads;              // last read whose offset is <= j
        while (hi - lo > 1) {
            const long long mid = (lo + hi) >> 1;
            if (off[mid] <= j) lo = mid; else hi = mid;
        }
        const long long k = j - off[lo];
        const long long p = rev[lo] ? start[lo] + (off[lo + 1] - off[lo]) - 1 - k : start[lo] + k;
        const unsigned long long kk = (unsigned long long)(p - kmin);
        key[j] = kk;
        val[j] = vals[j];
        for (int d = 0; d < BT_DIGITS; ++d) atomicAdd(h + d * 256 + (int)((kk >> (8 * d)) & 255u), 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < BT_DIGITS * 256; i += blockDim.x)
        if (h[i]) atomicAdd(ghist + i, (unsigned long long)h[i]);
}

// one thread per touched position (the first entry of each run of equal keys, stably sorted):
// continues the stored running sum with the position's values in read order, one fp64 add each,
// and counts them.  A count above 2^31 - 1 sets *overflow.
__global__ void k_bt_accumulate(const unsigned long long *key, const double *val, long long n, long long kmin,
                                double *sums, int *cov, int *overflow)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (i > 0 && key[i - 1] == key[i])) return;
    const long long p = kmin + (long long)key[i];
    double s = sums[p];
    long long c = cov[p];
    for (long long j = i; j < n && key[j] == key[i]; ++j) {
        s += val[j];
        ++c;
    }
    sums[p] = s;
    if (c > INT_MAX) {
        *overflow = 1;
        c = INT_MAX;
    }
    cov[p] = (int)c;
}

// base_sums / base_cov of get_mean_slot_genome_centric: 0 / 0 is NaN
__global__ void k_bt_means(const double *sums, const int *cov, long long n, double *out)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) out[p] = sums[p] / (double)cov[p];
}
