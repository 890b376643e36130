// select.cuh -- exact order statistics for a 256-thread block (np.median semantics).
//
// Radix select on the order-preserving 64-bit image of fp64 values, 8 bits per
// pass, values produced by a functor (recomputed each pass, nothing is sorted or
// copied).  np.median = middle order statistic, or (a + b) / 2 of the two middle
// ones (numpy lib/_function_base_impl.py:_median) -- both are returned exactly.
#pragma once
#include "common.cuh"

#define TB2_SEL_THREADS 256
#define TB2_SEL_SMALL 64      // candidates left at which the select finishes by ranking

__device__ __forceinline__ unsigned long long tb2_key(double v)
{
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
__device__ __forceinline__ double tb2_unkey(unsigned long long k)
{
    const unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffULL) : ~k;
    return __longlong_as_double((long long)u);
}

struct Sum4 { unsigned int x, y, z, w; };

struct SelectSmem {
    unsigned int hist[256];
    unsigned int warp_tot[8];
    unsigned int sel_bin, sel_below, sel_cnt;
    unsigned long long red_u64[8], red_and[8];
    unsigned int red_u32[8];
    Sum4 red_sum4[8];
    unsigned long long small[TB2_SEL_SMALL];   // finishing list of the radix select
    unsigned long long result, result2;   // rank k; rank k + 1 when it sat in the same list
    unsigned int n_small, have2;
};

// block-wide sum of an unsigned (all threads get the result)
__device__ __forceinline__ unsigned int tb2_block_sum(unsigned int v, SelectSmem &sm)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(TB2_FULL_MASK, v, off);
    __syncthreads();
    if (lane == 0) sm.red_u32[warp] = v;
    __syncthreads();
    unsigned int t = 0;
#pragma unroll
    for (int w = 0; w < TB2_SEL_THREADS / 32; ++w) t += sm.red_u32[w];
    return t;
}

// four block-wide sums at once, for the barriers of one
__device__ __forceinline__ Sum4 tb2_block_sum4(Sum4 v, SelectSmem &sm)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        v.x += __shfl_xor_sync(TB2_FULL_MASK, v.x, off);
        v.y += __shfl_xor_sync(TB2_FULL_MASK, v.y, off);
        v.z += __shfl_xor_sync(TB2_FULL_MASK, v.z, off);
        v.w += __shfl_xor_sync(TB2_FULL_MASK, v.w, off);
    }
    __syncthreads();
    if (lane == 0) sm.red_sum4[warp] = v;
    __syncthreads();
    Sum4 t = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int w = 0; w < TB2_SEL_THREADS / 32; ++w) {
        const Sum4 q = sm.red_sum4[w];
        t.x += q.x; t.y += q.y; t.z += q.z; t.w += q.w;
    }
    return t;
}

__device__ __forceinline__ unsigned long long tb2_block_min_u64(unsigned long long v,
                                                                SelectSmem &sm)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const unsigned long long o = __shfl_xor_sync(TB2_FULL_MASK, v, off);
        v = o < v ? o : v;
    }
    __syncthreads();
    if (lane == 0) sm.red_u64[warp] = v;
    __syncthreads();
    unsigned long long t = sm.red_u64[0];
#pragma unroll
    for (int w = 1; w < TB2_SEL_THREADS / 32; ++w) t = sm.red_u64[w] < t ? sm.red_u64[w] : t;
    return t;
}

// Key of the element of ascending rank k (0-based) among the n values f(i) with
// pred(i) true.  Requires 0 <= k < count(pred).  All 256 threads participate.
template <class F, class Pred>
__device__ unsigned long long tb2_block_select_key(F f, Pred pred, int n, int k, SelectSmem &sm)
{
    unsigned long long prefix = 0, mask = 0;
    unsigned int kk = (unsigned int)k;
    const int tid = threadIdx.x;
    if (tid == 0) sm.have2 = 0u;     // published by the barriers below
    // digits shared by every key need no pass: start below the common leading bytes, and
    // skip every later byte in which no two keys differ (integer-valued signal -- the int16
    // DAC dtype -- has five constant trailing bytes)
    int shift0 = 56;
    unsigned long long diff_bits = ~0ULL, common_bits = 0ULL;
    {
        unsigned long long all_or = 0, all_and = ~0ULL;
        for (int i = tid; i < n; i += TB2_SEL_THREADS) {
            if (!pred(i)) continue;
            const unsigned long long key = tb2_key(f(i));
            all_or |= key; all_and &= key;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            all_or |= __shfl_xor_sync(TB2_FULL_MASK, all_or, off);
            all_and &= __shfl_xor_sync(TB2_FULL_MASK, all_and, off);
        }
        __syncthreads();
        if ((tid & 31) == 0) { sm.red_u64[tid >> 5] = all_or; sm.red_and[tid >> 5] = all_and; }
        __syncthreads();
        all_or = 0; all_and = ~0ULL;
#pragma unroll
        for (int w = 0; w < TB2_SEL_THREADS / 32; ++w) { all_or |= sm.red_u64[w]; all_and &= sm.red_and[w]; }
        const unsigned long long diff = all_or ^ all_and;      // bits that differ somewhere
        if (diff == 0ULL) { __syncthreads(); return all_or; }   // all keys equal
        const int top = 63 - __clzll((long long)diff);          // highest differing bit
        diff_bits = diff; common_bits = all_or;
        shift0 = (top >> 3) << 3;
        if (shift0 < 56) {
            mask = ~0ULL << (shift0 + 8);
            prefix = all_or & mask;
        }
        __syncthreads();
    }
    for (int shift = shift0; shift >= 0; shift -= 8) {
        if (((diff_bits >> shift) & 0xffULL) == 0ULL) {         // same digit in every key
            prefix |= common_bits & (0xffULL << shift);
            mask |= 0xffULL << shift;
            continue;
        }
        sm.hist[tid] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += TB2_SEL_THREADS) {
            if (!pred(i)) continue;
            const unsigned long long key = tb2_key(f(i));
            if ((key & mask) == prefix) {
                // warp-aggregated: the leading digits of real signals are almost all
                // equal, one atomic per distinct digit instead of one per lane
                const unsigned int dg = (unsigned int)(key >> shift) & 255u;
#ifdef TB2_EMUL   // the host emulation has full-mask collectives only; same histogram
                atomicAdd(&sm.hist[dg], 1u);
#else
                const unsigned int peers = __match_any_sync(__activemask(), dg);
                if ((threadIdx.x & 31) == (__ffs(peers) - 1)) atomicAdd(&sm.hist[dg], __popc(peers));
#endif
            }
        }
        __syncthreads();
        // exclusive scan of the 256 bins (thread t <-> bin t)
        const unsigned int h = sm.hist[tid];
        unsigned int total;
        const unsigned int exc = tb2_block_excl_scan<TB2_SEL_THREADS>(h, sm.warp_tot, total);
        const unsigned int inc = exc + h;
        if (h > 0 && exc <= kk && kk < inc) { sm.sel_bin = tid; sm.sel_below = exc; sm.sel_cnt = h; }
        __syncthreads();
        prefix |= (unsigned long long)sm.sel_bin << shift;
        mask |= 0xffULL << shift;
        kk -= sm.sel_below;
        const unsigned int left = sm.sel_cnt;
        if (tid == 0) sm.n_small = 0;
        __syncthreads();
        if (left <= TB2_SEL_SMALL && shift > 0) {
            // few candidates share the digits fixed so far: list them and rank directly
            for (int i = tid; i < n; i += TB2_SEL_THREADS) {
                if (!pred(i)) continue;
                const unsigned long long key = tb2_key(f(i));
                if ((key & mask) == prefix) sm.small[atomicAdd(&sm.n_small, 1u)] = key;
            }
            __syncthreads();
            if (tid < (int)left) {
                const unsigned long long mine = sm.small[tid];
                unsigned int rank = 0;
                for (unsigned int q = 0; q < left; ++q) {
                    const unsigned long long o = sm.small[q];
                    rank += (o < mine) || (o == mine && q < (unsigned int)tid);
                }
                if (rank == kk) sm.result = mine;
                if (rank == kk + 1u) { sm.result2 = mine; sm.have2 = 1u; }
            }
            __syncthreads();
            const unsigned long long res = sm.result;
            __syncthreads();
            return res;
        }
    }
    return prefix;
}

// values of rank k and k+1 (k+1 only if want2); exact
template <class F, class Pred>
__device__ void tb2_block_select2(F f, Pred pred, int n, int k, bool want2, double *v0,
                                  double *v1, SelectSmem &sm)
{
    const unsigned long long K = tb2_block_select_key(f, pred, n, k, sm);
    *v0 = tb2_unkey(K);
    *v1 = *v0;
    if (!want2) return;
    // the finishing list usually holds rank k + 1 as well
    const unsigned int h2 = sm.have2;
    const unsigned long long r2 = sm.result2;
    __syncthreads();
    if (h2) { *v1 = tb2_unkey(r2); return; }
    unsigned int cnt_le = 0;
    unsigned long long min_gt = ~0ULL;
    for (int i = threadIdx.x; i < n; i += TB2_SEL_THREADS) {
        if (!pred(i)) continue;
        const unsigned long long key = tb2_key(f(i));
        if (key <= K) ++cnt_le;
        else if (key < min_gt) min_gt = key;
    }
    cnt_le = tb2_block_sum(cnt_le, sm);
    min_gt = tb2_block_min_u64(min_gt, sm);
    if (cnt_le <= (unsigned int)(k + 1)) *v1 = tb2_unkey(min_gt);
}

struct PredAll { __device__ __forceinline__ bool operator()(int) const { return true; } };

// np.median of f(0..n-1)
template <class F>
__device__ double tb2_block_median(F f, int n, SelectSmem &sm)
{
    double a, b;
    if (n & 1) {
        tb2_block_select2(f, PredAll(), n, n / 2, false, &a, &b, sm);
        return a;
    }
    tb2_block_select2(f, PredAll(), n, n / 2 - 1, true, &a, &b, sm);
    return (a + b) / 2.0;
}
