// radix_sort.cuh -- the stable LSD radix sort of accuracy.cu and stats_file.cu: 64-bit keys,
// 8-bit digits, a payload carried with each key.  One pass is three launches over tiles of
// RADIX_TILE items: per-tile digit histograms, their digit-major prefix, and a stable scatter.
// The caller skips a digit whose global histogram is a single bin: it keeps the order.
#pragma once
#include "common.cuh"

namespace {

constexpr int RADIX_NT = 256;                  // threads per block
constexpr int RADIX_IPT = 16;                  // items per thread of a tile
constexpr int RADIX_TILE = RADIX_NT * RADIX_IPT;

// float64 bits -> uint64 whose unsigned order is numpy's order of the values; -0.0 folds
// onto +0.0 (numpy compares them equal).  NaN maps above +inf.
__device__ __forceinline__ unsigned long long order_key(double x)
{
    unsigned long long u = (unsigned long long)__double_as_longlong(x);
    if (u == 0x8000000000000000ull) u = 0;
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// digit of one pass: shift 64 is a pass over the payload itself (a u8 label), else 8 bits of
// the key
template <class V> __device__ __forceinline__ int radix_digit(unsigned long long k, V v, int shift)
{
    return shift == 64 ? (int)v : (int)((k >> shift) & 255u);
}

// tile histograms, digit-major: th[d * n_tiles + t]
template <class V>
__global__ void __launch_bounds__(RADIX_NT)
k_radix_tile_hist(const unsigned long long *key, const V *val, long long n, int shift, unsigned int *th,
                  long long n_tiles)
{
    __shared__ unsigned int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const long long t = blockIdx.x, i0 = t * RADIX_TILE;
    for (int r = 0; r < RADIX_IPT; ++r) {
        const long long i = i0 + r * RADIX_NT + threadIdx.x;
        if (i < n) atomicAdd(h + radix_digit(key[i], val[i], shift), 1u);
    }
    __syncthreads();
    th[(size_t)threadIdx.x * n_tiles + t] = h[threadIdx.x];
}

// one block per digit: toff[d * n_tiles + t] = (entries of smaller digits, from the pass's
// global histogram) + (entries of digit d in tiles before t)
__global__ void __launch_bounds__(RADIX_NT)
k_radix_tile_scan(const unsigned int *th, long long n_tiles, const unsigned long long *pass_hist,
                  unsigned long long *toff)
{
    __shared__ unsigned int warp_tot[RADIX_NT / 32];
    __shared__ unsigned long long base_sh;
    const int d = blockIdx.x;
    if (threadIdx.x == 0) {
        unsigned long long s = 0;
        for (int e = 0; e < d; ++e) s += pass_hist[e];
        base_sh = s;
    }
    __syncthreads();
    unsigned long long base = base_sh;
    const unsigned int *row = th + (size_t)d * n_tiles;
    unsigned long long *orow = toff + (size_t)d * n_tiles;
    for (long long t0 = 0; t0 < n_tiles; t0 += RADIX_NT) {
        const long long t = t0 + threadIdx.x;
        const unsigned int x = t < n_tiles ? row[t] : 0;
        unsigned int total;
        __syncthreads();
        const unsigned long long o = base + tb2_block_excl_scan<RADIX_NT>(x, warp_tot, total);
        base += total;
        if (t < n_tiles) orow[t] = o;
    }
}

// stable scatter of one tile: RADIX_IPT rounds of RADIX_NT items in index order; within a
// round, an item's rank among equal digits is its rank in its warp (match_any) plus the counts
// of the same digit in earlier warps and earlier rounds
template <class V>
__global__ void __launch_bounds__(RADIX_NT)
k_radix_scatter_pass(const unsigned long long *kin, const V *vin, unsigned long long *kout, V *vout,
                     long long n, int shift, const unsigned long long *toff, long long n_tiles)
{
    __shared__ unsigned long long run[256];
    __shared__ unsigned int wcnt[RADIX_NT / 32][256];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long t = blockIdx.x, i0 = t * RADIX_TILE;
    run[tid] = toff[(size_t)tid * n_tiles + t];
    for (int w = 0; w < RADIX_NT / 32; ++w) wcnt[w][tid] = 0;
    __syncthreads();
    for (int r = 0; r < RADIX_IPT; ++r) {
        const long long i = i0 + r * RADIX_NT + tid;
        const bool live = i < n;
        unsigned long long k = 0;
        V v = 0;
        int d = 256 + lane;                              // a bin of its own for dead lanes
        if (live) { k = kin[i]; v = vin[i]; d = radix_digit(k, v, shift); }
        const unsigned int peers = __match_any_sync(0xffffffffu, d);
        const unsigned int rank = __popc(peers & ((1u << lane) - 1u));
        if (live && rank == 0) wcnt[warp][d] = __popc(peers);
        __syncthreads();
        if (live) {
            unsigned long long o = run[d] + rank;
            for (int w = 0; w < warp; ++w) o += wcnt[w][d];
            kout[o] = k;
            vout[o] = v;
        }
        __syncthreads();
        unsigned int s = 0;
        for (int w = 0; w < RADIX_NT / 32; ++w) { s += wcnt[w][tid]; wcnt[w][tid] = 0; }
        run[tid] += s;
        __syncthreads();
    }
}

}  // namespace
