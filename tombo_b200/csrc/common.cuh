// common.cuh -- shared device helpers for the tombo_b200 CUDA kernels (sm_90a).
//
// Arithmetic contract: everything that feeds an integer decision (event
// boundaries, band placement, traceback moves) is evaluated in fp64 with the
// reference's operation order and WITHOUT fused multiply-add (compile with
// -fmad=false); the reference's Cython objects contain no FMA (SURVEY.md s7).
#pragma once
#ifndef TB2_EMUL   // tests/emul/cuda_emul.h stands in for the CUDA headers on the host
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <math.h>
#include "../../include/tombo_b200.h"

#define TB2_FULL_MASK 0xffffffffu

// dynamic shared memory of a kernel (tests/emul substitutes its arena)
#ifdef TB2_EMUL
#define TB2_DYN_SMEM(T, name) T *name = (T *)emul::B->smem
#else
#define TB2_DYN_SMEM(T, name) extern __shared__ T name[]
#endif

__device__ __forceinline__ double tb2_neg_inf()
{
    return __longlong_as_double((long long)0xfff0000000000000ULL);
}

__device__ __forceinline__ int tb2_lane() { return threadIdx.x & 31; }

// Correctly rounded a / b for a divisor b that is reused (one k-mer level SD per DP
// row).  Once per divisor: y = RN(1/b) (__drcp_rn), e = 1 - b*y (exact in one FMA) and
// ylo = RN(e*y), so that y + ylo = (1/b)(1 + eps), |eps| <= 2 u^2.  Per quotient four
// fp64 operations:
//   t = RN(a*ylo); q0 = RN(a*y + t)   one rounding of (a/b)(1 + 3 u^2): q0 is a/b rounded
//                                     to nearest unless a/b lies within 3 u^2 of a midpoint,
//                                     and then still one of its two neighbours (faithful)
//   r = a - b*q0                      exact by FMA for a faithful q0
//   q1 = RN(q0 + r*y)                 = RN(a/b) by Markstein's theorem (Markstein 1990;
//                                     Muller et al., Handbook of Floating-Point Arithmetic,
//                                     "division by software": y = RN(1/b), q0 faithful),
//                                     barring over/underflow
// i.e. exactly what the IEEE division of the reference (_c_dynamic_programming.pyx:366)
// returns, for 4 operations instead of ~25 (round 1 used RN(a*y) and two corrections: 5).
// tests/test_div_gpu.py checks it against `/` on 2^31 adversarial and random pairs.
struct tb2_rcp { double hi, lo; };
__device__ __forceinline__ tb2_rcp tb2_rcp_of(double b)
{
    tb2_rcp y;
    y.hi = __drcp_rn(b);
    y.lo = __dmul_rn(__fma_rn(-b, y.hi, 1.0), y.hi);
    return y;
}
__device__ __forceinline__ double tb2_div_by(double a, double b, const tb2_rcp &y)
{
    const double q = __fma_rn(a, y.hi, __dmul_rn(a, y.lo));
    const double r = __fma_rn(-b, q, a);
    return __fma_rn(r, y.hi, q);
}

// keyed bijection on [0, n) (mirror of tombo_b200/synthetic.py perm_index):
// stands in for np.random.choice(n, 1000, replace=False), tombo_stats.py:413
__host__ __device__ __forceinline__ uint32_t tb2_mix32(uint32_t x)
{
    x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
    return x;
}
__host__ __device__ __forceinline__ uint32_t tb2_subsample_key(uint32_t seed, uint32_t read_index,
                                                              uint32_t call)
{
    return tb2_mix32(tb2_mix32(seed ^ 0x9E3779B9u) + tb2_mix32(read_index * 2654435761u + 1u) +
                     call * 0x632BE5ABu);
}
__host__ __device__ __forceinline__ int tb2_perm_index(int i, int n, uint32_t key)
{
    int bits = 0;
    for (int t = n - 1; t > 0; t >>= 1) bits++;
    if (bits < 2) bits = 2;
    int half = (bits + 1) / 2;
    uint32_t mask = (1u << half) - 1u;
    uint32_t x = (uint32_t)i;
    for (;;) {
        uint32_t l = x >> half, r = x & mask;
        for (uint32_t rnd = 0; rnd < 4; rnd++) {
            uint32_t f = tb2_mix32(r ^ key ^ (rnd * 0x9E3779B9u)) & mask;
            uint32_t nl = r, nr = l ^ f;
            l = nl; r = nr;
        }
        x = (l << half) | r;
        if ((int)x < n) return (int)x;
    }
}

// numpy DOUBLE_pairwise_sum (np.add.reduce on contiguous float64): used by
// np.mean in score_valid_bases / get_read_seg_score (tombo_stats.py:2338,2359).
// Serial, executed by one thread.  The numpy routine is recursive; the recursion
// is unrolled onto an explicit frame stack (device stacks are small).  The one definition
// of that order: the summands are a[0 .. n), where `a` is an array or anything with
// a[i] and a + k (csrc/model_est.cu sums values computed on the fly).
template <class A> __device__ __forceinline__ double tb2_pairwise_leaf(A a, int n)
{
    if (n < 8) {
        double res = 0.;
        for (int i = 0; i < n; i++) res += a[i];
        return res;
    }
    double r0 = a[0], r1 = a[1], r2 = a[2], r3 = a[3], r4 = a[4], r5 = a[5], r6 = a[6],
           r7 = a[7];
    int i;
    for (i = 8; i < n - (n % 8); i += 8) {
        r0 += a[i + 0]; r1 += a[i + 1]; r2 += a[i + 2]; r3 += a[i + 3];
        r4 += a[i + 4]; r5 += a[i + 5]; r6 += a[i + 6]; r7 += a[i + 7];
    }
    double res = ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7));
    for (; i < n; i++) res += a[i];
    return res;
}

// where numpy splits n > 128 summands: the size of the left part
__host__ __device__ __forceinline__ int tb2_pairwise_split(int n)
{
    int n2 = n / 2;
    n2 -= n2 % 8;
    return n2;
}

template <class A> __device__ inline double tb2_pairwise_sum(A a, int n)
{
    if (n <= 128) return tb2_pairwise_leaf(a, n);
    // frames: (offset, n, stage, left)
    int f_off[24], f_n[24], f_stage[24];
    double f_left[24];
    int sp = 0;
    f_off[0] = 0; f_n[0] = n; f_stage[0] = 0; f_left[0] = 0.0;
    double ret = 0.0;
    while (sp >= 0) {
        const int fn = f_n[sp];
        if (fn <= 128) { ret = tb2_pairwise_leaf(a + f_off[sp], fn); --sp; continue; }
        const int n2 = tb2_pairwise_split(fn);
        if (f_stage[sp] == 0) {
            f_stage[sp] = 1;
            f_off[sp + 1] = f_off[sp]; f_n[sp + 1] = n2; f_stage[sp + 1] = 0;
            ++sp;
        } else if (f_stage[sp] == 1) {
            f_left[sp] = ret;
            f_stage[sp] = 2;
            f_off[sp + 1] = f_off[sp] + n2; f_n[sp + 1] = fn - n2; f_stage[sp + 1] = 0;
            ++sp;
        } else {
            ret = f_left[sp] + ret;
            --sp;
        }
    }
    return ret;
}

// np.linspace(start, stop, num)[i] (endpoint=True) -- numpy
// _core/function_base.py: y = arange(num) * step + start; y[-1] = stop
__device__ __forceinline__ double tb2_linspace_at(double start, double stop, int num, int i)
{
    int div = num - 1;
    if (div <= 0) return 0.0 * (stop - start) + start;
    if (i == num - 1) return stop;
    double delta = stop - start;
    double step = delta / (double)div;
    if (step == 0.0) return ((double)i / (double)div) * delta + start;
    return (double)i * step + start;
}
