// cuda_emul.h -- TEST INFRASTRUCTURE ONLY.  A minimal host emulation of the CUDA
// execution model for warp-synchronous device code: every thread of a block is a
// user-level fiber (ucontext), warp collectives (__shfl*_sync, __any_sync,
// __ballot_sync, __syncwarp) and __syncthreads are rendezvous points between the
// fibers.  It lets the CPU test-suite run the *same device source* (csrc/*.cuh) that
// nvcc compiles for sm_90a and compare it with the oracle -- an algorithm check for
// index / band / edge-case logic before GPU time is spent.  Never linked into
// libtombo_b200.so; the product path has no CPU fallback.
#pragma once
#include <ucontext.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <cmath>
#include <functional>
#include <type_traits>
#include <vector>

#define TB2_EMUL 1
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __restrict__
#define __shared__ static

namespace emul {
struct Idx3 { unsigned x, y, z; };
struct Fiber {
    ucontext_t uc;
    char *stack = nullptr;
    int tid = 0;
    bool done = false;
    uint64_t wgen = 0, bgen = 0;   // warp / block collective generation
};
struct Warp { uint64_t slot[2][32]; uint64_t arrived[2]; };
struct Block {
    std::vector<Fiber> f;
    std::vector<Warp> w;
    int cur = 0;
    Idx3 bidx{0, 0, 0}, bdim{1, 1, 1}, gdim{1, 1, 1};
    char *smem = nullptr;
    size_t smem_bytes = 0;
    ucontext_t sched;
    uint64_t blk_arrived[2] = {0, 0};
    uint64_t progress = 0;
    std::function<void()> body;
};
extern Block *B;
inline Fiber &me() { return B->f[B->cur]; }
inline void yield() { swapcontext(&me().uc, &B->sched); }
inline Idx3 tidx() { return Idx3{(unsigned)me().tid, 0, 0}; }

// all lanes of the calling warp deposit v; returns after every lane has arrived.
// out (optional) receives the 32 deposited values.
inline uint64_t xchg(uint64_t v, int src, uint64_t *all = nullptr)
{
    Fiber &f = me();
    const int lane = f.tid & 31;
    Warp &w = B->w[f.tid >> 5];
    const unsigned b = (unsigned)(f.wgen & 1);
    const uint64_t target = 32ull * (f.wgen / 2 + 1);
    f.wgen++;
    w.slot[b][lane] = v;
    w.arrived[b]++;
    B->progress++;
    while (w.arrived[b] < target) yield();
    if (all) memcpy(all, w.slot[b], sizeof(w.slot[b]));
    return w.slot[b][src & 31];
}
inline void block_barrier()
{
    Fiber &f = me();
    const unsigned b = (unsigned)(f.bgen & 1);
    const uint64_t target = (uint64_t)B->f.size() * (f.bgen / 2 + 1);
    f.bgen++;
    B->blk_arrived[b]++;
    B->progress++;
    while (B->blk_arrived[b] < target) yield();
}
template <class T> inline uint64_t bits_of(T v)
{
    static_assert(sizeof(T) <= 8, "");
    uint64_t u = 0;
    memcpy(&u, &v, sizeof(T));
    return u;
}
template <class T> inline T from_bits(uint64_t u)
{
    T v;
    memcpy(&v, &u, sizeof(T));
    return v;
}
inline void check_mask(unsigned m)
{
    if (m != 0xffffffffu) { fprintf(stderr, "emul: partial-mask collective\n"); abort(); }
}
void launch(Idx3 grid, unsigned block_threads, size_t smem_bytes, std::function<void()> body);
}  // namespace emul

#define threadIdx (emul::tidx())
#define blockIdx (emul::B->bidx)
#define blockDim (emul::B->bdim)
#define gridDim (emul::B->gdim)

template <class T> inline T __shfl_sync(unsigned m, T v, int src)
{
    emul::check_mask(m);
    return emul::from_bits<T>(emul::xchg(emul::bits_of(v), src));
}
template <class T> inline T __shfl_up_sync(unsigned m, T v, unsigned d)
{
    emul::check_mask(m);
    const int lane = emul::me().tid & 31;
    const int src = lane - (int)d;
    return emul::from_bits<T>(emul::xchg(emul::bits_of(v), src < 0 ? lane : src));
}
template <class T> inline T __shfl_down_sync(unsigned m, T v, unsigned d)
{
    emul::check_mask(m);
    const int lane = emul::me().tid & 31;
    const int src = lane + (int)d;
    return emul::from_bits<T>(emul::xchg(emul::bits_of(v), src > 31 ? lane : src));
}
template <class T> inline T __shfl_xor_sync(unsigned m, T v, int x)
{
    emul::check_mask(m);
    const int lane = emul::me().tid & 31;
    return emul::from_bits<T>(emul::xchg(emul::bits_of(v), lane ^ x));
}
inline unsigned __ballot_sync(unsigned m, int pred)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg(pred ? 1 : 0, 0, all);
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) if (all[i]) r |= 1u << i;
    return r;
}
inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0; }
inline int __all_sync(unsigned m, int pred) { return __ballot_sync(m, pred) == 0xffffffffu; }
inline void __syncwarp(unsigned m = 0xffffffffu) { emul::check_mask(m); emul::xchg(0, 0); }
inline void __syncthreads() { emul::block_barrier(); }
namespace emul {
// block-wide reductions of a predicate (two barriers: deposit, read)
inline int block_reduce(int v, int mode)
{
    static std::vector<int> slots;
    Block *blk = B;
    if (slots.size() < blk->f.size()) slots.resize(blk->f.size());
    slots[me().tid] = v;
    block_barrier();
    int orv = 0, andv = 1, cnt = 0;
    for (size_t i = 0; i < blk->f.size(); ++i) { orv |= slots[i] != 0; andv &= slots[i] != 0; cnt += slots[i] != 0; }
    block_barrier();
    return mode == 0 ? orv : (mode == 1 ? andv : cnt);
}
}
inline int __syncthreads_or(int p) { return emul::block_reduce(p, 0); }
inline int __syncthreads_and(int p) { return emul::block_reduce(p, 1); }
inline int __syncthreads_count(int p) { return emul::block_reduce(p, 2); }
inline int __reduce_add_sync(unsigned m, int v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)(uint32_t)v, 0, all);
    int s = 0;
    for (int i = 0; i < 32; ++i) s += (int)(uint32_t)all[i];
    return s;
}
inline unsigned __reduce_or_sync(unsigned m, unsigned v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg(v, 0, all);
    unsigned s = 0;
    for (int i = 0; i < 32; ++i) s |= (unsigned)all[i];
    return s;
}
inline unsigned __reduce_and_sync(unsigned m, unsigned v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg(v, 0, all);
    unsigned s = 0xffffffffu;
    for (int i = 0; i < 32; ++i) s &= (unsigned)all[i];
    return s;
}
inline unsigned __reduce_max_sync(unsigned m, unsigned v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)v, 0, all);
    unsigned s = (unsigned)all[0];
    for (int i = 1; i < 32; ++i) s = s > (unsigned)all[i] ? s : (unsigned)all[i];
    return s;
}
inline unsigned __reduce_min_sync(unsigned m, unsigned v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)v, 0, all);
    unsigned s = (unsigned)all[0];
    for (int i = 1; i < 32; ++i) s = s < (unsigned)all[i] ? s : (unsigned)all[i];
    return s;
}
inline unsigned __reduce_add_sync(unsigned m, unsigned v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)v, 0, all);
    unsigned s = 0;
    for (int i = 0; i < 32; ++i) s += (unsigned)all[i];
    return s;
}
inline int __reduce_max_sync(unsigned m, int v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)(uint32_t)v, 0, all);
    int s = (int)(uint32_t)all[0];
    for (int i = 1; i < 32; ++i) s = s > (int)(uint32_t)all[i] ? s : (int)(uint32_t)all[i];
    return s;
}
inline int __reduce_min_sync(unsigned m, int v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)(uint32_t)v, 0, all);
    int s = (int)(uint32_t)all[0];
    for (int i = 1; i < 32; ++i) s = s < (int)(uint32_t)all[i] ? s : (int)(uint32_t)all[i];
    return s;
}

// ---- scalar intrinsics (compile the emulation with -ffp-contract=off) ----
template <class T> inline T __ldg(const T *p) { return *p; }
inline double __drcp_rn(double x) { return 1.0 / x; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
inline double __dsqrt_rn(double a) { return sqrt(a); }
inline double __fma_rn(double a, double b, double c) { return fma(a, b, c); }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float __fdividef(float a, float b) { return a / b; }
struct float4 { float x, y, z, w; };
inline float4 make_float4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
struct float2 { float x, y; };
inline float2 make_float2(float x, float y) { float2 r; r.x = x; r.y = y; return r; }
using std::isfinite;
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline double __longlong_as_double(long long v) { return emul::from_bits<double>((uint64_t)v); }
inline long long __double_as_longlong(double v) { return (long long)emul::bits_of(v); }
inline float __int_as_float(int v) { return emul::from_bits<float>((uint64_t)(uint32_t)v); }
inline int __float_as_int(float v) { return (int)(uint32_t)emul::bits_of(v); }
inline unsigned __float_as_uint(float v) { return (uint32_t)emul::bits_of(v); }
inline float __uint_as_float(unsigned v) { return emul::from_bits<float>((uint64_t)v); }
inline int __double2hiint(double v) { return (int)(emul::bits_of(v) >> 32); }
inline int __double2loint(double v) { return (int)(uint32_t)emul::bits_of(v); }
inline double __hiloint2double(int hi, int lo)
{
    return emul::from_bits<double>(((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo);
}
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __ffsll(long long x) { return __builtin_ffsll(x); }
inline unsigned __brev(unsigned x)
{
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) if (x & (1u << i)) r |= 1u << (31 - i);
    return r;
}
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s)
{
    return (unsigned)((((uint64_t)hi << 32) | lo) >> (s & 31));
}
inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned s)
{
    return (unsigned)(((((uint64_t)hi << 32) | lo) << (s & 31)) >> 32);
}
inline bool __isShared(const void *p)
{
    const char *c = (const char *)p;
    return emul::B->smem && c >= emul::B->smem && c < emul::B->smem + emul::B->smem_bytes;
}
#define EMUL_SMEM_BIAS 4096u
inline size_t __cvta_generic_to_shared(const void *p)
{
    return (size_t)((const char *)p - emul::B->smem) + EMUL_SMEM_BIAS;
}
inline char *emul_shared_ptr(unsigned a) { return emul::B->smem + (a - EMUL_SMEM_BIAS); }

template <class T, class U> inline T atomicAdd(T *p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> inline T atomicMax(T *p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class U> inline T atomicMin(T *p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> inline T atomicOr(T *p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> inline T atomicAnd(T *p, U v) { T o = *p; *p = (T)(o & (T)v); return o; }
template <class T, class U> inline T atomicExch(T *p, U v) { T o = *p; *p = (T)v; return o; }
template <class T, class U, class V> inline T atomicCAS(T *p, U c, V v) { T o = *p; if (o == (T)c) *p = (T)v; return o; }
inline void __threadfence() {}
inline void __threadfence_block() {}

template <class A, class B_> inline typename std::common_type<A, B_>::type min(A a, B_ b)
{
    typedef typename std::common_type<A, B_>::type T;
    return (T)b < (T)a ? (T)b : (T)a;
}
template <class A, class B_> inline typename std::common_type<A, B_>::type max(A a, B_ b)
{
    typedef typename std::common_type<A, B_>::type T;
    return (T)a < (T)b ? (T)b : (T)a;
}
using std::isnan;
using std::isinf;
