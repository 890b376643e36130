// debug.cu -- self-checks exposed for the GPU test-suite
#include "common.cuh"
#include "ctx.h"

namespace {
__device__ __forceinline__ unsigned long long xs(unsigned long long &s)
{
    s ^= s >> 12; s ^= s << 25; s ^= s >> 27;
    return s * 0x2545F4914F6CDD1DULL;
}
__device__ __forceinline__ double mk(unsigned long long mant, int e)
{
    // 1.mant * 2^e
    return __longlong_as_double((long long)(((unsigned long long)(e + 1023) << 52) |
                                            (mant & 0xFFFFFFFFFFFFFULL)));
}

// tb2_div_by(a, b, tb2_rcp_of(b)) must equal a / b bit for bit
__global__ void k_div_check(unsigned long long seed, int per_thread, unsigned long long *mism,
                            double *example)
{
    unsigned long long s = seed ^ (0x9E3779B97F4A7C15ULL * (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x + 1));
    unsigned long long bad = 0;
    for (int it = 0; it < per_thread; ++it) {
        const unsigned long long r0 = xs(s), r1 = xs(s), r2 = xs(s);
        // divisor: random / all-ones / power of two / near-one significands
        unsigned long long mb = r0;
        switch (r2 & 7) {
        case 0: mb = 0xFFFFFFFFFFFFFULL; break;
        case 1: mb = 0; break;
        case 2: mb = 0xFFFFFFFFFFFFFULL - (r0 & 15); break;
        case 3: mb = r0 & 15; break;
        default: break;
        }
        const double b = mk(mb, (int)((r2 >> 8) % 21) - 10);
        double a;
        if ((r2 >> 16) & 1) {
            // quotient next to a representable number or a midpoint: a = RN(b*q) +- k ulp
            const double q = mk(r1, (int)((r2 >> 20) % 31) - 20);
            a = b * q;
            const long long k = (long long)((r2 >> 32) % 5) - 2;
            a = __longlong_as_double(__double_as_longlong(a) + k);
        } else {
            a = mk(r1, (int)((r2 >> 20) % 43) - 30);
        }
        if ((r2 >> 40) % 97 == 0) a = 0.0;
        const double want = a / b;
        const double got = tb2_div_by(a, b, tb2_rcp_of(b));
        if (__double_as_longlong(want) != __double_as_longlong(got)) {
            if (bad == 0) { example[0] = a; example[1] = b; example[2] = want; example[3] = got; }
            ++bad;
        }
    }
    if (bad) atomicAdd(mism, bad);
}
}  // namespace

// per-call scratch of tb2_debug_div_check: the mismatch count, then the first example
struct DebugState { DevBuf out; };

extern "C" int tb2_debug_div_check(tb2_ctx *ctx, uint64_t seed, int blocks, int per_thread,
                                   uint64_t *mismatches, double *example4)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!mismatches || !example4 || blocks < 1 || per_thread < 1) return TB2_ERR_INVALID_ARG;
    DevBuf &out = tb2_state(ctx->debug).out;
    TB2_CUDA_TRY(ctx, out.reserve(64));
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(out.p, 0, 64, ctx->stream));
    k_div_check<<<blocks, 256, 0, ctx->stream>>>(seed, per_thread, out.as<unsigned long long>(),
                                                 out.as<double>() + 1);
    TB2_CHECK_LAUNCH(ctx);
    unsigned long long h[5];
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(h, out.p, 40, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *mismatches = h[0];
    memcpy(example4, &h[1], 32);
    return TB2_OK;
}
