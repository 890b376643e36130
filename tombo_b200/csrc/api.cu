// api.cu -- context management of libtombo_b200.so
#include "ctx.h"
#include <string.h>

extern "C" int tb2_abi_version(void) { return TB2_ABI_VERSION; }

extern "C" int tb2_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" int tb2_ctx_create(int device, tb2_ctx **out)
{
    if (!out) return TB2_ERR_INVALID_ARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) {
        cudaGetLastError();
        return TB2_ERR_CUDA;  // no CPU fallback: fail loudly
    }
    if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return TB2_ERR_CUDA; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return TB2_ERR_CUDA;
    cudaDeviceSetLimit(cudaLimitStackSize, 4096);
    tb2_ctx *ctx = new tb2_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&ctx->ev0) != cudaSuccess || cudaEventCreate(&ctx->ev1) != cudaSuccess ||
        cudaEventCreate(&ctx->ev2) != cudaSuccess || cudaEventCreate(&ctx->ev3) != cudaSuccess) {
        delete ctx;
        return TB2_ERR_CUDA;
    }
    *out = ctx;
    return TB2_OK;
}

extern "C" void tb2_ctx_destroy(tb2_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (tb2_ctx *ln : ctx->lanes) tb2_ctx_destroy(ln);
    ctx->lanes.clear();
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    cudaEventDestroy(ctx->ev0); cudaEventDestroy(ctx->ev1);
    cudaEventDestroy(ctx->ev2); cudaEventDestroy(ctx->ev3);
    if (ctx->ev_t0) { cudaEventDestroy(ctx->ev_t0); cudaEventDestroy(ctx->ev_t1); }
    cudaStreamDestroy(ctx->stream);
    delete ctx;   // the DevBuf destructors free the model tables and every module's buffers
}

extern "C" const char *tb2_last_error(tb2_ctx *ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

// page-locked host memory for callers that want full-rate H2D / D2H copies
extern "C" void *tb2_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

extern "C" void tb2_host_free(void *p)
{
    if (p) cudaFreeHost(p);
}

extern "C" int64_t tb2_launch_count(tb2_ctx *ctx) { return ctx ? ctx->launches : 0; }

extern "C" int tb2_last_timing(tb2_ctx *ctx, double *out3 /* 4 values */)
{
    if (!ctx || !out3) return TB2_ERR_INVALID_ARG;
    out3[0] = ctx->last_ms_total; out3[1] = ctx->last_ms_dp; out3[2] = ctx->last_dp_launches;
    out3[3] = ctx->last_dp_reads;
    return TB2_OK;
}

// device-side stopwatch on the context's stream (CUDA events): brackets any sequence of
// library calls issued on this context
extern "C" int tb2_timer_start(tb2_ctx *ctx)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!ctx->ev_t0) {
        TB2_CUDA_TRY(ctx, cudaEventCreate(&ctx->ev_t0));
        TB2_CUDA_TRY(ctx, cudaEventCreate(&ctx->ev_t1));
    }
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev_t0, ctx->stream));
    return TB2_OK;
}

extern "C" int tb2_timer_stop(tb2_ctx *ctx, double *ms_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!ctx->ev_t0 || !ms_out) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev_t1, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_t1));
    float ms = 0;
    TB2_CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_t0, ctx->ev_t1));
    *ms_out = ms;
    return TB2_OK;
}

extern "C" const char *tb2_status_message(int s)
{
    switch (s) {
    case TB2_OK: return "";
    case TB2_ERR_FEWER_CPTS: return "Fewer changepoints found than requested";
    case TB2_ERR_BEYOND_BANDWIDTH: return "Read event to sequence alignment extends beyond bandwidth";
    case TB2_ERR_ADAPTIVE_BEYOND_SIGNAL: return "Adaptive signal to seqeunce alignment extended beyond raw signal";
    case TB2_ERR_NOT_ENOUGH_DEL_SIGNAL: return "Not enough raw signal around potential genomic deletion(s)";
    case TB2_ERR_TOO_MANY_DELS: return "Read contains too many potential genomic deletions";
    case TB2_ERR_INVALID_SEG: return "Invalid segmentation results.";
    case TB2_ERR_ZERO_LEN_SEG: return "New segments include zero length events";
    case TB2_ERR_NEG_SEG: return "New segments start with negative index";
    case TB2_ERR_SEG_PAST_END: return "New segments end past raw signal values";
    case TB2_ERR_START_TOO_FAR: return "Read sequence to signal matching starts too far into events for full adaptive assignment";
    case TB2_ERR_MASKED_TOO_FEW: return "Masked z-score contains too few events.";
    case TB2_ERR_READ_TOO_SHORT_START: return "Read too short for start/end discovery";
    case TB2_ERR_MAP_TOO_SHORT_START: return "Genomic mapping too short for start/end discovery";
    case TB2_ERR_POOR_START_MATCH: return "Poor raw to expected signal matching in beginning of read.";
    case TB2_ERR_DISCORDANT_LEN: return "Discordant reference and seqeunce lengths.";
    case TB2_ERR_OPEN_PORE: return "Very poor signal quality. Read likely includes open pore.";
    case TB2_ERR_NO_RAW: return "Must have raw signal in order to complete re-squiggle algorithm";
    case TB2_ERR_TOO_MUCH_SIGNAL: return "Too much raw signal for mapped sequence";
    case TB2_ERR_SEG_COUNT: return "Aligned sequence does not match number of segments produced";
    case TB2_ERR_THEIL_SEN_ZERO: return "Read failed sequence-based signal re-scaling parameter estimation.";
    case TB2_ERR_INVALID_START_PATH: return "Invalid path through read start";
    case TB2_ERR_READ_TOO_SHORT_IN_REGION: return "Read sequence too short in this region.";
    case TB2_ERR_NO_INFO_IN_REGION: return "Read does not contain information in this region.";
    case TB2_ERR_FISHER_TOO_SHORT: return "P-values vector too short for Fisher's Method window compuation.";
    case TB2_ERR_NO_VALID_Z: return "No valid z-scores in read.";
    case TB2_ERR_UNEXPECTED: return "UNEXPECTED";
    case TB2_ERR_CUDA: return "CUDA error";
    case TB2_ERR_INVALID_ARG: return "invalid argument";
    case TB2_ERR_CAPACITY: return "problem exceeds compiled-in capacity";
    case TB2_ERR_INVALID_SEQ: return "Invalid sequence encountered from genome sequence.";
    default: return "unknown status";
    }
}
