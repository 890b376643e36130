// kernels.h -- internal launch interfaces between translation units
#pragma once
#ifdef TB2_EMUL   // host emulation of the device code (tests/emul): no CUDA runtime types
#include <stddef.h>
#include "../../include/tombo_b200.h"
struct tb2_ctx;
#else
#include "ctx.h"
#endif

// Device-resident batch description for the event->sequence assignment kernel.
// All arrays live in device memory.  Read r owns
//   cpts/em        at ev_off[r]   (n_cpts[r] changepoints, n_cpts[r]-1 event means)
//   rm/rs/starts   at base_off[r] (nb = base_off[r+1]-base_off[r])
//   read_tb/segs   at base_off[r] + r   (nb + 1 entries)
struct AlignBatch {
    int n_reads;
    const int *order;   // work order (longest first), null = index order
    const int *cpts;
    const double *em;
    const long long *ev_off;
    const int *n_cpts;        // n_cpts[r * stride]
    const int *num_events;    // requested events (class filter), may be null
    const double *rm, *rs;
    const long long *base_off;
    int *starts, *read_tb, *segs;
    int *rsrtr;        // rsrtr[r * stride]
    int *status;       // status[r * stride] in/out: processed only where TB2_OK on entry
    const int *active; // active[r * stride] != 0, may be null (all)
    int stride;        // element stride (ints) of n_cpts / rsrtr / status / active
    int *dbg;          // 3 ints per read or null
    tb2_params params;
    double sig_match_thresh;
};

struct AlignLaunchCfg {
    int smem_cells;       // per-warp row-buffer capacity in shared memory (cells)
    size_t tb_words;      // per-warp packed-move scratch (uint32 words)
    int grow_cells;       // per-warp global row scratch capacity (0 = none)
    int klass;            // 0: all reads; 1: static-band kernel, short reads only;
                          // 2: general kernel, long reads only
};

// launches the persistent warp-per-read kernel on ctx->stream
int tb2_launch_align(tb2_ctx *ctx, const AlignBatch &b, const AlignLaunchCfg &cfg);

#ifndef TB2_EMUL
// per-warp scratch of k_align (tb2_launch_align) and k_resolve (tb2_launch_resolve).  It holds
// nothing between launches, and launches on one context are stream-ordered, so the resident
// batch and the single-read mirrors share it.
struct LaunchScratch {
    DevBuf tb, grow, align_cnt;      // k_align: packed moves, global rows, work counter
    DevBuf raw_dp, resolve_cnt, raw_big;   // k_resolve: per-warp slabs, counters, overflow arena
};
#endif

// chunk width of the register engine for the adaptive band (dp_row2.cuh), 0 = band too wide
#if defined(__CUDACC__) || defined(TB2_EMUL)
__host__ __device__
#endif
static inline int tb2_abs_chunk_host(long long W)
{
    return W <= 218 ? 7 : (W <= 311 ? 10 : (W <= 404 ? 13 : (W <= 528 ? 17 : 0)));
}
// wide bands: three chunks per lane (dp_row2.cuh, multi-slab engine); chunk width or 0
#if defined(__CUDACC__) || defined(TB2_EMUL)
__host__ __device__
#endif
static inline int tb2_abs_ms_chunk_host(long long W)
{
    return (W > 528 && W <= 95 * 13 + 1) ? 13 : ((W > 528 && W <= 95 * 17 + 1) ? 17 : 0);
}
#define TB2_ABS_MS_SLABS 3
// packed-move words per adaptive row and lane for band width W (register engines), 0 if the
// band runs on the lane-chunk engine
#if defined(__CUDACC__) || defined(TB2_EMUL)
__host__ __device__
#endif
static inline int tb2_abs_words_per_row(long long W)
{
    const int c1 = tb2_abs_chunk_host(W);
    if (c1) return c1 > 16 ? 2 : 1;
    const int c3 = tb2_abs_ms_chunk_host(W);
    return c3 ? TB2_ABS_MS_SLABS * (c3 > 16 ? 2 : 1) : 0;
}
// capacity helper (host): packed-move words needed for (rows, W)
#define TB2_MAX_CHUNK 256   // cells per lane: band widths up to 8192 (dp_align.cuh)
// wavefront engine: step-space move words, 32 * (strip span / 16 + 1) per 32-row strip
// (dp_row.cuh tb2_wf_strip_words); drift = upper bound of last band start - first
static inline size_t tb2_wf_words_bound(long long rows, long long W, long long drift)
{
    const long long strips = (rows + 31) / 32;
    return (size_t)(strips * 32 * ((W + 30) / 16 + 2) + 2 * (drift < 0 ? 0 : drift) + 64);
}
static inline size_t tb2_tb_words(long long rows, long long W, long long drift)
{
    long long chunk = (W + 31) / 32;
    long long wpl = (chunk + 15) / 16;
    wpl = wpl <= 5 ? wpl : (wpl <= 8 ? 8 : 16);   // instantiated widths (tb2_wpl_of)
    if (tb2_abs_words_per_row(W) > wpl) wpl = tb2_abs_words_per_row(W);
    // lane-chunk rows (wpl * 32 words) plus wavefront rows: an upper bound valid for
    // every mix of the two engines
    return (size_t)(rows * wpl * 32) + tb2_wf_words_bound(rows, W, drift);
}
// doubles of shared memory per warp for the wavefront engine's lane-to-lane exchange
// (dp_row.cuh TB2_WF_FAST_STEP): 32 lanes + 16 steps on the diagonal
#define TB2_WF_RING 48
static inline int tb2_row_cells(long long W) { return (int)(((W + 31) / 32) * 32); }
