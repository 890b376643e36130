// pipeline.cu -- host orchestration of the batched resquiggle path and the C-ABI
// entry points built on the stage kernels.  The worker policy of the reference
// (iterate while norm_params_changed, retry failed reads once with the save
// bandwidth; resquiggle.py:1492-1504, 1578-1588) is a host loop over kernel
// launches on the whole batch; every kernel skips reads that are not active.
#include "batch.h"
#include <chrono>
#include <exception>
#include <string>
#include <cstdio>
#include <cstdlib>
#include "kernels.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

int tb2_launch_start_attempt(tb2_ctx *ctx, const BatchView &b, int attempt);
int tb2_launch_end_call(tb2_ctx *ctx, const BatchView &b, int max_iters);

// device arrays behind one BatchView (build_view).  The resident batch owns one set; the
// single-read mirrors build their views in a second set, so they never touch a resident batch.
struct BatchBuffers {
    DevBuf raw_off, seq_off, base_off, ev_off, seq, rawf, norm, cs, scores, cstate, cpts, em, rm, rs,
        bm, tmp_b, starts, read_tb, segs_dp, segs, stalls, state, order;
    DevBuf dbg;        // k_align: 3 ints per read
    DevBuf counters;   // tb2_launch_count_active
};

namespace {

// optional caller-provided per-read inputs of resquiggle_read: map_res.scale_values
// and map_res.stall_ints (resquiggle.py:1079-1084, 1101-1103)
__global__ void k_apply_inputs(BatchView b, const tb2_scale_values *sv_in, const int *n_stalls)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= b.n_reads) return;
    ReadState &s = b.st[r];
    if (n_stalls) s.n_stalls = n_stalls[r];
    if (sv_in && s.active && !isnan(sv_in[r].shift)) { s.use_sv = 1; s.sv = sv_in[r]; }
}

struct HostBatch {
    int n = 0;
    std::vector<long long> base_off, ev_off;
    long long total_s = 0, total_seq = 0, total_b = 0, total_e = 0;
};

long long num_events_of(long long n_raw, long long nb, const tb2_params &p, double ratio)
{
    const long long a = n_raw / p.mean_obs_per_event;
    const long long c = (long long)((double)nb * ratio);
    return a > c ? a : c;
}

// fills B for n reads and points v into it
int build_view(tb2_ctx *ctx, BatchBuffers &B, int n, const int64_t *raw_off, const int64_t *seq_off,
               int K, const tb2_params &p, double ratio, int is_rna, HostBatch &hb, BatchView &v)
{
    hb.n = n;
    long long max_raw_pre = 0;
    for (int r = 0; r < n; ++r) max_raw_pre = std::max<long long>(max_raw_pre, raw_off[r + 1] - raw_off[r]);
    hb.base_off.assign(n + 1, 0);
    hb.ev_off.assign(n + 1, 0);
    for (int r = 0; r < n; ++r) {
        const long long s = raw_off[r + 1] - raw_off[r];
        long long nb = (seq_off[r + 1] - seq_off[r]) - (K - 1);
        if (nb < 0) nb = 0;
        if (s < 0 || s > 0x3fffffff || nb > 0x3fffffff || seq_off[r + 1] < seq_off[r])
            return TB2_ERR_INVALID_ARG;
        hb.base_off[r + 1] = hb.base_off[r] + nb;
        hb.ev_off[r + 1] = hb.ev_off[r] + std::max<long long>(2, num_events_of(s, nb, p, ratio)) + 1;
    }
    const long long max_raw = max_raw_pre;
    v.max_raw = (int)max_raw;
    hb.total_s = raw_off[n] - raw_off[0];
    hb.total_seq = seq_off[n] - seq_off[0];
    hb.total_b = hb.base_off[n];
    hb.total_e = hb.ev_off[n];
    if (raw_off[0] != 0 || seq_off[0] != 0) return TB2_ERR_INVALID_ARG;
    const size_t S = (size_t)hb.total_s, Bn = (size_t)hb.total_b, E = (size_t)hb.total_e;
    // a stall needs > 200 consecutive observations (MEAN_STALL_PARAMS), so a read of S
    // samples holds at most S / 200 + 1 intervals: size the slots from the longest read
    const int stall_cap = (int)std::max<long long>(8, max_raw_pre / 200 + 4);
    TB2_CUDA_TRY(ctx, B.seq.reserve((size_t)hb.total_seq + 8));
    TB2_CUDA_TRY(ctx, B.rawf.reserve(S * 8 + 8));
    TB2_CUDA_TRY(ctx, B.norm.reserve(S * 8 + 8));
    TB2_CUDA_TRY(ctx, B.cs.reserve((S + n) * 8 + 8));
    TB2_CUDA_TRY(ctx, B.scores.reserve(S * 8 + 8));
    TB2_CUDA_TRY(ctx, B.cstate.reserve(2 * S + 128 * (size_t)n + 16));
    TB2_CUDA_TRY(ctx, B.cpts.reserve(E * 4 + 8));
    TB2_CUDA_TRY(ctx, B.em.reserve(E * 8 + 8));
    TB2_CUDA_TRY(ctx, B.rm.reserve(Bn * 8 + 8));
    TB2_CUDA_TRY(ctx, B.rs.reserve(Bn * 8 + 8));
    TB2_CUDA_TRY(ctx, B.bm.reserve(Bn * 8 + 8));
    TB2_CUDA_TRY(ctx, B.tmp_b.reserve((Bn + n) * 8 + 8));
    TB2_CUDA_TRY(ctx, B.starts.reserve(Bn * 4 + 8));
    TB2_CUDA_TRY(ctx, B.read_tb.reserve((Bn + n) * 4 + 8));
    TB2_CUDA_TRY(ctx, B.segs_dp.reserve((Bn + n) * 4 + 8));
    TB2_CUDA_TRY(ctx, B.segs.reserve((Bn + n) * 4 + 8));
    TB2_CUDA_TRY(ctx, B.stalls.reserve(is_rna ? (size_t)n * 2 * stall_cap * 4 + 8 : 8));
    TB2_CUDA_TRY(ctx, B.state.reserve((size_t)n * sizeof(ReadState)));
    TB2_CUDA_TRY(ctx, B.dbg.reserve((size_t)n * 3 * 4));
    TB2_CUDA_TRY(ctx, B.counters.reserve(64));
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, B.raw_off.upload(raw_off, (size_t)n + 1, s));
    TB2_CUDA_TRY(ctx, B.seq_off.upload(seq_off, (size_t)n + 1, s));
    TB2_CUDA_TRY(ctx, B.base_off.upload(hb.base_off.data(), (size_t)n + 1, s));
    TB2_CUDA_TRY(ctx, B.ev_off.upload(hb.ev_off.data(), (size_t)n + 1, s));
    // launch order: longest reads first, so that the persistent DP warps and the
    // CTA-per-read kernels do not end on a straggler (length bucketing of mixed batches)
    v.order = nullptr;
    {
        long long mn = max_raw;
        for (int r = 0; r < n; ++r) mn = std::min<long long>(mn, raw_off[r + 1] - raw_off[r]);
        if (mn != max_raw && n > 1) {
            std::vector<int> order((size_t)n);
            for (int r = 0; r < n; ++r) order[r] = r;
            std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
                return raw_off[a + 1] - raw_off[a] > raw_off[b + 1] - raw_off[b];
            });
            TB2_CUDA_TRY(ctx, B.order.upload(order.data(), (size_t)n, s));
            TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));   // order is a local
            v.order = B.order.as<int>();
        }
    }
    v.n_reads = n;
    v.kmer_width = K;
    v.raw_off = B.raw_off.as<long long>();
    v.seq_off = B.seq_off.as<long long>();
    v.base_off = B.base_off.as<long long>();
    v.ev_off = B.ev_off.as<long long>();
    v.seq = B.seq.as<unsigned char>();
    v.rawf = B.rawf.as<double>();
    v.norm = B.norm.as<double>();
    v.cs = B.cs.as<double>();
    v.scores = B.scores.as<double>();
    v.cstate = B.cstate.as<unsigned char>();
    v.cpts = B.cpts.as<int>();
    v.em = B.em.as<double>();
    v.rm = B.rm.as<double>();
    v.rs = B.rs.as<double>();
    v.bm = B.bm.as<double>();
    v.tmp_b = B.tmp_b.as<double>();
    v.starts = B.starts.as<int>();
    v.read_tb = B.read_tb.as<int>();
    v.segs_dp = B.segs_dp.as<int>();
    v.segs = B.segs.as<int>();
    v.stall_ints = is_rna ? B.stalls.as<int>() : nullptr;
    v.stall_cap = stall_cap;
    v.st = B.state.as<ReadState>();
    return TB2_OK;
}

// capacity plan per read class: short reads (static band only) get the lean kernel
void plan_align_batch(const tb2_params &p, const HostBatch &hb, const int64_t *raw_off, double ratio,
                      AlignLaunchCfg *cs, AlignLaunchCfg *cl, int *n_short, int *n_long)
{
    cs->smem_cells = 32; cs->tb_words = 32; cs->grow_cells = 0; cs->klass = 1;
    cl->smem_cells = 32; cl->tb_words = 32; cl->grow_cells = 0; cl->klass = 2;
    *n_short = *n_long = 0;
    for (int r = 0; r < hb.n; ++r) {
        const long long nb = hb.base_off[r + 1] - hb.base_off[r];
        const long long n_em = num_events_of(raw_off[r + 1] - raw_off[r], nb, p, ratio) - 1;
        if (nb < 1 || n_em < 1) continue;
        const long long mask_len = std::min(nb, n_em) / 4;
        const long long w_static = std::max<long long>(1, n_em - mask_len);
        const bool is_short = n_em < p.start_bw + p.start_n_bases || nb < p.start_n_bases;
        if (is_short) {
            ++*n_short;
            if (tb2_row_cells(w_static) / 32 > TB2_MAX_CHUNK) continue;  // CAPACITY status on device
            // static band: one plain row (wavefront engine); smem_cells counts pairs
            cs->smem_cells = std::max(cs->smem_cells, tb2_row_cells((w_static + 1) / 2));
            cs->tb_words = std::max(cs->tb_words, tb2_wf_words_bound(nb, w_static, mask_len + 1));
        } else {
            ++*n_long;
            // start search: one plain row; adaptive rows: four transposed rows when the
            // band is narrow enough for the fast path (<= 512 cells), else two
            // adaptive rows up to 528 cells live in registers (dp_row2.cuh) and only the masked
            // start rows need one plain row; wider bands keep two (four up to 512) transposed
            // rows for the lane-chunk engine
            const long long bw_cells = tb2_row_cells(p.bandwidth);
            const long long bw_pairs =
                tb2_abs_chunk_host(p.bandwidth) != 0 ? (p.bandwidth + 1) / 2
                : tb2_abs_ms_chunk_host(p.bandwidth) != 0
                    ? std::max<long long>((p.bandwidth + 1) / 2,
                                          (long long)TB2_ABS_MS_SLABS * tb2_abs_ms_chunk_host(p.bandwidth) * 16)
                    : (p.bandwidth <= 512 ? 2 * bw_cells : bw_cells);
            cl->smem_cells = std::max(cl->smem_cells,
                                      tb2_row_cells(std::max<long long>((p.start_bw + 1) / 2, bw_pairs)));
            cl->tb_words = std::max(cl->tb_words, std::max(tb2_tb_words(nb, p.bandwidth, n_em + p.bandwidth),
                                                           tb2_tb_words(p.start_n_bases, p.start_bw, p.start_n_bases)));
            if (n_em >= p.start_save_bw + p.start_n_bases) {
                cl->tb_words = std::max(cl->tb_words, tb2_tb_words(p.start_n_bases, p.start_save_bw, p.start_n_bases));
                cl->grow_cells = std::max(cl->grow_cells, tb2_row_cells(p.start_save_bw));
            }
            // long reads may fall back to the static band (failed start search with
            // too few events for the save bandwidth, or a start too close to the
            // read end: resquiggle.py:996-999, 1024-1027); rows live in global memory
            if (tb2_row_cells(w_static) / 32 <= TB2_MAX_CHUNK) {
                cl->tb_words = std::max(cl->tb_words, tb2_tb_words(nb, w_static, mask_len + 1));
                cl->grow_cells = std::max(cl->grow_cells, tb2_row_cells(w_static));
            }
        }
    }
}

__global__ void k_export(BatchView b, const int *dbg, long long *segs64, long long *rsrtr64,
                         tb2_scale_values *sv, double *score, int *status, int *n_iters,
                         int *flags)
{
    const int r = blockIdx.x;
    const ReadState &s = b.st[r];
    const long long bo = b.base_off[r];
    const int nb = (int)(b.base_off[r + 1] - bo);
    const bool ok = s.status == TB2_OK && s.done;
    for (int i = threadIdx.x; i <= nb; i += blockDim.x)
        segs64[bo + r + i] = ok ? (long long)b.segs[bo + r + i] : 0;
    if (threadIdx.x == 0) {
        rsrtr64[r] = ok ? s.rsrtr : 0;
        sv[r] = s.sv;
        score[r] = ok ? s.score : NAN;
        status[r] = s.status;
        n_iters[r] = s.n_iters;
        flags[r] = (s.changed ? 1 : 0) | (s.attempt ? 2 : 0) | ((dbg && dbg[3 * r] == 0) ? 4 : 0);
    }
}

StagePolicy stage_policy(const tb2_policy &pl)
{
    StagePolicy sp;
    sp.outlier_thresh = pl.outlier_thresh;
    sp.max_raw_cpts = pl.max_raw_cpts;
    sp.min_event_to_seq_ratio = pl.min_event_to_seq_ratio;
    sp.sig_match_thresh = pl.sig_match_thresh;
    sp.max_scaling_iters = (int)pl.max_scaling_iters;
    sp.is_rna = (int)pl.is_rna;
    sp.skip_seq_scaling = (int)pl.skip_seq_scaling;
    sp.const_scale = pl.const_scale;
    sp.subsample_seed = pl.subsample_seed;
    sp.literal_key = 0;
    sp.read_index_base = 0;
    return sp;
}

AlignBatch make_align_batch(const BatchBuffers &B, const BatchView &v, const tb2_params &p,
                            double thresh)
{
    AlignBatch ab;
    ab.n_reads = v.n_reads;
    ab.order = v.order;
    ab.cpts = v.cpts; ab.em = v.em; ab.ev_off = v.ev_off;
    ab.rm = v.rm; ab.rs = v.rs; ab.base_off = v.base_off;
    ab.starts = v.starts; ab.read_tb = v.read_tb; ab.segs = v.segs_dp;
    ab.stride = (int)(sizeof(ReadState) / sizeof(int));
    ab.n_cpts = &v.st[0].n_cpts;
    ab.num_events = &v.st[0].num_events;
    ab.rsrtr = &v.st[0].rsrtr;
    ab.status = &v.st[0].status;
    ab.active = &v.st[0].active;
    ab.dbg = B.dbg.as<int>();
    ab.params = p;
    ab.sig_match_thresh = thresh;
    return ab;
}

// one resquiggle_read call over the batch (all active reads)
int run_call(tb2_ctx *ctx, const BatchBuffers &B, const BatchView &v, const tb2_params &p,
             const StagePolicy &sp,
             const AlignLaunchCfg *acfg /* [2]: short, long; tb_words 0 = class empty */,
             int first_call, double *norm_mean_dev,
             double *norm_sig_dev, size_t rawdp_cap)
{
    int rc;
    if ((rc = tb2_launch_begin_call(ctx, v, p, sp))) return rc;
    if (p.use_t_test_seg) {
        // RNA: t-test changepoints on the raw signal, event-based scaling
        // (segment_signal resquiggle.py:1072-1098)
        if ((rc = tb2_launch_cpts(ctx, v, p, 1))) return rc;
        if ((rc = tb2_launch_rna_scale(ctx, v, sp))) return rc;
        if ((rc = tb2_launch_normalize(ctx, v, sp, first_call))) return rc;
    } else {
        if ((rc = tb2_launch_normalize(ctx, v, sp, first_call))) return rc;
        if ((rc = tb2_launch_cpts(ctx, v, p, 0))) return rc;
    }
    if ((rc = tb2_launch_event_means(ctx, v))) return rc;
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev2, ctx->stream));
    for (int k = 0; k < 2; ++k)
        if (acfg[k].tb_words > 0 &&
            (rc = tb2_launch_align(ctx, make_align_batch(B, v, p, sp.sig_match_thresh), acfg[k])))
            return rc;
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev3, ctx->stream));
    if ((rc = tb2_launch_resolve(ctx, v, p, sp, rawdp_cap))) return rc;
    if ((rc = tb2_launch_base_means(ctx, v))) return rc;
    if ((rc = tb2_launch_theil_sen(ctx, v, sp, first_call))) return rc;
    if ((rc = tb2_launch_finalize(ctx, v, sp, first_call, norm_mean_dev, norm_sig_dev))) return rc;
    if ((rc = tb2_launch_end_call(ctx, v, sp.max_scaling_iters))) return rc;
    return TB2_OK;
}

}  // namespace

// ---------------------------------------------------------------------------
extern "C" int tb2_set_model(tb2_ctx *ctx, const double *means, const double *sds, int kmer_width,
                             int central_pos)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!means || !sds || kmer_width < 1 || kmer_width > 12 || central_pos < 0 ||
        central_pos >= kmer_width)
        return TB2_ERR_INVALID_ARG;
    const size_t n = (size_t)1 << (2 * kmer_width);
    TB2_CUDA_TRY(ctx, ctx->model_means.upload(means, n, ctx->stream));
    TB2_CUDA_TRY(ctx, ctx->model_sds.upload(sds, n, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->kmer_width = kmer_width;
    ctx->central_pos = central_pos;
    return TB2_OK;
}

// ---------------------------------------------------------------------------
// batched hot path in three stages: upload (H2D), compute (kernels only; results
// stay on the device), download (D2H).  tb2_resquiggle_batch = all three.
// ---------------------------------------------------------------------------
struct BatchHolder {
    HostBatch hb;
    BatchView v;
    std::vector<int64_t> raw_off;
    int raw_dtype = 0;
    bool uploaded = false, computed = false, has_norm_sig = false;
    bool has_sv_in = false, has_stalls_in = false;
    BatchBuffers buf;                  // behind v
    DevBuf raw_in, sv_in, n_stall;     // uploaded signal, tb2_batch_set_read_inputs
    // export staging: segs (int64), norm_mean, norm_signal, and the per-read results (SmallOut)
    DevBuf out_segs, out_norm_mean, out_norm_sig, out_small;
};

namespace {
BatchHolder *holder_of(tb2_ctx *ctx) { return &tb2_state(ctx->batch); }

// layout of BatchHolder::out_small: six per-read arrays back to back
struct SmallOut {
    long long *rsrtr;
    tb2_scale_values *sv;
    double *score;
    int *status, *n_iters, *flags;
};
size_t small_out_bytes(int n) { return (size_t)n * (8 + sizeof(tb2_scale_values) + 8 + 4 + 4 + 4); }
SmallOut small_out(const DevBuf &b, int n)
{
    SmallOut o;
    o.rsrtr = b.as<long long>();
    o.sv = (tb2_scale_values *)(o.rsrtr + n);
    o.score = (double *)(o.sv + n);
    o.status = (int *)(o.score + n);
    o.n_iters = o.status + n;
    o.flags = o.n_iters + n;
    return o;
}
}  // namespace

static int batch_upload_impl(tb2_ctx *ctx, int64_t n_reads, const void *raw, int raw_dtype,
                                const int64_t *raw_off, const uint8_t *seq, const int64_t *seq_off,
                                const tb2_params *params, const tb2_policy *policy)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n_reads < 1 || n_reads > 0x7ffffff0 || !raw || !seq || !raw_off || !seq_off || !params ||
        !policy || (raw_dtype != 0 && raw_dtype != 1))
        return TB2_ERR_INVALID_ARG;
    if (ctx->kmer_width <= 0) { ctx->err = "tb2_set_model has not been called"; return TB2_ERR_INVALID_ARG; }
    BatchHolder *h = holder_of(ctx);
    h->uploaded = h->computed = false;
    const int n = (int)n_reads;
    rc = build_view(ctx, h->buf, n, raw_off, seq_off, ctx->kmer_width, *params,
                    policy->min_event_to_seq_ratio, (int)policy->is_rna, h->hb, h->v);
    if (rc) return rc;
    h->raw_off.assign(raw_off, raw_off + n + 1);
    h->raw_dtype = raw_dtype;
    cudaStream_t s = ctx->stream;
    const size_t esz = raw_dtype == 0 ? 8 : 2;
    TB2_CUDA_TRY(ctx, h->raw_in.reserve((size_t)h->hb.total_s * esz + 8));
    // the (small, possibly pageable) sequence copy goes first: a pageable source blocks the
    // host until the copy has run, and behind the big signal copy that would serialise
    // the pipelined path (H2D of chunk k+1 must overlap the kernels of chunk k)
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(h->buf.seq.p, seq, (size_t)h->hb.total_seq, cudaMemcpyHostToDevice, s));
    if (getenv("TB2_TRACE")) {
        if (!ctx->ev_h0) { cudaEventCreate(&ctx->ev_h0); cudaEventCreate(&ctx->ev_h1); }
        cudaEventRecord(ctx->ev_h0, s);
    }
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(h->raw_in.p, raw, (size_t)h->hb.total_s * esz, cudaMemcpyHostToDevice, s));
    if (ctx->ev_h1) cudaEventRecord(ctx->ev_h1, s);
    if (!ctx->async_mode) TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    h->uploaded = true;
    h->has_sv_in = h->has_stalls_in = false;
    return TB2_OK;
}

static int batch_set_read_inputs_impl(tb2_ctx *ctx, const tb2_scale_values *sv_in,
                                         const int64_t *stall_ints, const int64_t *stall_off)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    BatchHolder *h = holder_of(ctx);
    if (!h->uploaded) { ctx->err = "tb2_batch_upload has not been called"; return TB2_ERR_INVALID_ARG; }
    const int n = h->hb.n;
    cudaStream_t s = ctx->stream;
    h->has_sv_in = sv_in != nullptr;
    if (sv_in) {
        TB2_CUDA_TRY(ctx, h->sv_in.upload(sv_in, (size_t)n, s));
    }
    h->has_stalls_in = stall_off != nullptr;
    if (stall_off) {
        int cap = 1;
        for (int r = 0; r < n; ++r) cap = std::max<int>(cap, (int)(stall_off[r + 1] - stall_off[r]));
        std::vector<int> flat((size_t)n * 2 * cap, 0), cnt((size_t)n, 0);
        for (int r = 0; r < n; ++r) {
            cnt[r] = (int)(stall_off[r + 1] - stall_off[r]);
            for (int k = 0; k < cnt[r]; ++k) {
                flat[((size_t)r * cap + k) * 2] = (int)stall_ints[2 * (stall_off[r] + k)];
                flat[((size_t)r * cap + k) * 2 + 1] = (int)stall_ints[2 * (stall_off[r] + k) + 1];
            }
        }
        TB2_CUDA_TRY(ctx, h->buf.stalls.upload(flat.data(), flat.size(), s));
        TB2_CUDA_TRY(ctx, h->n_stall.upload(cnt.data(), (size_t)n, s));
        h->v.stall_ints = h->buf.stalls.as<int>();
        h->v.stall_cap = cap;
    }
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

static int batch_compute_impl(tb2_ctx *ctx, const tb2_params *params,
                                 const tb2_params *save_params, const tb2_policy *policy,
                                 int want_norm_signal)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!params || !policy) return TB2_ERR_INVALID_ARG;
    if (policy->rescue && !save_params) return TB2_ERR_INVALID_ARG;
    BatchHolder *h = holder_of(ctx);
    if (!h->uploaded) { ctx->err = "tb2_batch_upload has not been called"; return TB2_ERR_INVALID_ARG; }
    h->computed = false;
    StagePolicy sp = stage_policy(*policy);
    sp.read_index_base = ctx->read_index_base;
    const HostBatch &hb = h->hb;
    const BatchView &v = h->v;
    const int n = hb.n;
    cudaStream_t s = ctx->stream;
    const bool trace = getenv("TB2_TRACE") != nullptr;
    auto now_ms = [] {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    };
    const double tc0 = now_ms();
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, s));
    TB2_CUDA_TRY(ctx, h->out_norm_mean.reserve((size_t)hb.total_b * 8 + 8));
    double *norm_sig_dev = nullptr;
    if (want_norm_signal) {
        TB2_CUDA_TRY(ctx, h->out_norm_sig.reserve((size_t)hb.total_s * 8 + 8));
        norm_sig_dev = h->out_norm_sig.as<double>();
    }
    h->has_norm_sig = want_norm_signal != 0;
    double *norm_mean_dev = h->out_norm_mean.as<double>();
    if ((rc = tb2_launch_prep(ctx, v, h->raw_in.p, h->raw_dtype, sp.is_rna, hb.total_s, hb.total_b))) return rc;
    if (sp.is_rna && !h->has_stalls_in && (rc = tb2_launch_stalls(ctx, v))) return rc;
    const size_t rawdp_cap = (size_t)1 << 15;
    double ms_dp = 0, dp_reads = 0;
    int dp_launches = 0;
    int counters[2] = {0, 0};
    for (int attempt = 0; attempt < 2; ++attempt) {
        if (attempt == 1 && (!policy->rescue || counters[1] == 0)) break;
        const tb2_params &p = attempt == 0 ? *params : *save_params;
        AlignLaunchCfg acfg[2];
        int n_short = 0, n_long = 0;
        plan_align_batch(p, hb, h->raw_off.data(), sp.min_event_to_seq_ratio, &acfg[0], &acfg[1],
                         &n_short, &n_long);
        if (n_short == 0) acfg[0].tb_words = 0;
        if (n_long == 0) acfg[1].tb_words = 0;
        if ((rc = tb2_launch_start_attempt(ctx, v, attempt))) return rc;
        if (h->has_sv_in || h->has_stalls_in) {
            k_apply_inputs<<<(n + 255) / 256, 256, 0, s>>>(
                v, h->has_sv_in ? h->sv_in.as<tb2_scale_values>() : nullptr,
                h->has_stalls_in ? h->n_stall.as<int>() : nullptr);
            TB2_CHECK_LAUNCH(ctx);
        }
        double active_now = attempt == 0 ? n : counters[1];
        for (int it = 0; it < std::max(1, sp.max_scaling_iters); ++it) {
            if ((rc = run_call(ctx, h->buf, v, p, sp, acfg, it == 0, norm_mean_dev, norm_sig_dev, rawdp_cap)))
                return rc;
            if ((rc = tb2_launch_count_active(ctx, v, h->buf.counters.as<int>()))) return rc;
            if (attempt == 0 && it == 0 && ctx->after_first_launch) {
                auto fn = std::move(ctx->after_first_launch);
                ctx->after_first_launch = nullptr;
                if ((rc = fn())) return rc;
            }
            // read back through page-locked memory: a pageable destination would make the
            // driver stage the copy and stall behind the other lane's bulk transfers
            if (!ctx->pinned) {
                TB2_CUDA_TRY(ctx, cudaHostAlloc(&ctx->pinned, 256, cudaHostAllocPortable));
                ctx->pinned_cap = 256;
            }
            const double th0 = trace ? now_ms() : 0;
            TB2_CUDA_TRY(ctx, cudaMemcpyAsync(ctx->pinned, h->buf.counters.p, 8, cudaMemcpyDeviceToHost, s));
            TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
            memcpy(counters, ctx->pinned, 8);
            if (trace) fprintf(stderr, "[tb2]   call %d.%d: enqueued at +%.2f ms, synced at +%.2f ms\n", attempt, it, th0 - tc0, now_ms() - tc0);
            float ms = 0;
            if (cudaEventElapsedTime(&ms, ctx->ev2, ctx->ev3) == cudaSuccess) {
                ms_dp += ms; ++dp_launches; dp_reads += active_now;
            }
            active_now = counters[0];
            if (counters[0] == 0) break;
        }
    }
    // ---- export into device staging ----
    const size_t nsegs = (size_t)hb.total_b + n;
    TB2_CUDA_TRY(ctx, h->out_segs.reserve(nsegs * 8 + 8));
    TB2_CUDA_TRY(ctx, h->out_small.reserve(small_out_bytes(n) + 64));
    const SmallOut o = small_out(h->out_small, n);
    k_export<<<n, 128, 0, s>>>(v, h->buf.dbg.as<int>(), h->out_segs.as<long long>(), o.rsrtr, o.sv,
                               o.score, o.status, o.n_iters, o.flags);
    TB2_CHECK_LAUNCH(ctx);
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev1, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    ctx->last_ms_total = ms;
    ctx->last_ms_dp = ms_dp;
    ctx->last_dp_launches = dp_launches;
    ctx->last_dp_reads = dp_reads;
    h->computed = true;
    return TB2_OK;
}

int tb2_batch_result_view(tb2_ctx *ctx, BatchResultView *out)
{
    BatchHolder *h = holder_of(ctx);
    if (!h->computed) { ctx->err = "tb2_batch_compute has not been called"; return TB2_ERR_INVALID_ARG; }
    out->n_reads = h->hb.n;
    out->total_bases = h->hb.total_b;
    out->norm_mean = h->out_norm_mean.as<double>();
    out->base_off = h->v.base_off;
    out->seq_off = h->v.seq_off;
    out->seq = h->v.seq;
    out->status = &h->v.st[0].status;
    out->stride = (int)(sizeof(ReadState) / sizeof(int));
    return TB2_OK;
}

static int batch_download_impl(tb2_ctx *ctx, int64_t *segs, int64_t *read_start_rel_to_raw,
                                  tb2_scale_values *scale_out, double *sig_match_score,
                                  double *norm_mean, double *norm_signal, int32_t *status,
                                  int32_t *n_iters, int32_t *flags)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    BatchHolder *h = holder_of(ctx);
    if (!h->computed) { ctx->err = "tb2_batch_compute has not been called"; return TB2_ERR_INVALID_ARG; }
    if (!segs || !read_start_rel_to_raw || !scale_out || !sig_match_score || !status || !n_iters ||
        !flags || (norm_signal && !h->has_norm_sig))
        return TB2_ERR_INVALID_ARG;
    const HostBatch &hb = h->hb;
    const int n = hb.n;
    cudaStream_t s = ctx->stream;
    const size_t nsegs = (size_t)hb.total_b + n;
    const SmallOut o = small_out(h->out_small, n);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(segs, h->out_segs.p, nsegs * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(read_start_rel_to_raw, o.rsrtr, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(scale_out, o.sv, (size_t)n * sizeof(tb2_scale_values), cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(sig_match_score, o.score, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(status, o.status, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(n_iters, o.n_iters, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(flags, o.flags, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    if (norm_mean)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(norm_mean, h->out_norm_mean.p, (size_t)hb.total_b * 8, cudaMemcpyDeviceToHost, s));
    if (norm_signal)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(norm_signal, h->out_norm_sig.p, (size_t)hb.total_s * 8, cudaMemcpyDeviceToHost, s));
    if (!ctx->async_mode) TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

// Chunk schedule of the pipelined batch call (host only).  U = one read per resident DP
// warp of the lean kernel.  Up to 6 U reads go as one batch (returns 1 chunk); larger
// batches start with short chunks (the first upload is the only exposed one), continue
// with chunks of 6 U (the best of 6 / 8 / 12 on configs[1]) and end with the remainder.
static std::vector<int64_t> pipeline_chunk_starts(int sm_count, int64_t n_reads)
{
    std::vector<int64_t> cs;
    const int64_t U = (int64_t)std::max(1, sm_count) * 32, CH = 6 * U;
    int64_t at = 0;
    if (n_reads > 6 * U) {
        const int64_t ramp[2] = {2 * U, 4 * U};
        for (int q = 0; q < 2 && n_reads - at > ramp[q]; ++q) { cs.push_back(at); at += ramp[q]; }
        while (at < n_reads) { cs.push_back(at); at += CH; }
    } else {
        cs.push_back(0);
    }
    cs.push_back(n_reads);
    return cs;
}

extern "C" int tb2_pipeline_chunks(int sm_count, int64_t n_reads, int64_t *starts_out, int cap)
{
    if (n_reads < 0 || !starts_out || cap < 2) return -TB2_ERR_INVALID_ARG;
    try {
        const std::vector<int64_t> cs = pipeline_chunk_starts(sm_count, n_reads);
        if ((int)cs.size() > cap) return -TB2_ERR_CAPACITY;
        for (size_t i = 0; i < cs.size(); ++i) starts_out[i] = cs[i];
        return (int)cs.size() - 1;
    } catch (...) {
        return -TB2_ERR_UNEXPECTED;
    }
}

static int resquiggle_batch_impl(tb2_ctx *ctx, int64_t n_reads, const void *raw, int raw_dtype,
                                    const int64_t *raw_off, const uint8_t *seq,
                                    const int64_t *seq_off, const tb2_params *params,
                                    const tb2_params *save_params, const tb2_policy *policy,
                                    int64_t *segs, int64_t *read_start_rel_to_raw,
                                    tb2_scale_values *scale_out, double *sig_match_score,
                                    double *norm_mean, double *norm_signal, int32_t *status,
                                    int32_t *n_iters, int32_t *flags)
{
    if (n_reads == 0) return tb2_use(ctx);
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!raw_off || !seq_off || !params || !policy || !raw || !seq || !segs ||
        !read_start_rel_to_raw || !scale_out || !sig_match_score || !status || !n_iters || !flags ||
        (raw_dtype != 0 && raw_dtype != 1) || n_reads > 0x7ffffff0)
        return TB2_ERR_INVALID_ARG;
    const std::vector<int64_t> cstart = pipeline_chunk_starts(ctx->sm_count, n_reads);
    if (cstart.size() <= 2) {
        rc = tb2_batch_upload(ctx, n_reads, raw, raw_dtype, raw_off, seq, seq_off, params, policy);
        if (rc) return rc;
        if ((rc = tb2_batch_compute(ctx, params, save_params, policy, norm_signal != nullptr))) return rc;
        return tb2_batch_download(ctx, segs, read_start_rel_to_raw, scale_out, sig_match_score,
                                  norm_mean, norm_signal, status, n_iters, flags);
    }
    // ---- pipelined: chunk k+1 is uploaded (pinned host memory -> async DMA) while the
    // kernels of chunk k run; results stream back on the chunk's own stream ----
    while (ctx->lanes.size() < 2) {
        tb2_ctx *ln = new tb2_ctx();
        ln->device = ctx->device; ln->sm_count = ctx->sm_count;
        if (cudaStreamCreateWithFlags(&ln->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreate(&ln->ev0) != cudaSuccess || cudaEventCreate(&ln->ev1) != cudaSuccess ||
            cudaEventCreate(&ln->ev2) != cudaSuccess || cudaEventCreate(&ln->ev3) != cudaSuccess) {
            delete ln;
            ctx->err = "cannot create pipeline lane";
            return TB2_ERR_CUDA;
        }
        ctx->lanes.push_back(ln);
    }
    for (tb2_ctx *ln : ctx->lanes) {
        ln->model_means.p = ctx->model_means.p; ln->model_means.cap = ctx->model_means.cap;
        ln->model_sds.p = ctx->model_sds.p; ln->model_sds.cap = ctx->model_sds.cap;
        ln->model_means.owned = ln->model_sds.owned = false;
        ln->kmer_width = ctx->kmer_width; ln->central_pos = ctx->central_pos;
        ln->async_mode = true;
    }
    const int K = ctx->kmer_width;
    const int n = (int)n_reads;
    const int n_chunks = (int)cstart.size() - 1;
    std::vector<int64_t> base_off((size_t)n + 1, 0);
    for (int r = 0; r < n; ++r)
        base_off[r + 1] = base_off[r] + std::max<int64_t>(0, (seq_off[r + 1] - seq_off[r]) - (K - 1));
    std::vector<std::vector<int64_t>> ro((size_t)n_chunks), so((size_t)n_chunks);
    const size_t esz = raw_dtype == 0 ? 8 : 2;
    auto bounds = [&](int k, int *a, int *b) { *a = (int)cstart[k]; *b = (int)cstart[k + 1]; };
    auto upload = [&](int k) -> int {
        int a, b;
        bounds(k, &a, &b);
        tb2_ctx *ln = ctx->lanes[k & 1];
        if (cudaStreamSynchronize(ln->stream) != cudaSuccess) return TB2_ERR_CUDA;  // lane free again
        ro[k].resize((size_t)(b - a) + 1);
        so[k].resize((size_t)(b - a) + 1);
        for (int r = a; r <= b; ++r) { ro[k][r - a] = raw_off[r] - raw_off[a]; so[k][r - a] = seq_off[r] - seq_off[a]; }
        return tb2_batch_upload(ln, b - a, (const char *)raw + (size_t)raw_off[a] * esz, raw_dtype,
                                ro[k].data(), seq + seq_off[a], so[k].data(), params, policy);
    };
    double ms_total = 0, ms_dp = 0, dp_launches = 0, dp_reads = 0;
    const bool trace = getenv("TB2_TRACE") != nullptr;
    auto now_ms = [] {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    };
    const double t00 = now_ms();
    // (One host thread drives both lanes.  A thread per lane -- kernels of two chunks resident
    // side by side, optionally with the persistent DP grids sized to half an SM each -- was
    // slower end to end on configs[1]: the long
    // persistent DP kernels of one lane stall the short kernels of the other, and nothing is
    // gained back because the device is already never idle in this schedule.)
    rc = upload(0);
    for (int k = 0; k < n_chunks && rc == TB2_OK; ++k) {
        int a, b;
        bounds(k, &a, &b);
        tb2_ctx *ln = ctx->lanes[k & 1];
        const double t0 = now_ms();
        // the next chunk's upload is enqueued from inside compute(), right after this
        // chunk's first kernels: work submitted behind a bulk copy (even on another
        // stream) was observed to wait for it, work submitted ahead of it overlaps
        if (k + 1 < n_chunks) ln->after_first_launch = [&upload, k]() { return upload(k + 1); };
        const double t1 = now_ms();
        ln->read_index_base = a;
        rc = tb2_batch_compute(ln, params, save_params, policy, norm_signal != nullptr);
        ln->after_first_launch = nullptr;
        if (rc) break;
        if (trace && ln->ev_h0) {
            float h2d = 0, gap = 0;
            cudaEventElapsedTime(&h2d, ln->ev_h0, ln->ev_h1);
            cudaEventElapsedTime(&gap, ln->ev_h1, ln->ev0);
            fprintf(stderr, "[tb2]   own H2D took %.2f ms, ended %.2f ms before compute began on the device\n", h2d, gap);
        }
        if (trace)
            fprintf(stderr, "[tb2] chunk %d: t=%.1f upload(k+1) %.2f ms, compute %.2f ms (device %.2f)\n", k,
                    t0 - t00, t1 - t0, now_ms() - t1, ln->last_ms_total);
        ms_total += ln->last_ms_total; ms_dp += ln->last_ms_dp;
        dp_launches += ln->last_dp_launches; dp_reads += ln->last_dp_reads;
        rc = tb2_batch_download(ln, segs + base_off[a] + a, read_start_rel_to_raw + a, scale_out + a,
                                sig_match_score + a, norm_mean ? norm_mean + base_off[a] : nullptr,
                                norm_signal ? norm_signal + raw_off[a] : nullptr, status + a,
                                n_iters + a, flags + a);
    }
    for (tb2_ctx *ln : ctx->lanes) {
        if (cudaStreamSynchronize(ln->stream) != cudaSuccess && rc == TB2_OK) rc = TB2_ERR_CUDA;
        ctx->launches += ln->launches;
        ln->launches = 0;
        if (rc != TB2_OK && ctx->err.empty()) ctx->err = ln->err;
    }
    ctx->last_ms_total = ms_total; ctx->last_ms_dp = ms_dp;
    ctx->last_dp_launches = dp_launches; ctx->last_dp_reads = dp_reads;
    return rc;
}

// ---------------------------------------------------------------------------
// single-array mirror entry points (batch of one over the same kernels)
// ---------------------------------------------------------------------------
namespace {

// a one-read view over caller supplied signal; no sequence / model needed.  It lives in the
// context's single-read buffer set, never in the resident batch's.
struct OneRead {
    HostBatch hb;
    BatchView v;
    int64_t raw_off[2], seq_off[2];
    BatchBuffers *buf;
};

ReadState active_read()
{
    ReadState st;
    memset(&st, 0, sizeof(st));
    st.active = 1;
    return st;
}

// st: the read's initial state
int one_read_view(tb2_ctx *ctx, OneRead &o, const double *sig, int64_t n, int64_t nb,
                  const tb2_params &p, int64_t ev_cap, const ReadState &st)
{
    o.raw_off[0] = 0; o.raw_off[1] = n;
    o.seq_off[0] = 0; o.seq_off[1] = nb;   // K = 1
    o.buf = &tb2_state(ctx->one_read);
    int rc = build_view(ctx, *o.buf, 1, o.raw_off, o.seq_off, 1, p, 1.1, 0, o.hb, o.v);
    if (rc) return rc;
    if (ev_cap + 2 > o.hb.ev_off[1]) {
        // enlarge the event slots
        o.hb.ev_off[1] = ev_cap + 2;
        TB2_CUDA_TRY(ctx, o.buf->cpts.reserve((size_t)(ev_cap + 2) * 4 + 8));
        TB2_CUDA_TRY(ctx, o.buf->em.reserve((size_t)(ev_cap + 2) * 8 + 8));
        o.v.cpts = o.buf->cpts.as<int>();
        o.v.em = o.buf->em.as<double>();
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.buf->ev_off.p, o.hb.ev_off.data(), 16, cudaMemcpyHostToDevice, ctx->stream));
    }
    if (sig)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.rawf, sig, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.st, &st, sizeof(st), cudaMemcpyHostToDevice, ctx->stream));
    return TB2_OK;
}

tb2_params default_params()
{
    tb2_params p;
    memset(&p, 0, sizeof(p));
    p.bandwidth = 1; p.mean_obs_per_event = 1; p.running_stat_width = 1; p.min_obs_per_base = 1;
    p.raw_min_obs_per_base = 1; p.max_half_z_score = NAN;
    return p;
}

int fetch_state(tb2_ctx *ctx, const BatchView &v, ReadState *st)
{
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(st, v.st, sizeof(ReadState), cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return TB2_OK;
}

}  // namespace

extern "C" int tb2_normalize_raw_signal(tb2_ctx *ctx, const double *raw, int64_t n, int norm_type,
                                        double outlier_thresh, double const_scale,
                                        const tb2_scale_values *sv_in, double *norm_out,
                                        tb2_scale_values *sv_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!raw || !norm_out || !sv_out || n < 1 || (norm_type != 0 && norm_type != 1))
        return TB2_ERR_INVALID_ARG;
    ReadState st = active_read();
    if (sv_in) { st.use_sv = 1; st.sv = *sv_in; }
    OneRead o;
    if ((rc = one_read_view(ctx, o, raw, n, 1, default_params(), 2, st))) return rc;
    StagePolicy sp;
    memset(&sp, 0, sizeof(sp));
    sp.outlier_thresh = outlier_thresh;
    sp.const_scale = norm_type == 1 ? const_scale : NAN;
    if ((rc = tb2_launch_normalize(ctx, o.v, sp, 1))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(norm_out, o.v.norm, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = fetch_state(ctx, o.v, &st))) return rc;
    *sv_out = st.sv;
    if (sv_in == nullptr) sv_out->outlier_thresh = outlier_thresh;
    return st.status;
}

extern "C" int tb2_valid_cpts_w_cap(tb2_ctx *ctx, const double *sig, int64_t n,
                                    int64_t min_base_obs, int64_t running_stat_width,
                                    int64_t num_cpts, int t_test, int64_t *cpts_out,
                                    int *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!sig || !cpts_out || n < 1 || num_cpts < 1 || min_base_obs < 1 || running_stat_width < 1)
        return TB2_ERR_INVALID_ARG;
    tb2_params p = default_params();
    p.min_obs_per_base = min_base_obs;
    p.running_stat_width = running_stat_width;
    p.use_t_test_seg = t_test ? 1 : 0;
    ReadState st = active_read();
    st.num_events = (int)num_cpts;
    OneRead o;
    if ((rc = one_read_view(ctx, o, sig, n, 1, p, num_cpts, st))) return rc;
    if ((rc = tb2_launch_cpts(ctx, o.v, p, 1))) return rc;
    if ((rc = fetch_state(ctx, o.v, &st))) return rc;
    if (read_status) *read_status = st.status;
    if (st.status == TB2_OK) {
        std::vector<int> c32((size_t)num_cpts);
        TB2_CUDA_TRY(ctx, cudaMemcpy(c32.data(), o.v.cpts, (size_t)num_cpts * 4, cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < num_cpts; ++i) cpts_out[i] = c32[i];
    }
    return TB2_OK;
}

extern "C" int tb2_new_means(tb2_ctx *ctx, const double *sig, int64_t n_sig, const int64_t *segs,
                             int64_t n_segs, double *means_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!sig || !segs || !means_out || n_sig < 1 || n_segs < 1) return TB2_ERR_INVALID_ARG;
    ReadState st = active_read();
    st.n_cpts = (int)n_segs + 1;
    OneRead o;
    if ((rc = one_read_view(ctx, o, nullptr, n_sig, 1, default_params(), n_segs + 1, st))) return rc;
    // event means kernel reads `norm`
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.norm, sig, (size_t)n_sig * 8, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<int> s32((size_t)n_segs + 1);
    for (int64_t i = 0; i <= n_segs; ++i) {
        if (segs[i] < 0 || segs[i] > n_sig) return TB2_ERR_INVALID_ARG;
        s32[i] = (int)segs[i];
    }
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.cpts, s32.data(), (size_t)(n_segs + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = tb2_launch_event_means(ctx, o.v))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(means_out, o.v.em, (size_t)n_segs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return TB2_OK;
}

extern "C" int tb2_theil_sen(tb2_ctx *ctx, double prev_shift, double prev_scale,
                             const double *event_means, const double *model_means, int64_t n,
                             uint32_t subsample_key, double *out4, int *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!event_means || !model_means || !out4 || n < 1) return TB2_ERR_INVALID_ARG;
    ReadState st = active_read();
    st.sv.shift = prev_shift; st.sv.scale = prev_scale;
    OneRead o;
    // K = 1: seq_off = n gives n mapped bases
    if ((rc = one_read_view(ctx, o, nullptr, 1, n, default_params(), 2, st))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.bm, event_means, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.rm, model_means, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    StagePolicy sp;
    memset(&sp, 0, sizeof(sp));
    sp.outlier_thresh = NAN;
    sp.subsample_seed = subsample_key;
    sp.literal_key = 1;
    if ((rc = tb2_launch_theil_sen(ctx, o.v, sp, 0))) return rc;
    if ((rc = fetch_state(ctx, o.v, &st))) return rc;
    if (read_status) *read_status = st.status;
    out4[0] = st.sv.shift; out4[1] = st.sv.scale; out4[2] = st.shc; out4[3] = st.scc;
    return TB2_OK;
}

extern "C" int tb2_resolve_skipped_bases_with_raw(tb2_ctx *ctx, const int64_t *segs,
                                                  int64_t n_bases, const double *ref_means,
                                                  const double *ref_sds, const double *norm_signal,
                                                  int64_t n_norm, const tb2_params *params,
                                                  int64_t max_raw_cpts, int64_t *segs_out,
                                                  int *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!segs || !ref_means || !ref_sds || !norm_signal || !params || !segs_out || n_bases < 1 ||
        n_norm < 1)
        return TB2_ERR_INVALID_ARG;
    OneRead o;
    if ((rc = one_read_view(ctx, o, nullptr, n_norm, n_bases, default_params(), 2, active_read()))) return rc;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.norm, norm_signal, (size_t)n_norm * 8, cudaMemcpyHostToDevice, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.rm, ref_means, (size_t)n_bases * 8, cudaMemcpyHostToDevice, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.rs, ref_sds, (size_t)n_bases * 8, cudaMemcpyHostToDevice, s));
    std::vector<int> s32((size_t)n_bases + 1);
    for (int64_t i = 0; i <= n_bases; ++i) s32[i] = (int)segs[i];
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(o.v.segs_dp, s32.data(), (size_t)(n_bases + 1) * 4, cudaMemcpyHostToDevice, s));
    StagePolicy sp;
    memset(&sp, 0, sizeof(sp));
    sp.max_raw_cpts = max_raw_cpts;
    if ((rc = tb2_launch_resolve(ctx, o.v, *params, sp, (size_t)1 << 20))) return rc;
    ReadState st;
    if ((rc = fetch_state(ctx, o.v, &st))) return rc;
    if (read_status) *read_status = st.status;
    if (st.status == TB2_OK) {
        TB2_CUDA_TRY(ctx, cudaMemcpy(s32.data(), o.v.segs, (size_t)(n_bases + 1) * 4, cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i <= n_bases; ++i) segs_out[i] = s32[i];
    }
    return TB2_OK;
}

extern "C" int tb2_identify_stalls(tb2_ctx *ctx, const double *raw, int64_t n, int64_t *ints_out,
                                   int64_t cap, int64_t *n_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!raw || !ints_out || !n_out || n < 1 || cap < 1) return TB2_ERR_INVALID_ARG;
    OneRead o;
    if ((rc = one_read_view(ctx, o, raw, n, 1, default_params(), 2, active_read()))) return rc;
    const int scap = 4096;
    TB2_CUDA_TRY(ctx, o.buf->stalls.reserve((size_t)2 * scap * 4));
    o.v.stall_ints = o.buf->stalls.as<int>();
    o.v.stall_cap = scap;
    if ((rc = tb2_launch_stalls(ctx, o.v))) return rc;
    ReadState st;
    if ((rc = fetch_state(ctx, o.v, &st))) return rc;
    if (st.status != TB2_OK) return st.status;
    if (st.n_stalls > cap) return TB2_ERR_CAPACITY;
    std::vector<int> h((size_t)2 * std::max(1, st.n_stalls));
    if (st.n_stalls > 0)
        TB2_CUDA_TRY(ctx, cudaMemcpy(h.data(), o.v.stall_ints, (size_t)2 * st.n_stalls * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < 2 * st.n_stalls; ++i) ints_out[i] = h[i];
    *n_out = st.n_stalls;
    return TB2_OK;
}

// ---------------------------------------------------------------------------
// C ABI entry points of the batch path: no C++ exception may cross the boundary
// ---------------------------------------------------------------------------
#define TB2_GUARD(ctx, call)                                                        \
    try {                                                                           \
        return call;                                                                \
    } catch (const std::exception &e) {                                             \
        if (ctx) (ctx)->err = std::string("host exception: ") + e.what();           \
        return TB2_ERR_UNEXPECTED;                                                  \
    } catch (...) {                                                                 \
        if (ctx) (ctx)->err = "host exception";                                     \
        return TB2_ERR_UNEXPECTED;                                                  \
    }

extern "C" int tb2_batch_upload(tb2_ctx *ctx, int64_t n_reads, const void *raw, int raw_dtype,
                                const int64_t *raw_off, const uint8_t *seq, const int64_t *seq_off,
                                const tb2_params *params, const tb2_policy *policy)
{
    TB2_GUARD(ctx, batch_upload_impl(ctx, n_reads, raw, raw_dtype, raw_off, seq, seq_off, params, policy));
}

extern "C" int tb2_batch_set_read_inputs(tb2_ctx *ctx, const tb2_scale_values *sv_in,
                                         const int64_t *stall_ints, const int64_t *stall_off)
{
    TB2_GUARD(ctx, batch_set_read_inputs_impl(ctx, sv_in, stall_ints, stall_off));
}

extern "C" int tb2_batch_compute(tb2_ctx *ctx, const tb2_params *params,
                                 const tb2_params *save_params, const tb2_policy *policy,
                                 int want_norm_signal)
{
    TB2_GUARD(ctx, batch_compute_impl(ctx, params, save_params, policy, want_norm_signal));
}

extern "C" int tb2_batch_download(tb2_ctx *ctx, int64_t *segs, int64_t *read_start_rel_to_raw,
                                  tb2_scale_values *scale_out, double *sig_match_score,
                                  double *norm_mean, double *norm_signal, int32_t *status,
                                  int32_t *n_iters, int32_t *flags)
{
    TB2_GUARD(ctx, batch_download_impl(ctx, segs, read_start_rel_to_raw, scale_out, sig_match_score, norm_mean, norm_signal, status, n_iters, flags));
}

extern "C" int tb2_resquiggle_batch(tb2_ctx *ctx, int64_t n_reads, const void *raw, int raw_dtype,
                                    const int64_t *raw_off, const uint8_t *seq,
                                    const int64_t *seq_off, const tb2_params *params,
                                    const tb2_params *save_params, const tb2_policy *policy,
                                    int64_t *segs, int64_t *read_start_rel_to_raw,
                                    tb2_scale_values *scale_out, double *sig_match_score,
                                    double *norm_mean, double *norm_signal, int32_t *status,
                                    int32_t *n_iters, int32_t *flags)
{
    TB2_GUARD(ctx, resquiggle_batch_impl(ctx, n_reads, raw, raw_dtype, raw_off, seq, seq_off, params, save_params, policy, segs, read_start_rel_to_raw, scale_out, sig_match_score, norm_mean, norm_signal, status, n_iters, flags));
}
