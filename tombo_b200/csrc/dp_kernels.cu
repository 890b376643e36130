// dp_kernels.cu -- banded DP kernels (sm_90a) and their C-ABI entry points.
#include "kernels.h"
#include <algorithm>
#include <cstdlib>

#include "dp_align_kernel.cuh"

int tb2_launch_align(tb2_ctx *ctx, const AlignBatch &b, const AlignLaunchCfg &cfg_in)
{
    AlignLaunchCfg cfg = cfg_in;
    // shared memory per warp: 2 * smem_cells doubles of rows + the wavefront exchange ring
    const size_t max_smem = 200 * 1024;
    const auto smem_of = [](int cells) {
        return (size_t)ALIGN_WARPS * (2 * (size_t)cells + TB2_WF_RING) * sizeof(double);
    };
    size_t smem = smem_of(cfg.smem_cells);
    if (smem > max_smem) {
        // rows that do not fit go to the global row scratch
        const int cap = (int)((max_smem / (ALIGN_WARPS * sizeof(double)) - TB2_WF_RING) / 2 / 32) * 32;
        cfg.grow_cells = std::max(cfg.grow_cells, cfg.smem_cells);
        cfg.smem_cells = cap;
        smem = smem_of(cfg.smem_cells);
    }
    // resident CTAs per SM: 8 for the static-band kernel (64 registers), 4 for the general
    // one (128 registers; a 5-CTA build with 102 registers was slower on the configs[2] mix
    // and configs[4]).  228 KB of shared memory per SM (H100), 1 KB of it reserved per CTA.
    const int max_blocks = cfg.klass == 1 ? 8 : 4;
    int blocks_per_sm = (int)std::max<size_t>(1, std::min<size_t>(max_blocks, (228 * 1024) / (smem + 1024)));
    int grid = ctx->sm_count * blocks_per_sm;
    const int max_useful = (b.n_reads + ALIGN_WARPS - 1) / ALIGN_WARPS;
    if (grid > max_useful) grid = std::max(1, max_useful);
    const size_t slots = (size_t)grid * ALIGN_WARPS;
    LaunchScratch &ls = tb2_state(ctx->launch_scratch);
    TB2_CUDA_TRY(ctx, ls.tb.reserve(slots * cfg.tb_words * sizeof(uint32_t)));
    TB2_CUDA_TRY(ctx, ls.grow.reserve(slots * 2 * (size_t)cfg.grow_cells * sizeof(double) + 8));
    TB2_CUDA_TRY(ctx, ls.align_cnt.reserve(sizeof(int)));
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(ls.align_cnt.p, 0, sizeof(int), ctx->stream));
    auto kern = cfg.klass == 1 ? k_align<1> : (cfg.klass == 2 ? k_align<2> : k_align<0>);
    // (a constant, not this launch's size: contexts launch concurrently from several host
    // threads and the attribute is per function, not per context)
    TB2_CUDA_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           227 * 1024));
    // the static-band kernel needs 8 CTAs x (rows + ring) of shared memory per SM and touches
    // L1 only for its streaming event loads; the general kernel keeps the default split
    if (cfg.klass == 1)
        TB2_CUDA_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                                               (int)cudaSharedmemCarveoutMaxShared));
    kern<<<grid, ALIGN_WARPS * 32, smem, ctx->stream>>>(
        b, cfg, ls.tb.as<uint32_t>(), ls.grow.as<double>(), ls.align_cnt.as<int>());
    TB2_CHECK_LAUNCH(ctx);
    return TB2_OK;
}

// ---------------------------------------------------------------------------
// mirror-API kernels (single warp, full matrices dumped for parity tests)
// ---------------------------------------------------------------------------
__global__ void k_banded_forward_dbg(const double *z, const long long *starts64, int nb, int W,
                                     double skip_pen, double stay_pen, double *fwd,
                                     long long *tb64, int *starts32, uint32_t *tbp,
                                     double *grow, int grow_cells, int smem_cells, int *status)
{
    extern __shared__ double smem[];
    const int lane = tb2_lane();
    WarpRes wr;
    wr.smem_rows = smem; wr.smem_cap = 2 * smem_cells; wr.grow = grow; wr.grow_cap = grow_cells;
    wr.ring = smem + 2 * smem_cells;
    wr.tb = tbp; wr.tb_words = (size_t)nb * TB2_MAX_WPL * 32;
    DpConsts c;
    c.z_shift = 0; c.stay_pen = stay_pen; c.skip_pen = skip_pen; c.mhz = 0; c.winsor = 0;
    PassCtx pc;
    pc.em = nullptr; pc.n_em = 0; pc.rm = nullptr; pc.rs_ = nullptr; pc.zmat = z;
    pc.mso = 0; pc.msp_start = 0; pc.msp_stop = 0; pc.mask_fill = 0; pc.mask_shifted = 0;
    pc.starts = starts32; pc.tb = tbp; pc.dbg_fwd = fwd; pc.dbg_tb = tb64;
    pc.zbuf = nullptr; pc.cbuf = nullptr; pc.ring = wr.ring;
    int st = TB2_OK;
    pc.W = W; pc.chunk = (W + 31) / 32; pc.buf0 = nullptr; pc.buf1 = nullptr;
    double *rowbuf = tb2_wf_rowbuf(wr, W);
    if (rowbuf == nullptr) st = TB2_ERR_CAPACITY;
    if (st == TB2_OK) {
        for (int r = lane; r < nb; r += 32) starts32[r] = (int)starts64[r];
        for (int j = lane; j < W; j += 32) { fwd[j] = 0.0; tb64[j] = 0; }
        __syncwarp();
        int amax = 0;
        st = tb2_wavefront_rows(pc, c, TB2_MODE_EXPLICIT, nb, rowbuf, tbp, &amax);
    }
    if (lane == 0) *status = st;
}

__global__ void k_adaptive_dbg(double *fwd, long long *tb64, long long *starts64, int nb, int W,
                               const double *em, int n_em, const double *rm, const double *rs,
                               double z_shift, double skip_pen, double stay_pen, int ssp,
                               double mask_fill, int winsor, double mhz, int *starts32,
                               uint32_t *tbp, double *grow, int grow_cells, int smem_cells,
                               int *status)
{
    extern __shared__ double smem[];
    const int lane = tb2_lane();
    WarpRes wr;
    wr.smem_rows = smem; wr.smem_cap = 2 * smem_cells; wr.grow = grow; wr.grow_cap = grow_cells;
    wr.ring = smem + 2 * smem_cells;
    wr.tb = tbp; wr.tb_words = (size_t)nb * TB2_MAX_WPL * 32;
    DpConsts c;
    c.z_shift = z_shift; c.stay_pen = stay_pen; c.skip_pen = skip_pen; c.mhz = mhz;
    c.winsor = winsor;
    PassCtx pc;
    pc.em = em; pc.n_em = n_em; pc.rm = rm; pc.rs_ = rs; pc.zmat = nullptr;
    pc.mso = 0; pc.msp_start = 0; pc.msp_stop = 0; pc.mask_fill = mask_fill; pc.mask_shifted = 0;
    pc.starts = starts32; pc.tb = tbp; pc.dbg_fwd = fwd; pc.dbg_tb = tb64;
    pc.zbuf = nullptr; pc.cbuf = nullptr; pc.ring = wr.ring;
    int st = TB2_OK;
    if (!tb2_setup_geom(pc, wr, W)) st = TB2_ERR_CAPACITY;
    const int wpl = tb2_wpl_of(pc.chunk);
    if (wpl > TB2_MAX_WPL) st = TB2_ERR_CAPACITY;
    if (ssp < 1 || ssp > nb) st = TB2_ERR_INVALID_ARG;
    if (st == TB2_OK) {
        for (int r = lane; r < ssp; r += 32) starts32[r] = (int)starts64[r];
        __syncwarp();
        int sel;
        tb2_load_row(pc, fwd + (size_t)ssp * W, &sel);
        // arg-max of the seed row (first maximum)
        double best = tb2_neg_inf();
        int bi = 0x7fffffff;
        for (int j = lane; j < W; j += 32) {
            const double v = fwd[(size_t)ssp * W + j];
            if (v > best) { best = v; bi = j; }
        }
        int amax = tb2_warp_argmax(best, bi);
        st = tb2_run_rows_dyn(wpl, pc, c, TB2_MODE_ADAPTIVE, ssp, nb, nb, &sel, &amax);
        __syncwarp();
        // the reference leaves event_starts filled up to the failing row
        for (int r = ssp + lane; r < nb; r += 32) starts64[r] = starts32[r];
    }
    if (lane == 0) *status = st;
}

// c_banded_traceback on an unpacked int64 move matrix (mirror API only)
__global__ void k_traceback_dbg(const long long *tb, const long long *es, int nb, int bw,
                                long long band_pos, long long thresh, long long *seq_poss,
                                int *status)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    long long cur_event = band_pos + es[nb - 1];
    seq_poss[nb] = cur_event + 1;
    for (int sp = nb; sp > 0; --sp) {
        band_pos = cur_event - es[sp - 1];
        if (band_pos < 0 || band_pos >= bw) { *status = TB2_ERR_UNEXPECTED; return; }
        while (tb[(size_t)sp * bw + band_pos] == 0) {
            --band_pos;
            if (band_pos < 0) { *status = TB2_ERR_UNEXPECTED; return; }
        }
        if (tb[(size_t)sp * bw + band_pos] == 2) --band_pos;
        if (thresh >= 0) {
            const long long a = band_pos, b = bw - band_pos - 1;
            if ((a < b ? a : b) < thresh) { *status = TB2_ERR_BEYOND_BANDWIDTH; return; }
        }
        cur_event = es[sp - 1] + band_pos;
        seq_poss[sp - 1] = cur_event + 1;
    }
    *status = TB2_OK;
}

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
namespace {
// per-call scratch of the mirror entry points; nothing reads it after a call returns
enum { S_A = 0, S_B, S_C, S_D, S_E, S_F, S_G, S_H, S_I, S_J, S_COUNT };
}  // namespace
struct DpMirrorState { DevBuf buf[S_COUNT]; };

namespace {
struct DbgGeom { int smem_cells, grow_cells; size_t smem_bytes; };
DbgGeom dbg_geom(long long W)
{
    DbgGeom g;
    const int cells = tb2_row_cells(W);
    if ((size_t)cells * 2 * sizeof(double) <= 96 * 1024) {
        g.smem_cells = cells; g.grow_cells = 0;
    } else {
        g.smem_cells = 32; g.grow_cells = cells;
    }
    g.smem_bytes = ((size_t)g.smem_cells * 2 + TB2_WF_RING) * sizeof(double);
    return g;
}
}  // namespace

extern "C" int tb2_banded_forward_pass(tb2_ctx *ctx, const double *z, const int64_t *event_starts,
                                       int64_t n_bases, int64_t bw, double skip_pen,
                                       double stay_pen, double *fwd_out, int64_t *tb_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!z || !event_starts || !fwd_out || !tb_out || n_bases < 1 || bw < 1)
        return TB2_ERR_INVALID_ARG;
    if (tb2_row_cells(bw) / 32 > TB2_MAX_WPL * 16) return TB2_ERR_CAPACITY;
    const size_t nz = (size_t)n_bases * bw, nf = (size_t)(n_bases + 1) * bw;
    auto &P = tb2_state(ctx->dp).buf;
    TB2_CUDA_TRY(ctx, P[S_A].upload(z, nz, ctx->stream));
    TB2_CUDA_TRY(ctx, P[S_B].upload(event_starts, (size_t)n_bases, ctx->stream));
    TB2_CUDA_TRY(ctx, P[S_C].reserve(nf * 8));
    TB2_CUDA_TRY(ctx, P[S_D].reserve(nf * 8));
    TB2_CUDA_TRY(ctx, P[S_E].reserve(n_bases * 4));
    TB2_CUDA_TRY(ctx, P[S_F].reserve((size_t)n_bases * TB2_MAX_WPL * 32 * 4));
    TB2_CUDA_TRY(ctx, P[S_G].reserve(4));
    const DbgGeom g = dbg_geom(bw);
    TB2_CUDA_TRY(ctx, P[S_H].reserve((size_t)g.grow_cells * 2 * 8 + 8));
    TB2_CUDA_TRY(ctx, cudaFuncSetAttribute(k_banded_forward_dbg,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)g.smem_bytes));
    k_banded_forward_dbg<<<1, 32, g.smem_bytes, ctx->stream>>>(
        P[S_A].as<double>(), P[S_B].as<long long>(), (int)n_bases, (int)bw, skip_pen, stay_pen,
        P[S_C].as<double>(), P[S_D].as<long long>(), P[S_E].as<int>(), P[S_F].as<uint32_t>(),
        P[S_H].as<double>(), g.grow_cells, g.smem_cells, P[S_G].as<int>());
    TB2_CHECK_LAUNCH(ctx);
    int st = 0;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(fwd_out, P[S_C].p, nf * 8, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(tb_out, P[S_D].p, nf * 8, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(&st, P[S_G].p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return st;
}

extern "C" int tb2_banded_traceback(tb2_ctx *ctx, const int64_t *tb, const int64_t *event_starts,
                                    int64_t n_bases, int64_t bw, int64_t band_pos,
                                    int64_t band_boundary_thresh, int64_t *seq_poss_out,
                                    int *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!tb || !event_starts || !seq_poss_out || n_bases < 1 || bw < 1) return TB2_ERR_INVALID_ARG;
    const size_t nf = (size_t)(n_bases + 1) * bw;
    auto &P = tb2_state(ctx->dp).buf;
    TB2_CUDA_TRY(ctx, P[S_A].upload(tb, nf, ctx->stream));
    TB2_CUDA_TRY(ctx, P[S_B].upload(event_starts, (size_t)n_bases, ctx->stream));
    TB2_CUDA_TRY(ctx, P[S_C].reserve((n_bases + 1) * 8));
    TB2_CUDA_TRY(ctx, P[S_G].reserve(4));
    k_traceback_dbg<<<1, 32, 0, ctx->stream>>>(P[S_A].as<long long>(), P[S_B].as<long long>(),
                                               (int)n_bases, (int)bw, band_pos,
                                               band_boundary_thresh, P[S_C].as<long long>(),
                                               P[S_G].as<int>());
    TB2_CHECK_LAUNCH(ctx);
    int st = 0;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(seq_poss_out, P[S_C].p, (n_bases + 1) * 8,
                                      cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(&st, P[S_G].p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (read_status) *read_status = st;
    return TB2_OK;
}

extern "C" int tb2_adaptive_banded_forward_pass(
    tb2_ctx *ctx, double *fwd, int64_t *tb, int64_t *event_starts, int64_t n_bases, int64_t bw,
    const double *event_means, int64_t n_events, const double *ref_means, const double *ref_sds,
    double z_shift, double skip_pen, double stay_pen, int64_t start_seq_pos,
    double mask_fill_z_score, int do_winsorize_z, double max_half_z_score, int *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!fwd || !tb || !event_starts || !event_means || !ref_means || !ref_sds || n_bases < 1 ||
        bw < 1 || n_events < 1 || start_seq_pos < 1 || start_seq_pos > n_bases)
        return TB2_ERR_INVALID_ARG;
    if (tb2_row_cells(bw) / 32 > TB2_MAX_WPL * 16) return TB2_ERR_CAPACITY;
    const size_t nf = (size_t)(n_bases + 1) * bw;
    auto &P = tb2_state(ctx->dp).buf;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, P[S_A].upload(fwd, nf, s));
    TB2_CUDA_TRY(ctx, P[S_B].upload(tb, nf, s));
    TB2_CUDA_TRY(ctx, P[S_C].upload(event_starts, (size_t)n_bases, s));
    TB2_CUDA_TRY(ctx, P[S_D].upload(event_means, (size_t)n_events, s));
    TB2_CUDA_TRY(ctx, P[S_E].upload(ref_means, (size_t)n_bases, s));
    TB2_CUDA_TRY(ctx, P[S_F].upload(ref_sds, (size_t)n_bases, s));
    TB2_CUDA_TRY(ctx, P[S_G].reserve(4));
    TB2_CUDA_TRY(ctx, P[S_I].reserve(n_bases * 4));
    TB2_CUDA_TRY(ctx, P[S_J].reserve((size_t)n_bases * TB2_MAX_WPL * 32 * 4));
    const DbgGeom g = dbg_geom(bw);
    TB2_CUDA_TRY(ctx, P[S_H].reserve((size_t)g.grow_cells * 2 * 8 + 8));
    TB2_CUDA_TRY(ctx, cudaFuncSetAttribute(k_adaptive_dbg, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)g.smem_bytes));
    k_adaptive_dbg<<<1, 32, g.smem_bytes, s>>>(
        P[S_A].as<double>(), P[S_B].as<long long>(), P[S_C].as<long long>(), (int)n_bases, (int)bw,
        P[S_D].as<double>(), (int)n_events, P[S_E].as<double>(), P[S_F].as<double>(), z_shift,
        skip_pen, stay_pen, (int)start_seq_pos, mask_fill_z_score, do_winsorize_z ? 1 : 0,
        max_half_z_score, P[S_I].as<int>(), P[S_J].as<uint32_t>(), P[S_H].as<double>(),
        g.grow_cells, g.smem_cells, P[S_G].as<int>());
    TB2_CHECK_LAUNCH(ctx);
    int st = 0;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(fwd, P[S_A].p, nf * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(tb, P[S_B].p, nf * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(event_starts, P[S_C].p, n_bases * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(&st, P[S_G].p, 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    if (read_status) *read_status = st;
    return TB2_OK;
}

// capacity planning for one read of the assignment kernel (host)
static void plan_align(const tb2_params &p, long long n_em, long long nb, int *smem_cells,
                       size_t *tb_words, int *grow_cells)
{
    const long long mask_len = std::min(nb, n_em) / 4;
    const long long w_static = std::max<long long>(1, n_em - mask_len);
    const bool is_short = n_em < p.start_bw + p.start_n_bases || nb < p.start_n_bases;
    long long w_main = is_short ? w_static : std::max<long long>(p.start_bw, p.bandwidth);
    *smem_cells = std::max(*smem_cells, tb2_row_cells(w_main));
    size_t tw = is_short ? tb2_tb_words(nb, w_static, mask_len + 1)
                         : std::max(tb2_tb_words(nb, p.bandwidth, n_em + p.bandwidth),
                                    tb2_tb_words(p.start_n_bases, p.start_bw, p.start_n_bases));
    if (!is_short) {
        // rare fall-backs keep their rows in global memory
        long long w_rare = p.start_save_bw;
        if (n_em >= p.start_save_bw + p.start_n_bases)
            tw = std::max(tw, tb2_tb_words(p.start_n_bases, p.start_save_bw, p.start_n_bases));
        *grow_cells = std::max(*grow_cells, tb2_row_cells(w_rare));
    }
    *tb_words = std::max(*tb_words, tw);
}

extern "C" int tb2_find_adaptive_base_assignment(
    tb2_ctx *ctx, const int64_t *valid_cpts, int64_t n_cpts, const double *event_means,
    const tb2_params *params, const double *ref_means, const double *ref_sds, int64_t n_bases,
    double sig_match_thresh, int64_t *segs_out, int64_t *read_start_rel_to_raw, int64_t *dbg,
    int *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!valid_cpts || !event_means || !params || !ref_means || !ref_sds || !segs_out ||
        !read_start_rel_to_raw || n_cpts < 2 || n_bases < 1)
        return TB2_ERR_INVALID_ARG;
    auto &P = tb2_state(ctx->dp).buf;
    cudaStream_t s = ctx->stream;
    const long long nb = n_bases, n_em = n_cpts - 1;
    std::vector<int> cp32((size_t)n_cpts);
    for (int64_t i = 0; i < n_cpts; ++i) cp32[i] = (int)valid_cpts[i];
    long long offs[4] = {0, n_cpts, 0, nb};
    int ncp = (int)n_cpts, zero = 0;
    TB2_CUDA_TRY(ctx, P[S_A].upload(cp32.data(), (size_t)n_cpts, s));
    TB2_CUDA_TRY(ctx, P[S_B].upload(event_means, (size_t)n_em, s));
    TB2_CUDA_TRY(ctx, P[S_C].upload(ref_means, (size_t)nb, s));
    TB2_CUDA_TRY(ctx, P[S_D].upload(ref_sds, (size_t)nb, s));
    TB2_CUDA_TRY(ctx, P[S_E].upload(offs, 4, s));
    TB2_CUDA_TRY(ctx, P[S_F].reserve((nb + 1) * 4 * 3 + 64));  // starts, read_tb, segs
    // small ints: [0]=n_cpts [1]=status [2]=rsrtr [3..5]=dbg
    int small[8] = {ncp, zero, 0, 0, 0, 0, 0, 0};
    TB2_CUDA_TRY(ctx, P[S_G].reserve(64));
    TB2_CUDA_TRY(ctx, P[S_G].upload(small, 8, s));
    AlignBatch b;
    b.n_reads = 1;
    b.order = nullptr;
    b.cpts = P[S_A].as<int>();
    b.em = P[S_B].as<double>();
    b.ev_off = P[S_E].as<long long>();
    b.n_cpts = P[S_G].as<int>();
    b.rm = P[S_C].as<double>();
    b.rs = P[S_D].as<double>();
    b.base_off = P[S_E].as<long long>() + 2;
    int *scr = P[S_F].as<int>();
    b.starts = scr;
    b.read_tb = scr + (nb + 1);
    b.segs = scr + 2 * (nb + 1);
    b.rsrtr = P[S_G].as<int>() + 2;
    b.status = P[S_G].as<int>() + 1;
    b.active = nullptr;
    b.num_events = nullptr;
    b.stride = 1;
    b.dbg = P[S_G].as<int>() + 3;
    b.params = *params;
    b.sig_match_thresh = sig_match_thresh;
    AlignLaunchCfg cfg = {32, 32, 0, 0};
    plan_align(*params, n_em, nb, &cfg.smem_cells, &cfg.tb_words, &cfg.grow_cells);
    // the single-read mirror also covers the rare static fall-back of long reads
    cfg.tb_words = std::max(cfg.tb_words, tb2_tb_words(nb, std::max<long long>(1, n_em - std::min(nb, n_em) / 4), n_em));
    cfg.grow_cells = std::max(cfg.grow_cells, tb2_row_cells(std::max<long long>(1, n_em)));
    rc = tb2_launch_align(ctx, b, cfg);
    if (rc) return rc;
    std::vector<int> segs32((size_t)nb + 1);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(segs32.data(), b.segs, (nb + 1) * 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(small, P[S_G].p, 32, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    if (read_status) *read_status = small[1];
    if (small[1] == TB2_OK) {
        for (long long i = 0; i <= nb; ++i) segs_out[i] = segs32[i];
        *read_start_rel_to_raw = small[2];
    }
    if (dbg) { dbg[0] = small[3]; dbg[1] = small[4]; dbg[2] = small[5]; }
    return TB2_OK;
}

// ---------------------------------------------------------------------------
// single-read mirrors of find_static_base_assignment (resquiggle.py:547-600) and
// find_seq_start_in_events (resquiggle.py:685-752)
// ---------------------------------------------------------------------------
__global__ void k_single(int mode, const double *em, int n_em, const double *rm, const double *rs,
                         int nb, tb2_params p, int num_bases, int num_events, int check_score,
                         double sig_match_thresh, int *starts, int *read_tb, uint32_t *tbp,
                         size_t tb_words, double *grow, int grow_cells, int smem_cells,
                         int *out_int /* status, start_loc */, double *out_epb)
{
    extern __shared__ double smem[];
    const int lane = tb2_lane();
    WarpRes wr;
    wr.smem_rows = smem; wr.smem_cap = 2 * smem_cells; wr.grow = grow; wr.grow_cap = grow_cells;
    wr.ring = smem + 2 * smem_cells;
    wr.tb = tbp; wr.tb_words = tb_words;
    DpConsts c;
    c.z_shift = p.z_shift; c.stay_pen = p.stay_pen; c.skip_pen = p.skip_pen;
    c.winsor = !isnan(p.max_half_z_score);
    c.mhz = c.winsor ? p.max_half_z_score : 0.0;
    AlignRead a;
    a.cpts = nullptr; a.n_cpts = n_em + 1; a.em = em; a.rm = rm; a.rs = rs; a.nb = nb;
    a.starts = starts; a.read_tb = read_tb; a.segs = nullptr; a.rsrtr = nullptr; a.dbg = nullptr;
    int st, sloc = 0;
    double epb = 0;
    if (mode == 0) st = tb2_static_assign(a, wr, c, /*emit_segs=*/false);
    else st = tb2_start_find(a, wr, c, num_bases, num_events, check_score != 0, sig_match_thresh,
                             &sloc, &epb);
    if (lane == 0) { out_int[0] = st; out_int[1] = sloc; *out_epb = epb; }
}

static int run_single(tb2_ctx *ctx, int mode, const double *em, int64_t n_em, const double *rm,
                      const double *rs, int64_t nb, const tb2_params *p, int64_t num_bases,
                      int64_t num_events, int check, double thresh, int64_t *tb_out,
                      int64_t n_tb_out, int64_t *start_loc, double *epb, int *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!em || !rm || !rs || !p || n_em < 1 || nb < 1 || (mode == 0 ? !tb_out : (!start_loc || !epb)))
        return TB2_ERR_INVALID_ARG;
    auto &P = tb2_state(ctx->dp).buf;
    cudaStream_t s = ctx->stream;
    const long long W = mode == 0 ? std::max<long long>(1, n_em - std::min<long long>(nb, n_em) / 4)
                                  : num_events;
    const long long rows = mode == 0 ? nb : num_bases;
    if (W < 1 || rows < 1) return TB2_ERR_INVALID_ARG;
    if (tb2_row_cells(W) / 32 > TB2_MAX_CHUNK) { if (read_status) *read_status = TB2_ERR_CAPACITY; return TB2_OK; }
    const DbgGeom g = dbg_geom(W);
    const size_t tbw = tb2_tb_words(rows, W, n_em);
    TB2_CUDA_TRY(ctx, P[S_A].upload(em, (size_t)n_em, s));
    TB2_CUDA_TRY(ctx, P[S_B].upload(rm, (size_t)nb, s));
    TB2_CUDA_TRY(ctx, P[S_C].upload(rs, (size_t)nb, s));
    TB2_CUDA_TRY(ctx, P[S_D].reserve((size_t)(nb + 1) * 4 * 2 + 64));
    TB2_CUDA_TRY(ctx, P[S_E].reserve(tbw * 4 + 64));
    TB2_CUDA_TRY(ctx, P[S_G].reserve(64));
    TB2_CUDA_TRY(ctx, P[S_H].reserve((size_t)g.grow_cells * 2 * 8 + 8));
    TB2_CUDA_TRY(ctx, cudaFuncSetAttribute(k_single, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)g.smem_bytes));
    int *ints = P[S_D].as<int>();
    k_single<<<1, 32, g.smem_bytes, s>>>(mode, P[S_A].as<double>(), (int)n_em, P[S_B].as<double>(),
                                         P[S_C].as<double>(), (int)nb, *p, (int)num_bases,
                                         (int)num_events, check, thresh, ints, ints + (nb + 1),
                                         P[S_E].as<uint32_t>(), tbw, P[S_H].as<double>(),
                                         g.grow_cells, g.smem_cells, P[S_G].as<int>(),
                                         (double *)(P[S_G].as<int>() + 4));
    TB2_CHECK_LAUNCH(ctx);
    int small[6];
    std::vector<int> tb32((size_t)nb + 1);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(small, P[S_G].p, 24, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(tb32.data(), ints + (nb + 1), (size_t)(nb + 1) * 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    if (read_status) *read_status = small[0];
    if (small[0] == TB2_OK) {
        if (tb_out) for (int64_t i = 0; i < n_tb_out; ++i) tb_out[i] = tb32[i];
        if (start_loc) *start_loc = small[1];
        if (epb) memcpy(epb, &small[4], 8);
    }
    return TB2_OK;
}

extern "C" int tb2_find_static_base_assignment(tb2_ctx *ctx, const double *event_means,
                                               int64_t n_events, const double *ref_means,
                                               const double *ref_sds, int64_t n_bases,
                                               const tb2_params *params, int64_t *read_tb_out,
                                               int *read_status)
{
    return run_single(ctx, 0, event_means, n_events, ref_means, ref_sds, n_bases, params, 0, 0, 0,
                      0.0, read_tb_out, n_bases + 1, nullptr, nullptr, read_status);
}

extern "C" int tb2_find_seq_start_in_events(tb2_ctx *ctx, const double *event_means,
                                            int64_t n_events, const double *ref_means,
                                            const double *ref_sds, int64_t n_ref,
                                            const tb2_params *params, int64_t num_bases,
                                            int64_t num_events, int check_score,
                                            double sig_match_thresh, int64_t *start_loc,
                                            double *events_per_base, int *read_status)
{
    return run_single(ctx, 1, event_means, n_events, ref_means, ref_sds, n_ref, params, num_bases,
                      num_events, check_score, sig_match_thresh, nullptr, 0, start_loc,
                      events_per_base, read_status);
}

extern "C" int tb2_debug_dp_counters(tb2_ctx *ctx, unsigned long long *out8, int reset)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!out8) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, cudaDeviceSynchronize());
    TB2_CUDA_TRY(ctx, cudaMemcpyFromSymbol(out8, g_tb2_dp_counters, 64));
    if (reset) {
        unsigned long long z[8] = {0};
        TB2_CUDA_TRY(ctx, cudaMemcpyToSymbol(g_tb2_dp_counters, z, 64));
    }
    return TB2_OK;
}
