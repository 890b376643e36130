// stats_file.cu -- the statistics file (tombo detect_modifications aggregate_per_read_stats and
// the writer of test_significance) on the device.
//
//   tb2_stats_file_aggregate  _agg_stats_worker tombo_stats.py:4699-4725 with
//                             apply_per_read_thresh :4084-4122 and the block table of
//                             ModelStats._write_stat_block :2737-2773, many blocks per launch:
//                             one CTA per block counts coverage, valid coverage and stats >=
//                             threshold per position (shared memory when the block's three
//                             int32 counter arrays fit, global memory otherwise), then emits the
//                             covered positions in order without the NaN damp_frac rows
//   tb2_most_signif_*         the running most-significant table of ModelStats / LevelStats
//                             (_add_to_most_signif :2722-2735, _update_most_signif :2714-2720,
//                             _close_write :2775-2795)
//
// The most-significant table.  Each _update_most_signif sorts [running rows, then the queued
// blocks in arrival order] with numpy's stable mergesort on a structured array, keeping the
// first N.  numpy orders structured rows by the `order` field first and breaks ties with the
// remaining fields in dtype order, so rows compare as the tuple
//   model: (damp_frac, frac, pos, cov, control_cov, valid_cov, chrm, strand)
//   level: (stat, pos, cov, control_cov, chrm, strand)
// with floats compared as numbers (-0.0 == +0.0), and only rows equal in every field keep
// their arrival order.  The running rows always precede the queued ones and hold every earlier
// row that can still be among the first N, so by induction the table is the first N rows of
// one stable sort of all rows in arrival order, whatever the update cadence (DESIGN.md §3).
// Here every row is K 64-bit words whose unsigned order, most significant word first, is that
// tuple order (floats through order_key, the integer fields packed two per word); the table
// keeps its rows in arrival order behind its sorted front and sorts them with the stable LSD
// radix sort of radix_sort.cuh when it holds more than it may keep or is read.
#include "ctx.h"
#include "stats_file.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

static_assert(sizeof(tb2_sf_block) == TB2_SF_BLOCK_FIELDS * 8, "tb2_sf_block rows");

namespace {

// global-memory counters of the fallback path: blocks per launch are cut to this many bytes
constexpr size_t GCNT_BUDGET = 256u << 20;

enum { G_BLK = 0, G_POS, G_STAT, G_UB, G_CNT, G_OFF, G_GCNT, G_ERR,
       G_UPOS, G_UDAMP, G_UFRAC, G_UCOV, G_UVALID, G_POSO, G_DAMP, G_FRAC, G_COV, G_VALID, G_COUNT };
enum { T_RAW = 0, T_OUT, T_KEY0, T_KEY1, T_IDX0, T_IDX1, T_THIST, T_TOFF, T_HIST, T_COUNT };

}  // namespace

struct StatsFileState {
    // last aggregation: rows of block b at [off[b], off[b + 1]) of the G_POSO .. G_VALID columns
    DevBuf agg[G_COUNT];
    long long agg_blocks = -1, agg_rows = 0;
    // most-significant table: rows word-major, raw[w * cap + i]; the first `sorted` rows are the
    // table in order, the rest arrived since
    DevBuf tab[T_COUNT];
    int kind = -1, K = 0, nf = 0;     // 0 model (5 words, 2 floats), 1 level (4 words, 1 float)
    long long N = 0, n = 0, cap = 0, sorted = 0;
};

namespace {

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
unsigned grid_of(long long n) { return (unsigned)std::max<long long>(1, (n + 255) / 256); }

// room for `need` rows, keeping the first S.n
int table_reserve(tb2_ctx *ctx, StatsFileState &S, long long need)
{
    if (need <= S.cap) return TB2_OK;
    if (need >= (1LL << 32)) {                       // the sort carries 32-bit row indices
        ctx->err = "most-significant table: more than 2^32 - 1 rows between two sorts";
        return TB2_ERR_CAPACITY;
    }
    const long long cap = std::min<long long>((1LL << 32) - 1, std::max(need + need / 4, 2 * S.N));
    DevBuf nb;
    TB2_RESERVE(ctx, "stats file", nb, (size_t)S.K * cap * 8);
    for (int w = 0; w < S.K && S.n; ++w)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(nb.as<unsigned long long>() + (size_t)w * cap,
                                          S.tab[T_RAW].as<unsigned long long>() + (size_t)w * S.cap,
                                          (size_t)S.n * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    std::swap(S.tab[T_RAW].p, nb.p);
    std::swap(S.tab[T_RAW].cap, nb.cap);
    S.cap = cap;
    return TB2_OK;
}

// sort every row held and keep the first N
int table_reduce(tb2_ctx *ctx, StatsFileState &S)
{
    if (S.n == S.sorted && S.n <= S.N) return TB2_OK;
    cudaStream_t q = ctx->stream;
    DevBuf *T = S.tab;
    const long long n = S.n, m = std::min(S.n, S.N), cap = S.cap;
    const int K = S.K;
    const long long n_tiles = (n + RADIX_TILE - 1) / RADIX_TILE;
    TB2_RESERVE(ctx, "stats file", T[T_OUT], (size_t)K * cap * 8);
    TB2_RESERVE(ctx, "stats file", T[T_KEY0], (size_t)n * 8);
    TB2_RESERVE(ctx, "stats file", T[T_KEY1], (size_t)n * 8);
    TB2_RESERVE(ctx, "stats file", T[T_IDX0], (size_t)n * 4);
    TB2_RESERVE(ctx, "stats file", T[T_IDX1], (size_t)n * 4);
    TB2_RESERVE(ctx, "stats file", T[T_THIST], (size_t)256 * n_tiles * 4);
    TB2_RESERVE(ctx, "stats file", T[T_TOFF], (size_t)256 * n_tiles * 8);
    TB2_RESERVE(ctx, "stats file", T[T_HIST], (size_t)MAXW * 8 * 256 * 8);
    unsigned long long *raw = T[T_RAW].as<unsigned long long>(), *gh = T[T_HIST].as<unsigned long long>();
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(gh, 0, (size_t)K * 8 * 256 * 8, q));
    const unsigned hgrid = (unsigned)std::min<long long>(grid_of(n), 4LL * ctx->sm_count);
    k_sf_hist<<<hgrid, 256, 0, q>>>(raw, cap, n, K, S.nf, gh);
    TB2_CHECK_LAUNCH(ctx);
    std::vector<unsigned long long> h((size_t)K * 8 * 256);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(h.data(), gh, h.size() * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    // least significant word first; a digit held by one bin keeps the order and is skipped
    int cur = 0;
    bool any = false;
    for (int w = K - 1; w >= 0; --w) {
        bool live[8];
        if (!sf_live_digits(h.data(), n, w, live)) continue;
        k_sf_word_keys<<<grid_of(n), 256, 0, q>>>(raw + (size_t)w * cap, w < S.nf,
                                                  any ? T[T_IDX0 + cur].as<unsigned int>() : nullptr, n,
                                                  T[T_KEY0 + cur].as<unsigned long long>(),
                                                  any ? nullptr : T[T_IDX0 + cur].as<unsigned int>());
        TB2_CHECK_LAUNCH(ctx);
        any = true;
        for (int d = 0; d < 8; ++d) {
            if (!live[d]) continue;
            unsigned long long *kin = T[T_KEY0 + cur].as<unsigned long long>();
            unsigned long long *kout = T[T_KEY1 - cur].as<unsigned long long>();
            unsigned int *vin = T[T_IDX0 + cur].as<unsigned int>(), *vout = T[T_IDX1 - cur].as<unsigned int>();
            k_radix_tile_hist<<<(unsigned)n_tiles, RADIX_NT, 0, q>>>(kin, vin, n, 8 * d,
                                                                     T[T_THIST].as<unsigned int>(), n_tiles);
            TB2_CHECK_LAUNCH(ctx);
            k_radix_tile_scan<<<256, RADIX_NT, 0, q>>>(T[T_THIST].as<unsigned int>(), n_tiles,
                                                       gh + (size_t)(w * 8 + d) * 256,
                                                       T[T_TOFF].as<unsigned long long>());
            TB2_CHECK_LAUNCH(ctx);
            k_radix_scatter_pass<<<(unsigned)n_tiles, RADIX_NT, 0, q>>>(
                kin, vin, kout, vout, n, 8 * d, T[T_TOFF].as<unsigned long long>(), n_tiles);
            TB2_CHECK_LAUNCH(ctx);
            cur ^= 1;
        }
    }
    k_sf_gather<<<grid_of(m), 256, 0, q>>>(raw, T[T_OUT].as<unsigned long long>(), cap, K,
                                           any ? T[T_IDX0 + cur].as<unsigned int>() : nullptr, m);
    TB2_CHECK_LAUNCH(ctx);
    std::swap(T[T_RAW].p, T[T_OUT].p);
    std::swap(T[T_RAW].cap, T[T_OUT].cap);
    S.n = S.sorted = m;
    return TB2_OK;
}

int table_open(tb2_ctx *ctx, StatsFileState &S)
{
    if (S.kind >= 0) return TB2_OK;
    ctx->err = "tb2_most_signif_begin has not been called";
    return TB2_ERR_INVALID_ARG;
}

}  // namespace

// ---------------------------------------------------------------------------
// C ABI: aggregation
// ---------------------------------------------------------------------------
extern "C" int tb2_stats_file_aggregate(tb2_ctx *ctx, int64_t n_blocks, const int64_t *block_rows,
                                        int64_t region_size, int64_t n_stat, const uint32_t *pos,
                                        const double *stat, double single_read_thresh, double lower_thresh,
                                        int stat_type, double unmod_count, double mod_count, int64_t *row_off)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    S.agg_blocks = -1;
    const tb2_sf_block *blk = (const tb2_sf_block *)block_rows;
    if (n_blocks < 0 || n_blocks > INT32_MAX || (n_blocks > 0 && !blk) || !row_off || region_size < 1 ||
        region_size > (1LL << 28) || n_stat < 0 || (n_stat > 0 && (!pos || !stat)) ||
        isnan(single_read_thresh) || isnan(unmod_count) || isnan(mod_count) || (stat_type != 0 && stat_type != 1))
        return TB2_ERR_INVALID_ARG;
    std::vector<long long> ub((size_t)n_blocks + 1, 0);
    for (int64_t b = 0; b < n_blocks; ++b) {
        const tb2_sf_block &B = blk[b];
        if (B.stat_off < 0 || B.n_stat < 0 || B.stat_off > n_stat - B.n_stat || B.chrm < 0 ||
            B.chrm > (int64_t)UINT32_MAX || B.strand < 0 || B.strand > 255) {
            ctx->err = "a block's statistics range, chromosome id or strand is invalid";
            return TB2_ERR_INVALID_ARG;
        }
        ub[b + 1] = ub[b] + std::min<long long>(B.n_stat, region_size);
    }
    DevBuf *G = S.agg;
    cudaStream_t q = ctx->stream;
    const long long U = ub[n_blocks];
    TB2_RESERVE(ctx, "stats file", G[G_BLK], (size_t)n_blocks * sizeof(tb2_sf_block) + 8);
    TB2_RESERVE(ctx, "stats file", G[G_POS], (size_t)n_stat * 4 + 8);
    TB2_RESERVE(ctx, "stats file", G[G_STAT], (size_t)n_stat * 8 + 8);
    TB2_RESERVE(ctx, "stats file", G[G_UB], (size_t)(n_blocks + 1) * 8);
    TB2_RESERVE(ctx, "stats file", G[G_CNT], (size_t)n_blocks * 8 + 8);
    TB2_RESERVE(ctx, "stats file", G[G_OFF], (size_t)(n_blocks + 1) * 8);
    TB2_RESERVE(ctx, "stats file", G[G_ERR], 8);
    const int cols[5] = {G_UPOS, G_UDAMP, G_UFRAC, G_UCOV, G_UVALID}, pcols[5] = {G_POSO, G_DAMP, G_FRAC, G_COV, G_VALID};
    const int width[5] = {4, 8, 8, 4, 4};
    for (int c = 0; c < 5; ++c) {
        TB2_RESERVE(ctx, "stats file", G[cols[c]], (size_t)U * width[c] + 8);
        TB2_RESERVE(ctx, "stats file", G[pcols[c]], (size_t)U * width[c] + 8);
    }
    if (n_blocks)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(G[G_BLK].p, blk, (size_t)n_blocks * sizeof(tb2_sf_block),
                                          cudaMemcpyHostToDevice, q));
    if (n_stat) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(G[G_POS].p, pos, (size_t)n_stat * 4, cudaMemcpyHostToDevice, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(G[G_STAT].p, stat, (size_t)n_stat * 8, cudaMemcpyHostToDevice, q));
    }
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(G[G_UB].p, ub.data(), ub.size() * 8, cudaMemcpyHostToDevice, q));
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));          // kernel time: tb2_last_timing
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(G[G_ERR].p, 0, 4, q));
    AggArgs a;
    memset(&a, 0, sizeof(a));
    a.blk = G[G_BLK].as<tb2_sf_block>();
    a.pos = G[G_POS].as<unsigned int>();
    a.stat = G[G_STAT].as<double>();
    a.R = region_size;
    a.thresh = single_read_thresh; a.lower = lower_thresh; a.unmod = unmod_count; a.mod = mod_count;
    a.llr = stat_type == 0;
    a.ub = G[G_UB].as<long long>();
    a.o_pos = G[G_UPOS].as<unsigned int>(); a.o_damp = G[G_UDAMP].as<double>(); a.o_frac = G[G_UFRAC].as<double>();
    a.o_cov = G[G_UCOV].as<unsigned int>(); a.o_valid = G[G_UVALID].as<unsigned int>();
    a.n_rows = G[G_CNT].as<long long>();
    a.err = G[G_ERR].as<int>();
    int optin = 0;
    TB2_CUDA_TRY(ctx, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    const size_t smem = (size_t)region_size * 12;
    if (n_blocks && smem + sizeof(int) * (AGG_NT / 32) <= (size_t)optin) {
        TB2_CUDA_TRY(ctx, cudaFuncSetAttribute(k_sf_aggregate<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)smem));
        k_sf_aggregate<true><<<(unsigned)n_blocks, AGG_NT, smem, q>>>(a);
        TB2_CHECK_LAUNCH(ctx);
    } else if (n_blocks) {
        const long long per = std::max<long long>(1, std::min<long long>(n_blocks, (long long)(GCNT_BUDGET / smem)));
        TB2_RESERVE(ctx, "stats file", G[G_GCNT], (size_t)per * smem);
        a.gcnt = G[G_GCNT].as<int>();
        for (long long b0 = 0; b0 < n_blocks; b0 += per) {
            a.blk0 = (int)b0;
            k_sf_aggregate<false><<<(unsigned)std::min(per, n_blocks - b0), AGG_NT, 0, q>>>(a);
            TB2_CHECK_LAUNCH(ctx);
        }
    }
    k_scan_offsets<<<1, 1024, 0, q>>>(G[G_CNT].as<long long>(), G[G_OFF].as<long long>(), n_blocks);
    TB2_CHECK_LAUNCH(ctx);
    if (n_blocks) {
        k_sf_pack_rows<<<(unsigned)n_blocks, 256, 0, q>>>(
            G[G_UB].as<long long>(), G[G_OFF].as<long long>(), G[G_UPOS].as<unsigned int>(), G[G_UDAMP].as<double>(),
            G[G_UFRAC].as<double>(), G[G_UCOV].as<unsigned int>(), G[G_UVALID].as<unsigned int>(),
            G[G_POSO].as<unsigned int>(), G[G_DAMP].as<double>(), G[G_FRAC].as<double>(), G[G_COV].as<unsigned int>(),
            G[G_VALID].as<unsigned int>());
        TB2_CHECK_LAUNCH(ctx);
    }
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    int err = 0;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(&err, G[G_ERR].p, 4, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(row_off, G[G_OFF].p, (size_t)(n_blocks + 1) * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    if (err) {
        ctx->err = "a statistic's position lies outside its block [start, start + region_size)";
        return TB2_ERR_INVALID_ARG;
    }
    S.agg_blocks = n_blocks;
    S.agg_rows = row_off[n_blocks];
    return TB2_OK;
}

extern "C" int tb2_stats_file_aggregate_download(tb2_ctx *ctx, uint32_t *pos_out, double *damp_frac_out,
                                                 double *frac_out, uint32_t *cov_out, uint32_t *valid_cov_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    if (S.agg_blocks < 0) {
        ctx->err = "no successful tb2_stats_file_aggregate call";
        return TB2_ERR_INVALID_ARG;
    }
    const size_t n = (size_t)S.agg_rows;
    if (!n) return TB2_OK;
    if (!pos_out || !damp_frac_out || !frac_out || !cov_out || !valid_cov_out) return TB2_ERR_INVALID_ARG;
    DevBuf *G = S.agg;
    cudaStream_t q = ctx->stream;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, G[G_POSO].p, n * 4, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(damp_frac_out, G[G_DAMP].p, n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(frac_out, G[G_FRAC].p, n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cov_out, G[G_COV].p, n * 4, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(valid_cov_out, G[G_VALID].p, n * 4, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}

// ---------------------------------------------------------------------------
// C ABI: most-significant table
// ---------------------------------------------------------------------------
extern "C" int tb2_most_signif_begin(tb2_ctx *ctx, int kind, int64_t num_most_signif)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if ((kind != 0 && kind != 1) || num_most_signif < 1 || num_most_signif >= (1LL << 31)) return TB2_ERR_INVALID_ARG;
    StatsFileState &S = tb2_state(ctx->stats_file);
    if (S.kind >= 0) {
        ctx->err = "a most-significant table is open on this context: tb2_most_signif_end it first";
        return TB2_ERR_INVALID_ARG;
    }
    if (S.K != (kind == 0 ? 5 : 4)) S.cap = 0;       // the row layout changes: start the buffer over
    S.kind = kind;
    S.K = kind == 0 ? 5 : 4;
    S.nf = kind == 0 ? 2 : 1;
    S.N = num_most_signif;
    S.n = S.sorted = 0;
    return TB2_OK;
}

extern "C" int tb2_most_signif_end(tb2_ctx *ctx)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    S.kind = -1;
    S.n = S.sorted = 0;
    return TB2_OK;
}

extern "C" int tb2_most_signif_reset(tb2_ctx *ctx)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    if ((rc = table_open(ctx, S))) return rc;
    S.n = S.sorted = 0;
    return TB2_OK;
}

extern "C" int tb2_most_signif_add_rows(tb2_ctx *ctx, int64_t n, const double *key, const double *frac,
                                        const uint32_t *pos, const uint32_t *cov, const uint32_t *control_cov,
                                        const uint32_t *valid_cov, uint32_t chrm, uint8_t strand)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    if ((rc = table_open(ctx, S))) return rc;
    const bool model = S.kind == 0;
    if (n < 0 || (n > 0 && (!key || !pos || !cov || !control_cov || (model && (!frac || !valid_cov)))))
        return TB2_ERR_INVALID_ARG;
    for (int64_t i = 0; i < n; ++i)
        if (std::isnan(key[i])) { ctx->err = "NaN key: the writer drops those rows"; return TB2_ERR_INVALID_ARG; }
    if (n == 0) return TB2_OK;
    if (sf_reduce_before_add(S.n, n, S.cap, S.N) && (rc = table_reduce(ctx, S))) return rc;
    if ((rc = table_reserve(ctx, S, S.n + n))) return rc;
    std::vector<unsigned long long> w((size_t)S.K * n);
    for (int64_t i = 0; i < n; ++i)
        sf_pack_row(S.kind, key[i], model ? frac[i] : 0.0, pos[i], cov[i], control_cov[i], model ? valid_cov[i] : 0,
                    chrm, strand, w.data() + i, n);
    for (int k = 0; k < S.K; ++k)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(S.tab[T_RAW].as<unsigned long long>() + (size_t)k * S.cap + S.n,
                                          w.data() + (size_t)k * n, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));   // the host rows may go away
    S.n += n;
    return TB2_OK;
}

extern "C" int tb2_most_signif_add_aggregate(tb2_ctx *ctx)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    if ((rc = table_open(ctx, S))) return rc;
    if (S.kind != 0 || S.agg_blocks < 0) {
        ctx->err = "the table holds level statistics, or there is no aggregation to add";
        return TB2_ERR_INVALID_ARG;
    }
    const long long n = S.agg_rows;
    if (n == 0) return TB2_OK;
    if (sf_reduce_before_add(S.n, n, S.cap, S.N) && (rc = table_reduce(ctx, S))) return rc;
    if ((rc = table_reserve(ctx, S, S.n + n))) return rc;
    DevBuf *G = S.agg;
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    k_sf_table_from_agg<<<(unsigned)S.agg_blocks, 256, 0, ctx->stream>>>(
        G[G_BLK].as<tb2_sf_block>(), G[G_OFF].as<long long>(), G[G_POSO].as<unsigned int>(), G[G_DAMP].as<double>(),
        G[G_FRAC].as<double>(), G[G_COV].as<unsigned int>(), G[G_VALID].as<unsigned int>(),
        S.tab[T_RAW].as<unsigned long long>(), S.cap, S.n);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    S.n += n;
    return TB2_OK;
}

extern "C" int tb2_most_signif_count(tb2_ctx *ctx, int64_t *n_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    if ((rc = table_open(ctx, S))) return rc;
    if (!n_out) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    if ((rc = table_reduce(ctx, S))) return rc;
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    *n_out = S.n;
    return TB2_OK;
}

extern "C" int tb2_most_signif_get(tb2_ctx *ctx, double *key_out, double *frac_out, uint32_t *pos_out,
                                   uint32_t *cov_out, uint32_t *control_cov_out, uint32_t *valid_cov_out,
                                   uint32_t *chrm_out, uint8_t *strand_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    StatsFileState &S = tb2_state(ctx->stats_file);
    if ((rc = table_open(ctx, S))) return rc;
    const bool model = S.kind == 0;
    if (!key_out || !pos_out || !cov_out || !control_cov_out || !chrm_out || !strand_out ||
        (model && (!frac_out || !valid_cov_out)))
        return TB2_ERR_INVALID_ARG;
    if ((rc = table_reduce(ctx, S))) return rc;
    const long long n = S.n;
    if (!n) return TB2_OK;
    std::vector<unsigned long long> w((size_t)S.K * n);
    for (int k = 0; k < S.K; ++k)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(w.data() + (size_t)k * n, S.tab[T_RAW].as<unsigned long long>() + (size_t)k * S.cap,
                                          (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    for (long long i = 0; i < n; ++i) {
        memcpy(key_out + i, &w[i], 8);
        if (model) {
            memcpy(frac_out + i, &w[n + i], 8);
            pos_out[i] = (uint32_t)(w[2 * n + i] >> 32); cov_out[i] = (uint32_t)w[2 * n + i];
            control_cov_out[i] = (uint32_t)(w[3 * n + i] >> 32); valid_cov_out[i] = (uint32_t)w[3 * n + i];
            chrm_out[i] = (uint32_t)(w[4 * n + i] >> 8); strand_out[i] = (uint8_t)w[4 * n + i];
        } else {
            pos_out[i] = (uint32_t)(w[n + i] >> 32); cov_out[i] = (uint32_t)w[n + i];
            control_cov_out[i] = (uint32_t)(w[2 * n + i] >> 32); chrm_out[i] = (uint32_t)w[2 * n + i];
            strand_out[i] = (uint8_t)w[3 * n + i];
        }
    }
    return TB2_OK;
}
