// llr.cu -- per-read alternative-model log-likelihood ratios:
// compute_alt_model_read_stats tombo_stats.py:3972-4082 with trim_seq_and_means
// (:3888-3970), c_calc_scaled_llh_ratio_const_var _c_helper.pyx:313-358 (default) and
// c_calc_llh_ratio_const_var :298-311.  tb2_alt_model_llr_batch / tb2_batch_alt_llr score
// whole '+' strand reads with a single-base motif TomboMotif(alt_base, 1);
// tb2_alt_model_llr_motif_batch / tb2_batch_alt_llr_motif take any motif, both strands and
// a region (the kernels are in motif_llr.cuh).  Also c_new_mean_stds :38-57.
#include "batch.h"
#include "motif_llr.cuh"
#include <cstring>

namespace {
// per-call scratch of the entry points below; nothing reads it after a call returns
enum { L_MEAN = 0, L_MOFF, L_SEQ, L_SOFF, L_START, L_CNT, L_SITEOFF, L_LLR, L_POS, L_A, L_B, L_C, L_D,
       L_STRAND, L_STATUS, L_COUNT };
}  // namespace

struct LlrState {
    DevBuf scratch[L_COUNT];
    // resident LLRs of the last tb2_batch_alt_llr, for tb2_batch_llr_download and
    // tb2_region_stats_add_batch_llr
    DevBuf site_off, llr, pos;
    long long sites = 0;
    int reads = 0;
};

namespace {
// FILL = false: count sites per read; FILL = true: write llr / pos
template <bool FILL>
__global__ void __launch_bounds__(256)
k_llr(LlrArgs a, int *counts, const long long *site_off, double *llr_out, long long *pos_out)
{
    __shared__ unsigned int warp_tot[8];
    const int r = blockIdx.x, tid = threadIdx.x;
    const long long mo = a.mean_off[r];
    const int nb = (int)(a.mean_off[r + 1] - mo);
    const int K = a.K;
    // trimmed read sequence: base i = seq[so + cpos + i]
    const unsigned char *bases = a.seq + a.seq_off[r] + a.cpos;
    const double *means = a.norm_mean + mo;
    int testable = nb - 2 * (K - 1);            // len(motif_search_seq)
    if (a.status && a.status[(size_t)r * a.status_stride] != TB2_OK) testable = 0;
    if (testable <= 0) { if (!FILL && tid == 0) counts[r] = 0; return; }
    const int per = (testable + 255) / 256;
    const int i0 = min(testable, tid * per), i1 = min(testable, i0 + per);
    unsigned int mine = 0;
    for (int i = i0; i < i1; ++i) mine += (bases[i + K - 1] == a.alt_code);
    const int lane = tid & 31, warp = tid >> 5;
    unsigned int inc = mine;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const unsigned int o = __shfl_up_sync(0xffffffffu, inc, off);
        if (lane >= off) inc += o;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    unsigned int base = 0, total = 0;
    for (int q = 0; q < 8; ++q) { if (q < warp) base += warp_tot[q]; total += warp_tot[q]; }
    if (!FILL) { if (tid == 0) counts[r] = (int)total; return; }
    long long o = site_off[r] + base + inc - mine;
    for (int i = i0; i < i1; ++i) {
        if (bases[i + K - 1] != a.alt_code) continue;
        // alt_pos = i: k-mers i .. i+K-1 of the trimmed sequence, means' = means[cpos + .]
        llr_out[o] = llr_site(a, bases, means, i);
        pos_out[o] = a.read_start[r] + (K - 1) + i;
        ++o;
    }
}

__global__ void k_mean_stds(const double *sig, const long long *segs, long long n_segs,
                            double *means, double *sds)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_segs) return;
    const long long a = segs[i], z = segs[i + 1];
    double s = 0, v = 0;
    for (long long k = a; k < z; ++k) s += sig[k];
    const double m = s / (double)(z - a);
    means[i] = m;
    for (long long k = a; k < z; ++k) { const double d = sig[k] - m; v += d * d; }
    sds[i] = sqrt(v / (double)(z - a));
}

// exclusive scan of the per-read site counts (one block; n is a batch, <= ~1e6)
__global__ void __launch_bounds__(1024) k_scan_sites(const int *cnt, long long *site_off, int n)
{
    __shared__ long long warp_tot[32];
    __shared__ long long base_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { base_s = 0; site_off[0] = 0; }
    __syncthreads();
    for (int c0 = 0; c0 < n; c0 += 1024) {
        const int i = c0 + tid;
        long long v = i < n ? cnt[i] : 0, inc = v;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const long long o = __shfl_up_sync(0xffffffffu, inc, off);
            if (lane >= off) inc += o;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        long long before = 0, total = 0;
        for (int q = 0; q < 32; ++q) { if (q < warp) before += warp_tot[q]; total += warp_tot[q]; }
        if (i < n) site_off[i + 1] = base_s + before + inc;
        __syncthreads();
        if (tid == 0) base_s += total;
        __syncthreads();
    }
}
}  // namespace

extern "C" int tb2_set_alt_model(tb2_ctx *ctx, const double *alt_means, int kmer_width)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!alt_means || kmer_width < 1 || kmer_width > 12) return TB2_ERR_INVALID_ARG;
    const size_t n = ((size_t)1 << (2 * kmer_width)) * kmer_width;
    TB2_CUDA_TRY(ctx, ctx->alt_means.upload(alt_means, n, ctx->stream));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->alt_kmer_width = kmer_width;
    return TB2_OK;
}

namespace {
bool alt_model_ok(tb2_ctx *ctx)
{
    if (ctx->kmer_width > 0 && ctx->alt_kmer_width == ctx->kmer_width) return true;
    ctx->err = "standard and alternative models must be set with the same k-mer width";
    return false;
}

// everything of LlrArgs but the reads
LlrArgs llr_args(tb2_ctx *ctx, int alt_code, int use_standard_llhr, double sf, double hf, double hp)
{
    LlrArgs a;
    memset(&a, 0, sizeof(a));
    a.K = ctx->kmer_width; a.cpos = ctx->central_pos; a.alt_code = alt_code;
    a.use_std = use_standard_llhr ? 1 : 0;
    a.sf = sf; a.hf = hf; a.hp = hp;
    a.kmeans = ctx->model_means.as<double>();
    a.ksds = ctx->model_sds.as<double>();
    a.alt = ctx->alt_means.as<double>();
    return a;
}

// the reads of the resident batch (after tb2_batch_compute): sequence, per-base means and
// per-read status are already in HBM; only the read starts are uploaded
int resident_reads(tb2_ctx *ctx, const int64_t *read_start, BatchResultView *v, LlrArgs &a)
{
    int rc = tb2_batch_result_view(ctx, v);
    if (rc) return rc;
    DevBuf &start = tb2_state(ctx->llr).scratch[L_START];
    TB2_CUDA_TRY(ctx, start.upload(read_start, (size_t)v->n_reads, ctx->stream));
    a.n_reads = v->n_reads;
    a.norm_mean = v->norm_mean; a.mean_off = v->base_off; a.seq_off = v->seq_off; a.seq = v->seq;
    a.read_start = start.as<long long>();
    a.status = v->status; a.status_stride = v->stride;
    return TB2_OK;
}

// k_llr<FILL> or k_llr_motif<FILL>
template <class A> using LlrKernel = void (*)(A, int *, const long long *, double *, long long *);

// count -> scan -> fill over the n reads of `a`: site offsets (n + 1) into site_off, LLRs and
// positions into llr / pos, which get room for max_sites sites.  Reads back the site count
// and, where read_status is given, the per-read status the motif count pass wrote.
template <class A>
int run_llr(tb2_ctx *ctx, LlrKernel<A> count, LlrKernel<A> fill, const A &a, int n,
            size_t max_sites, DevBuf &site_off, DevBuf &llr, DevBuf &pos, int32_t *read_status,
            long long *total)
{
    auto &P = tb2_state(ctx->llr).scratch;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, P[L_CNT].reserve((size_t)n * 4));
    TB2_CUDA_TRY(ctx, site_off.reserve((size_t)(n + 1) * 8));
    TB2_CUDA_TRY(ctx, llr.reserve(max_sites * 8 + 8));
    TB2_CUDA_TRY(ctx, pos.reserve(max_sites * 8 + 8));
    count<<<n, 256, 0, s>>>(a, P[L_CNT].as<int>(), nullptr, nullptr, nullptr);
    TB2_CHECK_LAUNCH(ctx);
    k_scan_sites<<<1, 1024, 0, s>>>(P[L_CNT].as<int>(), site_off.as<long long>(), n);
    TB2_CHECK_LAUNCH(ctx);
    fill<<<n, 256, 0, s>>>(a, nullptr, site_off.as<long long>(), llr.as<double>(), pos.as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(total, site_off.as<long long>() + n, 8, cudaMemcpyDeviceToHost, s));
    if (read_status)
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(read_status, P[L_STATUS].p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

// host-array calls: sites in the per-call scratch, copied out to the caller
template <class A>
int run_host(tb2_ctx *ctx, LlrKernel<A> count, LlrKernel<A> fill, const A &a, int n,
             size_t max_sites, double *llr_out, int64_t *pos_out, int64_t *site_off,
             int32_t *read_status)
{
    auto &P = tb2_state(ctx->llr).scratch;
    cudaStream_t s = ctx->stream;
    long long total = 0;
    int rc = run_llr(ctx, count, fill, a, n, max_sites, P[L_SITEOFF], P[L_LLR], P[L_POS],
                     read_status, &total);
    if (rc) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(site_off, P[L_SITEOFF].p, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, s));
    if (total) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(llr_out, P[L_LLR].p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, P[L_POS].p, (size_t)total * 8, cudaMemcpyDeviceToHost, s));
    }
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

// resident calls: the LLRs stay in LlrState for tb2_batch_llr_download and
// tb2_region_stats_add_batch_llr
template <class A>
int run_resident(tb2_ctx *ctx, LlrKernel<A> count, LlrKernel<A> fill, const A &a,
                 const BatchResultView &v, int32_t *read_status, int64_t *n_sites_total)
{
    LlrState &L = tb2_state(ctx->llr);
    long long total = 0;
    // every site is a base: the batch's base count bounds the site count (no size round trip)
    int rc = run_llr(ctx, count, fill, a, v.n_reads, (size_t)v.total_bases, L.site_off, L.llr,
                     L.pos, read_status, &total);
    if (rc) return rc;
    L.sites = total;
    L.reads = v.n_reads;
    if (n_sites_total) *n_sites_total = total;
    return TB2_OK;
}
}  // namespace

extern "C" int tb2_alt_model_llr_batch(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                                       const int64_t *mean_off, const uint8_t *seq,
                                       const int64_t *seq_off, const int64_t *read_start,
                                       int alt_base_code, int use_standard_llhr,
                                       double scale_factor, double height_factor,
                                       double height_power, double *llr_out, int64_t *pos_out,
                                       int64_t *site_off)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!site_off || alt_base_code < 0 || alt_base_code > 3 || !alt_model_ok(ctx))
        return TB2_ERR_INVALID_ARG;
    LlrArgs a = llr_args(ctx, alt_base_code, use_standard_llhr, scale_factor, height_factor, height_power);
    if ((rc = tb2_stage_reads(ctx, n_reads, norm_mean, mean_off, seq, seq_off, read_start,
                              tb2_state(ctx->llr).scratch + L_MEAN, a)))
        return rc;
    const int n = a.n_reads = (int)n_reads;
    site_off[0] = 0;
    if (n == 0) return TB2_OK;
    if (!norm_mean || !seq || !llr_out || !pos_out) return TB2_ERR_INVALID_ARG;
    // every site is a base of its read: the mean count bounds the site count
    return run_host(ctx, k_llr<false>, k_llr<true>, a, n, (size_t)mean_off[n], llr_out, pos_out,
                    site_off, nullptr);
}

extern "C" int tb2_batch_alt_llr(tb2_ctx *ctx, const int64_t *read_start, int alt_base_code,
                                 int use_standard_llhr, double scale_factor, double height_factor,
                                 double height_power, int64_t *n_sites_total)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!read_start || alt_base_code < 0 || alt_base_code > 3 || !alt_model_ok(ctx))
        return TB2_ERR_INVALID_ARG;
    LlrArgs a = llr_args(ctx, alt_base_code, use_standard_llhr, scale_factor, height_factor, height_power);
    BatchResultView v;
    if ((rc = resident_reads(ctx, read_start, &v, a))) return rc;
    return run_resident(ctx, k_llr<false>, k_llr<true>, a, v, nullptr, n_sites_total);
}

// ---------------------------------------------------------------------------
// motif models, both strands, region clipping (k_llr_motif, motif_llr.cuh)
// ---------------------------------------------------------------------------
namespace {
// checks shared by both motif entry points; fills everything of `a` but the reads and strands
int motif_args(tb2_ctx *ctx, const tb2_motif *motif, int64_t max_motif_bb, int64_t max_motif_ab,
               int64_t reg_start, int64_t reg_end, int use_standard_llhr, double sf, double hf,
               double hp, MotifArgs *a)
{
    if (!motif || motif->len < 1 || motif->len > 32 || motif->mod_pos < 1 ||
        motif->mod_pos > motif->len)
        return TB2_ERR_INVALID_ARG;
    for (int j = 0; j < motif->len; ++j)
        if (motif->mask[j] == 0 || motif->mask[j] > 15) return TB2_ERR_INVALID_ARG;
    if (max_motif_bb < motif->mod_pos - 1 || max_motif_ab < motif->len - motif->mod_pos)
        return TB2_ERR_INVALID_ARG;
    if (!alt_model_ok(ctx)) return TB2_ERR_INVALID_ARG;
    memset(a, 0, sizeof(*a));
    a->m.len = motif->len;
    a->m.mod_pos = motif->mod_pos;
    for (int j = 0; j < motif->len; ++j) a->m.mask[j] = motif->mask[j];
    a->m.overlap = motif_can_overlap(a->m.mask, a->m.len) ? 1 : 0;
    a->max_ab = max_motif_ab;
    a->reg_start = reg_start;
    a->reg_end = reg_end;
    a->s = llr_args(ctx, -1, use_standard_llhr, sf, hf, hp);
    return TB2_OK;
}

// checks and uploads the strand of each of n reads; the count pass writes each read's status
int motif_strands(tb2_ctx *ctx, int n, const int8_t *strand, MotifArgs &a)
{
    for (int r = 0; r < n; ++r)
        if (strand[r] < -1 || strand[r] > 1) return TB2_ERR_INVALID_ARG;
    auto &P = tb2_state(ctx->llr).scratch;
    TB2_CUDA_TRY(ctx, P[L_STRAND].upload(strand, (size_t)n, ctx->stream));
    TB2_CUDA_TRY(ctx, P[L_STATUS].reserve((size_t)n * 4));
    a.strand = P[L_STRAND].as<signed char>();
    a.read_status = P[L_STATUS].as<int>();
    return TB2_OK;
}
}  // namespace

extern "C" int tb2_alt_model_llr_motif_batch(
    tb2_ctx *ctx, int64_t n_reads, const double *norm_mean, const int64_t *mean_off,
    const uint8_t *seq, const int64_t *seq_off, const int64_t *read_start, const int8_t *strand,
    const tb2_motif *motif, int64_t max_motif_bb, int64_t max_motif_ab, int64_t reg_start,
    int64_t reg_end, int use_standard_llhr, double scale_factor, double height_factor,
    double height_power, double *llr_out, int64_t *pos_out, int64_t *site_off, int32_t *read_status)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!strand || !site_off) return TB2_ERR_INVALID_ARG;
    MotifArgs a;
    if ((rc = motif_args(ctx, motif, max_motif_bb, max_motif_ab, reg_start, reg_end,
                         use_standard_llhr, scale_factor, height_factor, height_power, &a)))
        return rc;
    if ((rc = tb2_stage_reads(ctx, n_reads, norm_mean, mean_off, seq, seq_off, read_start,
                              tb2_state(ctx->llr).scratch + L_MEAN, a.s)))
        return rc;
    const int n = a.s.n_reads = (int)n_reads;
    if ((rc = motif_strands(ctx, n, strand, a))) return rc;
    site_off[0] = 0;
    if (n == 0) return TB2_OK;
    if (!norm_mean || !seq || !llr_out || !pos_out) return TB2_ERR_INVALID_ARG;
    return run_host(ctx, k_llr_motif<false>, k_llr_motif<true>, a, n, (size_t)mean_off[n], llr_out,
                    pos_out, site_off, read_status);
}

extern "C" int tb2_batch_alt_llr_motif(tb2_ctx *ctx, const int64_t *read_start, const int8_t *strand,
                                       const tb2_motif *motif, int64_t max_motif_bb,
                                       int64_t max_motif_ab, int64_t reg_start, int64_t reg_end,
                                       int use_standard_llhr, double scale_factor,
                                       double height_factor, double height_power,
                                       int32_t *read_status, int64_t *n_sites_total)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!read_start || !strand) return TB2_ERR_INVALID_ARG;
    MotifArgs a;
    if ((rc = motif_args(ctx, motif, max_motif_bb, max_motif_ab, reg_start, reg_end,
                         use_standard_llhr, scale_factor, height_factor, height_power, &a)))
        return rc;
    BatchResultView v;
    if ((rc = resident_reads(ctx, read_start, &v, a.s))) return rc;
    if ((rc = motif_strands(ctx, v.n_reads, strand, a))) return rc;
    return run_resident(ctx, k_llr_motif<false>, k_llr_motif<true>, a, v, read_status, n_sites_total);
}

extern "C" int tb2_batch_llr_download(tb2_ctx *ctx, double *llr_out, int64_t *pos_out, int64_t *site_off)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    const LlrState &L = tb2_state(ctx->llr);
    if (L.reads <= 0 || !site_off) return TB2_ERR_INVALID_ARG;
    cudaStream_t s = ctx->stream;
    const size_t t = (size_t)L.sites;
    if (t && (!llr_out || !pos_out)) return TB2_ERR_INVALID_ARG;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(site_off, L.site_off.p, (size_t)(L.reads + 1) * 8, cudaMemcpyDeviceToHost, s));
    if (t) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(llr_out, L.llr.p, t * 8, cudaMemcpyDeviceToHost, s));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, L.pos.p, t * 8, cudaMemcpyDeviceToHost, s));
    }
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

// the resident LLRs feed the region counters without leaving the device
extern "C" int tb2_region_stats_add_batch_llr(tb2_ctx *ctx, double single_read_thresh,
                                              double lower_thresh, int stat_type)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    LlrState &L = tb2_state(ctx->llr);
    if (L.reads <= 0 || isnan(single_read_thresh)) return TB2_ERR_INVALID_ARG;
    return tb2_region_accumulate_dev(ctx, L.sites, L.llr.as<double>(), L.pos.as<long long>(),
                                     single_read_thresh, lower_thresh, stat_type);
}

extern "C" int tb2_new_mean_stds(tb2_ctx *ctx, const double *sig, int64_t n_sig,
                                 const int64_t *segs, int64_t n_segs, double *means_out,
                                 double *sds_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (!sig || !segs || !means_out || !sds_out || n_sig < 1 || n_segs < 1) return TB2_ERR_INVALID_ARG;
    for (int64_t i = 0; i <= n_segs; ++i)
        if (segs[i] < 0 || segs[i] > n_sig) return TB2_ERR_INVALID_ARG;
    auto &P = tb2_state(ctx->llr).scratch;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, P[L_A].upload(sig, (size_t)n_sig, s));
    TB2_CUDA_TRY(ctx, P[L_B].upload(segs, (size_t)n_segs + 1, s));
    TB2_CUDA_TRY(ctx, P[L_C].reserve((size_t)n_segs * 8));
    TB2_CUDA_TRY(ctx, P[L_D].reserve((size_t)n_segs * 8));
    k_mean_stds<<<(unsigned)((n_segs + 127) / 128), 128, 0, s>>>(
        P[L_A].as<double>(), P[L_B].as<long long>(), n_segs, P[L_C].as<double>(), P[L_D].as<double>());
    TB2_CHECK_LAUNCH(ctx);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(means_out, P[L_C].p, (size_t)n_segs * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(sds_out, P[L_D].p, (size_t)n_segs * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}

// ---------------------------------------------------------------------------
// batched mirrors of the three Cython scorers over explicit windows:
// mode 0 c_calc_scaled_llh_ratio_const_var (_c_helper.pyx:313-358)
// mode 1 c_calc_llh_ratio_const_var (:298-311), mode 2 c_calc_llh_ratio (:277-296)
// means / ref_means / alt_means: n x K row-major; var_a: const_var[n] (modes 0,1)
// or ref_vars[n x K] (mode 2); var_b: alt_vars[n x K] (mode 2)
// ---------------------------------------------------------------------------
namespace {
__global__ void k_llh_windows(int mode, long long n, int K, const double *m, const double *rm,
                              const double *am, const double *va, const double *vb, double sf,
                              double hf, double hp, double *out)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const double *pm = m + s * K, *pr = rm + s * K, *pa = am + s * K;
    double acc = 0.0;
    if (mode == 2) {
        double rz = 0, rl = 0, az = 0, al = 0;
        for (int i = 0; i < K; ++i) {
            const double rd = pm[i] - pr[i];
            rz += (rd * rd) / va[s * K + i];
            rl += log(va[s * K + i]);
            const double ad = pm[i] - pa[i];
            az += (ad * ad) / vb[s * K + i];
            al += log(vb[s * K + i]);
        }
        out[s] = az + al - rz - rl;
        return;
    }
    const double cv = va[s];
    for (int i = 0; i < K; ++i) {
        const double obs = pm[i], ref_mean = pr[i], alt_mean = pa[i];
        if (mode == 1) {
            const double rd = obs - ref_mean, ad = obs - alt_mean;
            acc += ((ad * ad) - (rd * rd)) / cv;
        } else {
            if (ref_mean == alt_mean) continue;
            const double scale_mean = (alt_mean + ref_mean) / 2;
            const double ref_diff = obs - ref_mean, alt_diff = obs - alt_mean;
            const double scale_diff = obs - scale_mean;
            double means_diff = alt_mean - ref_mean;
            if (means_diff < 0) means_diff = means_diff * -1;
            acc += exp(-(scale_diff * scale_diff) / (sf * cv)) *
                   ((alt_diff * alt_diff) - (ref_diff * ref_diff)) / (cv * pow(means_diff, hp) * hf);
        }
    }
    out[s] = acc;
}
}  // namespace

extern "C" int tb2_calc_llh_ratio_windows(tb2_ctx *ctx, int mode, int64_t n_sites, int kmer_width,
                                          const double *means, const double *ref_means,
                                          const double *alt_means, const double *var_a,
                                          const double *var_b, double scale_factor,
                                          double height_factor, double height_power,
                                          double *llr_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (mode < 0 || mode > 2 || n_sites < 0 || kmer_width < 1 || !var_a || (mode == 2 && !var_b))
        return TB2_ERR_INVALID_ARG;
    if (n_sites == 0) return TB2_OK;
    if (!means || !ref_means || !alt_means || !llr_out) return TB2_ERR_INVALID_ARG;
    auto &P = tb2_state(ctx->llr).scratch;
    cudaStream_t s = ctx->stream;
    const size_t nk = (size_t)n_sites * kmer_width, nv = (size_t)n_sites;
    TB2_CUDA_TRY(ctx, P[L_MEAN].upload(means, nk, s));
    TB2_CUDA_TRY(ctx, P[L_A].upload(ref_means, nk, s));
    TB2_CUDA_TRY(ctx, P[L_B].upload(alt_means, nk, s));
    TB2_CUDA_TRY(ctx, P[L_C].upload(var_a, mode == 2 ? nk : nv, s));
    TB2_CUDA_TRY(ctx, P[L_D].upload(var_b, mode == 2 ? nk : 0, s));
    TB2_CUDA_TRY(ctx, P[L_LLR].reserve(nv * 8));
    k_llh_windows<<<(unsigned)((n_sites + 127) / 128), 128, 0, s>>>(
        mode, n_sites, kmer_width, P[L_MEAN].as<double>(), P[L_A].as<double>(), P[L_B].as<double>(),
        P[L_C].as<double>(), P[L_D].as<double>(), scale_factor, height_factor, height_power,
        P[L_LLR].as<double>());
    TB2_CHECK_LAUNCH(ctx);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(llr_out, P[L_LLR].p, nv * 8, cudaMemcpyDeviceToHost, s));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return TB2_OK;
}
