// accuracy.cu -- accuracy of modified-base calls on the device (tombo plot roc, per_read_roc,
// sample_compare_roc, per_read_sample_compare_roc).
//
//   tb2_accuracy_label_motif  _compute_motif_stats tombo_stats.py:2406-2456: a window around
//                             each statistic, the mod-base check and the motif prefix match
//   tb2_accuracy_label_truth  _compute_ground_truth_stats :2458-2483: binary search in the
//                             sorted mod / unmod locations of the block's (chrm, strand)
//   tb2_accuracy_label_ctrl   _compute_ctrl_motif_stats :2485-2535: re.finditer motif sites per
//                             block, sample statistics at a site True, control ones False
//   tb2_accuracy_curve        prep_accuracy_rates _plot_commands.py:60-82 with
//                             compute_accuracy_rates :2384-2404 on one slot: Python's tuple
//                             order by a stable LSD radix sort, then the sampled rates
//   tb2_accuracy_rates_ordered  compute_accuracy_rates on labels already in order
//
// Labelling appends (stat, label) entries to slots (one per modification name) that stay
// on the device until tb2_accuracy_reset.  Every labelling call is a count pass (one block
// of 256 threads per statistics block, counts per block and motif), a host-side prefix over
// the counts, and one ordered scatter pass per slot, so each slot receives its entries in
// exactly the reference's append order (DESIGN.md §3 "Accuracy of modified-base calls").
#include "ctx.h"
#include "motif_llr.cuh"
#include "radix_sort.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <utility>

static_assert(sizeof(tb2_acc_block) == TB2_ACC_BLOCK_FIELDS * 8, "tb2_acc_block rows");

namespace {

constexpr int AT = 256;                 // threads per block of every accuracy kernel
constexpr int MAXM = 8;                 // motifs per labelling call
constexpr int MAXSLOT = 16;             // slots (modification names)
constexpr int IPT = RADIX_IPT;          // radix sort: items per thread of a tile
constexpr int TILE = RADIX_TILE;
static_assert(AT == RADIX_NT, "the curve kernels share the radix sort's tiles");

enum { A_BLK = 0, A_SEQ, A_POS, A_STAT, A_CPOS, A_CSTAT, A_MOD, A_UNMOD, A_SITE, A_CNT, A_OFF,
       A_KEY0, A_KEY1, A_LAB0, A_LAB1, A_THIST, A_TOFF, A_GHIST, A_IDX, A_OUT, A_COUNT };

struct Slot {
    DevBuf stat, lab;
    long long n = 0;
};

}  // namespace

struct AccuracyState {
    DevBuf buf[A_COUNT];
    Slot slot[MAXSLOT];
};

namespace {

enum { MODE_MOTIF = 0, MODE_TRUTH = 1, MODE_CTRL = 2 };

struct AccArgs {
    const tb2_acc_block *blk;
    const unsigned char *seq;              // codes: A C G T = 0..3, anything else 4
    const unsigned int *pos, *cpos;
    const double *stat, *cstat;
    const long long *mod, *unmod;
    const unsigned char *site;             // ctrl: site[m * n_seq + seq_off + r]
    long long n_seq, bb, ab;
    int n_motifs;
    MotifDev fw[MAXM], rc[MAXM];           // motif and reverse-complement masks
    unsigned char mod_base[MAXM];          // code of the motif's mod base
};

__device__ __forceinline__ bool class_has(unsigned char mask, int code)
{
    return code < 4 && ((mask >> code) & 1u);
}

// the window of one statistic (tombo_stats.py:2432-2440): reg_seq[lo:hi] clipped to the
// sequence, reverse-complemented on '-'.  lo < 0 is the uint32 wrap of the reference (an empty
// slice); a window of at most bb bases makes window[bb] raise IndexError.
struct Win {
    const unsigned char *s;
    long long lo, len;
    int minus;
};

__device__ __forceinline__ bool window_of(const AccArgs &a, const tb2_acc_block &B, unsigned int pos, Win &w)
{
    const long long r = (long long)pos - B.seq_start;
    w.s = a.seq + B.seq_off;
    w.minus = B.strand;
    const long long lo = B.strand ? r - a.ab : r - a.bb;
    const long long hi = B.strand ? r + a.bb + 1 : r + a.ab + 1;
    if (lo < 0) return false;
    const long long end = hi < B.seq_len ? hi : B.seq_len;
    w.lo = lo;
    w.len = end > lo ? end - lo : 0;
    return w.len > a.bb;
}

__device__ __forceinline__ int win_at(const Win &w, long long k)
{
    if (!w.minus) return w.s[w.lo + k];
    const int c = w.s[w.lo + w.len - 1 - k];
    return c < 4 ? 3 - c : c;
}

// -1: motif m skipped (window[bb] is not its mod base), else whether motif_pat.match holds
// at window[bb - mod_pos + 1:]
__device__ __forceinline__ int motif_hit(const AccArgs &a, const Win &w, int m)
{
    if (win_at(w, a.bb) != a.mod_base[m]) return -1;
    const MotifDev &md = a.fw[m];
    const long long s = a.bb - md.mod_pos + 1;
    if (s + md.len > w.len) return 0;
    for (int j = 0; j < md.len; ++j)
        if (!class_has(md.mask[j], win_at(w, s + j))) return 0;
    return 1;
}

__device__ __forceinline__ bool in_sorted(const long long *v, long long n, long long x)
{
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (v[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo < n && v[lo] == x;
}

// ctrl: -1 no site, else the label of item j of motif block (sample j < n_stat: True)
__device__ __forceinline__ int ctrl_hit(const AccArgs &a, const tb2_acc_block &B, int m, long long j,
                                        double &v)
{
    unsigned int p;
    int lab;
    if (j < B.n_stat) { p = a.pos[B.stat_off + j]; v = a.stat[B.stat_off + j]; lab = 1; }
    else { p = a.cpos[B.ctrl_off + j - B.n_stat]; v = a.cstat[B.ctrl_off + j - B.n_stat]; lab = 0; }
    const long long r = (long long)p - B.seq_start;
    if (r < 0 || r >= B.seq_len) return -1;
    return a.site[(size_t)m * a.n_seq + B.seq_off + r] ? lab : -1;
}

template <int MODE> __device__ __forceinline__ long long n_items(const AccArgs &a, const tb2_acc_block &B)
{
    return MODE == MODE_CTRL ? (long long)a.n_motifs * (B.n_stat + B.n_ctrl) : B.n_stat;
}

// count pass: cnt[b * n_motifs + m] entries of block b for motif m; *fail = 1 when a motif
// window raises in the reference
template <int MODE>
__global__ void __launch_bounds__(AT) k_acc_count(AccArgs a, long long *cnt, int *fail)
{
    __shared__ unsigned int sh[MAXM];
    const int b = blockIdx.x, tid = threadIdx.x;
    const tb2_acc_block B = a.blk[b];
    if (tid < MAXM) sh[tid] = 0;
    __syncthreads();
    const long long n = n_items<MODE>(a, B);
    for (long long i = tid; i < n; i += AT) {
        if (MODE == MODE_MOTIF) {
            Win w;
            if (!window_of(a, B, a.pos[B.stat_off + i], w)) { *fail = 1; continue; }
            for (int m = 0; m < a.n_motifs; ++m)
                if (motif_hit(a, w, m) >= 0) atomicAdd(sh + m, 1u);
        } else if (MODE == MODE_TRUTH) {
            const long long p = a.pos[B.stat_off + i];
            if (in_sorted(a.mod + B.mod_off, B.n_mod, p) || in_sorted(a.unmod + B.unmod_off, B.n_unmod, p))
                atomicAdd(sh, 1u);
        } else {
            const long long per = B.n_stat + B.n_ctrl;
            const int m = (int)(i / per);
            double v;
            if (ctrl_hit(a, B, m, i - m * per, v) >= 0) atomicAdd(sh + m, 1u);
        }
    }
    __syncthreads();
    const int nm = MODE == MODE_TRUTH ? 1 : a.n_motifs;
    if (tid < nm) cnt[(size_t)b * nm + tid] = (long long)sh[tid];
}

// scatter pass of one slot (motifs `mask`): block b's entries go to out[off[b] ...] in the
// reference's append order
template <int MODE>
__global__ void __launch_bounds__(AT)
k_acc_scatter(AccArgs a, unsigned int mask, const long long *off, double *out_stat, unsigned char *out_lab)
{
    __shared__ unsigned int warp_tot[AT / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const tb2_acc_block B = a.blk[b];
    const long long n = n_items<MODE>(a, B);
    long long base = off[b];
    for (long long i0 = 0; i0 < n; i0 += AT) {
        const long long i = i0 + tid;
        unsigned int c = 0;
        Win w;
        w.len = 0;
        double v = 0;
        int lab = -1;
        if (i < n) {
            if (MODE == MODE_MOTIF) {
                if (window_of(a, B, a.pos[B.stat_off + i], w)) {
                    v = a.stat[B.stat_off + i];
                    for (int m = 0; m < a.n_motifs; ++m)
                        if (((mask >> m) & 1u) && motif_hit(a, w, m) >= 0) ++c;
                }
            } else if (MODE == MODE_TRUTH) {
                const long long p = a.pos[B.stat_off + i];
                v = a.stat[B.stat_off + i];
                lab = in_sorted(a.mod + B.mod_off, B.n_mod, p) ? 1
                      : (in_sorted(a.unmod + B.unmod_off, B.n_unmod, p) ? 0 : -1);
                c = lab >= 0;
            } else {
                const long long per = B.n_stat + B.n_ctrl;
                const int m = (int)(i / per);
                if ((mask >> m) & 1u) lab = ctrl_hit(a, B, m, i - m * per, v);
                c = lab >= 0;
            }
        }
        unsigned int total;
        __syncthreads();          // here rather than after the fills: a warp's fills overlap the next lookups
        long long o = base + tb2_block_excl_scan<AT>(c, warp_tot, total);
        base += total;
        if (c) {
            if (MODE == MODE_MOTIF) {
                for (int m = 0; m < a.n_motifs; ++m) {
                    if (!((mask >> m) & 1u)) continue;
                    const int h = motif_hit(a, w, m);
                    if (h < 0) continue;
                    out_stat[o] = v;
                    out_lab[o] = (unsigned char)h;
                    ++o;
                }
            } else {
                out_stat[o] = v;
                out_lab[o] = (unsigned char)lab;
            }
        }
    }
}

// finditer sites of motif blockIdx.y over block blockIdx.x's sequence: a motif that cannot
// overlap itself takes every match; one that can is walked left to right by warp 0
__global__ void __launch_bounds__(AT) k_acc_sites(AccArgs a, unsigned char *site)
{
    const int b = blockIdx.x, m = blockIdx.y, tid = threadIdx.x;
    const tb2_acc_block B = a.blk[b];
    const MotifDev &md = B.strand ? a.rc[m] : a.fw[m];
    const unsigned char *s = a.seq + B.seq_off;
    const long long L = B.seq_len, n = L - md.len + 1;
    const int shift = B.strand ? md.len - md.mod_pos : md.mod_pos - 1;
    unsigned char *out = site + (size_t)m * a.n_seq + B.seq_off + shift;
    if (n <= 0) return;
    if (!md.overlap) {
        for (long long p = tid; p < n; p += AT) {
            bool ok = true;
            for (int j = 0; j < md.len && ok; ++j) ok = class_has(md.mask[j], s[p + j]);
            if (ok) out[p] = 1;
        }
        return;
    }
    if (tid >= 32) return;
    long long next = 0;
    for (long long c0 = 0; c0 < n; c0 += 32) {
        const long long p = c0 + tid;
        bool ok = p < n;
        for (int j = 0; j < md.len && ok; ++j) ok = class_has(md.mask[j], s[p + j]);
        unsigned int bits = __ballot_sync(0xffffffffu, ok);
        unsigned int take = 0;
        while (bits) {                                   // every lane walks the same bits
            const int q = __ffs(bits) - 1;
            bits &= bits - 1;
            if (c0 + q < next) continue;
            take |= 1u << q;
            next = c0 + q + md.len;
        }
        if ((take >> tid) & 1u) out[p] = 1;
    }
}

// ---------------------------------------------------------------------------
// curve: order-preserving keys (radix_sort.cuh), stable LSD radix sort carrying the label, rates
// ---------------------------------------------------------------------------
// keys, NaN flag, and the histograms of all eight key digits (ghist[d * 256 + v]) and of
// the label (ghist[8 * 256 + l]); a histogram does not depend on the order, so every pass
// that a single bin holds is known before the sort starts
__global__ void __launch_bounds__(AT)
k_acc_keys(const double *stat, long long n, unsigned long long *key, unsigned long long *ghist, int *nan_flag)
{
    __shared__ unsigned int h[9 * 256];
    for (int i = threadIdx.x; i < 9 * 256; i += AT) h[i] = 0;
    __syncthreads();
    for (long long i = (long long)blockIdx.x * AT + threadIdx.x; i < n; i += (long long)gridDim.x * AT) {
        const double x = stat[i];
        if (x != x) { *nan_flag = 1; continue; }
        const unsigned long long k = order_key(x);
        key[i] = k;
#pragma unroll
        for (int d = 0; d < 8; ++d) atomicAdd(h + d * 256 + (int)((k >> (8 * d)) & 255u), 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * 256; i += AT)
        if (h[i]) atomicAdd(ghist + i, (unsigned long long)h[i]);
}

__global__ void k_acc_label_hist(const unsigned char *lab, long long n, unsigned long long *ghist)
{
    unsigned int t = 0;
    for (long long i = (long long)blockIdx.x * AT + threadIdx.x; i < n; i += (long long)gridDim.x * AT)
        t += lab[i];
    t = __reduce_add_sync(0xffffffffu, t);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(ghist + 8 * 256 + 1, (unsigned long long)t);
}

// per-tile label sums
__global__ void __launch_bounds__(AT) k_acc_lab_tiles(const unsigned char *lab, long long n, unsigned long long *tsum)
{
    __shared__ unsigned int warp_tot[AT / 32];
    const long long t = blockIdx.x, i0 = t * TILE;
    unsigned int s = 0;
    for (int r = 0; r < IPT; ++r) {
        const long long i = i0 + r * AT + threadIdx.x;
        if (i < n) s += lab[i];
    }
    unsigned int total;
    tb2_block_excl_scan<AT>(s, warp_tot, total);
    if (threadIdx.x == 0) tsum[t] = total;
}

// tp_cumsum at index q: one warp per query
__device__ __forceinline__ long long tp_at(const unsigned char *lab, const unsigned long long *texcl, long long q)
{
    const long long t = q / TILE;
    unsigned int s = 0;
    for (long long i = t * TILE + (threadIdx.x & 31); i <= q; i += 32) s += lab[i];
    s = __reduce_add_sync(0xffffffffu, s);
    return (long long)texcl[t] + s;
}

// compute_accuracy_rates at the host's sample indices: IEEE float64 divisions of exact
// integer counts; a class that is absent gives 0 / 0 = NaN as numpy does
__global__ void __launch_bounds__(AT)
k_acc_rates(const unsigned char *lab, const unsigned long long *texcl, long long n_tiles, long long n,
            const long long *ridx, const long long *pidx, long long n_points, double *tp, double *fp, double *prec)
{
    const long long j = ((long long)blockIdx.x * AT + threadIdx.x) >> 5;
    if (j >= 2 * n_points) return;
    const long long tp_tot = (long long)texcl[n_tiles], fp_tot = n - tp_tot;
    if (j < n_points) {
        const long long q = ridx[j];
        const long long c = tp_at(lab, texcl, q);
        if ((threadIdx.x & 31) == 0) {
            tp[j] = (double)c / (double)tp_tot;
            fp[j] = (double)(q + 1 - c) / (double)fp_tot;
        }
    } else {
        const long long q = pidx[j - n_points];
        const long long c = tp_at(lab, texcl, q);
        if ((threadIdx.x & 31) == 0) prec[j - n_points] = (double)c / (double)(q + 1);
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
// grow a slot to hold `need` entries, keeping its first s.n
int slot_reserve(tb2_ctx *ctx, Slot &s, long long need)
{
    if ((size_t)need * 8 + 8 <= s.stat.cap && (size_t)need + 8 <= s.lab.cap) return TB2_OK;
    DevBuf st, lb;
    const size_t want = (size_t)need + (size_t)need / 2;
    TB2_RESERVE(ctx, "accuracy", st, want * 8 + 8);
    TB2_RESERVE(ctx, "accuracy", lb, want + 8);
    if (s.n) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(st.p, s.stat.p, (size_t)s.n * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(lb.p, s.lab.p, (size_t)s.n, cudaMemcpyDeviceToDevice, ctx->stream));
        TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    }
    std::swap(s.stat.p, st.p); std::swap(s.stat.cap, st.cap);
    std::swap(s.lab.p, lb.p); std::swap(s.lab.cap, lb.cap);
    return TB2_OK;
}

template <class T> int acc_upload(tb2_ctx *ctx, DevBuf &b, const T *host, long long n)
{
    TB2_RESERVE(ctx, "accuracy", b, (size_t)n * sizeof(T) + 8);
    if (n) TB2_CUDA_TRY(ctx, cudaMemcpyAsync(b.p, host, (size_t)n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return TB2_OK;
}

bool motif_ok(const tb2_motif &m)
{
    if (m.len < 1 || m.len > 32 || m.mod_pos < 1 || m.mod_pos > m.len) return false;
    for (int j = 0; j < m.len; ++j)
        if (m.mask[j] == 0 || m.mask[j] > 15) return false;
    const unsigned char mb = m.mask[m.mod_pos - 1];
    return mb == 1 || mb == 2 || mb == 4 || mb == 8;      // a single base (TomboMotif)
}

unsigned char comp_bits(unsigned char x)
{
    return (unsigned char)(((x & 1) << 3) | ((x & 2) << 1) | ((x & 4) >> 1) | ((x & 8) >> 3));
}

void set_motifs(AccArgs &a, int n_motifs, const tb2_motif *motifs)
{
    a.n_motifs = n_motifs;
    for (int m = 0; m < n_motifs; ++m) {
        const tb2_motif &t = motifs[m];
        MotifDev &f = a.fw[m], &r = a.rc[m];
        memset(&f, 0, sizeof(f));
        memset(&r, 0, sizeof(r));
        f.len = r.len = t.len;
        f.mod_pos = r.mod_pos = t.mod_pos;
        for (int j = 0; j < t.len; ++j) {
            f.mask[j] = t.mask[j];
            r.mask[j] = comp_bits(t.mask[t.len - 1 - j]);
        }
        f.overlap = motif_can_overlap(f.mask, f.len);
        r.overlap = motif_can_overlap(r.mask, r.len);
        const unsigned char mb = t.mask[t.mod_pos - 1];
        a.mod_base[m] = (unsigned char)(mb == 1 ? 0 : mb == 2 ? 1 : mb == 4 ? 2 : 3);
    }
}

int check_blocks(long long n_blocks, const tb2_acc_block *blk, long long n_seq, long long n_stat, long long n_ctrl,
                 long long n_mod, long long n_unmod)
{
    if (n_blocks < 0 || n_blocks > INT32_MAX || (n_blocks > 0 && !blk)) return TB2_ERR_INVALID_ARG;
    for (long long b = 0; b < n_blocks; ++b) {
        const tb2_acc_block &B = blk[b];
        if (B.strand != 0 && B.strand != 1) return TB2_ERR_INVALID_ARG;
        if (B.seq_off < 0 || B.seq_len < 0 || B.seq_off > n_seq - B.seq_len || B.seq_start < 0) return TB2_ERR_INVALID_ARG;
        if (B.stat_off < 0 || B.n_stat < 0 || B.stat_off > n_stat - B.n_stat) return TB2_ERR_INVALID_ARG;
        if (B.ctrl_off < 0 || B.n_ctrl < 0 || B.ctrl_off > n_ctrl - B.n_ctrl) return TB2_ERR_INVALID_ARG;
        if (B.mod_off < 0 || B.n_mod < 0 || B.mod_off > n_mod - B.n_mod) return TB2_ERR_INVALID_ARG;
        if (B.unmod_off < 0 || B.n_unmod < 0 || B.unmod_off > n_unmod - B.n_unmod) return TB2_ERR_INVALID_ARG;
    }
    return TB2_OK;
}

// the shared tail of the three labelling calls: count, per-slot offsets, ordered scatter
template <int MODE>
int label(tb2_ctx *ctx, AccArgs &a, long long n_blocks, const int32_t *slot_of, int64_t *counts_out)
{
    AccuracyState &S = tb2_state(ctx->accuracy);
    DevBuf *P = S.buf;
    cudaStream_t q = ctx->stream;
    const int nm = MODE == MODE_TRUTH ? 1 : a.n_motifs;
    std::vector<long long> cnt((size_t)n_blocks * nm);
    TB2_RESERVE(ctx, "accuracy", P[A_CNT], cnt.size() * 8 + 16);
    int *fail = (int *)(P[A_CNT].as<long long>() + cnt.size());
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));          // kernel time: tb2_last_timing
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(fail, 0, 4, q));
    if (MODE == MODE_CTRL && n_blocks && a.n_seq) {
        TB2_RESERVE(ctx, "accuracy", P[A_SITE], (size_t)nm * a.n_seq);
        TB2_CUDA_TRY(ctx, cudaMemsetAsync(P[A_SITE].p, 0, (size_t)nm * a.n_seq, q));
        a.site = P[A_SITE].as<unsigned char>();
        k_acc_sites<<<dim3((unsigned)n_blocks, (unsigned)nm), AT, 0, q>>>(a, P[A_SITE].as<unsigned char>());
        TB2_CHECK_LAUNCH(ctx);
    }
    int h_fail = 0;
    if (n_blocks) {
        k_acc_count<MODE><<<(unsigned)n_blocks, AT, 0, q>>>(a, P[A_CNT].as<long long>(), fail);
        TB2_CHECK_LAUNCH(ctx);
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cnt.data(), P[A_CNT].p, cnt.size() * 8, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(&h_fail, fail, 4, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    }
    if (h_fail) {
        ctx->err = "string index out of range";
        return TB2_ERR_UNEXPECTED;
    }
    // per slot: block offsets after the slot's current entries
    int slots[MAXM];
    int n_slots = 0;
    for (int m = 0; m < nm; ++m) {
        bool seen = false;
        for (int k = 0; k < n_slots; ++k) seen = seen || slots[k] == slot_of[m];
        if (!seen) slots[n_slots++] = slot_of[m];
    }
    std::vector<long long> off((size_t)n_slots * (n_blocks + 1));
    for (int k = 0; k < n_slots; ++k) {
        long long o = S.slot[slots[k]].n;
        for (long long b = 0; b < n_blocks; ++b) {
            off[(size_t)k * (n_blocks + 1) + b] = o;
            for (int m = 0; m < nm; ++m)
                if (slot_of[m] == slots[k]) o += cnt[(size_t)b * nm + m];
        }
        off[(size_t)k * (n_blocks + 1) + n_blocks] = o;
        int rc = slot_reserve(ctx, S.slot[slots[k]], o);
        if (rc) return rc;
    }
    int rc = acc_upload(ctx, P[A_OFF], off.data(), (long long)off.size());
    if (rc) return rc;
    for (int k = 0; k < n_slots && n_blocks; ++k) {
        unsigned int mask = 0;
        for (int m = 0; m < nm; ++m)
            if (slot_of[m] == slots[k]) mask |= 1u << m;
        Slot &s = S.slot[slots[k]];
        k_acc_scatter<MODE><<<(unsigned)n_blocks, AT, 0, q>>>(
            a, mask, P[A_OFF].as<long long>() + (size_t)k * (n_blocks + 1), s.stat.as<double>(),
            s.lab.as<unsigned char>());
        TB2_CHECK_LAUNCH(ctx);
    }
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    for (int k = 0; k < n_slots; ++k) S.slot[slots[k]].n = off[(size_t)k * (n_blocks + 1) + n_blocks];
    if (counts_out) memcpy(counts_out, cnt.data(), cnt.size() * 8);
    return TB2_OK;
}

int check_slots(int n, const int32_t *slot)
{
    if (!slot) return TB2_ERR_INVALID_ARG;
    for (int m = 0; m < n; ++m)
        if (slot[m] < 0 || slot[m] >= MAXSLOT) return TB2_ERR_INVALID_ARG;
    return TB2_OK;
}

int upload_common(tb2_ctx *ctx, AccArgs &a, long long n_blocks, const tb2_acc_block *blk, long long n_seq,
                  const uint8_t *seq, long long n_stat, const uint32_t *pos, const double *stat)
{
    DevBuf *P = tb2_state(ctx->accuracy).buf;
    int rc;
    if ((rc = acc_upload(ctx, P[A_BLK], blk, n_blocks))) return rc;
    if ((rc = acc_upload(ctx, P[A_SEQ], seq, n_seq))) return rc;
    if ((rc = acc_upload(ctx, P[A_POS], pos, n_stat))) return rc;
    if ((rc = acc_upload(ctx, P[A_STAT], stat, n_stat))) return rc;
    memset(&a, 0, sizeof(a));
    a.blk = P[A_BLK].as<tb2_acc_block>();
    a.seq = P[A_SEQ].as<unsigned char>();
    a.pos = P[A_POS].as<unsigned int>();
    a.stat = P[A_STAT].as<double>();
    a.n_seq = n_seq;
    return TB2_OK;
}

// ordered labels in P[lab_buf] (n entries) -> the sampled rates
int rates(tb2_ctx *ctx, const unsigned char *lab, long long n, long long n_points, const int64_t *ridx,
          const int64_t *pidx, double *tp, double *fp, double *prec)
{
    DevBuf *P = tb2_state(ctx->accuracy).buf;
    cudaStream_t q = ctx->stream;
    const long long n_tiles = (n + TILE - 1) / TILE;
    int rc;
    TB2_RESERVE(ctx, "accuracy", P[A_GHIST], (size_t)(n_tiles + 1) * 8);
    TB2_RESERVE(ctx, "accuracy", P[A_IDX], (size_t)2 * n_points * 8 + 8);
    TB2_RESERVE(ctx, "accuracy", P[A_OUT], (size_t)3 * n_points * 8 + 8);
    unsigned long long *tsum = P[A_GHIST].as<unsigned long long>();
    long long *idx = P[A_IDX].as<long long>();
    double *out = P[A_OUT].as<double>();
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(idx, ridx, (size_t)n_points * 8, cudaMemcpyHostToDevice, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(idx + n_points, pidx, (size_t)n_points * 8, cudaMemcpyHostToDevice, q));
    k_acc_lab_tiles<<<(unsigned)n_tiles, AT, 0, q>>>(lab, n, tsum);
    TB2_CHECK_LAUNCH(ctx);
    k_scan_offsets<<<1, 1024, 0, q>>>(tsum, (long long *)tsum, n_tiles);   // in place
    TB2_CHECK_LAUNCH(ctx);
    const long long threads = 2 * n_points * 32;
    k_acc_rates<<<(unsigned)((threads + AT - 1) / AT), AT, 0, q>>>(lab, tsum, n_tiles, n, idx, idx + n_points,
                                                                 n_points, out, out + n_points, out + 2 * n_points);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(tp, out, (size_t)n_points * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(fp, out + n_points, (size_t)n_points * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(prec, out + 2 * n_points, (size_t)n_points * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}

int check_points(long long n, long long n_points, const int64_t *ridx, const int64_t *pidx, const double *tp,
                 const double *fp, const double *prec)
{
    if (n_points < 1 || n_points > (1LL << 24) || !ridx || !pidx || !tp || !fp || !prec) return TB2_ERR_INVALID_ARG;
    for (long long j = 0; j < n_points; ++j)
        if (ridx[j] < 0 || ridx[j] >= n || pidx[j] < 0 || pidx[j] >= n) return TB2_ERR_INVALID_ARG;
    return TB2_OK;
}

}  // namespace

extern "C" int tb2_accuracy_reset(tb2_ctx *ctx)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    AccuracyState &S = tb2_state(ctx->accuracy);
    for (int k = 0; k < MAXSLOT; ++k) S.slot[k].n = 0;
    return TB2_OK;
}

extern "C" int tb2_accuracy_count(tb2_ctx *ctx, int slot, int64_t *n_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (slot < 0 || slot >= MAXSLOT || !n_out) return TB2_ERR_INVALID_ARG;
    *n_out = tb2_state(ctx->accuracy).slot[slot].n;
    return TB2_OK;
}

extern "C" int tb2_accuracy_download(tb2_ctx *ctx, int slot, double *stat_out, uint8_t *label_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (slot < 0 || slot >= MAXSLOT || !stat_out || !label_out) return TB2_ERR_INVALID_ARG;
    Slot &s = tb2_state(ctx->accuracy).slot[slot];
    if (s.n) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(stat_out, s.stat.p, (size_t)s.n * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(label_out, s.lab.p, (size_t)s.n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return TB2_OK;
}

extern "C" int tb2_accuracy_load(tb2_ctx *ctx, int slot, int64_t n, const double *stat, const uint8_t *label)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (slot < 0 || slot >= MAXSLOT || n < 0 || (n > 0 && (!stat || !label))) return TB2_ERR_INVALID_ARG;
    for (int64_t i = 0; i < n; ++i)
        if (label[i] > 1) return TB2_ERR_INVALID_ARG;
    Slot &s = tb2_state(ctx->accuracy).slot[slot];
    s.n = 0;
    if ((rc = slot_reserve(ctx, s, n))) return rc;
    if (n) {
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(s.stat.p, stat, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(s.lab.p, label, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        TB2_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    }
    s.n = n;
    return TB2_OK;
}

extern "C" int tb2_accuracy_label_motif(tb2_ctx *ctx, int64_t n_blocks, const int64_t *block_rows, int64_t n_seq,
                                        const uint8_t *seq, int64_t n_stat, const uint32_t *pos, const double *stat,
                                        int n_motifs, const tb2_motif *motifs, const int32_t *slot, int64_t bb,
                                        int64_t ab, int64_t *counts_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    const tb2_acc_block *blocks = (const tb2_acc_block *)block_rows;
    if (n_motifs < 1 || n_motifs > MAXM || !motifs || n_seq < 0 || n_stat < 0 ||
        (n_seq > 0 && !seq) || (n_stat > 0 && (!pos || !stat)) || bb < 0 || ab < 0 || !counts_out)
        return TB2_ERR_INVALID_ARG;
    if ((rc = check_slots(n_motifs, slot))) return rc;
    long long mbb = 0, mab = 0;
    for (int m = 0; m < n_motifs; ++m) {
        if (!motif_ok(motifs[m])) return TB2_ERR_INVALID_ARG;
        mbb = std::max<long long>(mbb, motifs[m].mod_pos - 1);
        mab = std::max<long long>(mab, motifs[m].len - motifs[m].mod_pos);
    }
    if (bb != mbb || ab != mab) return TB2_ERR_INVALID_ARG;
    if ((rc = check_blocks(n_blocks, blocks, n_seq, n_stat, 0, 0, 0))) return rc;
    AccArgs a;
    if ((rc = upload_common(ctx, a, n_blocks, blocks, n_seq, seq, n_stat, pos, stat))) return rc;
    set_motifs(a, n_motifs, motifs);
    a.bb = bb; a.ab = ab;
    return label<MODE_MOTIF>(ctx, a, n_blocks, slot, counts_out);
}

extern "C" int tb2_accuracy_label_truth(tb2_ctx *ctx, int64_t n_blocks, const int64_t *block_rows, int64_t n_stat,
                                        const uint32_t *pos, const double *stat, int64_t n_mod,
                                        const int64_t *mod_locs, int64_t n_unmod, const int64_t *unmod_locs,
                                        int slot, int64_t *counts_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    const tb2_acc_block *blocks = (const tb2_acc_block *)block_rows;
    if (n_stat < 0 || (n_stat > 0 && (!pos || !stat)) || n_mod < 0 || n_unmod < 0 ||
        (n_mod > 0 && !mod_locs) || (n_unmod > 0 && !unmod_locs) || !counts_out)
        return TB2_ERR_INVALID_ARG;
    const int32_t slots[1] = {slot};
    if ((rc = check_slots(1, slots))) return rc;
    if ((rc = check_blocks(n_blocks, blocks, 0, n_stat, 0, n_mod, n_unmod))) return rc;
    // each block's ranges are sorted and unique: the binary search relies on it
    for (int64_t b = 0; b < n_blocks; ++b) {
        for (int64_t i = blocks[b].mod_off + 1; i < blocks[b].mod_off + blocks[b].n_mod; ++i)
            if (mod_locs[i] <= mod_locs[i - 1]) return TB2_ERR_INVALID_ARG;
        for (int64_t i = blocks[b].unmod_off + 1; i < blocks[b].unmod_off + blocks[b].n_unmod; ++i)
            if (unmod_locs[i] <= unmod_locs[i - 1]) return TB2_ERR_INVALID_ARG;
    }
    AccArgs a;
    if ((rc = upload_common(ctx, a, n_blocks, blocks, 0, nullptr, n_stat, pos, stat))) return rc;
    DevBuf *P = tb2_state(ctx->accuracy).buf;
    if ((rc = acc_upload(ctx, P[A_MOD], mod_locs, n_mod))) return rc;
    if ((rc = acc_upload(ctx, P[A_UNMOD], unmod_locs, n_unmod))) return rc;
    a.mod = P[A_MOD].as<long long>();
    a.unmod = P[A_UNMOD].as<long long>();
    a.n_motifs = 1;
    return label<MODE_TRUTH>(ctx, a, n_blocks, slots, counts_out);
}

extern "C" int tb2_accuracy_label_ctrl(tb2_ctx *ctx, int64_t n_blocks, const int64_t *block_rows, int64_t n_seq,
                                       const uint8_t *seq, int64_t n_stat, const uint32_t *pos, const double *stat,
                                       int64_t n_ctrl, const uint32_t *ctrl_pos, const double *ctrl_stat,
                                       int n_motifs, const tb2_motif *motifs, const int32_t *slot,
                                       int64_t *counts_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    const tb2_acc_block *blocks = (const tb2_acc_block *)block_rows;
    if (n_motifs < 1 || n_motifs > MAXM || !motifs || n_seq < 0 || n_stat < 0 || n_ctrl < 0 ||
        (n_seq > 0 && !seq) || (n_stat > 0 && (!pos || !stat)) || (n_ctrl > 0 && (!ctrl_pos || !ctrl_stat)) ||
        !counts_out)
        return TB2_ERR_INVALID_ARG;
    if ((rc = check_slots(n_motifs, slot))) return rc;
    for (int m = 0; m < n_motifs; ++m)
        if (!motif_ok(motifs[m])) return TB2_ERR_INVALID_ARG;
    if ((rc = check_blocks(n_blocks, blocks, n_seq, n_stat, n_ctrl, 0, 0))) return rc;
    AccArgs a;
    if ((rc = upload_common(ctx, a, n_blocks, blocks, n_seq, seq, n_stat, pos, stat))) return rc;
    DevBuf *P = tb2_state(ctx->accuracy).buf;
    if ((rc = acc_upload(ctx, P[A_CPOS], ctrl_pos, n_ctrl))) return rc;
    if ((rc = acc_upload(ctx, P[A_CSTAT], ctrl_stat, n_ctrl))) return rc;
    a.cpos = P[A_CPOS].as<unsigned int>();
    a.cstat = P[A_CSTAT].as<double>();
    set_motifs(a, n_motifs, motifs);
    return label<MODE_CTRL>(ctx, a, n_blocks, slot, counts_out);
}

extern "C" int tb2_accuracy_curve(tb2_ctx *ctx, int slot, int64_t n_points, const int64_t *rate_idx,
                                  const int64_t *prec_idx, double *tp_rate, double *fp_rate, double *precision)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (slot < 0 || slot >= MAXSLOT) return TB2_ERR_INVALID_ARG;
    AccuracyState &S = tb2_state(ctx->accuracy);
    Slot &s = S.slot[slot];
    const long long n = s.n;
    if (n < 1) return TB2_ERR_INVALID_ARG;
    if ((rc = check_points(n, n_points, rate_idx, prec_idx, tp_rate, fp_rate, precision))) return rc;
    DevBuf *P = S.buf;
    cudaStream_t q = ctx->stream;
    const long long n_tiles = (n + TILE - 1) / TILE;
    TB2_RESERVE(ctx, "accuracy", P[A_KEY0], (size_t)n * 8);
    TB2_RESERVE(ctx, "accuracy", P[A_KEY1], (size_t)n * 8);
    TB2_RESERVE(ctx, "accuracy", P[A_LAB0], (size_t)n);
    TB2_RESERVE(ctx, "accuracy", P[A_LAB1], (size_t)n);
    TB2_RESERVE(ctx, "accuracy", P[A_THIST], (size_t)256 * n_tiles * 4);
    TB2_RESERVE(ctx, "accuracy", P[A_TOFF], (size_t)256 * n_tiles * 8);
    TB2_RESERVE(ctx, "accuracy", P[A_CNT], (size_t)9 * 256 * 8 + 8);
    unsigned long long *gh = P[A_CNT].as<unsigned long long>();
    int *nan_flag = (int *)(gh + 9 * 256);
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));          // kernel time: tb2_last_timing
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(gh, 0, (size_t)9 * 256 * 8 + 8, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(P[A_LAB0].p, s.lab.p, (size_t)n, cudaMemcpyDeviceToDevice, q));
    const unsigned grid = (unsigned)std::min<long long>((n + AT - 1) / AT, 4LL * ctx->sm_count);
    k_acc_keys<<<grid, AT, 0, q>>>(s.stat.as<double>(), n, P[A_KEY0].as<unsigned long long>(), gh, nan_flag);
    TB2_CHECK_LAUNCH(ctx);
    k_acc_label_hist<<<grid, AT, 0, q>>>(s.lab.as<unsigned char>(), n, gh);
    TB2_CHECK_LAUNCH(ctx);
    std::vector<unsigned long long> h(9 * 256 + 1);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(h.data(), gh, h.size() * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    if (((const int *)(h.data() + 9 * 256))[0]) {
        ctx->err = "NaN statistic";
        return TB2_ERR_INVALID_ARG;
    }
    h[8 * 256] = (unsigned long long)n - h[8 * 256 + 1];      // False count
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(gh + 8 * 256, h.data() + 8 * 256, 8, cudaMemcpyHostToDevice, q));
    // the label first (False before True among equal keys), then the key digits upward
    const int order[9] = {8, 0, 1, 2, 3, 4, 5, 6, 7};
    int cur = 0;
    for (int pi = 0; pi < 9; ++pi) {
        const int d = order[pi];
        const unsigned long long *ph = h.data() + d * 256;
        bool single = false;
        for (int v = 0; v < 256 && !single; ++v) single = ph[v] == (unsigned long long)n;
        if (single) continue;
        const int shift = d == 8 ? 64 : 8 * d;
        unsigned long long *kin = P[A_KEY0 + cur].as<unsigned long long>();
        unsigned long long *kout = P[A_KEY1 - cur].as<unsigned long long>();
        unsigned char *lin = P[A_LAB0 + cur].as<unsigned char>(), *lout = P[A_LAB1 - cur].as<unsigned char>();
        k_radix_tile_hist<<<(unsigned)n_tiles, AT, 0, q>>>(kin, lin, n, shift, P[A_THIST].as<unsigned int>(), n_tiles);
        TB2_CHECK_LAUNCH(ctx);
        k_radix_tile_scan<<<256, AT, 0, q>>>(P[A_THIST].as<unsigned int>(), n_tiles, gh + d * 256,
                                           P[A_TOFF].as<unsigned long long>());
        TB2_CHECK_LAUNCH(ctx);
        k_radix_scatter_pass<<<(unsigned)n_tiles, AT, 0, q>>>(kin, lin, kout, lout, n, shift,
                                                            P[A_TOFF].as<unsigned long long>(), n_tiles);
        TB2_CHECK_LAUNCH(ctx);
        cur ^= 1;
    }
    return rates(ctx, P[A_LAB0 + cur].as<unsigned char>(), n, n_points, rate_idx, prec_idx, tp_rate, fp_rate,
                 precision);
}

extern "C" int tb2_accuracy_rates_ordered(tb2_ctx *ctx, int64_t n, const uint8_t *labels, int64_t n_points,
                                          const int64_t *rate_idx, const int64_t *prec_idx, double *tp_rate,
                                          double *fp_rate, double *precision)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n < 1 || !labels) return TB2_ERR_INVALID_ARG;
    if ((rc = check_points(n, n_points, rate_idx, prec_idx, tp_rate, fp_rate, precision))) return rc;
    for (int64_t i = 0; i < n; ++i)
        if (labels[i] > 1) return TB2_ERR_INVALID_ARG;
    DevBuf *P = tb2_state(ctx->accuracy).buf;
    if ((rc = acc_upload(ctx, P[A_LAB0], labels, n))) return rc;
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    return rates(ctx, P[A_LAB0].as<unsigned char>(), n, n_points, rate_idx, prec_idx, tp_rate, fp_rate, precision);
}
