// stats_file.cuh -- device code of stats_file.cu (aggregation and most-significant table
// kernels) and the host-side decisions its entry points make: which radix digits a sort runs,
// when the table sorts, and how a row packs into words.  tests/emul runs the same source on
// the host.
#pragma once
#include "radix_sort.cuh"

namespace {

constexpr int AGG_NT = 1024;          // threads per aggregation block
constexpr int MAXW = 5;               // words of a model row

// a model row (kind 0): damp_frac, frac, pos << 32 | cov, control_cov << 32 | valid_cov,
// chrm << 8 | strand; a level row (kind 1): stat, pos << 32 | cov, control_cov << 32 | chrm,
// strand.  Words [0, nf) are float64 bits, compared through order_key.
inline void sf_pack_row(int kind, double key, double frac, uint32_t pos, uint32_t cov, uint32_t ctrl,
                        uint32_t valid, uint32_t chrm, uint8_t strand, unsigned long long *w, long long stride)
{
    unsigned long long kb, fb;
    memcpy(&kb, &key, 8);
    memcpy(&fb, &frac, 8);
    const unsigned long long pc = ((unsigned long long)pos << 32) | cov;
    if (kind == 0) {
        w[0] = kb; w[stride] = fb; w[2 * stride] = pc;
        w[3 * stride] = ((unsigned long long)ctrl << 32) | valid;
        w[4 * stride] = ((unsigned long long)chrm << 8) | strand;
    } else {
        w[0] = kb; w[stride] = pc;
        w[2 * stride] = ((unsigned long long)ctrl << 32) | chrm;
        w[3 * stride] = strand;
    }
}

// the table sorts before `add` more rows when they would pass max(2N, its capacity) and it
// holds more than it keeps
inline bool sf_reduce_before_add(long long held, long long add, long long cap, long long N)
{
    return held + add > (cap > 2 * N ? cap : 2 * N) && held > N;
}

// live[d]: digit d of word w takes more than one value over the n rows (hist: the digit
// histograms of k_sf_hist); returns whether any digit of the word is live
inline bool sf_live_digits(const unsigned long long *hist, long long n, int w, bool live[8])
{
    bool any = false;
    for (int d = 0; d < 8; ++d) {
        const unsigned long long *ph = hist + (size_t)(w * 8 + d) * 256;
        live[d] = true;
        for (int v = 0; v < 256; ++v) if (ph[v] == (unsigned long long)n) live[d] = false;
        any = any || live[d];
    }
    return any;
}

struct AggArgs {
    const tb2_sf_block *blk;
    const unsigned int *pos;
    const double *stat;
    long long R;                      // region_size
    double thresh, lower, unmod, mod; // lower NaN: None
    int llr;                          // stat_type: alternative-model LLRs
    int blk0;                         // first block of this launch
    const long long *ub;              // block b's rows go to [ub[b], ...) first
    int *gcnt;                        // global counters: 3 * R ints per block of the launch
    unsigned int *o_pos, *o_cov, *o_valid;
    double *o_damp, *o_frac;
    long long *n_rows;
    int *err;                         // a position outside [start, start + R)
};

// _agg_stats_worker + apply_per_read_thresh + calc_damp_fraction for one block per CTA.
// Unlike collate_reg_stats, a NaN statistic is kept: it counts in cov, and in valid_cov when
// neither lower_thresh nor the LLR filter applies (valid_cov = reg_cov, :4106), but never as
// >= thresh.
template <bool SMEM>
__global__ void __launch_bounds__(AGG_NT) k_sf_aggregate(AggArgs a)
{
    TB2_DYN_SMEM(int, sh_cnt);
    __shared__ int warp_tot[AGG_NT / 32];
    const int tid = threadIdx.x, b = a.blk0 + blockIdx.x;
    const tb2_sf_block B = a.blk[b];
    const long long R = a.R;
    int *cov = SMEM ? sh_cnt : a.gcnt + (size_t)blockIdx.x * 3 * R;
    int *val = cov + R, *ge = cov + 2 * R;
    for (long long i = tid; i < 3 * R; i += AGG_NT) cov[i] = 0;
    __syncthreads();
    for (long long i = tid; i < B.n_stat; i += AGG_NT) {
        const long long p = (long long)a.pos[B.stat_off + i] - B.start;
        if (p < 0 || p >= R) { *a.err = 1; continue; }
        const double s = a.stat[B.stat_off + i];
        atomicAdd(cov + p, 1);                                         // reg_cov
        bool valid = true;
        if (!isnan(a.lower)) valid = (s <= a.lower) || (s >= a.thresh);  // :4089-4097
        else if (a.llr) valid = fabs(s) >= a.thresh;                   // :4098-4104
        if (!valid) continue;
        atomicAdd(val + p, 1);
        if (s >= a.thresh) atomicAdd(ge + p, 1);
    }
    __syncthreads();
    const long long o0 = a.ub[b];
    int base = 0;
    for (long long c0 = 0; c0 < R; c0 += AGG_NT) {
        const long long p = c0 + tid;
        const int c = p < R ? cov[p] : 0;
        double frac = NAN, damp = NAN;
        int v = 0;
        if (c) {
            v = val[p];
            // np.greater_equal(...).sum() / base_stats.shape[0], NaN on empty (:4116-4120)
            frac = v > 0 ? (double)ge[p] / (double)v : NAN;
            // calc_damp_fraction :2545-2550: np.round = round half to even = rint
            damp = (rint(frac * (double)v) + a.unmod) / ((double)v + (a.unmod + a.mod));
        }
        const int keep = c > 0 && !isnan(damp);                        // :2760
        int total;
        const int o = base + tb2_block_excl_scan<AGG_NT>(keep, warp_tot, total);
        base += total;
        if (keep) {
            a.o_pos[o0 + o] = (unsigned int)(B.start + p);
            a.o_damp[o0 + o] = damp;
            a.o_frac[o0 + o] = frac;
            a.o_cov[o0 + o] = (unsigned int)c;
            a.o_valid[o0 + o] = (unsigned int)v;
        }
        __syncthreads();
    }
    if (tid == 0) a.n_rows[b] = base;
}

// block b's rows from its upper-bound slot to its place in the packed output
__global__ void __launch_bounds__(256)
k_sf_pack_rows(const long long *ub, const long long *off, const unsigned int *ipos, const double *idamp,
               const double *ifrac, const unsigned int *icov, const unsigned int *ivalid, unsigned int *opos,
               double *odamp, double *ofrac, unsigned int *ocov, unsigned int *ovalid)
{
    const int b = blockIdx.x;
    const long long s = ub[b], d = off[b], n = off[b + 1] - off[b];
    for (long long i = threadIdx.x; i < n; i += 256) {
        opos[d + i] = ipos[s + i];
        odamp[d + i] = idamp[s + i];
        ofrac[d + i] = ifrac[s + i];
        ocov[d + i] = icov[s + i];
        ovalid[d + i] = ivalid[s + i];
    }
}

// ---------------------------------------------------------------------------
// most-significant table
// ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long word_key(unsigned long long raw, bool is_float)
{
    return is_float ? order_key(__longlong_as_double((long long)raw)) : raw;
}

// histograms of all 8 digits of every word's key: hist[(w * 8 + d) * 256 + v]
__global__ void __launch_bounds__(256)
k_sf_hist(const unsigned long long *raw, long long cap, long long n, int K, int nf, unsigned long long *hist)
{
    __shared__ unsigned int h[MAXW * 8 * 256];
    for (int i = threadIdx.x; i < K * 8 * 256; i += 256) h[i] = 0;
    __syncthreads();
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        for (int w = 0; w < K; ++w) {
            const unsigned long long k = word_key(raw[(size_t)w * cap + i], w < nf);
#pragma unroll
            for (int d = 0; d < 8; ++d) atomicAdd(h + (w * 8 + d) * 256 + (int)((k >> (8 * d)) & 255u), 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K * 8 * 256; i += 256)
        if (h[i]) atomicAdd(hist + i, (unsigned long long)h[i]);
}

// the key of one word in the current order: idx null -> arrival order (and idx_out = identity)
__global__ void k_sf_word_keys(const unsigned long long *word, bool is_float, const unsigned int *idx, long long n,
                               unsigned long long *key, unsigned int *idx_out)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const long long j = idx ? idx[i] : i;
    key[i] = word_key(word[j], is_float);
    if (idx_out) idx_out[i] = (unsigned int)i;
}

// the first m rows in sorted order into `out` (idx null: arrival order)
__global__ void k_sf_gather(const unsigned long long *raw, unsigned long long *out, long long cap, int K,
                            const unsigned int *idx, long long m)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= m) return;
    const long long j = idx ? idx[i] : i;
    for (int w = 0; w < K; ++w) out[(size_t)w * cap + i] = raw[(size_t)w * cap + j];
}

// rows of the last aggregation into the table (model rows, control_cov 0), block order
__global__ void __launch_bounds__(256)
k_sf_table_from_agg(const tb2_sf_block *blk, const long long *off, const unsigned int *pos, const double *damp,
                    const double *frac, const unsigned int *cov, const unsigned int *valid,
                    unsigned long long *raw, long long cap, long long n0)
{
    const int b = blockIdx.x;
    const long long s = off[b], n = off[b + 1] - off[b];
    const unsigned long long cs = ((unsigned long long)(unsigned int)blk[b].chrm << 8) |
                                  (unsigned long long)(blk[b].strand & 255);
    for (long long i = threadIdx.x; i < n; i += 256) {
        const size_t r = (size_t)(n0 + s + i);
        raw[r] = (unsigned long long)__double_as_longlong(damp[s + i]);
        raw[cap + r] = (unsigned long long)__double_as_longlong(frac[s + i]);
        raw[2 * cap + r] = ((unsigned long long)pos[s + i] << 32) | cov[s + i];
        raw[3 * cap + r] = valid[s + i];
        raw[4 * cap + r] = cs;
    }
}

}  // namespace
