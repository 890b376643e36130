// motif_llr.cuh -- device code of the per-read alternative-model LLRs
// (compute_alt_model_read_stats tombo_stats.py:3972-4082 with trim_seq_and_means :3888-3970):
// the per-site score shared by every LLR kernel, and the motif site finder for motif models
// (TomboMotif tombo_helper.py:542-640), both strands and region clipping.  Included by
// llr.cu and, for the host emulation, by tests/emul/emul_motif.cpp.
#pragma once

struct LlrArgs {
    int n_reads, K, cpos, alt_code, use_std;
    double sf, hf, hp;
    const double *norm_mean;
    const long long *mean_off, *seq_off, *read_start;
    const unsigned char *seq;
    const double *kmeans, *ksds, *alt;   // alt[code * K + pos]
    const int *status;                   // resident batch: reads that failed hold no sites
    int status_stride;
};

__device__ __forceinline__ int kmer_code(const unsigned char *bases, int K)
{
    int c = 0;
    for (int j = 0; j < K; ++j) c = c * 4 + (bases[j] & 3);
    return c;
}

// LLR of the site at alt_pos = i: k-mers i .. i+K-1 of `bases` (the trimmed read sequence)
// and levels means[cpos + i + t], alternative level of k-mer t at position K - 1 - t,
// const_var = sd(k-mer i)^2; c_calc_llh_ratio_const_var (_c_helper.pyx:298-311) with
// use_std, else c_calc_scaled_llh_ratio_const_var (:313-358), in their operation order
__device__ __forceinline__ double llr_site(const LlrArgs &a, const unsigned char *bases,
                                           const double *means, int i)
{
    const int K = a.K;
    const double const_var = a.ksds[kmer_code(bases + i, K)];
    const double cv = const_var * const_var;                 // np.square(r_ref_sds)[alt_pos]
    double acc = 0.0;
    for (int t = 0; t < K; ++t) {
        const int code = kmer_code(bases + i + t, K);
        const double obs = means[a.cpos + i + t];
        const double ref_mean = a.kmeans[code];
        const double alt_mean = a.alt[(size_t)code * K + (K - 1 - t)];
        if (a.use_std) {
            const double rd = obs - ref_mean, ad = obs - alt_mean;
            acc += ((ad * ad) - (rd * rd)) / cv;
        } else {
            if (ref_mean == alt_mean) continue;
            const double scale_mean = (alt_mean + ref_mean) / 2;
            const double ref_diff = obs - ref_mean, alt_diff = obs - alt_mean;
            const double scale_diff = obs - scale_mean;
            double means_diff = alt_mean - ref_mean;
            if (means_diff < 0) means_diff = means_diff * -1;
            acc += exp(-(scale_diff * scale_diff) / (a.sf * cv)) *
                   ((alt_diff * alt_diff) - (ref_diff * ref_diff)) /
                   (cv * pow(means_diff, a.hp) * a.hf);
        }
    }
    return acc;
}

// ---------------------------------------------------------------------------
// motif models
// ---------------------------------------------------------------------------
// tb2_motif on the device; `overlap`: two matches can lie closer than len (decided on the
// host by motif_can_overlap), so matches are chosen left to right like re.finditer
struct MotifDev {
    int len, mod_pos, overlap;
    unsigned char mask[32];               // IUPAC bit sets, A = 1, C = 2, G = 4, T = 8
};

// some shift 0 < s < len lets two matches overlap: every pair of aligned classes
// mask[j], mask[j - s] (s <= j < len) shares a base
__host__ __device__ inline bool motif_can_overlap(const unsigned char *mask, int len)
{
    for (int s = 1; s < len; ++s) {
        bool all = true;
        for (int j = s; j < len && all; ++j) all = (mask[j] & mask[j - s]) != 0;
        if (all) return true;
    }
    return false;
}

struct MotifArgs {
    LlrArgs s;
    MotifDev m;
    const signed char *strand;            // 0 '+', 1 '-', -1 skip
    long long max_ab;                     // over all alt models of the call
    long long reg_start, reg_end;
    int *read_status;                     // written by the count pass
};

// one read clipped to the region (trim_seq_and_means).  Candidate alt_pos = i (0 <= i <
// n_cand) has its motif at read bases s0 + i .. s0 + i + len - 1 and is scored on the read
// shifted by clip5; its genome position is g0 + i ('+') or g0 - i ('-').  Of the call's
// motif context only max_ab decides anything: max_bb pads the search string with 'N' where
// it reaches past the read, and 'N' never matches.
struct MotifRead {
    int status;                           // TB2_OK or TB2_ERR_READ_TOO_SHORT_IN_REGION
    int clip5, s0, n_cand;
    long long g0;
};

__host__ __device__ inline MotifRead motif_read(long long nb, int K, int cpos, long long r_start,
                                                int minus, long long reg_start, long long reg_end,
                                                int len, int mod_pos, long long max_ab)
{
    MotifRead g;
    g.status = TB2_OK; g.clip5 = 0; g.s0 = 0; g.n_cand = 0; g.g0 = 0;
    const long long flank = K - 1, r_end = r_start + nb;
    long long clip5 = 0, clip3 = 0;
    if (r_start + flank < reg_start) {
        (minus ? clip3 : clip5) = reg_start - (r_start + flank);
        r_start = reg_start - flank;
    }
    if (r_end - flank > reg_end) (minus ? clip5 : clip3) = r_end - flank - reg_end;
    // means[clip5 + cpos:][:-(clip3 + K - cpos - 1)]; a zero count empties the array
    const long long head = nb - clip5 - cpos > 0 ? nb - clip5 - cpos : 0;
    const long long tail = clip3 + K - cpos - 1;
    const long long n_means = (tail == 0 || head <= tail) ? 0 : head - tail;
    if (n_means < K) { g.status = TB2_ERR_READ_TOO_SHORT_IN_REGION; return g; }
    // n_means >= K bounds clip5 and clip3 by nb, so the rest fits an int
    const long long testable = n_means - K + 1;
    g.clip5 = (int)clip5;
    g.s0 = (int)(clip5 + K - mod_pos);
    g.g0 = minus ? r_start + flank + testable - 1 : r_start + flank;
    // motif_search_seq[:-(clip3 + K - 1 - max_ab)]: a zero count leaves no sites
    g.n_cand = (clip3 + flank - max_ab == 0) ? 0 : (int)testable;
    return g;
}

// the motif matches at trimmed-read base p (bases outside the read's nb bases are 'N',
// which no IUPAC class matches)
__device__ __forceinline__ bool motif_at(const MotifDev &m, const unsigned char *bases, int nb, int p)
{
    if (p < 0 || p + m.len > nb) return false;
    bool ok = true;
    for (int j = 0; j < m.len; ++j) ok = ok && (m.mask[j] & (1u << (bases[p + j] & 3)));
    return ok;
}

// one block (256 threads) per read.  FILL = false: counts[r] and read_status[r];
// FILL = true: llr_out / pos_out from site_off[r].  A motif that cannot overlap itself
// takes every candidate that matches (chunks per thread, block scan, as k_llr); one that can
// is resolved by warp 0 left to right, 32 candidates per ballot.
template <bool FILL>
__global__ void __launch_bounds__(256)
k_llr_motif(MotifArgs a, int *counts, const long long *site_off, double *llr_out, long long *pos_out)
{
    __shared__ unsigned int warp_tot[8];
    const int r = blockIdx.x, tid = threadIdx.x;
    const long long mo = a.s.mean_off[r];
    const int nb = (int)(a.s.mean_off[r + 1] - mo);
    const unsigned char *bases = a.s.seq + a.s.seq_off[r] + a.s.cpos;   // the read's nb bases
    const int strand = a.strand[r];
    int rs = TB2_OK;
    if (a.s.status && a.s.status[(size_t)r * a.s.status_stride] != TB2_OK)
        rs = a.s.status[(size_t)r * a.s.status_stride];
    MotifRead g;
    g.n_cand = 0;
    if (rs == TB2_OK && strand >= 0) {
        g = motif_read(nb, a.s.K, a.s.cpos, a.s.read_start[r], strand, a.reg_start, a.reg_end,
                       a.m.len, a.m.mod_pos, a.max_ab);
        rs = g.status;
    }
    if (!FILL && tid == 0) a.read_status[r] = rs;
    const int n = g.n_cand;
    if (n <= 0) { if (!FILL && tid == 0) counts[r] = 0; return; }
    const unsigned char *tb = bases + g.clip5;          // trimmed read: k-mers and levels
    const double *tm = a.s.norm_mean + mo + g.clip5;
    const long long step = strand ? -1 : 1;
    const int lane = tid & 31, warp = tid >> 5;
    if (!a.m.overlap) {
        const int per = (n + 255) / 256;
        const int i0 = min(n, tid * per), i1 = min(n, i0 + per);
        unsigned int mine = 0;
        for (int i = i0; i < i1; ++i) mine += motif_at(a.m, bases, nb, g.s0 + i);
        unsigned int inc = mine;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const unsigned int o = __shfl_up_sync(0xffffffffu, inc, off);
            if (lane >= off) inc += o;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        unsigned int before = 0, total = 0;
        for (int q = 0; q < 8; ++q) { if (q < warp) before += warp_tot[q]; total += warp_tot[q]; }
        if (!FILL) { if (tid == 0) counts[r] = (int)total; return; }
        long long o = site_off[r] + before + inc - mine;
        for (int i = i0; i < i1; ++i) {
            if (!motif_at(a.m, bases, nb, g.s0 + i)) continue;
            llr_out[o] = llr_site(a.s, tb, tm, i);
            pos_out[o] = g.g0 + step * i;
            ++o;
        }
        return;
    }
    // re.finditer: leftmost match, then the next one that starts at or after its end
    if (warp != 0) return;
    long long o = FILL ? site_off[r] : 0;
    int next = 0;                                        // first candidate still allowed
    unsigned int total = 0;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int i = c0 + lane;
        unsigned int m = __ballot_sync(0xffffffffu, i < n && motif_at(a.m, bases, nb, g.s0 + i));
        unsigned int acc = 0;
        while (m) {                                      // every lane walks the same bits
            const int b = __ffs(m) - 1;
            m &= m - 1;
            if (c0 + b < next) continue;
            acc |= 1u << b;
            next = c0 + b + a.m.len;
        }
        if (FILL && ((acc >> lane) & 1u)) {
            const long long w = o + __popc(acc & ((1u << lane) - 1u));
            llr_out[w] = llr_site(a.s, tb, tm, i);
            pos_out[w] = g.g0 + step * i;
        }
        o += __popc(acc);
        total += __popc(acc);
    }
    if (!FILL && lane == 0) counts[r] = (int)total;
}
