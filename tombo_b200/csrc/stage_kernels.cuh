// stage_kernels.cuh -- (device code; stage_kernels.cu holds the launch wrappers; tests/emul
// runs this file on the host)  the non-DP stages of resquiggle_read as batched kernels
// (sm_90a): signal conversion + k-mer lookup, normalisation, changepoint
// detection, event means, skipped-base raw-signal DP, base means, Theil-Sen
// rescaling, final scoring.  One CTA (or warp) per read; arithmetic follows the
// reference operation for operation (see DESIGN.md "Arithmetic contract").
#pragma once
#include "batch.h"
#include "select.cuh"

#define ST_THREADS TB2_SEL_THREADS

__device__ __forceinline__ bool rd_active(const ReadState &s) { return s.active && s.status == TB2_OK; }

// ===========================================================================
// prep: raw -> fp64 (reversed for RNA), k-mer level lookup, state init
// TomboModel.get_exp_levels_from_seq tombo_stats.py:834-862; RNA flip
// resquiggle.py:1516
// ===========================================================================
template <class T>
__global__ void __launch_bounds__(ST_THREADS)
k_prep(BatchView b, const T *raw, int is_rna, const double *kmeans, const double *ksds)
{
    const int r = blockIdx.x;
    const long long ro = b.raw_off[r];
    const int n = (int)(b.raw_off[r + 1] - ro);
    for (int i = threadIdx.x; i < n; i += ST_THREADS)
        b.rawf[ro + i] = (double)raw[ro + (is_rna ? n - 1 - i : i)];
    const long long so = b.seq_off[r], bo = b.base_off[r];
    const int nb = (int)(b.base_off[r + 1] - bo);
    const int K = b.kmer_width;
    int bad = 0;
    for (int i = threadIdx.x; i < nb; i += ST_THREADS) {
        int code = 0;
        for (int j = 0; j < K; ++j) {
            const int c = b.seq[so + i + j];
            if (c > 3) bad = 1;
            code = code * 4 + (c & 3);
        }
        b.rm[bo + i] = kmeans[code];
        b.rs[bo + i] = ksds[code];
    }
    const int any_bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) {
        ReadState s;
        memset(&s, 0, sizeof(s));
        s.status = TB2_OK;
        if (n <= 0) s.status = TB2_ERR_NO_RAW;
        if (nb <= 0 || (int)(b.seq_off[r + 1] - so) != nb + K - 1) s.status = TB2_ERR_DISCORDANT_LEN;
        if (any_bad) s.status = TB2_ERR_INVALID_SEQ;
        s.done = (s.status != TB2_OK);
        b.st[r] = s;
    }
}

// worker policy bookkeeping (resquiggle.py:1492-1504, 1578-1588)
__global__ void k_start_attempt(BatchView b, int attempt)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= b.n_reads) return;
    ReadState &s = b.st[r];
    if (s.done) { s.active = 0; return; }
    if (attempt == 0) {
        s.active = 1;
    } else {
        if (s.status == TB2_OK) { s.active = 0; s.done = 1; return; }  // defensive
        // capacity overruns are library limits, not read failures: never rescued
        if (s.status == TB2_ERR_CAPACITY) { s.active = 0; s.done = 1; return; }
        s.first_status = s.status;
        s.status = TB2_OK;
        s.active = 1;
    }
    s.attempt = attempt;
    s.n_iters = 0;
    s.use_sv = 0;
}

// compute_num_events (tombo_stats.py:1558-1574) + the signal/sequence guard of
// resquiggle_read (resquiggle.py:1154-1160)
__global__ void k_begin_call(BatchView b, tb2_params p, StagePolicy pol)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= b.n_reads) return;
    ReadState &s = b.st[r];
    if (!rd_active(s)) return;
    const int n = (int)(b.raw_off[r + 1] - b.raw_off[r]);
    const int nb = (int)(b.base_off[r + 1] - b.base_off[r]);
    const long long a = (long long)n / p.mean_obs_per_event;
    const long long c = (long long)((double)nb * pol.min_event_to_seq_ratio);
    const long long ne = a > c ? a : c;
    if ((double)ne / (double)p.bandwidth > (double)nb) { s.status = TB2_ERR_TOO_MUCH_SIGNAL; return; }
    if (ne > b.ev_off[r + 1] - b.ev_off[r] || ne < 2) { s.status = TB2_ERR_CAPACITY; return; }
    s.num_events = (int)ne;
}

__global__ void k_end_call(BatchView b, int max_iters)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= b.n_reads) return;
    ReadState &s = b.st[r];
    if (!s.active) return;
    s.calls += 1;
    if (s.status != TB2_OK) { s.active = 0; return; }  // attempt failed
    s.n_iters += 1;
    if (s.changed && s.n_iters < max_iters) { s.use_sv = 1; return; }  // iterate
    s.active = 0;
    s.done = 1;
}

__global__ void k_count_active(BatchView b, int *counters)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    int act = 0, fail = 0;
    if (r < b.n_reads) {
        act = b.st[r].active != 0;
        fail = (!b.st[r].done && b.st[r].status != TB2_OK);
    }
    act = __syncthreads_count(act);
    fail = __syncthreads_count(fail);
    if (threadIdx.x == 0) {
        if (act) atomicAdd(&counters[0], act);
        if (fail) atomicAdd(&counters[1], fail);
    }
}

// ===========================================================================
// normalize_raw_signal tombo_stats.py:482-573 (+ c_apply_outlier_thresh
// _c_helper.pyx:73-87)
// ===========================================================================
__global__ void __launch_bounds__(ST_THREADS)
k_normalize(BatchView b, StagePolicy pol, int first_call)
{
    __shared__ SelectSmem sm;
    const int r = b.order ? b.order[blockIdx.x] : blockIdx.x;
    ReadState &s = b.st[r];
    if (!rd_active(s)) return;
    const long long ro = b.raw_off[r];
    const int n = (int)(b.raw_off[r + 1] - ro);
    const double *raw = b.rawf + ro;
    double *norm = b.norm + ro;
    double shift, scale, lo = NAN, hi = NAN;
    const bool given = s.use_sv != 0;
    const bool use_const = first_call && !isnan(pol.const_scale);
    double mid_a = 0.0, mid_b = 0.0;     // the middle order statistic(s) of raw
    if (!given) {
        auto f_raw = [&](int i) { return raw[i]; };
        if (n & 1) {
            tb2_block_select2(f_raw, PredAll(), n, n / 2, false, &mid_a, &mid_b, sm);
            shift = mid_a;                                                            // :541/:545
        } else {
            tb2_block_select2(f_raw, PredAll(), n, n / 2 - 1, true, &mid_a, &mid_b, sm);
            shift = (mid_a + mid_b) / 2.0;
        }
        if (use_const) scale = pol.const_scale;                                       // :546
        else scale = tb2_block_median([&](int i) { return fabs(raw[i] - shift); }, n, sm);  // :542
    } else {
        shift = s.sv.shift; scale = s.sv.scale;
    }
    if (scale == 0.0 || isnan(scale)) {  // FloatingPointError under np.seterr(all='raise')
        if (threadIdx.x == 0) s.status = TB2_ERR_UNEXPECTED;
        return;
    }
    for (int i = threadIdx.x; i < n; i += ST_THREADS) norm[i] = (raw[i] - shift) / scale;  // :554
    __syncthreads();
    const double thresh = given ? NAN : pol.outlier_thresh;
    if (!isnan(thresh)) {                                                             // :559-563
        double med, mad;
        if ((n & 1) && !use_const) {
            // odd n: shift is an element of raw and scale an element of |raw - shift|.
            // x -> (x - shift) / scale is monotone (each rounding is), so the middle
            // order statistic of norm is the image of shift: (shift - shift) / scale = +0;
            // |norm - 0| = |x - shift| / scale is monotone in |x - shift|, so its middle
            // order statistic is scale / scale = 1 -- the values np.median returns.
            med = 0.0;
            mad = 1.0;
        } else {
            // even n: the two middle elements of norm are the images of raw's
            if (n & 1) med = tb2_block_median([&](int i) { return norm[i]; }, n, sm);
            else med = (((mid_a - shift) / scale) + ((mid_b - shift) / scale)) / 2.0;
            mad = tb2_block_median([&](int i) { return fabs(norm[i] - med); }, n, sm);
        }
        lo = med - (mad * thresh);
        hi = med + (mad * thresh);
    } else if (given) { lo = s.sv.lower_lim; hi = s.sv.upper_lim; }                   // :565-566
    if (!isnan(lo) && !isnan(hi)) {
        for (int i = threadIdx.x; i < n; i += ST_THREADS) {
            const double v = norm[i];
            norm[i] = v > hi ? hi : (v < lo ? lo : v);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        s.sv.shift = shift; s.sv.scale = scale; s.sv.lower_lim = lo; s.sv.upper_lim = hi;
        s.sv.outlier_thresh = thresh;
    }
}

// ===========================================================================
// changepoints: c_valid_cpts_w_cap / c_valid_cpts_w_cap_t_test
// (_c_helper.pyx:89-120 / 144-202) + sort (tombo_helper.py:76-91)
// + remove_stall_cpts (tombo_stats.py:1576-1597)
//
// The reference ranks all candidates (argsort, descending) and picks greedily
// with a +-(min_base_obs-1) exclusion zone until num_cpts are found.  Here the
// same set is obtained without a sort: a candidate is accepted iff every
// higher-ranked candidate inside its zone is rejected (iterated to the fixed
// point, which is the greedy result), then the num_cpts best accepted ones are
// kept via an exact radix select.  Rank order: score descending, ties -> larger
// position first (the pinned rule of SURVEY.md 8c-7).
// ===========================================================================
__device__ __forceinline__ bool cand_gt(double si, int i, double sk, int k)
{
    return si > sk || (si == sk && i > k);
}

// np.cumsum(concatenate([[0.0], signal])) (_c_helper.pyx:93-94): strictly sequential
// fp64 sums, one warp per read.  The warp stages 256 samples in shared memory
// (coalesced), then every lane carries the same running sum through them (broadcast
// reads issued ahead of the adds, so the serial chain is the add latency alone); lane
// k keeps the prefix sums of elements k, k + 32, ... for a coalesced store.
#define CS_WARPS 4
__global__ void __launch_bounds__(CS_WARPS * 32, 8)
k_cumsum(BatchView b, int on_raw)
{
    __shared__ double s_all[CS_WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = blockIdx.x * CS_WARPS + warp;
    if (r >= b.n_reads) return;
    if (!rd_active(b.st[r])) return;
    double *s_x = s_all[warp];
    const long long ro = b.raw_off[r];
    const int n = (int)(b.raw_off[r + 1] - ro);
    const double *sig = (on_raw ? b.rawf : b.norm) + ro;
    double *cs = b.cs + ro + r;
    double acc = 0.0;
    if (lane == 0) cs[0] = 0.0;
    for (int base = 0; base < n; base += 256) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int i = base + q * 32 + lane;
            s_x[q * 32 + lane] = (i < n) ? sig[i] : 0.0;
        }
        __syncwarp();
        double mine[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            double m_q = 0.0;
#pragma unroll
            for (int k = 0; k < 32; ++k) {
                acc = acc + s_x[q * 32 + k];
                if (lane == k) m_q = acc;
            }
            mine[q] = m_q;
        }
        __syncwarp();
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int i = base + q * 32 + lane;
            if (i < n) cs[i + 1] = mine[q];
        }
    }
}

// bit i of word w <-> candidate 32 w + i.  X(i + o) / X(i - o) as words aligned to i.
__device__ __forceinline__ uint32_t cp_shr(const uint32_t *x, int w, int nw, int o)
{
    const uint32_t hi = (w + 1 < nw) ? x[w + 1] : 0u;
    return (x[w] >> o) | (hi << (32 - o));
}
__device__ __forceinline__ uint32_t cp_shl(const uint32_t *x, int w, int o)
{
    const uint32_t lo = (w > 0) ? x[w - 1] : 0u;
    return (x[w] << o) | (lo >> (32 - o));
}

#define CP_MAX_OFF 12   // exclusion zones up to +-12 candidates run bit-parallel

__global__ void __launch_bounds__(ST_THREADS, 5)
k_cpts(BatchView b, tb2_params p, int on_raw, int smem_words)
{
    TB2_DYN_SMEM(uint32_t, cp_smem);
    __shared__ SelectSmem sm;
    __shared__ int s_pos;
    const int r = b.order ? b.order[blockIdx.x] : blockIdx.x;
    ReadState &s = b.st[r];
    if (!rd_active(s)) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long ro = b.raw_off[r];
    const int n = (int)(b.raw_off[r + 1] - ro);
    const double *sig = (on_raw ? b.rawf : b.norm) + ro;
    double *cs = b.cs + ro + r;
    double *sc = b.scores + ro;
    const int w = (int)p.running_stat_width, m = (int)p.min_obs_per_base;
    const int N = s.num_events;
    int n_cand, bound;
    if (!p.use_t_test_seg) {
        n_cand = n + 1 - 2 * w;
        bound = n_cand - 2 * w;  // num_cands = candidate_poss.shape[0] - 2*w (:105-106)
        if (n_cand <= 0) { if (tid == 0) s.status = TB2_ERR_UNEXPECTED; return; }
        // cs = np.cumsum(concatenate([[0.0], signal])) comes from k_cumsum
        for (int i = tid; i < n_cand; i += ST_THREADS)
            sc[i] = fabs(((2 * cs[i + w]) - cs[i]) - cs[i + 2 * w]);   // :95-98
    } else {
        n_cand = n - 2 * w;
        bound = n_cand;      // :199
        if (n_cand <= 0) { if (tid == 0) s.status = TB2_ERR_UNEXPECTED; return; }
        for (int pos = tid; pos < n_cand; pos += ST_THREADS) {           // :153-179
            double m1 = 0, m2 = 0, var1 = 0, var2 = 0, d;
            for (int k = 0; k < w; ++k) m1 += sig[pos + k];
            m1 /= (double)w;
            for (int k = 0; k < w; ++k) m2 += sig[pos + w + k];
            m2 /= (double)w;
            for (int k = 0; k < w; ++k) { d = sig[pos + k] - m1; var1 += d * d; }
            for (int k = 0; k < w; ++k) { d = sig[pos + w + k] - m2; var2 += d * d; }
            double t;
            if (var1 + var2 == 0) t = 0.0;
            else if (m1 > m2) t = (m1 - m2) / sqrt(var1 + var2);
            else t = (m2 - m1) / sqrt(var1 + var2);
            sc[pos] = t;
        }
    }
    if (N < 1 || N > n_cand) { if (tid == 0) s.status = (N < 1) ? TB2_ERR_UNEXPECTED : TB2_ERR_FEWER_CPTS; return; }
    __syncthreads();
    // ---- greedy exclusion as a fixed point, 32 candidates per word ----
    // A = accepted, D = decided, G_o bit i = "candidate i + o outranks candidate i".
    // A round accepts every undecided candidate whose zone holds no accepted and no
    // undecided higher-ranked candidate, and rejects those with an accepted one in
    // their zone (Jacobi sweep on double buffers: decisions are final and are exactly
    // the ranked greedy's, whatever the sweep order).
    const int nw = (n_cand + 31) >> 5;
    const int no = m - 1;                       // zone half-width
    uint32_t *bits;
    if ((4 + max(no, 0)) * nw <= smem_words) bits = cp_smem;
    else bits = reinterpret_cast<uint32_t *>(b.cstate + ((2 * ro + 128LL * r + 3) & ~3LL));
    if (no > CP_MAX_OFF) { if (tid == 0) s.status = TB2_ERR_CAPACITY; return; }
    uint32_t *A0 = bits, *A1 = bits + nw, *D0 = bits + 2 * nw, *D1 = bits + 3 * nw, *G = bits + 4 * nw;
    for (int wd = warp; wd < nw; wd += ST_THREADS / 32) {
        const int i = wd * 32 + lane;
        const bool valid = i < n_cand;
        const double si = valid ? sc[i] : 0.0;
        for (int o = 1; o <= no; ++o) {
            const bool gt = valid && (i + o < n_cand) && cand_gt(sc[i + o], i + o, si, i);
            const uint32_t g = __ballot_sync(TB2_FULL_MASK, gt);
            if (lane == 0) G[(o - 1) * nw + wd] = g;
        }
        const uint32_t inv = __ballot_sync(TB2_FULL_MASK, !valid);
        if (lane == 0) { A0[wd] = 0u; D0[wd] = inv; }
    }
    __syncthreads();
    uint32_t *Ac = A0, *An = A1, *Dc = D0, *Dn = D1;
    for (;;) {
        int undecided = 0;
        for (int wd = tid; wd < nw; wd += ST_THREADS) {
            const uint32_t a = Ac[wd], dd = Dc[wd];
            const uint32_t U = ~dd;
            uint32_t na = a, nd = dd;
            if (U != 0u) {
                uint32_t accnb = 0u, blocked = 0u;
                for (int o = 1; o <= no; ++o) {
                    const uint32_t *Go = G + (o - 1) * nw;
                    accnb |= cp_shr(Ac, wd, nw, o) | cp_shl(Ac, wd, o);
                    // undecided neighbours: bits of ~D, out-of-range words read as decided
                    const uint32_t d_hi = (wd + 1 < nw) ? Dc[wd + 1] : ~0u;
                    const uint32_t d_lo = (wd > 0) ? Dc[wd - 1] : ~0u;
                    const uint32_t u_up = ~((dd >> o) | (d_hi << (32 - o)));
                    const uint32_t u_dn = ~((dd << o) | (d_lo >> (32 - o)));
                    const uint32_t g_up = Go[wd];
                    const uint32_t g_dn = ~cp_shl(Go, wd, o);     // i - o outranks i
                    blocked |= (u_up & g_up) | (u_dn & g_dn);
                }
                const uint32_t rej = U & accnb;
                const uint32_t acc = U & ~accnb & ~blocked;
                na = a | acc;
                nd = dd | rej | acc;
                if (~nd != 0u) undecided = 1;
            }
            An[wd] = na; Dn[wd] = nd;
        }
        const int again = __syncthreads_or(undecided);
        uint32_t *tA = Ac; Ac = An; An = tA;
        uint32_t *tD = Dc; Dc = Dn; Dn = tD;
        if (!again) break;
    }
    const uint32_t *A = Ac;      // final accepted set
    uint32_t *K = An;            // scratch: kept set
    // ---- keep the N best accepted ----
    unsigned int acc_cnt = 0;
    for (int wd = tid; wd < nw; wd += ST_THREADS) acc_cnt += __popc(A[wd]);
    acc_cnt = tb2_block_sum(acc_cnt, sm);
    if ((int)acc_cnt < N) { if (tid == 0) s.status = TB2_ERR_FEWER_CPTS; return; }
    double vN, dummy;
    auto f_score = [&](int i) { return sc[i]; };
    auto p_acc = [&](int i) { return (A[i >> 5] >> (i & 31)) & 1u; };
    tb2_block_select2(f_score, p_acc, n_cand, (int)acc_cnt - N, false, &vN, &dummy, sm);
    if (tid == 0) s_pos = -1;
    __syncthreads();
    unsigned int g = 0, e = 0, higher = 0, eq_all = 0;
    for (int i = tid; i < n_cand; i += ST_THREADS) {
        const double v = sc[i];
        const bool acc = p_acc(i);
        higher += v > vN;
        if (v == vN) {
            ++eq_all;
            if (acc) { ++e; atomicMax(&s_pos, i); }
        }
        g += acc && v > vN;
    }
    g = tb2_block_sum(g, sm);
    e = tb2_block_sum(e, sm);
    eq_all = tb2_block_sum(eq_all, sm);
    higher = tb2_block_sum(higher, sm);
    const int need = N - (int)g;   // 1 <= need <= e, taken from the largest positions
    int posN;
    if (e == 1u) {
        posN = s_pos;              // the usual case: the N-th score is unique
    } else {
        auto f_pos = [&](int i) { return (double)i; };
        auto p_tie = [&](int i) { return p_acc(i) && sc[i] == vN; };
        double pv, pd;
        tb2_block_select2(f_pos, p_tie, n_cand, (int)e - need, false, &pv, &pd, sm);
        posN = (int)pv;
    }
    // rank index of the N-th pick in the full candidate order (:109-118)
    if (eq_all > 1u) {
        unsigned int h2 = 0;
        for (int i = tid; i < n_cand; i += ST_THREADS) h2 += (sc[i] == vN && i > posN);
        higher += tb2_block_sum(h2, sm);
    }
    if (N > 1 && (int)higher + 1 >= bound) { if (tid == 0) s.status = TB2_ERR_FEWER_CPTS; return; }
    // ---- ordered compaction (+ w), dropping changepoints inside stalls ----
    const int *si = b.stall_ints ? b.stall_ints + 2 * (size_t)b.stall_cap * r : nullptr;
    const int ns = b.stall_ints ? s.n_stalls : 0;
    for (int wd = warp; wd < nw; wd += ST_THREADS / 32) {
        const int i = wd * 32 + lane;
        bool keep = (A[wd] >> lane) & 1u;
        if (keep) {
            const double v = sc[i];
            keep = v > vN || (v == vN && i >= posN);
            const int c = i + w;
            for (int k = 0; keep && k < ns; ++k) if (si[2 * k] < c && c < si[2 * k + 1]) keep = false;
        }
        const uint32_t kw = __ballot_sync(TB2_FULL_MASK, keep);
        if (lane == 0) K[wd] = kw;
    }
    __syncthreads();
    const int per = (nw + ST_THREADS - 1) / ST_THREADS;
    const int w0 = min(nw, tid * per), w1 = min(nw, w0 + per);
    unsigned int mine = 0;
    for (int wd = w0; wd < w1; ++wd) mine += __popc(K[wd]);
    unsigned int inc = mine;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const unsigned int o = __shfl_up_sync(TB2_FULL_MASK, inc, off);
        if (lane >= off) inc += o;
    }
    if (lane == 31) sm.warp_tot[warp] = inc;
    __syncthreads();
    unsigned int base = 0, total = 0;
    for (int q = 0; q < ST_THREADS / 32; ++q) { if (q < warp) base += sm.warp_tot[q]; total += sm.warp_tot[q]; }
    unsigned int o = base + inc - mine;
    int *cp = b.cpts + b.ev_off[r];
    for (int wd = w0; wd < w1; ++wd) {
        uint32_t kw = K[wd];
        while (kw) {
            const int bit = __ffs(kw) - 1;
            kw &= kw - 1u;
            cp[o++] = wd * 32 + bit + w;
        }
    }
    if (tid == 0) s.n_cpts = (int)total;
}

// ===========================================================================
// c_new_means _c_helper.pyx:59-71 over the changepoints (event means)
// ===========================================================================
__global__ void __launch_bounds__(ST_THREADS) k_event_means(BatchView b)
{
    const int r = blockIdx.x;
    const ReadState &s = b.st[r];
    if (!rd_active(s)) return;
    const double *norm = b.norm + b.raw_off[r];
    const int *cp = b.cpts + b.ev_off[r];
    double *em = b.em + b.ev_off[r];
    const int ne = s.n_cpts - 1;
    if (ne < 1) { if (threadIdx.x == 0) b.st[r].status = TB2_ERR_UNEXPECTED; return; }
    for (int e = threadIdx.x; e < ne; e += ST_THREADS) {
        const int a = cp[e], z = cp[e + 1];
        double acc = 0;
        for (int k = a; k < z; ++k) acc += norm[k];
        em[e] = acc / (double)(z - a);
    }
}

// get_scale_values_from_events tombo_stats.py:217-233 (RNA, first call)
__global__ void __launch_bounds__(ST_THREADS) k_rna_scale(BatchView b, StagePolicy pol)
{
    __shared__ SelectSmem sm;
    const int r = blockIdx.x;
    ReadState &s = b.st[r];
    if (!rd_active(s) || s.use_sv == 1) return;
    // a caller-supplied const_scale wins over the event-based scaling: segment_signal
    // takes the 'median_const_scale' branch (resquiggle.py:1084-1087), k_normalize does it
    if (!isnan(pol.const_scale)) return;
    const double *raw = b.rawf + b.raw_off[r];
    const int *cp = b.cpts + b.ev_off[r];
    double *em = b.em + b.ev_off[r];
    int ne = 10000;                                         // RNA_SCALE_NUM_EVENTS
    if ((double)s.n_cpts * 0.75 < (double)ne) ne = (int)((double)s.n_cpts * 0.75);
    if (ne < 2) { if (threadIdx.x == 0) s.status = TB2_ERR_UNEXPECTED; return; }
    for (int e = threadIdx.x; e < ne - 1; e += ST_THREADS) {
        const int a = cp[e], z = cp[e + 1];
        double acc = 0;
        for (int k = a; k < z; ++k) acc += raw[k];
        em[e] = acc / (double)(z - a);
    }
    __syncthreads();
    const double med = tb2_block_median([&](int i) { return em[i]; }, ne - 1, sm);
    const double mad = tb2_block_median([&](int i) { return fabs(em[i] - med); }, ne - 1, sm);
    __syncthreads();
    if (threadIdx.x == 0) {
        s.sv.shift = med; s.sv.scale = mad;
        s.sv.lower_lim = -pol.outlier_thresh; s.sv.upper_lim = pol.outlier_thresh;
        s.sv.outlier_thresh = NAN;
        s.use_sv = 2;   // consumed by k_normalize of this call
    }
}

// ===========================================================================
// identify_stalls (mean-window method) tombo_stats.py:269-368,
// MEAN_STALL_PARAMS _default_parameters.py:93-97.  Once per read (RNA).
// ===========================================================================
__global__ void __launch_bounds__(ST_THREADS) k_stalls(BatchView b)
{
    const int r = blockIdx.x;
    ReadState &s = b.st[r];
    if (s.done) return;
    const int tid = threadIdx.x;
    const long long ro = b.raw_off[r];
    const int n = (int)(b.raw_off[r + 1] - ro);
    const double *raw = b.rawf + ro;
    double *cs = b.cs + ro + r;        // cumsum, then moving averages
    double *metric = b.scores + ro;    // diff sums
    volatile unsigned char *below = b.cstate + ro;
    const int window = 350, mini = 50, nwin = 7, min_consec = 200, edge = 100;
    const double thresh = 40;
    if (tid == 0) s.n_stalls = 0;
    if (n < window) return;
    if (tid < 32) {   // np.cumsum(all_raw_signal): sequential
        double acc = 0.0;
        for (int base = 0; base < n; base += 32) {
            const double x = (base + tid < n) ? raw[base + tid] : 0.0;
            double mine = 0.0;
#pragma unroll
            for (int k = 0; k < 32; ++k) {
                acc = (base + k == 0) ? __shfl_sync(TB2_FULL_MASK, x, k)
                                      : acc + __shfl_sync(TB2_FULL_MASK, x, k);
                if (tid == k) mine = acc;
            }
            if (base + tid < n) cs[base + tid] = mine;
        }
    }
    __syncthreads();
    const int n_ma = n - (mini - 1);
    const int n_off = n_ma - mini * (nwin - 1);
    // mav[k] = (cs[k+49] - cs[k-1]) / 50 ; first window: cs[49] / 50   (:277-282)
    auto mav = [&](int k) {
        const int i = k + mini - 1;
        const double v = (i >= mini) ? cs[i] - cs[i - mini] : cs[i];
        return v / (double)mini;
    };
    for (int q = tid; q < n_off; q += ST_THREADS) {
        double off[7];
#pragma unroll
        for (int o = 0; o < 7; ++o) off[o] = mav(q + mini * o);
        double sum = fabs(off[0] - off[1]);                  // diffs[0].copy() (:298)
#pragma unroll
        for (int i = 0; i < 7; ++i)
#pragma unroll
            for (int j = i + 1; j < 7; ++j) sum += fabs(off[i] - off[j]);
        metric[q] = sum / 21.0;
    }
    const int start_off = (int)((double)window * 0.5);
    for (int i = tid; i < n; i += ST_THREADS) below[i] = 0;
    __syncthreads();
    for (int q = tid; q < n_off; q += ST_THREADS) below[start_off + q] = metric[q] <= thresh;
    __syncthreads();
    if (tid == 0) {
        int *out = b.stall_ints + 2 * (size_t)b.stall_cap * r;
        const int expand = window / 2 - edge;
        int no = 0, have = 0, ps = 0, pe = 0, i = 0, overflow = 0;
        while (i < n) {
            if (below[i]) {
                int j = i;
                while (j < n && below[j]) ++j;
                if (j - i > min_consec) {
                    const int a = i - expand, z = j + expand;
                    if (!have) { ps = a; pe = z; have = 1; }
                    else if (a > pe) {
                        if (no < b.stall_cap) { out[2 * no] = ps; out[2 * no + 1] = pe; } else overflow = 1;
                        ++no; ps = a; pe = z;
                    } else pe = z;
                }
                i = j;
            } else ++i;
        }
        if (have) {
            if (no < b.stall_cap) { out[2 * no] = ps; out[2 * no + 1] = pe; } else overflow = 1;
            ++no;
        }
        s.n_stalls = no;
        if (overflow) { s.status = TB2_ERR_CAPACITY; s.done = 1; }
    }
}

// ===========================================================================
// resolve_skipped_bases_with_raw resquiggle.py:402-540 with c_reg_z_scores,
// c_base_forward_pass, c_base_traceback (_c_dynamic_programming.pyx:34-182).
// Small serial DPs: one warp per read, lane 0 walks the windows.
// ===========================================================================
struct RawCtx {
    const double *sig;   // window signal (norm + rsrtr + sig_start)
    const double *rm, *rs;
    int n_ev, L, m;
    int winsor;
    double mhz;
    double *fwd;         // n_ev x L; on entry of raw_window row r holds the z-scores of base r
    double *cs;          // L
    int *ld0, *ld1;      // L each
};

__device__ __forceinline__ double raw_z(const RawCtx &c, int row, int i)
{
    // c_base_z_scores :17-32 on r_sig[b_start + i]
    double z = (c.sig[row * c.m + i] - c.rm[row]) / c.rs[row];
    if (z > 0) z = -z;
    if (c.winsor && z < -c.mhz) z = -c.mhz;
    return z;
}

// all lanes: the z-scores of every (base, sample) cell of the window, written where the
// forward values will go (the serial pass below consumes each one right before it overwrites
// it) -- the IEEE divisions leave the single-lane critical path
__device__ __forceinline__ void raw_fill_z(const RawCtx &c)
{
    const int lane = threadIdx.x & 31;
    for (int r = 0; r < c.n_ev; ++r) {
        double *row = c.fwd + (size_t)r * c.L;
        for (int i = lane; i < c.L; i += 32) row[i] = raw_z(c, r, i);
    }
    __syncwarp();
}

// lane 0 only: serial forward pass (any raw_min_obs_per_base)
__device__ int raw_window(RawCtx &c, int *new_segs)
{
    const int L = c.L, m = c.m, n_ev = c.n_ev;
    if (n_ev < 2 || L < 1) return TB2_ERR_UNEXPECTED;
    // with raw_min_obs_per_base > 1 a row needs the cumulative z-scores of the row above
    // (c_base_forward_pass :113, np.cumsum: sequential).  They are summed while that row is
    // consumed -- same values, same order -- into one half of cs; the halves alternate.
    const bool need_cs = m > 1;
    double *cs_prev = c.cs, *cs_next = c.cs + L;
    // raw_forward_pass resquiggle.py:345-380 -- first row is a cumsum of its z-scores
    {
        double acc = 0;
        for (int i = 0; i < L; ++i) {
            acc = (i == 0) ? c.fwd[0] : acc + c.fwd[i];
            c.fwd[i] = acc; c.ld0[i] = m;
            if (need_cs) cs_prev[i] = acc;
        }
    }
    int *pld = c.ld0, *cld = c.ld1;
    for (int r = 1; r < n_ev; ++r) {
        const double *pf = c.fwd + (size_t)(r - 1) * L;
        double *bf = c.fwd + (size_t)r * L;      // holds z(r, .) until overwritten below
        // c_base_forward_pass :99-163; rows: start r*m, end r*m + L
        const int b_start = r * m, p_start = (r - 1) * m, p_end = p_start + L, b_end = b_start + L;
        double zacc = 0;
        auto take_z = [&](int ix) {              // ix runs 0 .. L-1 in order over the row
            const double zv = bf[ix];
            if (need_cs) { zacc = (ix == 0) ? zv : zacc + zv; cs_next[ix] = zacc; }
            return zv;
        };
        if (b_start - p_start - 1 < 0 || b_start - p_start - 1 >= L) return TB2_ERR_UNEXPECTED;
        bf[0] = take_z(0) + pf[b_start - p_start - 1];
        cld[0] = 1;
        for (int pos = b_start + 1; pos < p_end + 1; ++pos) {
            int lag = 1;
            for (;;) {
                const int ix = pos - p_start - lag;
                if (ix < 0 || ix >= L) return TB2_ERR_UNEXPECTED;
                if (pld[ix] + lag <= m) ++lag; else break;
            }
            double diag = pf[pos - p_start - lag];
            if (lag > 1) {
                if (pos - p_start - 1 >= L) return TB2_ERR_UNEXPECTED;
                diag += cs_prev[pos - p_start - 1] - cs_prev[pos - p_start - lag];
            }
            if (pos - b_start >= L) return TB2_ERR_UNEXPECTED;
            const double stay = bf[pos - b_start - 1];
            double score; int dv;
            if (diag > stay) { score = diag; dv = 1; }
            else { score = stay; dv = cld[pos - b_start - 1] + 1; }
            bf[pos - b_start] = take_z(pos - b_start) + score;
            cld[pos - b_start] = dv;
        }
        if (b_end > p_end + 1) {
            double fv = bf[p_end - b_start];
            int cl = cld[p_end - b_start];
            const int left = b_end - p_end - 1;
            for (int i = 0; i < left; ++i) {
                fv += take_z(i + p_end - b_start + 1);
                cl += 1;
                bf[i + p_end - b_start + 1] = fv;
                cld[i + p_end - b_start + 1] = cl;
            }
        }
        int *t = pld; pld = cld; cld = t;
        double *tc = cs_prev; cs_prev = cs_next; cs_next = tc;
    }
    return TB2_OK;
}

// raw_min_obs_per_base == 1 (DNA): cell (r, i) needs (r, i-1) [stay] and (r-1, i) [diag]
// only (c_base_forward_pass :99-163 with lag == 1), so rows can be skewed against each other
// like the static band: lane l owns row s0 + l of a 32-row strip, one cell behind lane l-1;
// the cell above arrives by one shuffle, the stay value is the lane's own register.  Same
// operations in the same order as the serial pass (z + max(diag, stay), ties to stay; first
// row: running sum).  All lanes; forward values go to c.fwd.
__device__ void raw_forward_wf(const RawCtx &c)
{
    const int lane = threadIdx.x & 31;
    const int L = c.L, n_ev = c.n_ev;
    for (int s0 = 0; s0 < n_ev; s0 += 32) {
        const int r = s0 + lane;
        const bool row_ok = r < n_ev;
        double *bf = c.fwd + (size_t)(row_ok ? r : s0) * L;
        const double *above = (s0 > 0) ? c.fwd + (size_t)(s0 - 1) * L : nullptr;   // lane 0's diag source
        const int last = min(31, n_ev - 1 - s0);
        double x = 0.0, xout = 0.0;
        for (int t = 0; t < L + last; ++t) {
            double up = __shfl_up_sync(TB2_FULL_MASK, xout, 1);
            const int i = t - lane;
            if (row_ok && i >= 0 && i < L) {
                if (lane == 0 && above != nullptr) up = above[i];
                const double z = raw_z(c, r, i);
                double nx;
                if (r == 0) nx = (i == 0) ? z : x + z;                 // resquiggle.py:352-356
                else if (i == 0) nx = z + up;                          // :136
                else nx = z + ((up > x) ? up : x);                     // :141-150
                bf[i] = nx;
                x = nx; xout = nx;
            }
        }
        __syncwarp();      // the strip's last row is the next strip's row above
    }
}

// lane 0: raw_traceback over the forward values
__device__ int raw_traceback_rows(const RawCtx &c, int *new_segs)
{
    const int L = c.L, m = c.m, n_ev = c.n_ev;
    // raw_traceback resquiggle.py:382-400 with c_base_traceback :165-182
    int sig_start = (n_ev - 1) * m + L - 1;   // curr_end - 1
    for (int bp = n_ev - 2; bp >= 0; --bp) {
        const int cur = bp + 1;
        const double *cf = c.fwd + (size_t)cur * L, *nf = c.fwd + (size_t)bp * L;
        const int c_start = cur * m, n_start = bp * m, n_end = n_start + L;
        int cbs = 1, found = -1;
        for (int sp = sig_start; sp >= 0; --sp) {
            cbs += 1;
            if (cbs <= m || sp - 1 >= n_end) continue;
            if (sp <= c_start) { found = sp; break; }
            const int a = sp - n_start - 1, q = sp - c_start - 1;
            if (a < 0 || a >= L || q < 0 || q >= L) return TB2_ERR_UNEXPECTED;
            if (nf[a] > cf[q]) { found = sp; break; }
        }
        if (found < 0) return TB2_ERR_UNEXPECTED;   // reference: None -> TypeError
        new_segs[bp] = found;
        sig_start = found - 1;
    }
    return TB2_OK;
}

#define DEL_FIX_WINDOW 2
#define MAX_DEL_FIX_WINDOW 10
#define EXTRA_SIG_FACTOR 1.1

__global__ void __launch_bounds__(128)
k_resolve(BatchView b, tb2_params p, StagePolicy pol, double *pool, size_t cap, int *counter,
          double *big_pool, unsigned long long big_cap, unsigned long long *big_used)
{
    const int lane = threadIdx.x & 31;
    const size_t slot = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    double *scr = pool + slot * cap;
    for (;;) {
        int r = 0;
        if (lane == 0) r = atomicAdd(counter, 1);
        r = __shfl_sync(TB2_FULL_MASK, r, 0);
        if (r >= b.n_reads) break;
        ReadState &s = b.st[r];
        if (!rd_active(s)) continue;
        const long long bo = b.base_off[r];
        const int nb = (int)(b.base_off[r + 1] - bo);
        const int *segs = b.segs_dp + bo + r;
        int *out = b.segs + bo + r;
        for (int i = lane; i <= nb; i += 32) out[i] = segs[i];
        __syncwarp();
        const int n_norm = segs[nb];
        if (lane == 0) s.n_norm = n_norm;
        const double *norm = b.norm + b.raw_off[r] + s.rsrtr;
        const double *rm = b.rm + bo, *rs = b.rs + bo;
        int *ws = b.starts + bo, *we = b.read_tb + bo + r;   // scratch (>= nb entries each)
        const int n_segs = nb + 1;
        const int m = (int)p.raw_min_obs_per_base;
        int nw = 0, st = TB2_OK;
#define TOO_SMALL(a, z) ((double)(segs[z] - segs[a]) <= ((double)(((z) - (a) + 1) * m)) * EXTRA_SIG_FACTOR)
#define MERGE_TRIM() do { \
            int mm = 0; \
            for (int k = 0; k < nw; ++k) { \
                if (mm > 0 && ws[k] < we[mm - 1]) we[mm - 1] = we[k]; \
                else { ws[mm] = ws[k]; we[mm] = we[k]; ++mm; } } \
            nw = mm; \
            if (ws[0] < 0) ws[0] = 0; \
            if (we[nw - 1] > n_segs - 1) we[nw - 1] = n_segs - 1; } while (0)
        if (lane == 0) {
            // the windows (lane 0; a handful of integers per read)
            for (int d = 0; d < nb; ++d) {                                   // :465-472
                if (segs[d + 1] - segs[d] != 0) continue;
                if (nw > 0 && d < we[nw - 1] + DEL_FIX_WINDOW) we[nw - 1] = d + DEL_FIX_WINDOW + 1;
                else { ws[nw] = d - DEL_FIX_WINDOW; we[nw] = d + DEL_FIX_WINDOW + 1; ++nw; }
            }
            if (nw > 0) {
                MERGE_TRIM();
                int expanded = 0;
                for (int it = 0; it < MAX_DEL_FIX_WINDOW - DEL_FIX_WINDOW; ++it) {   // :481-486
                    expanded = 0;
                    for (int k = 0; k < nw; ++k)
                        if (TOO_SMALL(ws[k], we[k])) { expanded = 1; ws[k] -= 1; we[k] += 1; }
                    if (!expanded) break;
                    MERGE_TRIM();
                }
                if (expanded)
                    for (int k = 0; k < nw; ++k)
                        if (TOO_SMALL(ws[k], we[k])) { st = TB2_ERR_NOT_ENOUGH_DEL_SIGNAL; break; }
                if (st == TB2_OK && pol.max_raw_cpts >= 0) {
                    int mx = 0;
                    for (int k = 0; k < nw; ++k) mx = max(mx, we[k] - ws[k]);
                    if (mx > pol.max_raw_cpts) st = TB2_ERR_TOO_MANY_DELS;
                }
            }
        }
        nw = __shfl_sync(TB2_FULL_MASK, nw, 0);
        st = __shfl_sync(TB2_FULL_MASK, st, 0);
        if (nw == 0) continue;
        __syncwarp();                              // ws / we written by lane 0 are read by all
        for (int k = 0; k < nw && st == TB2_OK; ++k) {                    // :506-531
            const int a = ws[k], z = we[k], n_ev = z - a;
            const int sig_start = segs[a], sig_len = segs[z] - segs[a];
            if (sig_start < 0 || sig_start + sig_len > n_norm) { st = TB2_ERR_UNEXPECTED; break; }
            RawCtx c;
            c.sig = norm + sig_start; c.rm = rm + a; c.rs = rs + a;
            c.n_ev = n_ev; c.m = m;
            // c_reg_z_scores with max_base_shift = n_events: starts idx*m, ends
            // sig_len - (n_ev-1-idx)*m  (:56-81)  => every row has the same length
            c.L = sig_len - (n_ev - 1) * m;
            c.winsor = !isnan(p.max_half_z_score);
            c.mhz = c.winsor ? p.max_half_z_score : 0.0;
            if (c.L < 1) { st = TB2_ERR_UNEXPECTED; break; }
            const size_t need = (size_t)n_ev * c.L + 3 * (size_t)c.L + 8;
            unsigned long long woff = 0;           // 0: the warp's own slab
            if (need > cap) {
                // a window too large for the per-warp slab (e.g. a base carrying a 10k-sample
                // stall, BASELINE configs[4]): bump-allocate from the overflow arena of this
                // launch; only when that is exhausted too is the read a loud capacity failure
                if (lane == 0) woff = atomicAdd(big_used, (unsigned long long)need) + 1ULL;
                woff = __shfl_sync(TB2_FULL_MASK, woff, 0);
                if (woff - 1ULL + need > big_cap) { st = TB2_ERR_CAPACITY; break; }
            }
            double *win = woff ? big_pool + (woff - 1ULL) : scr;
            c.fwd = win;
            c.cs = win + (size_t)n_ev * c.L;       // two halves of L
            c.ld0 = (int *)(c.cs + 2 * (size_t)c.L);
            c.ld1 = c.ld0 + c.L;
            if (n_ev < 2) { st = TB2_ERR_UNEXPECTED; break; }
            // forward pass: 32-row wavefront when every base needs one observation (DNA),
            // else z-scores by all lanes and the serial recurrence by lane 0
            if (m == 1) raw_forward_wf(c);
            else raw_fill_z(c);
            // new segs land in out[a+1 .. z-1]
            if (lane == 0) {
                st = (m == 1) ? TB2_OK : raw_window(c, out + a + 1);
                if (st == TB2_OK) st = raw_traceback_rows(c, out + a + 1);
                if (st == TB2_OK) for (int i = 0; i < n_ev - 1; ++i) out[a + 1 + i] += sig_start;
            }
            st = __shfl_sync(TB2_FULL_MASK, st, 0);
            __syncwarp();
        }
        if (lane != 0) continue;
        if (st == TB2_OK) {
            for (int i = 0; i < nb; ++i) if (out[i + 1] - out[i] < 1) { st = TB2_ERR_ZERO_LEN_SEG; break; }
            if (st == TB2_OK && out[0] < 0) st = TB2_ERR_NEG_SEG;
            if (st == TB2_OK && out[nb] > n_norm) st = TB2_ERR_SEG_PAST_END;
        }
        if (st != TB2_OK) s.status = st;
    }
}

// ===========================================================================
// compute_base_means on the clipped signal (resquiggle.py:1185)
// ===========================================================================
__global__ void __launch_bounds__(ST_THREADS) k_base_means(BatchView b)
{
    const int r = blockIdx.x;
    const ReadState &s = b.st[r];
    if (!rd_active(s)) return;
    const long long bo = b.base_off[r];
    const int nb = (int)(b.base_off[r + 1] - bo);
    const double *norm = b.norm + b.raw_off[r] + s.rsrtr;
    const int *segs = b.segs + bo + r;
    for (int i = threadIdx.x; i < nb; i += ST_THREADS) {
        const int a = segs[i], z = segs[i + 1];
        double acc = 0;
        for (int k = a; k < z; ++k) acc += norm[k];
        b.bm[bo + i] = acc / (double)(z - a);
    }
}

// ===========================================================================
// calc_kmer_fitted_shift_scale(method='theil_sen') tombo_stats.py:401-450 with
// c_compute_slopes _c_helper.pyx:362-377: median of all pairwise slopes, then
// median intercept.  Exact: slopes are recomputed, never approximated; a
// 2048-bin histogram over a sample-derived bracket narrows the median to one
// bin, whose members are selected exactly (generic radix select as fall-back).
// ===========================================================================
// debug counters (tests / tuning): [0] Theil-Sen reads, [1] fp32 bracket over every pair,
// [2] exact histogram path, [3] generic select path, [4] fp32 bracket over sampled pairs,
// [5] sort-and-sweep finished, [6] sort-and-sweep abandoned (one of [1]-[4] then finishes),
// [7] odd-even sweep phases (TS_DEBUG builds only)
__device__ unsigned long long g_tb2_counters[8];

#define TS_MAX 1000
#define TS_BINS 2048
#define TS_BUF 2048

#define TS_ABINS 4096   // bins of the approximate (fp32) pre-pass

#define TS_PAD 1024     // TS_MAX rounded up to a power of two (bitonic sort by ev)

struct TsSmem {
    double ev[TS_PAD], md[TS_PAD];     // points, sorted by ev once the bracket sample is taken
    float4 pt[TS_PAD];                 // fp32 images: pass 1 (ev, md), pass 2 (qL, qH, ev)
    union {
        unsigned int hist[TS_ABINS + 2];   // also holds the TS_BINS + 2 exact bins
        double buf[TS_BUF];                // bracket sample, then the slopes inside the bracket
    };
    unsigned int nbuf, nout, b1, b2, below, maxabs_bits;
    int ok;
};

__device__ __forceinline__ double ts_slope(const TsSmem &t, int i, int j)
{
    // (i < j) -- combinations order, _c_helper.pyx:370-376
    return (t.ev[i] == t.ev[j]) ? 1000.0 : (t.md[i] - t.md[j]) / (t.ev[i] - t.ev[j]);
}

template <class Fn>
__device__ __forceinline__ void ts_for_pairs(int n, Fn fn)
{
    // balanced column pairing: column j holds pairs (i, j), i < j
    const int half = (n + 1) / 2;
    for (int c = threadIdx.x; c < half; c += ST_THREADS) {
        const int j0 = c, j1 = n - 1 - c;
        for (int i = 0; i < j0; ++i) fn(i, j0);
        if (j1 != j0) for (int i = 0; i < j1; ++i) fn(i, j1);
    }
}

// the same pairing, one call per column (the callee keeps column j in registers)
template <class Fn>
__device__ __forceinline__ void ts_for_cols(int n, Fn fn)
{
    const int half = (n + 1) / 2;
    for (int c = threadIdx.x; c < half; c += ST_THREADS) {
        const int j0 = c, j1 = n - 1 - c;
        fn(j0);
        if (j1 != j0) fn(j1);
    }
}

__device__ __forceinline__ void ts_pair_of(long long s, int n, int *pi, int *pj)
{
    // inverse of the combinations enumeration index
    double disc = (double)(2 * n - 1) * (double)(2 * n - 1) - 8.0 * (double)s;
    int i = (int)(((double)(2 * n - 1) - sqrt(disc)) / 2.0);
    if (i < 0) i = 0;
    auto row_start = [&](int q) { return (long long)q * (2 * n - q - 1) / 2; };
    while (i > 0 && row_start(i) > s) --i;
    while (row_start(i + 1) <= s) ++i;
    *pi = i;
    *pj = (int)(s - row_start(i)) + i + 1;
}


// ---------------------------------------------------------------------------
// Sort-and-sweep median of the pairwise slopes (round 2).  With the points sorted by ev,
// a pair a < b has slope < T  <=>  Q_T(a) > Q_T(b),  Q_T(k) = md_k - T * ev_k: the number
// of slopes below T is the inversion count of the sequence Q_T, and the pairs whose slope
// lies in [T1, T2) are exactly the adjacent transpositions that turn the Q_T1 order into
// the Q_T2 order.  So instead of testing all n(n-1)/2 pairs against a bracket:
//   1. a 2048-pair sample histogram places three thresholds L < H1 < H2 below / around the
//      median ranks (cheap; only has to be roughly right);
//   2. one merge sort by Q_L counts the slopes below L exactly (O(n log^2 n));
//   3. odd-even transposition passes re-sort to Q_H1 (counting swaps) and then to Q_H2
//      (listing the swapped pairs): a few dozen passes, since few pairs cross;
//   4. the listed pairs (~1 % of all) get the reference's exact fp64 quotient and one
//      radix select returns the order statistics np.median sees.
// Exactness: every comparison is made on fp64 Q values; after each (re)sort all adjacent
// gaps must exceed a guard g = 1e-12 * M * (1 + |T|) -- then NO pair is within g of the
// threshold, the computed order is the real-arithmetic order, and the reference's rounded
// quotient (within 3 ulp of the real slope) falls on the same side.  Any doubt (a gap within
// the guard, equal ev, thresholds that miss the median ranks, an overflowing list) abandons
// this path for the exhaustive one below -- never a different answer.
// ---------------------------------------------------------------------------
#define TS_SBINS 1024          // bins of the sample histogram over [lo, hi)
#define TS_SAMPLES 2048
#define TS_LIST 4096           // listed (swapped) pairs, u32 each
#define TS_MAX_PHASES 600

// stable merge sort of (key, id) by key ascending, ids are positions 0..P-1 in ev order; returns
// the number of inversions (pairs of positions a < b with key[a] > key[b]).  P is a power of
// two >= n, keys beyond n are +inf.  On return the sorted arrays are in (*ka, *pa).
__device__ long long ts_sort_count(double **ka, double **kb, unsigned short **pa, unsigned short **pb,
                                   int P, SelectSmem &sm)
{
    const int tid = threadIdx.x;
    unsigned int inv = 0;
    for (int w = 1; w < P; w <<= 1) {
        const double *src = *ka; const unsigned short *sp = *pa;
        double *dst = *kb; unsigned short *dp = *pb;
        for (int p = tid; p < P; p += ST_THREADS) {
            const int base = p & ~(2 * w - 1), mid = base + w;
            const double key = src[p];
            int lo, hi;
            if (p < mid) {                       // left run: count right elements < key
                lo = mid; hi = mid + w;
                while (lo < hi) { const int m = (lo + hi) >> 1; if (src[m] < key) lo = m + 1; else hi = m; }
                dst[p + (lo - mid)] = key; dp[p + (lo - mid)] = sp[p];
            } else {                             // right run: count left elements <= key
                lo = base; hi = mid;
                while (lo < hi) { const int m = (lo + hi) >> 1; if (src[m] <= key) lo = m + 1; else hi = m; }
                const int le = lo - base;
                dst[base + (p - mid) + le] = key; dp[base + (p - mid) + le] = sp[p];
                inv += (unsigned int)(w - le);   // left elements > key
            }
        }
        __syncthreads();
        double *tk = *ka; *ka = *kb; *kb = tk;
        unsigned short *tp = *pa; *pa = *pb; *pb = tp;
    }
    // block-wide sum in 64 bits (n <= 1000: < 5e5 inversions, a 32-bit sum is safe)
    return (long long)tb2_block_sum(inv, sm);
}

// odd-even transposition re-sort of `perm` (positions -> element ids) by q[] ascending.
// Returns the number of swaps (pairs that crossed) or -1 if it did not settle; swapped pairs
// are appended to list[*n_list] as (min id << 16 | max id) when list != nullptr.
__device__ long long ts_sweep(unsigned short *perm, const double *q, int n, unsigned int *list,
                              unsigned int *n_list, SelectSmem &sm)
{
    const int tid = threadIdx.x;
    unsigned int swaps = 0;
    int quiet = 0;
    for (int ph = 0; ph < TS_MAX_PHASES; ++ph) {
        int any = 0;
        for (int p = 2 * tid + (ph & 1); p + 1 < n; p += 2 * ST_THREADS) {
            const unsigned short x = perm[p], y = perm[p + 1];
            if (q[x] > q[y]) {
                perm[p] = y; perm[p + 1] = x;
                ++swaps; any = 1;
                if (list) {
                    const unsigned int slot = atomicAdd(n_list, 1u);
                    if (slot < TS_LIST) list[slot] = ((unsigned int)min(x, y) << 16) | (unsigned int)max(x, y);
                }
            }
        }
        any = __syncthreads_or(any);
        quiet = any ? 0 : quiet + 1;
        if (quiet >= 2) {
#ifdef TS_DEBUG
            if (tid == 0) atomicAdd(&g_tb2_counters[7], (unsigned long long)(ph + 1));
#endif
            return (long long)tb2_block_sum(swaps, sm);
        }
    }
    tb2_block_sum(swaps, sm);
    return -1;
}

// all adjacent gaps of the order `perm` by q exceed the guard (then no pair at all is within it)
__device__ bool ts_gaps_ok(const unsigned short *perm, const double *q, const double *ev, int n, double g)
{
    int bad = 0;
    for (int p = threadIdx.x; p + 1 < n; p += ST_THREADS) {
        const int x = perm[p], y = perm[p + 1];
        bad |= !(q[y] - q[x] > g) && (ev[x] != ev[y]);   // equal-ev neighbours are exempt
    }
    return !__syncthreads_or(bad);
}

__global__ void __launch_bounds__(ST_THREADS, 4)
k_theil_sen(BatchView b, StagePolicy pol, int first_call)
{
    TB2_DYN_SMEM(unsigned char, ts_raw);
    TsSmem &t = *reinterpret_cast<TsSmem *>(ts_raw);
    __shared__ SelectSmem sm;
    const int r = b.order ? b.order[blockIdx.x] : blockIdx.x;
    ReadState &s = b.st[r];
    if (!rd_active(s)) return;
    const int tid = threadIdx.x;
    if (first_call && pol.skip_seq_scaling) {       // resquiggle.py:1179-1180
        if (tid == 0) { s.changed = 0; s.shc = 0.0; s.scc = 1.0; }
        return;
    }
    const long long bo = b.base_off[r];
    const int nb = (int)(b.base_off[r + 1] - bo);
    const double *bm = b.bm + bo, *rm = b.rm + bo;
    int n = nb;
    if (nb > TS_MAX) {                              // tombo_stats.py:411-416
        n = TS_MAX;
        const unsigned int key = pol.literal_key
            ? pol.subsample_seed
            : tb2_subsample_key(pol.subsample_seed, (unsigned int)(r + pol.read_index_base),
                                (unsigned int)s.calls);
        for (int i = tid; i < n; i += ST_THREADS) {
            const int k = tb2_perm_index(i, nb, key);
            t.ev[i] = bm[k]; t.md[i] = rm[k];
        }
    } else {
        for (int i = tid; i < n; i += ST_THREADS) { t.ev[i] = bm[i]; t.md[i] = rm[i]; }
    }
    __syncthreads();
    const long long Np = (long long)n * (n - 1) / 2;
    if (Np <= 0) { if (tid == 0) s.status = TB2_ERR_UNEXPECTED; return; }
    if (tid == 0) atomicAdd(&g_tb2_counters[0], 1ULL);
    const bool even = (Np % 2) == 0;
    const long long k1 = even ? Np / 2 - 1 : Np / 2;   // ranks k1 (and k1+1 if even)
    double v1 = 0, v2 = 0;
    bool have = false;
    // ---- bracket [lo, hi] from a sample of n/2 independent pairs (original order) ----
    const int hs = n / 2;
    double lo = 0, hi = 0;
    if (hs >= 16) {
        for (int i = tid; i < hs; i += ST_THREADS) t.buf[i] = ts_slope(t, i, i + hs);
        __syncthreads();
        double d0;
        auto f_samp = [&](int i) { return t.buf[i]; };
        tb2_block_select2(f_samp, PredAll(), hs, (int)(hs * 0.30), false, &lo, &d0, sm);
        tb2_block_select2(f_samp, PredAll(), hs, (int)(hs * 0.70), false, &hi, &d0, sm);
    }
    // ---- sort the points by ev: slope(i, j) is symmetric in (i, j) (both differences
    // negate exactly), so the multiset of slopes is unchanged, and every pair a < b now
    // has ev_a - ev_b <= 0, which fixes the direction of the screening inequalities ----
    {
        int P = 2;
        while (P < n) P <<= 1;
        for (int i = n + tid; i < P; i += ST_THREADS) { t.ev[i] = __longlong_as_double(0x7ff0000000000000LL); t.md[i] = 0.0; }
        __syncthreads();
        for (int k = 2; k <= P; k <<= 1) {
            for (int jj = k >> 1; jj > 0; jj >>= 1) {
                for (int idx = tid; idx < (P >> 1); idx += ST_THREADS) {
                    const int a = ((idx & ~(jj - 1)) << 1) | (idx & (jj - 1)), c = a | jj;
                    // (ev, md) lexicographic: points of equal ev end up in ascending md, so that
                    // such a pair -- whose slope the reference defines as 1000.0 -- is never an
                    // inversion of any Q_T sequence
                    const double ea = t.ev[a], ec = t.ev[c];
                    const double ma = t.md[a], mc = t.md[c];
                    const bool gt = (ea > ec) || (ea == ec && ma > mc);
                    const bool ne = (ea != ec) || (ma != mc);
                    if (ne && (gt == ((a & k) == 0))) {
                        t.ev[a] = ec; t.ev[c] = ea;
                        t.md[a] = mc; t.md[c] = ma;
                    }
                }
                __syncthreads();
            }
        }
    }
    // ---- sort-and-sweep path (see the comment above ts_sort_count) ----
    if (hs >= 16 && n >= 128 && hi > lo && hi < 1000.0) {
        // shared-memory plan: pt (16 KB) = two key arrays for the merge sort, afterwards the
        // per-element Q (qa) and the start of the pair list (qb); the hist/buf union = sample
        // CDF (4.1 KB, later the rest of the pair list) and, in its last 4 KB, the two id
        // arrays; the exact slopes finally take pt + union (32 KB = 4096 doubles)
        double *qa = reinterpret_cast<double *>(t.pt), *qb = qa + TS_PAD;
        // ids: the last 4 KB of the union; pair list: from qb (8 KB) on through the union up to
        // the ids (12 KB) -- it overwrites the sample CDF, which is dead once the listing sweep's
        // threshold has been picked
        unsigned short *pa = reinterpret_cast<unsigned short *>(t.buf + (TS_BUF - 512)), *pb = pa + TS_PAD;
        unsigned int *list = reinterpret_cast<unsigned int *>(qb);
        static_assert(TS_LIST * 4 <= TS_PAD * 8 + (TS_BUF - 512) * 8, "pair list overlaps the id arrays");
        bool ok;
        double M;
        // sample size: about one sample per 24 pairs, 2048 .. 8192
        const int n_samples = (int)min(8192LL, max(2048LL, Np / 24));
        {
            // finite values; ev is non-decreasing after the sort.  Pairs of equal ev (common on
            // integer-valued signal: base means are ratios of small integers) have the
            // reference slope 1000.0 for every T: they sit above every threshold this path
            // uses (hi < 1000 is checked), never count as inversions (sorted by md inside a
            // tie group), never cross in a sweep (their Q difference does not depend on T) and
            // are exempt from the guard-gap test (any two elements within the guard are then
            // joined by a chain of equal-ev neighbours, i.e. are themselves an equal-ev pair)
            int bad = 0;
            double mx = 0.0;
            for (int i = tid; i < n; i += ST_THREADS) {
                const double e = t.ev[i], m = t.md[i];
                if (!(fabs(e) < 1e300) || !(fabs(m) < 1e300)) bad = 1;
                if (i + 1 < n && !(t.ev[i + 1] >= e)) bad = 1;
                mx = fmax(mx, fmax(fabs(e), fabs(m)));
            }
            ok = !__syncthreads_or(bad);
#ifdef TS_DEBUG
            if (!ok && tid == 0) { int c = 0; for (int i = 0; i + 1 < n; ++i) if (!(t.ev[i + 1] > t.ev[i])) { if (c++ < 3) printf("  ev order: i=%d %.17g %.17g\n", i, t.ev[i], t.ev[i + 1]); } }
#endif
            unsigned long long mk = (unsigned long long)__double_as_longlong(mx);   // mx >= 0: bit order
            mk = ~tb2_block_min_u64(~mk, sm);
            M = fmax(1.0, __longlong_as_double((long long)mk));
        }
        // 1. sample histogram of approximate slopes over [lo, hi), turned into a CDF table
        const float lo_f = (float)lo, hi_f = (float)hi;
        const float w_f = (hi_f - lo_f) / (float)TS_SBINS;
        ok = ok && (w_f > 0.0f) && isfinite(w_f);
        if (ok) {
            for (int i = tid; i < TS_SBINS + 2; i += ST_THREADS) t.hist[i] = 0;
            __syncthreads();
            const float inv_w = 1.0f / w_f;
            for (int q = tid; q < n_samples; q += ST_THREADS) {
                // a pseudo-random pair (i, j != i) without integer division: multiply-shift
                const uint32_t h1 = tb2_mix32((uint32_t)q * 2654435761u + 17u), h2 = tb2_mix32(h1 ^ 0x9E3779B9u);
                const int i = (int)(((unsigned long long)h1 * (unsigned long long)n) >> 32);
                int j = i + 1 + (int)(((unsigned long long)h2 * (unsigned long long)(n - 1)) >> 32);
                if (j >= n) j -= n;
                const double de = t.ev[i] - t.ev[j];
                const float sa = __fdividef((float)(t.md[i] - t.md[j]), (float)de);
                int bin = 0;                                 // bin 0: below lo
                if (sa >= hi_f || de == 0.0) bin = TS_SBINS + 1;   // last: at or above hi (equal ev: 1000.0)
                else if (sa >= lo_f) bin = min(TS_SBINS - 1, (int)((sa - lo_f) * inv_w)) + 1;
                atomicAdd(&t.hist[bin], 1u);
            }
            __syncthreads();
            const int per = (TS_SBINS + 2 + ST_THREADS - 1) / ST_THREADS;
            const int q0 = min(TS_SBINS + 2, tid * per), q1 = min(TS_SBINS + 2, q0 + per);
            unsigned int mine = 0;
            for (int q = q0; q < q1; ++q) mine += t.hist[q];
            const int lane = tid & 31, warp = tid >> 5;
            unsigned int inc = mine;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const unsigned int o = __shfl_up_sync(TB2_FULL_MASK, inc, off);
                if (lane >= off) inc += o;
            }
            if (lane == 31) sm.warp_tot[warp] = inc;
            __syncthreads();
            unsigned int run = inc - mine;
            for (int q = 0; q < warp; ++q) run += sm.warp_tot[q];
            for (int q = q0; q < q1; ++q) { run += t.hist[q]; t.hist[q] = run; }   // cum[q]: samples in bins <= q
            __syncthreads();
        }
        // threshold = upper edge of the first bin b (1..TS_SBINS) with cum[b] >= frac * samples
        auto pick = [&](double frac, int *bsel) -> bool {
            const double tf = frac * (double)n_samples;
            if (!(tf > (double)t.hist[0]) || !(tf < (double)t.hist[TS_SBINS])) return false;
            const unsigned int target = (unsigned int)tf;
            int blo = 1, bhi = TS_SBINS;
            while (blo < bhi) { const int m = (blo + bhi) >> 1; if (t.hist[m] >= target) bhi = m; else blo = m + 1; }
            *bsel = blo;
            return true;
        };
        auto thr = [&](int bsel) { return (double)lo_f + (double)w_f * (double)bsel; };
        const long long kT = even ? k1 + 1 : k1;
        const double sig = 0.5 / sqrt((double)n_samples);        // sd of a sample quantile near 0.5
        const double ppm = (double)Np / (double)n_samples;       // pairs per sample
        int bL = 0, bH1 = 0, bH2 = 0;
        long long invL = 0, inv1 = 0, inv2 = 0;
        if (ok) ok = pick((double)k1 / (double)Np - 3.0 * sig, &bL);
        if (ok) {
            // 2. exact count below L: merge sort by Q_L, certainty of the order
            const double TL = thr(bL);
            const double gL = 1e-12 * M * (1.0 + fabs(TL));
            int P = 2;
            while (P < n) P <<= 1;
            for (int i = tid; i < P; i += ST_THREADS) {
                qa[i] = (i < n) ? __fma_rn(-TL, t.ev[i], t.md[i]) : __longlong_as_double(0x7ff0000000000000LL);
                pa[i] = (unsigned short)i;
            }
            __syncthreads();
            double *ka = qa, *kb = qb;
            unsigned short *ia = pa, *ib = pb;
            invL = ts_sort_count(&ka, &kb, &ia, &ib, P, sm);
            int bad = 0;
            for (int p2 = tid; p2 + 1 < n; p2 += ST_THREADS)
                bad |= !(ka[p2 + 1] - ka[p2] > gL) && (t.ev[ia[p2]] != t.ev[ia[p2 + 1]]);
            ok = !__syncthreads_or(bad);
            if (ia != pa) for (int i = tid; i < n; i += ST_THREADS) pa[i] = ia[i];
            __syncthreads();
            ok = ok && invL <= k1;
        }
        // 3a. approach the median ranks from below with count-only sweeps.  Each exact count
        // re-calibrates the sample CDF; moving on by D pairs is then predictable to about
        // sqrt(D * pairs-per-sample), so every stage aims 3 of those sigmas short of rank k1
        // until the remaining distance fits the pair list
        bH1 = bL; inv1 = invL;
        for (int stage = 0; ok && stage < 5; ++stage) {
            const double D = (double)(k1 - inv1);
            const double rest = fmax(3.0 * sqrt(D * ppm), 150.0);
            if (D <= rest + 250.0 || D + 3.0 * sqrt(D * ppm) + 300.0 <= 0.8 * TS_LIST) break;
            const double delta = (double)inv1 / (double)Np - (double)t.hist[bH1] / (double)n_samples;
            int bn;
            if (!pick(((double)k1 - rest) / (double)Np - delta, &bn) || bn <= bH1) break;
            const double T1 = thr(bn);
            for (int i = tid; i < n; i += ST_THREADS) qa[i] = __fma_rn(-T1, t.ev[i], t.md[i]);
            __syncthreads();
            const long long sw = ts_sweep(pa, qa, n, nullptr, nullptr, sm);
            ok = sw >= 0 && ts_gaps_ok(pa, qa, t.ev, n, 1e-12 * M * (1.0 + fabs(T1)));
            bH1 = bn; inv1 += sw;
            ok = ok && inv1 <= k1;
#ifdef TS_DEBUG
            if (tid == 0) printf("  stage %d: D=%.0f aimed rest %.0f -> got rest %lld (swaps %lld)\n", stage, D, rest, k1 - inv1, sw);
#endif
        }
        if (ok) {
            // 3b. sweep past the median ranks, listing every pair that crosses
            const double D = (double)(kT - inv1);
            const double over = fmax(3.0 * sqrt(fmax(D, 1.0) * ppm), 150.0);
            const double delta = (double)inv1 / (double)Np - (double)t.hist[bH1] / (double)n_samples;
            ok = pick(((double)kT + over) / (double)Np - delta, &bH2) && bH2 > bH1;
            if (ok) {
                const double T2 = thr(bH2);
                for (int i = tid; i < n; i += ST_THREADS) qa[i] = __fma_rn(-T2, t.ev[i], t.md[i]);
                if (tid == 0) t.nbuf = 0;
                __syncthreads();
                const long long sw = ts_sweep(pa, qa, n, list, &t.nbuf, sm);
                ok = sw >= 0 && sw <= TS_LIST && ts_gaps_ok(pa, qa, t.ev, n, 1e-12 * M * (1.0 + fabs(T2)));
                inv2 = inv1 + sw;
                ok = ok && kT < inv2;
            }
        }
        if (ok) {
            // 4. the reference's own quotient for the listed pairs, then the order statistics
            const int K = (int)(inv2 - inv1);
            __syncthreads();
            double mine_v[TS_LIST / ST_THREADS];
#pragma unroll
            for (int u = 0; u < TS_LIST / ST_THREADS; ++u) {
                const int q = tid + u * ST_THREADS;
                mine_v[u] = 0.0;
                if (q < K) {
                    const int i = (int)(list[q] >> 16), j = (int)(list[q] & 0xffffu);
                    mine_v[u] = (t.md[i] - t.md[j]) / (t.ev[i] - t.ev[j]);      // _c_helper.pyx:371-376
                }
            }
            __syncthreads();
            double *outv = reinterpret_cast<double *>(t.pt);
#pragma unroll
            for (int u = 0; u < TS_LIST / ST_THREADS; ++u) {
                const int q = tid + u * ST_THREADS;
                if (q < K) outv[q] = mine_v[u];
            }
            __syncthreads();
            tb2_block_select2([&](int i) { return outv[i]; }, PredAll(), K, (int)(k1 - inv1), even,
                              &v1, &v2, sm);
            have = true;
            if (tid == 0) atomicAdd(&g_tb2_counters[5], 1ULL);
        } else if (tid == 0) {
            atomicAdd(&g_tb2_counters[6], 1ULL);
#ifdef TS_DEBUG
            printf("ts abandon: n=%d Np=%lld k1=%lld bL=%d bH1=%d bH2=%d invL=%lld inv1=%lld inv2=%lld nbuf=%u cum0=%u cumN=%u\n", n, Np, k1, bL, bH1, bH2, invL, inv1, inv2, t.nbuf, t.hist[0], t.hist[TS_SBINS]);
#endif
        }
        __syncthreads();
    }
    // ---- fast path: fp32 pre-pass picks a bracket [L, H), then ONE exact pass counts
    // the slopes below L and collects those inside; every decision of that pass is
    // exact (a guarded fp32 screen, the true fp64 division whenever a pair is within
    // the guard or inside the bracket), so the selected order statistics are the same
    // doubles np.median sees.  If the bracket misses, fall through.
    if (!have && hs >= 16 && Np > 4 * TS_ABINS) {
        const float lo_f = (float)lo, hi_f = (float)hi;
        const float w_f = (hi_f - lo_f) / (float)TS_ABINS;
        if (hi_f > lo_f && w_f > 0.0f && isfinite(w_f)) {
            const float inv_w = 1.0f / w_f;
            if (tid == 0) t.maxabs_bits = 0u;
            __syncthreads();
            {
                float mx = 0.0f;
                for (int i = tid; i < n; i += ST_THREADS)
                    mx = fmaxf(mx, fmaxf(fabsf((float)t.ev[i]), fabsf((float)t.md[i])));
                if (!(mx < 3.0e38f)) mx = 3.0e38f;          // inf / nan: everything is screened out
                atomicMax(&t.maxabs_bits, __float_as_uint(mx));
            }
            // The pre-pass only has to bracket the median ranks, so it looks at the pairs
            // with (i + j) % stride == 0 (every point takes part equally) and widens the
            // bracket by 2.5 sigma of the sampled rank; stride is chosen so that the
            // bracket still fits the buffer (2.5 * sqrt(Np * stride) <~ 1800).  A bracket
            // that misses or overflows is retried with every pair.
            int stride = (int)min(8LL, max(1LL, 518400LL / Np));
            for (; !have && stride >= 1; stride = (stride > 1) ? 1 : 0) {
                for (int i = tid; i < n; i += ST_THREADS)
                    t.pt[i] = make_float4((float)t.ev[i], (float)t.md[i], 0.0f, 0.0f);
                for (int i = tid; i < TS_ABINS + 2; i += ST_THREADS) t.hist[i] = 0;
                if (tid == 0) { t.nbuf = 0; t.ok = 0; t.below = 0; t.b1 = 0; t.b2 = 0; }
                __syncthreads();
                unsigned int n_under = 0, n_smp = 0;   // the underflow bin lives in a register
                ts_for_cols(n, [&](int j) {
                    const float4 pj = t.pt[j];
                    const int jm = j % stride;
                    int i = jm ? stride - jm : 0;
                    for (; i < j; i += stride) {
                        const float4 pi = t.pt[i];
                        const float de = pi.x - pj.x;
                        float sa = __fdividef(pi.y - pj.y, de);
                        if (de == 0.0f) sa = 1000.0f;
                        ++n_smp;
                        n_under += sa < lo_f;
                        if (sa >= lo_f && sa < hi_f)
                            atomicAdd(&t.hist[min(TS_ABINS - 1, (int)((sa - lo_f) * inv_w)) + 1], 1u);
                    }
                });
                n_under = tb2_block_sum(n_under, sm);
                n_smp = tb2_block_sum(n_smp, sm);
                if (tid == 0) t.hist[0] = n_under;
                __syncthreads();
                // sampled ranks that bracket the median ranks of the full set
                long long kA, kB;
                if (stride == 1) { kA = k1; kB = even ? k1 + 1 : k1; }
                else {
                    const long long kS = (long long)((double)k1 * (double)n_smp / (double)Np);
                    const long long mg = (long long)(1.25 * sqrt((double)n_smp)) + 2;
                    kA = kS - mg; kB = kS + mg;
                }
                if (tid == 0) { t.b1 = 0; t.b2 = TS_ABINS + 1; }   // "outside" unless located
                __syncthreads();
                if (kA >= 0 && kB < (long long)n_smp) {
                    // bins holding the sampled ranks kA and kB: 256 threads x 17 bins
                    const int per = (TS_ABINS + 2 + ST_THREADS - 1) / ST_THREADS;
                    const int q0 = min(TS_ABINS + 2, tid * per), q1 = min(TS_ABINS + 2, q0 + per);
                    unsigned int mine = 0;
                    for (int q = q0; q < q1; ++q) mine += t.hist[q];
                    const int lane = tid & 31, warp = tid >> 5;
                    unsigned int inc = mine;
#pragma unroll
                    for (int off = 1; off < 32; off <<= 1) {
                        const unsigned int o = __shfl_up_sync(TB2_FULL_MASK, inc, off);
                        if (lane >= off) inc += o;
                    }
                    if (lane == 31) sm.warp_tot[warp] = inc;
                    __syncthreads();
                    unsigned int base = 0;
                    for (int q = 0; q < warp; ++q) base += sm.warp_tot[q];
                    long long cum = (long long)base + inc - mine;
                    for (int q = q0; q < q1; ++q) {
                        const long long c = t.hist[q];
                        if (kA >= cum && kA < cum + c) t.b1 = q;
                        if (kB >= cum && kB < cum + c) t.b2 = q;
                        cum += c;
                    }
                }
                __syncthreads();
                const int bA = (int)t.b1, bB = (int)t.b2;
                if (bA >= 1 && bB <= TS_ABINS && bA <= bB) {
                    // exact bracket with a one-bin margin on both sides
                    const double L = (double)lo_f + (double)w_f * (double)(bA - 2);
                    const double H = (double)lo_f + (double)w_f * (double)(bB + 1);
                    // fp32 screen.  With Q_T(k) = md_k - T * ev_k, a pair a < b (ev_a <= ev_b)
                    // has slope < T  <=>  Q_T(a) > Q_T(b)  and  slope >= T  <=>  Q_T(a) <= Q_T(b)
                    // whenever ev_a != ev_b.  The fp32 images q = fma(-T_f, ev_f, md_f) carry an
                    // absolute error <= 1.8e-7 * M * (1 + |T|) each (|values| <= M), so a
                    // difference beyond g(T) = 1e-5 * M * (1 + |T|) settles the side of T with a
                    // margin far above the 3 ulp between the exact quotient and the reference's
                    // rounded one; anything closer, and every pair whose fp32 ev images
                    // coincide (ev_a == ev_b gives the reference's 1000.0), takes the exact
                    // fp64 path.
                    const float M = fmaxf(1.0f, __uint_as_float(t.maxabs_bits));
                    const float Lf = (float)L, Hf = (float)H;
                    const float gLf = 1e-5f * M * (1.0f + fabsf(Lf)), gHf = 1e-5f * M * (1.0f + fabsf(Hf));
                    __syncthreads();
                    for (int i = tid; i < n; i += ST_THREADS) {
                        const float ef = t.pt[i].x, mf = t.pt[i].y;
                        t.pt[i] = make_float4(fmaf(-Lf, ef, mf), fmaf(-Hf, ef, mf), ef, 0.0f);
                    }
                    __syncthreads();     // hist is dead from here on: buf takes its place
                    // screened pairs are settled in registers; the others (inside the
                    // bracket or within the guard) are queued as (i, j) and evaluated
                    // afterwards by all threads, so the fp64 divide never runs divergent
                    unsigned int below = 0;
                    unsigned int *queue = reinterpret_cast<unsigned int *>(t.buf);
                    const unsigned int QCAP = 2 * TS_BUF;
                    auto push = [&](int i, int j) {
                        const unsigned int slot = atomicAdd(&t.nbuf, 1u);
                        if (slot < QCAP) queue[slot] = ((unsigned int)i << 16) | (unsigned int)j;
                    };
                    {
                        // thread c owns columns ja = c and jb = n - 1 - c (ja <= jb): rows
                        // i < ja are tested against both with one load of point i
                        const int half = (n + 1) / 2;
                        for (int cidx = tid; cidx < half; cidx += ST_THREADS) {
                            const int ja = cidx, jb = n - 1 - cidx;
                            const float4 pa = t.pt[ja], pb = t.pt[jb];
                            const float xla = pa.x + gLf, yha = pa.y - gHf;
                            const float xlb = pb.x + gLf, yhb = pb.y - gHf;
                            int i = 0;
                            if (ja != jb) {
#pragma unroll 4
                                for (; i < ja; ++i) {
                                    const float4 pi = t.pt[i];
                                    const bool la = pi.x > xla, ha = pi.y < yha;
                                    const bool lb = pi.x > xlb, hb = pi.y < yhb;
                                    if ((la || ha) && pi.z != pa.z) below += la; else push(i, ja);
                                    if ((lb || hb) && pi.z != pb.z) below += lb; else push(i, jb);
                                }
                            }
#pragma unroll 4
                            for (; i < jb; ++i) {
                                const float4 pi = t.pt[i];
                                const bool lb = pi.x > xlb, hb = pi.y < yhb;
                                if ((lb || hb) && pi.z != pb.z) below += lb; else push(i, jb);
                            }
                        }
                    }
                    __syncthreads();
                    const unsigned int nq = t.nbuf;
                    double *outv = reinterpret_cast<double *>(t.pt);   // pt is dead now
                    if (tid == 0) t.nout = 0;
                    __syncthreads();
                    if (nq <= QCAP) {
                        for (unsigned int q = tid; q < nq; q += ST_THREADS) {
                            const int i = (int)(queue[q] >> 16), j = (int)(queue[q] & 0xffffu);
                            const double de = t.ev[i] - t.ev[j], dm = t.md[i] - t.md[j];
                            // the reference's value (_c_helper.pyx:371-376)
                            const double sv = (de == 0.0) ? 1000.0 : dm / de;
                            if (sv < L) ++below;
                            else if (sv < H) {
                                const unsigned int slot = atomicAdd(&t.nout, 1u);
                                if (slot < TS_BUF) outv[slot] = sv;
                            }
                        }
                    }
                    below = tb2_block_sum(below, sm);
                    __syncthreads();
                    const long long nbuf = t.nout;
                    const long long kT = even ? k1 + 1 : k1;
                    if (nq <= QCAP && nbuf <= TS_BUF && k1 >= (long long)below && kT < (long long)below + nbuf) {
                        tb2_block_select2([&](int i) { return outv[i]; }, PredAll(), (int)nbuf,
                                          (int)(k1 - (long long)below), even, &v1, &v2, sm);
                        have = true;
                        if (tid == 0) atomicAdd(&g_tb2_counters[stride == 1 ? 1 : 4], 1ULL);
                    }
                }
                __syncthreads();
            }
        }
    }
    if (!have && hs >= 16) {
        if (hi > lo) {
            const double inv_w = (double)TS_BINS / (hi - lo);
            auto bin_of = [&](double v) -> int {
                if (v < lo) return 0;                    // underflow bin
                if (!(v < hi)) return TS_BINS + 1;       // overflow bin
                int q = (int)((v - lo) * inv_w);
                if (q >= TS_BINS) q = TS_BINS - 1;
                return q + 1;
            };
            for (int i = tid; i < TS_BINS + 2; i += ST_THREADS) t.hist[i] = 0;
            if (tid == 0) { t.nbuf = 0; t.ok = 0; }
            __syncthreads();
            ts_for_pairs(n, [&](int i, int j) { atomicAdd(&t.hist[bin_of(ts_slope(t, i, j))], 1u); });
            __syncthreads();
            if (tid == 0) {
                // locate the bins holding ranks k1 and (if even) k1 + 1
                long long cum = 0;
                const long long kA = k1, kB = even ? k1 + 1 : k1;
                int bA = -1, bB = -1;
                long long belowA = 0;
                for (int q = 0; q < TS_BINS + 2; ++q) {
                    const long long c = t.hist[q];
                    if (bA < 0 && kA < cum + c) { bA = q; belowA = cum; }
                    if (bB < 0 && kB < cum + c) { bB = q; }
                    cum += c;
                    if (bA >= 0 && bB >= 0) break;
                }
                long long inrange = 0;
                if (bA >= 1 && bB <= TS_BINS && bA >= 0 && bB >= 0) {
                    for (int q = bA; q <= bB; ++q) inrange += t.hist[q];
                    if (inrange <= TS_BUF) { t.ok = 1; t.b1 = bA; t.b2 = bB; t.below = (unsigned int)belowA; }
                }
            }
            __syncthreads();
            if (t.ok) {
                const int bA = (int)t.b1, bB = (int)t.b2;
                ts_for_pairs(n, [&](int i, int j) {
                    const double v = ts_slope(t, i, j);
                    const int q = bin_of(v);
                    if (q >= bA && q <= bB) t.buf[atomicAdd(&t.nbuf, 1u)] = v;
                });
                __syncthreads();
                const int nbuf = (int)t.nbuf;
                tb2_block_select2([&](int i) { return t.buf[i]; }, PredAll(), nbuf,
                                  (int)(k1 - (long long)t.below), even, &v1, &v2, sm);
                have = true;
                if (tid == 0) atomicAdd(&g_tb2_counters[2], 1ULL);
            }
        }
    }
    if (!have) {
        if (tid == 0) { atomicAdd(&g_tb2_counters[3], 1ULL); }
        // generic exact fall-back: radix select over all pairs
        auto f_all = [&](int q) { int i, j; ts_pair_of(q, n, &i, &j); return ts_slope(t, i, j); };
        tb2_block_select2(f_all, PredAll(), (int)Np, (int)k1, even, &v1, &v2, sm);
    }
    const double slope = even ? (v1 + v2) / 2.0 : v1;                    // np.median (:418)
    const double inter = tb2_block_median([&](int i) { return t.md[i] - (slope * t.ev[i]); }, n, sm);  // :419
    if (tid == 0) {
        if (slope == 0) { s.status = TB2_ERR_THEIL_SEN_ZERO; return; }
        const double scc = 1 / slope;
        const double shc = -inter / slope;
        const double shift = s.sv.shift + (shc * s.sv.scale);            // :447
        const double scale = s.sv.scale * scc;                           // :448
        s.sv.shift = shift; s.sv.scale = scale; s.sv.outlier_thresh = pol.outlier_thresh;
        s.shc = shc; s.scc = scc;
        s.changed = (fabs(shc) > 0.1) || (fabs(scc - 1) > 0.1);         // resquiggle.py:1193-1195
    }
}

// ===========================================================================
// final re-normalisation + per-base means + sig_match_score
// (resquiggle.py:1190-1199, get_read_seg_score tombo_stats.py:2327-2338)
// ===========================================================================
__global__ void __launch_bounds__(ST_THREADS)
k_finalize(BatchView b, StagePolicy pol, int first_call, double *norm_mean_out,
           double *norm_signal_out)
{
    const int r = blockIdx.x;
    ReadState &s = b.st[r];
    if (!rd_active(s)) return;
    const long long bo = b.base_off[r];
    const int nb = (int)(b.base_off[r + 1] - bo);
    const double *norm = b.norm + b.raw_off[r] + s.rsrtr;
    const int *segs = b.segs + bo + r;
    const bool rescale = !(first_call && pol.skip_seq_scaling);
    const double shc = s.shc, scc = s.scc;
    double *t = b.tmp_b + bo + r;
    for (int i = threadIdx.x; i < nb; i += ST_THREADS) {
        const int a = segs[i], z = segs[i + 1];
        double acc = 0;
        if (rescale) for (int k = a; k < z; ++k) acc += (norm[k] - shc) / scc;
        else for (int k = a; k < z; ++k) acc += norm[k];
        const double mean = acc / (double)(z - a);
        b.bm[bo + i] = mean;
        if (norm_mean_out) norm_mean_out[bo + i] = mean;
        t[i] = fabs((mean - b.rm[bo + i]) / b.rs[bo + i]);
    }
    if (norm_signal_out) {
        double *o = norm_signal_out + b.raw_off[r];
        const int nn = s.n_norm;
        for (int k = threadIdx.x; k < nn; k += ST_THREADS)
            o[k] = rescale ? (norm[k] - shc) / scc : norm[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) s.score = tb2_pairwise_sum(t, nb) / (double)nb;
}

