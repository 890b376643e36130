// dp_row.cuh -- warp-per-read banded dynamic programming engine.
//
// One warp owns one read.  A band row (W cells, fp64) is split into 32
// contiguous chunks, one per lane; the row lives in shared memory in a
// lane-transposed layout (cell j -> buf[(j % chunk) * 32 + j / chunk]) so that
// the lanes' serial walks are bank-conflict free.
//
// Exactness (SURVEY.md s7 hard parts 1,2): the reference recurrence
//     x_j = max_tie( (x_{j-1} - stay_pen) + z_j ,  diag_j , skip_j )
// (_c_dynamic_programming.pyx:213-234) is a serial chain inside a row.  We do
// NOT re-associate it.  Every lane first walks its chunk speculatively with an
// unknown left neighbour (x_in = -inf), then lanes whose true x_in (the left
// lane's last cell) differs re-walk their prefix until the recomputed value is
// bit-identical to the stored one.  f_j is monotone in x_{j-1}, so from the first
// bit-identical cell on the speculative suffix is exactly what the serial
// reference computes; rounds repeat until no lane's input changed (<= 32, usually
// 2).  Every cell is evaluated with the reference's fp64 operations in the
// reference's order, so fwd values, move codes and arg-max are bit-exact.
#pragma once
#include "common.cuh"

struct DpConsts {
    double z_shift, stay_pen, skip_pen, mhz;
    int winsor;
};

// how to evaluate the shifted z-score of band cell j of one row
struct RowSpec {
    const double *em;    // event means (index e0 + j)
    const double *zrow;  // explicit z-scores of this row (mirror API) or nullptr
    double mu, sd;
    tb2_rcp inv_sd;      // reciprocal of sd (tb2_div_by)
    int e0;              // event index of band position 0 (may be negative)
    int lo, hi;          // cells outside [lo, hi) hold maskval
    double maskval;
};

__device__ __forceinline__ double tb2_zscore(const RowSpec &rs, const DpConsts &c, int j)
{
    if (rs.zrow) return rs.zrow[j];
    if (j < rs.lo || j >= rs.hi) return rs.maskval;
    // z_shift - min(max_half_z, |ev - mean| / sd)
    // (_c_dynamic_programming.pyx:366-372; resquiggle.py:574-582)
    double a = tb2_div_by(fabs(__ldg(rs.em + (rs.e0 + j)) - rs.mu), rs.sd, rs.inv_sd);
    if (c.winsor) a = (c.mhz < a) ? c.mhz : a;
    return c.z_shift - a;
}

// One lane walks its chunk left to right.  FIX=false: speculative first walk.
// FIX=true: re-walk from the true left input until bit-identical.
template <int WPL, bool FIX>
__device__ __forceinline__ void tb2_walk(const double *prev, double *cur, int W, int chunk,
                                         int lane, int nvalid, const RowSpec &rs,
                                         const DpConsts &c, int d, bool first_skip, double x,
                                         uint32_t (&codes)[WPL], double &best, int &best_idx,
                                         double &x_end)
{
    const int j0 = lane * chunk;
    int p = j0 + d;  // previous-row band position under cell j (skip source)
    int lane_p = p / chunk;
    int i_p = p - lane_p * chunk;
    double pm1 = tb2_neg_inf();  // previous-row value at p-1 (diag source)
    if (p >= 1 && p - 1 < W) {
        const int q = p - 1, lq = q / chunk;
        pm1 = prev[(q - lq * chunk) * 32 + lq];
    }
    bool done = false;
#pragma unroll
    for (int w = 0; w < WPL; ++w) {
        const int ibeg = w * 16;
        const int iend = min(nvalid, ibeg + 16);
        uint32_t cw = FIX ? codes[w] : 0u;
        for (int i = ibeg; i < iend && !done; ++i) {
            const int j = j0 + i;
            const double z = tb2_zscore(rs, c, j);
            const double pv = (p < W) ? prev[i_p * 32 + lane_p] : tb2_neg_inf();
            double nx;
            uint32_t code;
            if (j == 0) {
                // band position 0: skip if the band did not move, else diag
                // (_c_dynamic_programming.pyx:261-270, 393-401); never a stay
                if (first_skip) { nx = pv - c.skip_pen; code = 1u; }
                else { nx = pm1 + z; code = 2u; }
            } else {
                const double a = (x - c.stay_pen) + z;   // stay  (code 0)
                double cc = pm1 + z;                     // diag  (code 2)
                uint32_t cf = 2u;
                const double sk = pv - c.skip_pen;       // skip  (code 1)
                if (sk > cc) { cc = sk; cf = 1u; }
                if (cc > a) { nx = cc; code = cf; }
                else { nx = a; code = 0u; }
            }
            const int sh = 2 * (i - ibeg);
            if (FIX) {
                const double old = cur[i * 32 + lane];
                cw = (cw & ~(3u << sh)) | (code << sh);
                if (nx == old) done = true;
            } else {
                cw |= code << sh;
            }
            cur[i * 32 + lane] = nx;
            if (nx > best || (FIX && nx == best && j < best_idx)) { best = nx; best_idx = j; }
            x = nx;
            pm1 = pv;
            ++p;
            if (++i_p == chunk) { i_p = 0; ++lane_p; }
        }
        codes[w] = cw;
    }
    if (!done && nvalid > 0) x_end = x;
}

// One band row for the whole warp.  On return cur holds the row, codes the 2-bit
// moves of this lane's chunk, (best, best_idx) this lane's first arg-max.
template <int WPL>
__device__ __forceinline__ void tb2_dp_row(const double *prev, double *cur, int W, int chunk,
                                           int lane, const RowSpec &rs, const DpConsts &c,
                                           int d, bool first_skip, uint32_t (&codes)[WPL],
                                           double &best, int &best_idx)
{
    const int nvalid = max(0, min(chunk, W - lane * chunk));
    best = tb2_neg_inf();
    best_idx = 0x7fffffff;
    double x_end = tb2_neg_inf();
    tb2_walk<WPL, false>(prev, cur, W, chunk, lane, nvalid, rs, c, d, first_skip, tb2_neg_inf(),
                         codes, best, best_idx, x_end);
    double last_in = tb2_neg_inf();
    for (;;) {
        const double xin = __shfl_up_sync(TB2_FULL_MASK, x_end, 1);
        const bool need = (lane > 0) && (nvalid > 0) && (xin != last_in);
        if (!__any_sync(TB2_FULL_MASK, need)) break;
        if (need) {
            tb2_walk<WPL, true>(prev, cur, W, chunk, lane, nvalid, rs, c, d, first_skip, xin,
                                codes, best, best_idx, x_end);
            last_in = xin;
        }
    }
}

// warp arg-max with first-maximum semantics (c_argmax :186-197, np.argmax)
__device__ __forceinline__ int tb2_warp_argmax(double best, int best_idx)
{
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const double ob = __shfl_xor_sync(TB2_FULL_MASK, best, off);
        const int oi = __shfl_xor_sync(TB2_FULL_MASK, best_idx, off);
        if (ob > best || (ob == best && oi < best_idx)) { best = ob; best_idx = oi; }
    }
    return best_idx;
}

// ---------------------------------------------------------------------------
// Fast row for band widths <= 512 (chunk <= 16 cells per lane, one move word) with
// both row buffers in shared memory -- the adaptive band of real reads (bandwidth
// 200-500).  Same arithmetic as tb2_dp_row; the z-scores and the best
// diag/skip candidate of every cell stay in registers, so the re-walks that fix the
// speculation cost one add and one compare per cell instead of a division and two
// shared-memory reads.
// ---------------------------------------------------------------------------
// tuning counters of the lane-chunk engine: [0] rows, [1] fix-up rounds, [2] cells
// re-walked, [3] rows that needed more than 2 rounds
__device__ unsigned long long g_tb2_dp_counters[8];

#ifdef TB2_EMUL
__device__ __forceinline__ double tb2_lds(unsigned a) { return *(double *)emul_shared_ptr(a); }
__device__ __forceinline__ void tb2_sts(unsigned a, double v) { *(double *)emul_shared_ptr(a) = v; }
#else
__device__ __forceinline__ double tb2_lds(unsigned a)
{
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void tb2_sts(unsigned a, double v)
{
    asm volatile("st.shared.f64 [%0], %1;" ::"r"(a), "d"(v));
}
#endif

// prev_s / cur_s / z_s / c_s: shared-memory byte addresses of four lane-transposed
// row buffers (previous row, current row, z-scores, best diag/skip candidate)
__device__ __forceinline__ void tb2_dp_row_s(unsigned prev_s, unsigned cur_s, unsigned z_s,
                                             unsigned c_s, int W, int chunk, int lane,
                                             const RowSpec &rs, const DpConsts &c, int d,
                                             bool first_skip, uint32_t &codeword, double &best,
                                             int &best_idx)
{
    const double NEG = tb2_neg_inf();
    const double stay = c.stay_pen, skip = c.skip_pen;
    const int j0 = lane * chunk;
    const int nvalid = max(0, min(chunk, W - j0));
    const unsigned lo8 = 8u * (unsigned)lane;
    cur_s += lo8; z_s += lo8; c_s += lo8;
    uint32_t cfw = 0u, cw = 0u;
    int p = j0 + d;
    int lane_p = p / chunk;
    int i_p = p - lane_p * chunk;
    double pm1 = NEG;
    if (p >= 1 && p - 1 < W) {
        const int q = p - 1, lq = q / chunk;
        pm1 = tb2_lds(prev_s + 8u * (unsigned)((q - lq * chunk) * 32 + lq));
    }
    double x = NEG;
    best = NEG;
    best_idx = 0x7fffffff;
#pragma unroll 1
    for (int i = 0; i < nvalid; ++i) {
        const int j = j0 + i;
        const double zz = tb2_zscore(rs, c, j);
        const double pv = (p < W) ? tb2_lds(prev_s + 8u * (unsigned)(i_p * 32 + lane_p)) : NEG;
        double cand = pm1 + zz;               // diag (code 2)
        uint32_t cf = 2u;
        const double sk = pv - skip;          // skip (code 1)
        double a;
        if (j == 0) {
            // band position 0: skip if the band did not move, else diag; no stay
            a = NEG;
            if (first_skip) { cand = sk; cf = 1u; }
        } else {
            if (sk > cand) { cand = sk; cf = 1u; }
            a = (x - stay) + zz;              // stay (code 0)
        }
        double nx = a;
        uint32_t code = 0u;
        if (cand > a) { nx = cand; code = cf; }
        const unsigned off = 256u * (unsigned)i;
        tb2_sts(z_s + off, zz);
        tb2_sts(c_s + off, cand);
        tb2_sts(cur_s + off, nx);
        cfw |= cf << (2 * i);
        cw |= code << (2 * i);
        if (nx > best) { best = nx; best_idx = j; }
        x = nx;
        pm1 = pv;
        ++p;
        if (++i_p == chunk) { i_p = 0; ++lane_p; }
    }
    double x_end = x;
    double last_in = NEG;
    int n_rounds = 0, n_walked = 0;
    for (;;) {
        const double xin = __shfl_up_sync(TB2_FULL_MASK, x_end, 1);
        const bool need = (lane > 0) && (nvalid > 0) && (xin != last_in);
        if (!__any_sync(TB2_FULL_MASK, need)) break;
        ++n_rounds;
        if (need) {
            double xx = xin;
            bool done = false;
#pragma unroll 1
            for (int i = 0; i < nvalid; ++i) {
                ++n_walked;
                const unsigned off = 256u * (unsigned)i;
                const double a = (xx - stay) + tb2_lds(z_s + off);
                const double cand = tb2_lds(c_s + off);
                double nx = a;
                uint32_t code = 0u;
                if (cand > a) { nx = cand; code = (cfw >> (2 * i)) & 3u; }
                const double old = tb2_lds(cur_s + off);
                cw = (cw & ~(3u << (2 * i))) | (code << (2 * i));
                const int j = j0 + i;
                if (nx > best || (nx == best && j < best_idx)) { best = nx; best_idx = j; }
                xx = nx;
                if (nx == old) { done = true; break; }
                tb2_sts(cur_s + off, nx);
            }
            if (!done) x_end = xx;
            last_in = xin;
        }
    }
    codeword = cw;
#ifdef TB2_DP_COUNTERS   // tuning build only: four contended global atomics per row
    n_walked = __reduce_add_sync(TB2_FULL_MASK, n_walked);
    if (lane == 0) {
        atomicAdd(&g_tb2_dp_counters[0], 1ULL);
        atomicAdd(&g_tb2_dp_counters[1], (unsigned long long)n_rounds);
        atomicAdd(&g_tb2_dp_counters[2], (unsigned long long)n_walked);
        if (n_rounds > 2) atomicAdd(&g_tb2_dp_counters[3], 1ULL);
    }
#else
    (void)n_rounds; (void)n_walked;
#endif
}

// ---------------------------------------------------------------------------
// Pass description: a run of consecutive rows sharing one band width.
// ---------------------------------------------------------------------------
enum { TB2_MODE_PLAIN = 0, TB2_MODE_MASKED = 1, TB2_MODE_ADAPTIVE = 2, TB2_MODE_EXPLICIT = 3 };

struct PassCtx {
    // geometry
    int W, chunk;
    // row buffers (lane-transposed, >= chunk*32 doubles each)
    double *buf0, *buf1;
    double *zbuf, *cbuf;     // optional: z-score / candidate rows (fast adaptive path)
    // inputs
    const double *em;   // event means (already offset by events_start_clip)
    int n_em;
    const double *rm, *rs_;  // reference levels per base
    const double *zmat;      // EXPLICIT mode: n_rows x W z-scores
    // masked-start parameters (resquiggle.py:607-683)
    int mso;                 // mapped_start_offset
    double msp_start, msp_stop;  // mask_start_pos = linspace(msp_start, msp_stop, MASK_BASES)
    double mask_shifted;     // (mask_fill - z_shift) + z_shift
    double mask_fill;        // MASK_FILL_Z_SCORE (adaptive padding)
    // outputs
    int *starts;             // band event starts per base (global)
    uint32_t *tb;            // packed moves: row r at tb[r * wpl * 32 + w * 32 + lane]
    double *ring;            // TB2_WF_RING doubles of shared memory (wavefront exchange) or null
    // mirror-API dumps (may be null)
    double *dbg_fwd;         // (n_bases + 1) x W
    long long *dbg_tb;       // (n_bases + 1) x W
};

#define TB2_MASK_BASES 50

// Runs rows [r_begin, r_end).  `prev` must hold fwd row r_begin on entry (buf
// selected by *cur_sel), starts[r_begin-1] valid if r_begin > 0.  Returns status
// (TB2_OK or TB2_ERR_ADAPTIVE_BEYOND_SIGNAL); on return *cur_sel selects the
// buffer holding fwd row r_end and (best_idx_out) its first arg-max.
template <int WPL>
__device__ __noinline__ int tb2_run_rows(const PassCtx &pc, const DpConsts &c, int mode, int r_begin,
                            int r_end, int n_bases_total, int *cur_sel, int *argmax_out)
{
    const int lane = tb2_lane();
    const int W = pc.W, chunk = pc.chunk;
    double *prev = (*cur_sel) ? pc.buf1 : pc.buf0;
    double *cur = (*cur_sel) ? pc.buf0 : pc.buf1;
    int last_argmax = *argmax_out;
    // fast path: four row buffers in shared memory (rows, z-scores, candidates)
    const bool fast_s = (pc.zbuf != nullptr) && __isShared(pc.buf0);
    const unsigned z_s = fast_s ? (unsigned)__cvta_generic_to_shared(pc.zbuf) : 0u;
    const unsigned c_s = fast_s ? (unsigned)__cvta_generic_to_shared(pc.cbuf) : 0u;
    int prev_start = (r_begin > 0) ? pc.starts[r_begin - 1] : 0;
    const int half_bw = W / 2;
    for (int r = r_begin; r < r_end; ++r) {
        RowSpec rs;
        rs.em = pc.em; rs.zrow = nullptr;
        rs.mu = pc.rm ? __ldg(pc.rm + r) : 0.0;
        rs.sd = pc.rs_ ? __ldg(pc.rs_ + r) : 1.0;
        rs.inv_sd = tb2_rcp_of(rs.sd);
        rs.lo = 0; rs.hi = W; rs.maskval = pc.mask_fill;
        int cur_start;
        if (mode == TB2_MODE_ADAPTIVE) {
            // _c_dynamic_programming.pyx:344-358
            cur_start = prev_start + last_argmax - half_bw + 1;
            if (cur_start < prev_start) cur_start = prev_start;
            if (cur_start >= pc.n_em) {
                if (r < n_bases_total - 2) return TB2_ERR_ADAPTIVE_BEYOND_SIGNAL;
                cur_start = pc.n_em - 1;
            }
            if (lane == 0) pc.starts[r] = cur_start;
            rs.hi = min(W, pc.n_em - cur_start);
        } else {
            cur_start = pc.starts[r];
            if (mode == TB2_MODE_MASKED) {
                // get_start_mask_z_score resquiggle.py:647-673 (validated by caller)
                const int sml = max(pc.mso - cur_start, 0);
                int eml = 0;
                if (r < TB2_MASK_BASES) {
                    const int msp = (int)tb2_linspace_at(pc.msp_start, pc.msp_stop,
                                                         TB2_MASK_BASES, r);
                    eml = W - (msp - cur_start);
                }
                if (cur_start + W - eml > pc.n_em) eml = cur_start + W - pc.n_em;
                rs.lo = sml; rs.hi = W - eml; rs.maskval = pc.mask_shifted;
            } else if (mode == TB2_MODE_EXPLICIT) {
                rs.zrow = pc.zmat + (size_t)r * W;
            }
        }
        rs.e0 = cur_start;
        const int d = (r > 0) ? cur_start - prev_start : 0;
        const bool first_skip = (r == 0) || (d == 0);
        uint32_t codes[WPL];
        double best; int best_idx;
        if (WPL == 1 && fast_s)
            tb2_dp_row_s((unsigned)__cvta_generic_to_shared(prev), (unsigned)__cvta_generic_to_shared(cur),
                         z_s, c_s, W, chunk, lane, rs, c, d, first_skip, codes[0], best, best_idx);
        else
            tb2_dp_row<WPL>(prev, cur, W, chunk, lane, rs, c, d, first_skip, codes, best, best_idx);
#pragma unroll
        for (int w = 0; w < WPL; ++w)
            pc.tb[(size_t)r * (WPL * 32) + w * 32 + lane] = codes[w];
        if (mode == TB2_MODE_ADAPTIVE || r == r_end - 1 || r == n_bases_total - 1)
            last_argmax = tb2_warp_argmax(best, best_idx);
        __syncwarp();
        if (pc.dbg_fwd) {
            const int nvalid = max(0, min(chunk, W - lane * chunk));
            for (int i = 0; i < nvalid; ++i) {
                const int j = lane * chunk + i;
                pc.dbg_fwd[(size_t)(r + 1) * W + j] = cur[i * 32 + lane];
                uint32_t cwv = codes[0];
#pragma unroll
                for (int k = 1; k < WPL; ++k) if ((i >> 4) == k) cwv = codes[k];
                pc.dbg_tb[(size_t)(r + 1) * W + j] = (cwv >> (2 * (i & 15))) & 3u;
            }
        }
        double *t = prev; prev = cur; cur = t;
        *cur_sel ^= 1;
        prev_start = cur_start;
    }
    *argmax_out = last_argmax;
    return TB2_OK;
}

// fwd row 0 = zeros (_c_dynamic_programming.pyx:253-254)
__device__ __forceinline__ void tb2_init_row0(const PassCtx &pc, int *cur_sel)
{
    const int lane = tb2_lane();
    for (int i = 0; i < pc.chunk; ++i) pc.buf0[i * 32 + lane] = 0.0;
    *cur_sel = 0;
    __syncwarp();
}

// load an explicit fwd row (mirror API of the in-place adaptive pass)
__device__ __forceinline__ void tb2_load_row(const PassCtx &pc, const double *row, int *cur_sel)
{
    const int lane = tb2_lane();
    for (int j = lane; j < pc.W; j += 32) {
        const int lj = j / pc.chunk;
        pc.buf0[(j - lj * pc.chunk) * 32 + lj] = row[j];
    }
    *cur_sel = 0;
    __syncwarp();
}

// ---------------------------------------------------------------------------
// Traceback (c_banded_traceback _c_dynamic_programming.pyx:281-310), warp
// cooperative: every lane loads its own packed words of a row (coalesced, position
// independent, four rows in flight), cells are fetched with shuffles.
// ---------------------------------------------------------------------------
template <int WPL>
__device__ __forceinline__ uint32_t tb2_tb_code(const uint32_t (&w)[WPL], int bp, int chunk)
{
    const int lj = bp / chunk;
    const int i = bp - lj * chunk;
    uint32_t v = w[0];
#pragma unroll
    for (int k = 1; k < WPL; ++k) if ((i >> 4) == k) v = w[k];
    v = __shfl_sync(TB2_FULL_MASK, v, lj);
    return (v >> (2 * (i & 15))) & 3u;
}

// rows [row_lo, row_hi) in the lane-chunk layout; cur_event carried in and out
template <int WPL>
__device__ __noinline__ int tb2_tb_seg_chunk(const uint32_t *tb, const int *starts, int row_hi, int row_lo,
                                int W, int chunk, int thresh, int *cur_event_io, int *read_tb)
{
    const int lane = tb2_lane();
    int cur_event = *cur_event_io;
    int sp = row_hi;
    while (sp > row_lo) {
        const int nblk = min(4, sp - row_lo);
        uint32_t w[4][WPL];
        int st[4];
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            if (b < nblk) {
                const int row = sp - 1 - b;
#pragma unroll
                for (int k = 0; k < WPL; ++k)
                    w[b][k] = tb[(size_t)row * (WPL * 32) + k * 32 + lane];
                st[b] = starts[row];
            }
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            if (b < nblk) {
                int bp = cur_event - st[b];
                if (bp < 0 || bp >= W) return TB2_ERR_UNEXPECTED;
                uint32_t code = tb2_tb_code<WPL>(w[b], bp, chunk);
                while (code == 0u) {  // 0: stay in the current base
                    --bp;
                    if (bp < 0) return TB2_ERR_UNEXPECTED;
                    code = tb2_tb_code<WPL>(w[b], bp, chunk);
                }
                if (code == 2u) --bp;  // diagonal
                if (thresh >= 0 && min(bp, W - bp - 1) < thresh)
                    return TB2_ERR_BEYOND_BANDWIDTH;
                cur_event = st[b] + bp;
                if (lane == 0) read_tb[sp - 1 - b] = cur_event + 1;
            }
        }
        sp -= nblk;
    }
    *cur_event_io = cur_event;
    __syncwarp();
    return TB2_OK;
}

// ===========================================================================
// Wavefront engine for STATIC bands (band starts known up front: short-read
// static band, start search, masked start, mirror API).
//
// Lane L of a 32-row strip owns row s0+L and walks its band left to right; at
// step t it handles event e = t - L, so the cell above (row-1, e) was produced by
// lane L-1 one step earlier and arrives by a single shuffle, and (row-1, e-1) is
// the value received the step before.  Every cell is evaluated exactly once with
// the reference's operations (no speculation, no re-association): bit-exact by
// construction.  Strips are chained through one row buffer in shared memory
// (writes of the strip's last row trail the reads of its first row by >= 31
// cells).  Event means are read coalesced (32 consecutive events per step).
//
// Moves: 2 bits/cell packed in STEP space: word (strip, k, lane) holds lane's moves
// of steps t_begin + 16k .. +15 at  tb[strip_base + k * 32 + lane]  -- every 16
// steps the warp stores one coalesced 128-byte line, and a traceback path crossing
// a strip touches a handful of lines.  Strip sizes follow from the band starts
// (tb2_wf_strip_words), so forward pass and traceback agree without a table.
// ===========================================================================
__device__ __forceinline__ int tb2_wf_strip_words(const int *starts, int s0, int r_end, int W)
{
    const int last = min(31, r_end - 1 - s0);
    const int span = starts[s0 + last] - starts[s0] + W - 1 + last;   // t_end - t_begin
    return span < 0 ? -1 : ((span >> 4) + 1) * 32;
}

// total packed-move words of a wavefront pass over rows [0, r_end); -1 for band
// starts that move left by more than the strip skew can follow
__device__ long long tb2_wf_total_words(const int *starts, int r_end, int W)
{
    long long sum = 0;
    int bad = 0;
    for (int s0 = tb2_lane() * 32; s0 < r_end; s0 += 32 * 32) {
        const int w = tb2_wf_strip_words(starts, s0, r_end, W);
        if (w < 0) bad = 1; else sum += w;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(TB2_FULL_MASK, sum, off);
    return __any_sync(TB2_FULL_MASK, bad) ? -1 : sum;
}

// shifted z-score of one cell for the wavefront engine, from its event mean m (not read
// for a masked cell).  The divide is the exact reciprocal form (tb2_div_by): inv_sd =
// tb2_rcp_of(sd) once per row.
template <int MODE, bool WIN>
__device__ __forceinline__ double tb2_wf_z_of(double m, int j, double mu, double sd,
                                              tb2_rcp inv_sd, int lo, int hi, double maskval,
                                              double zs, double mhz)
{
    if (MODE == TB2_MODE_MASKED && (j < lo || j >= hi)) return maskval;
    double a = tb2_div_by(fabs(m - mu), sd, inv_sd);
    if (WIN) a = (mhz < a) ? mhz : a;
    return zs - a;
}

// the same with the event mean (or the explicit z-score) read here
template <int MODE, bool WIN>
__device__ __forceinline__ double tb2_wf_z(const double *ep, int j, double mu, double sd,
                                           tb2_rcp inv_sd, int lo, int hi, double maskval,
                                           const double *zrow, double zs, double mhz)
{
    if (MODE == TB2_MODE_EXPLICIT) return zrow[j];
    if (MODE == TB2_MODE_MASKED && (j < lo || j >= hi)) return maskval;
    return tb2_wf_z_of<MODE, WIN>(__ldg(ep), j, mu, sd, inv_sd, lo, hi, maskval, zs, mhz);
}

// strip-chaining row buffer: shared-memory accesses when it lives in shared memory
template <bool RBS>
__device__ __forceinline__ double tb2_rb_ld(const double *rb, unsigned rb_s, int i)
{
    if (RBS) return tb2_lds(rb_s + 8u * (unsigned)i);
    return rb[i];
}
template <bool RBS>
__device__ __forceinline__ void tb2_rb_st(double *rb, unsigned rb_s, int i, double v)
{
    if (RBS) tb2_sts(rb_s + 8u * (unsigned)i, v);
    else rb[i] = v;
}

// move word of one lane over 16 steps: bit q = "step q left the stay candidate behind",
// bit 16 + q = "its skip candidate beat the diagonal one" (meaningful when bit q is set):
// stay = 0x, diagonal = 01 (code 2), skip = 11 (code 1).  The steady state sets the two bits
// straight from its two compare predicates.
#define TB2_WF_MOVE_BITS(code, q) ((((code) != 0u ? 1u : 0u) << (q)) | (((code) == 1u ? 0x10000u : 0u) << (q)))

// one steady-state step (U = position inside the 16-step group).  Neighbouring lanes
// exchange the row above through a 48-slot ring in shared memory laid out on the
// diagonal: lane l stores its cell of step U at slot l + U and lane l + 1 loads it at step
// U + 1 from (l + 1) - 2 + (U + 1), so both addresses are "per-lane base + 8 * U" and fold
// into the instruction.  Lane 0 runs its load pointer along the chaining row instead (the
// tail row of the previous strip) and the tail lane runs its store pointer along it, which
// removes every predicate and register shuffle of the exchange.  Step 0 of a group takes
// the cell above by a shuffle (the ring only spans one group).  Within a group slot s is
// written at step U by lane s - U alone, read by lane s - U + 1 at step U + 1 and
// overwritten by lane s - U - 1 later in that same step: one __syncwarp() after the load
// and one after the store order the three (each compiles to a NOP in this converged loop).
//
// The event means are software-pipelined TB2_WF_MD = 3 steps deep: step U reads the mean of
// step U + 3 into m2 and turns the mean of step U + 1, which is already in m1, into the
// z-score of step U + 1, so that chain does not depend on step U's recurrence.  Every cell
// gets the z-score tb2_wf_z would give it, with the same operations in the same order.  At 64
// registers ptxas still schedules each load 16-32 instructions ahead of its first use (7-10
// without the pipeline) and the z-score chain next to the recurrence that consumes it.
// Loads that fall into the next group read from epn, which is ep + 16 when that group runs
// and ep (this group's own first steps, whose means are then simply not used) when it does
// not, and a masked row loads only unmasked cells: no address outside what the loop reads is
// touched, and no predicate stays live across the group.
#define TB2_WF_MD 3
#define TB2_WF_MLD(m, K)                                                                        \
    if (MODE != TB2_MODE_MASKED ||                                                              \
        (unsigned)(((K) < 16 ? j + (K) : j + nadv + (K) - 16) - lo) < (unsigned)(hi - lo))      \
        m = __ldg(((K) < 16 ? ep : epn) + ((K) < 16 ? (K) : (K) - 16));
#ifdef TB2_EMUL
#define TB2_WF_PLD(up, U) if (l0flag) up = tb2_lds(rd_a + 8 * (U));
#else
#define TB2_WF_PLD(up, U)                                                                       \
        asm volatile("{ .reg .pred p; setp.ne.u32 p, %2, 0; @p ld.shared.f64 %0, [%1+%3]; }"    \
                     : "+d"(up) : "r"(rd_a), "r"(l0flag), "n"(8 * (U)));
#endif
#define TB2_WF_FAST_STEP(U)                                                                     \
    {                                                                                           \
        const double mz = m1;                       /* mean of step U + 1 (arrived)  */       \
        m1 = m2;                                    /* mean of step U + 2 (in flight) */       \
        TB2_WF_MLD(m2, (U) + TB2_WF_MD)             /* mean of step U + 3             */       \
        double up;                                                                              \
        if ((U) == 0) {                                                                         \
            up = __shfl_up_sync(TB2_FULL_MASK, xout, 1);                                        \
            TB2_WF_PLD(up, U)                                                                   \
        } else up = tb2_lds(rd_a + 8u * (U));                                                   \
        __syncwarp();                                                                           \
        const double zn = tb2_wf_z_of<MODE, WIN>(mz, j + (U) + 1, mu, sd, inv_sd, lo, hi,       \
                                                 maskval, zs, mhz);                             \
        const double a = (x - stay) + z;                                                        \
        double cc = up_prev + z;                                                                \
        const double sk = up - skip;                                                            \
        if (sk > cc) { cc = sk; cw |= 0x10000u << (U); }                                        \
        double nx = a;                                                                          \
        if (cc > a) { nx = cc; cw |= 1u << (U); }                                               \
        up_prev = up;                                                                           \
        x = nx; xout = nx; z = zn;                                                              \
        tb2_sts(wr_a + 8u * (U), nx);                                                           \
        __syncwarp();                                                                           \
    }

template <int MODE, bool DBG, bool WIN, bool RBS>
__device__ __noinline__ int tb2_wavefront_rows_t(const PassCtx &pc, const DpConsts &c, int r_end,
                                                 double *rowbuf, uint32_t *tbw, int *argmax_out)
{
    const int lane = tb2_lane();
    const int W = pc.W;
    const double NEG = tb2_neg_inf();
    const double stay = c.stay_pen, skip = c.skip_pen, zs = c.z_shift, mhz = c.mhz;
    const unsigned rb_s = RBS ? (unsigned)__cvta_generic_to_shared(rowbuf) : 0u;
    const unsigned ring_s = (RBS && pc.ring) ? (unsigned)__cvta_generic_to_shared(pc.ring) : 0u;
    const double *em = pc.em;
    const int *starts = pc.starts;
    // the steady state is only built for the production modes with the row buffer in
    // shared memory; its first strip reads "the row above row 0" as zeros
    constexpr bool FAST_T = RBS && !DBG && MODE != TB2_MODE_EXPLICIT;
    const bool FAST = FAST_T && pc.ring != nullptr;
    if (FAST) {
        for (int jj = lane; jj < W; jj += 32) tb2_rb_st<RBS>(rowbuf, rb_s, jj, 0.0);
        __syncwarp();
    }
    uint32_t *tbs = tbw;
    for (int s0 = 0; s0 < r_end; s0 += 32) {
        const int r = s0 + lane;
        const bool row_ok = r < r_end;
        const int lane_last = min(31, r_end - 1 - s0);
        // lanes past the last row of a partial strip mirror that row (inactive in the
        // predicated steps, harmless passengers in the steady state)
        const int rr = min(r, r_end - 1);
        const int start = starts[rr];
        const int prev_start = rr > 0 ? starts[rr - 1] : start;
        const int d = start - prev_start;
        const double mu = pc.rm ? __ldg(pc.rm + rr) : 0.0;
        const double sd = pc.rs_ ? __ldg(pc.rs_ + rr) : 1.0;
        const tb2_rcp inv_sd = tb2_rcp_of(sd);
        int lo = 0, hi = W;
        double maskval = pc.mask_fill;
        if (MODE == TB2_MODE_MASKED && row_ok) {
            const int sml = max(pc.mso - start, 0);
            int eml = 0;
            if (r < TB2_MASK_BASES)
                eml = W - ((int)tb2_linspace_at(pc.msp_start, pc.msp_stop, TB2_MASK_BASES, r) - start);
            if (start + W - eml > pc.n_em) eml = start + W - pc.n_em;
            lo = sml; hi = W - eml; maskval = pc.mask_shifted;
        }
        const double *zrow = (MODE == TB2_MODE_EXPLICIT && row_ok) ? pc.zmat + (size_t)r * W : nullptr;
        const bool first_skip = (r == 0) || (d == 0);
        const bool is_tail = row_ok && (lane == lane_last);       // feeds the next strip
        // uniform time bounds of the strip
        const int start_first = __shfl_sync(TB2_FULL_MASK, start, 0);
        const int start_last = __shfl_sync(TB2_FULL_MASK, start, lane_last);
        int dmax = row_ok ? d : 0, dmin = row_ok ? d : 0;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            dmax = max(dmax, __shfl_xor_sync(TB2_FULL_MASK, dmax, off));
            dmin = min(dmin, __shfl_xor_sync(TB2_FULL_MASK, dmin, off));
        }
        // predicated ("lean") steps and the steady state need band starts that never
        // move left; anything else takes the fully general step
        const bool lean = FAST && dmin >= 0;
        const int t_begin = start_first;
        const int t_end = start_last + W - 1 + lane_last;
        // steady state: every lane of a full strip is inside its band with j >= 1 and
        // both cells of the row above available
        int t_lo = start_last + lane_last + 1, t_hi = start_first + W - 2 - dmax;
        if (!lean) { t_lo = t_end + 1; t_hi = t_end; }   // general path only
        double x = 0.0, xout = 0.0, up_prev = 0.0;
        uint32_t cw = 0u;
        const int lane_eff = min(lane, lane_last);
        int j = t_begin - lane_eff - start;
        const double *ep = em + (t_begin - lane_eff);
        int t = t_begin;
        // ---------- lean step: every band-edge rule of the general step folded into
        // three range tests (row active, cell above valid, cell above-left valid); the
        // first cell of a row falls out of x = -inf (stay impossible) and of the ranges:
        // d == 0 -> above-left invalid -> forced skip, d >= 1 -> above invalid at j = 0 ->
        // forced diagonal, exactly as _c_dynamic_programming.pyx:213-234 ----------
        const int w_act = row_ok ? W : 0;
        const int julo = d >= 1 ? 1 : 0, jllo = 1 - julo;
        const unsigned n_u = (unsigned)max(W - d - julo, 0), n_ul = (unsigned)max(W - d - jllo + 1, 0);
#define TB2_WF_LEAN_STEP()                                                                      \
        {                                                                                       \
            double up = __shfl_up_sync(TB2_FULL_MASK, xout, 1);                                 \
            if (lane == 0 && (unsigned)(j + d) < (unsigned)W) up = tb2_rb_ld<RBS>(rowbuf, rb_s, j + d); \
            const double upl = up_prev;                                                         \
            up_prev = up;                                                                       \
            const bool act = (unsigned)j < (unsigned)w_act;                                     \
            const double u = ((unsigned)(j - julo) < n_u) ? up : NEG;                           \
            const double ul = ((unsigned)(j - jllo) < n_ul) ? upl : NEG;                        \
            const double z = act ? tb2_wf_z<MODE, WIN>(ep, j, mu, sd, inv_sd, lo, hi, maskval,  \
                                                       zrow, zs, mhz) : 0.0;                    \
            const double a = (x - stay) + z;                                                    \
            double cc = ul + z;                                                                 \
            uint32_t code = 2u;                                                                 \
            const double sk = u - skip;                                                         \
            if (sk > cc) { cc = sk; code = 1u; }                                                \
            double nx = a;                                                                      \
            if (cc > a) nx = cc; else code = 0u;                                                \
            const int tq = (t - t_begin) & 15;                                                  \
            if (act) {                                                                          \
                x = nx; xout = nx;                                                              \
                cw |= TB2_WF_MOVE_BITS(code, tq);                                               \
                if (is_tail) tb2_rb_st<RBS>(rowbuf, rb_s, j, nx);                               \
            }                                                                                   \
            if (tq == 15 || t == t_end) {                                                       \
                tbs[((t - t_begin) >> 4) * 32 + lane] = cw;                                     \
                cw = 0u;                                                                        \
            }                                                                                   \
            /* lane 0 reads the chaining row, the tail lane rewrites it a few cells behind  */  \
            /* (one cell behind in a two-row strip): a barrier per step orders each pair    */  \
            __syncwarp();                                                                       \
            ++j; ++ep;                                                                          \
        }
        if (lean) {
            x = NEG;
            if (lane == 0 && d >= 1) up_prev = tb2_rb_ld<RBS>(rowbuf, rb_s, d - 1);
            for (; t <= t_end && (t < t_lo || ((t - t_begin) & 15) != 0); ++t) TB2_WF_LEAN_STEP()
        }
        // ---------- general step (prologue / epilogue / partial strips) ----------
#define TB2_WF_GENERAL_STEP()                                                                   \
        {                                                                                       \
            double up = __shfl_up_sync(TB2_FULL_MASK, xout, 1);                                 \
            const int p = j + d;                                                                \
            double upl = up_prev;                                                               \
            if (lane == 0) {                                                                    \
                if (s0 == 0) { up = 0.0; upl = 0.0; }                                           \
                else {                                                                          \
                    up = (p >= 0 && p < W) ? tb2_rb_ld<RBS>(rowbuf, rb_s, p) : NEG;             \
                    if (j == 0) upl = (p >= 1 && p - 1 < W) ? tb2_rb_ld<RBS>(rowbuf, rb_s, p - 1) : NEG; \
                }                                                                               \
            }                                                                                   \
            up_prev = up;                                                                       \
            const int tq = (t - t_begin) & 15;                                                  \
            if (row_ok && j >= 0 && j < W) {                                                    \
                const double z = tb2_wf_z<MODE, WIN>(ep, j, mu, sd, inv_sd, lo, hi, maskval,    \
                                                     zrow, zs, mhz);                            \
                const double u = (p < W) ? up : NEG;                                            \
                const double ul = (p >= 1 && p - 1 < W) ? upl : NEG;                            \
                double nx;                                                                      \
                uint32_t code;                                                                  \
                if (j == 0) {                                                                   \
                    if (first_skip) { nx = u - skip; code = 1u; }                               \
                    else { nx = ul + z; code = 2u; }                                            \
                } else {                                                                        \
                    const double a = (x - stay) + z;                                            \
                    double cc = ul + z;                                                         \
                    uint32_t cf = 2u;                                                           \
                    const double sk = u - skip;                                                 \
                    if (sk > cc) { cc = sk; cf = 1u; }                                          \
                    if (cc > a) { nx = cc; code = cf; }                                         \
                    else { nx = a; code = 0u; }                                                 \
                }                                                                               \
                x = nx;                                                                         \
                xout = nx;                                                                      \
                cw |= TB2_WF_MOVE_BITS(code, tq);                                               \
                if (is_tail) tb2_rb_st<RBS>(rowbuf, rb_s, j, nx);                               \
                if (DBG) {                                                                      \
                    pc.dbg_fwd[(size_t)(r + 1) * W + j] = nx;                                   \
                    pc.dbg_tb[(size_t)(r + 1) * W + j] = code;                                  \
                }                                                                               \
            }                                                                                   \
            if (!DBG && (tq == 15 || t == t_end)) {                                             \
                tbs[((t - t_begin) >> 4) * 32 + lane] = cw;                                     \
                cw = 0u;                                                                        \
            }                                                                                   \
            __syncwarp();                                                                       \
            ++j; ++ep;                                                                          \
        }
        if (lean && t + 15 <= t_hi) {
            // ---------- steady state: groups of 16 steps, no band-edge predicates, z one
            // step ahead and event means TB2_WF_MD steps ahead, one coalesced move-word
            // store per group ----------
            double z = tb2_wf_z<MODE, WIN>(ep, j, mu, sd, inv_sd, lo, hi, maskval, nullptr, zs, mhz);
            int nadv = 0;                        // the prologue stays inside the first group
            const double *epn = ep;
            double m1 = 0.0, m2 = 0.0;
            TB2_WF_MLD(m1, 1)
            TB2_WF_MLD(m2, 2)
            // lane 0 loads along the chaining row (cell above), the tail lane stores along
            // it (own cell); everyone else goes through the ring
            unsigned rd_a = lane == 0 ? rb_s + 8u * (unsigned)(j + d) : ring_s + 8u * (unsigned)(lane - 2);
            unsigned wr_a = is_tail ? rb_s + 8u * (unsigned)j : ring_s + 8u * (unsigned)lane;
            const unsigned rd_inc = lane == 0 ? 128u : 0u, wr_inc = is_tail ? 128u : 0u;
            const unsigned l0flag = lane == 0;
            uint32_t *tbp = tbs + ((t - t_begin) >> 4) * 32 + lane;
            for (; t + 15 <= t_hi; t += 16) {
                nadv = t + 31 <= t_hi ? 16 : 0;  // the next group runs: prefetch into it
                epn = ep + nadv;
                TB2_WF_FAST_STEP(0) TB2_WF_FAST_STEP(1) TB2_WF_FAST_STEP(2) TB2_WF_FAST_STEP(3)
                TB2_WF_FAST_STEP(4) TB2_WF_FAST_STEP(5) TB2_WF_FAST_STEP(6) TB2_WF_FAST_STEP(7)
                TB2_WF_FAST_STEP(8) TB2_WF_FAST_STEP(9) TB2_WF_FAST_STEP(10) TB2_WF_FAST_STEP(11)
                TB2_WF_FAST_STEP(12) TB2_WF_FAST_STEP(13) TB2_WF_FAST_STEP(14) TB2_WF_FAST_STEP(15)
                *tbp = cw;
                cw = 0u;
                tbp += 32;
                rd_a += rd_inc; wr_a += wr_inc;
                j += 16; ep += 16;
                // (the tail lane's writes to the chaining row trail lane 0's reads by >= 31
                // cells; the per-step barriers order every such pair)
            }
            cw = 0u;
        }
        if (lean) {
            for (; t <= t_end; ++t) TB2_WF_LEAN_STEP()
        } else {
            for (; t <= t_end; ++t) TB2_WF_GENERAL_STEP()
        }
#undef TB2_WF_GENERAL_STEP
#undef TB2_WF_LEAN_STEP
        tbs += (((t_end - t_begin) >> 4) + 1) * 32;
        __syncwarp();
    }
    // first arg-max of the last row (it is the tail row of the last strip: rowbuf)
    double best = NEG;
    int best_idx = 0x7fffffff;
    for (int jj = lane; jj < W; jj += 32) {
        const double v = tb2_rb_ld<RBS>(rowbuf, rb_s, jj);
        if (v > best) { best = v; best_idx = jj; }
    }
    *argmax_out = tb2_warp_argmax(best, best_idx);
    return TB2_OK;
}
#undef TB2_WF_FAST_STEP
#undef TB2_WF_MLD
#undef TB2_WF_MD

__device__ int tb2_wavefront_rows(const PassCtx &pc, const DpConsts &c, int mode, int r_end,
                                  double *rowbuf, uint32_t *tbw, int *argmax_out)
{
    const bool rbs = __isShared(rowbuf);
    const bool win = c.winsor != 0;
#define TB2_WF_CALL(M, D, WN, RB) tb2_wavefront_rows_t<M, D, WN, RB>(pc, c, r_end, rowbuf, tbw, argmax_out)
    if (mode == TB2_MODE_EXPLICIT) {
        // mirror API: explicit z matrix, optional full dumps
        if (pc.dbg_fwd) return rbs ? TB2_WF_CALL(TB2_MODE_EXPLICIT, true, false, true)
                                   : TB2_WF_CALL(TB2_MODE_EXPLICIT, true, false, false);
        return TB2_ERR_INVALID_ARG;
    }
    if (mode == TB2_MODE_MASKED) {
        if (win) return rbs ? TB2_WF_CALL(TB2_MODE_MASKED, false, true, true)
                            : TB2_WF_CALL(TB2_MODE_MASKED, false, true, false);
        return rbs ? TB2_WF_CALL(TB2_MODE_MASKED, false, false, true)
                   : TB2_WF_CALL(TB2_MODE_MASKED, false, false, false);
    }
    if (win) return rbs ? TB2_WF_CALL(TB2_MODE_PLAIN, false, true, true)
                        : TB2_WF_CALL(TB2_MODE_PLAIN, false, true, false);
    return rbs ? TB2_WF_CALL(TB2_MODE_PLAIN, false, false, true)
               : TB2_WF_CALL(TB2_MODE_PLAIN, false, false, false);
#undef TB2_WF_CALL
}

// traceback over rows [0, n_rows) stored in the wavefront layout (total_words =
// tb2_wf_total_words of the pass); cur_event is carried in and out
// (c_banded_traceback _c_dynamic_programming.pyx:295-308).  Strip by strip from the
// top: lanes prefetch three step-words around the expected position of their row.
__device__ __noinline__ int tb2_tb_seg_wf(const uint32_t *tbw, long long total_words, const int *starts,
                             int n_rows, int W, int thresh, int *cur_event_io, int *read_tb)
{
    const int lane = tb2_lane();
    int cur_event = *cur_event_io;
    const uint32_t *tbs = tbw + total_words;
    for (int s0 = ((n_rows - 1) >> 5) << 5; s0 >= 0; s0 -= 32) {
        const int nblk = min(32, n_rows - s0);
        const int sw = tb2_wf_strip_words(starts, s0, n_rows, W);
        if (sw < 0) return TB2_ERR_UNEXPECTED;
        tbs -= sw;
        const int nw = sw >> 5;
        const int t_begin = starts[s0];
        // lane L holds row s0 + L; the path is expected to keep its average slope down
        // to the first row
        const float slope = (float)(cur_event - starts[0]) / (float)(s0 + nblk);
        int my_start = 0, base = 0;
        uint32_t w0 = 0, w1 = 0, w2 = 0;
        if (lane < nblk) {
            my_start = starts[s0 + lane];
            const int est = cur_event - (int)((float)(nblk - 1 - lane) * slope) + lane - t_begin;
            base = min(max((est >> 4) - 1, 0), max(nw - 3, 0));
            const uint32_t *rw = tbs + lane;
            w0 = rw[base * 32];
            if (base + 1 < nw) w1 = rw[(base + 1) * 32];
            if (base + 2 < nw) w2 = rw[(base + 2) * 32];
        }
        for (int k = nblk - 1; k >= 0; --k) {
            const int row = s0 + k;
            const int st = __shfl_sync(TB2_FULL_MASK, my_start, k);
            const int bs = __shfl_sync(TB2_FULL_MASK, base, k);
            int bp = cur_event - st;
            if (bp < 0 || bp >= W) return TB2_ERR_UNEXPECTED;
            const int toff = st + k - t_begin;      // step = bp + toff
            uint32_t code;
            for (;;) {
                const int ts = bp + toff;
                const int wi = ts >> 4, rel = wi - bs, q = ts & 15;
                uint32_t v;
                if (rel >= 0 && rel < 3) {
                    const uint32_t mine = rel == 0 ? w0 : (rel == 1 ? w1 : w2);
                    v = __shfl_sync(TB2_FULL_MASK, mine, k);
                } else {
                    v = tbs[wi * 32 + k];
                }
                // a run of stays is skipped in one go: highest non-stay move at or below
                // position q of this word (TB2_WF_MOVE_BITS)
                const uint32_t nz = (v & 0xffffu) & (0xffffu >> (15 - q));
                if (nz != 0u) {
                    const int kq = 31 - __clz(nz);
                    bp -= q - kq;
                    code = ((v >> (16 + kq)) & 1u) ? 1u : 2u;
                    break;
                }
                bp -= q + 1;
                if (bp < 0) return TB2_ERR_UNEXPECTED;
            }
            if (code == 2u) --bp;
            if (thresh >= 0 && min(bp, W - bp - 1) < thresh) return TB2_ERR_BEYOND_BANDWIDTH;
            cur_event = st + bp;
            if (lane == 0) read_tb[row] = cur_event + 1;
        }
    }
    *cur_event_io = cur_event;
    __syncwarp();
    return TB2_OK;
}
