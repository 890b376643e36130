// level_gather.cuh -- ragged genome-ordered reads (levels, off, start) -> the levels of
// every covered position in CSR order, and the per-position median / std kernel.  Shared
// by group_stats.cu (level tests, control-sample reference levels) and kmer_model.cu
// (k-mer model estimation); DESIGN.md §3 "Level tests".
#pragma once
#include "kernels.h"
#include "common.cuh"
#include <algorithm>

// slots of a caller's workspace that gather() and upload_sample() use; a caller's own
// slots follow G_GATHER_COUNT
enum GatherSlot { G_INT = 0, G_IDX, G_VAL, G_RD, G_SQ, G_HDR, G_LV, G_OFF, G_ST, G_GATHER_COUNT };

namespace {

constexpr int BT = 256;            // threads of the per-position kernels
constexpr int R_SH = 1920;         // (level, square, read) triples per position (reference levels)
constexpr long long MAX_REG_LEN = 1LL << 24;

// ---------------------------------------------------------------------------
// gather
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_count(const double *lv, const long long *off, const long long *st, long long reg_start,
        long long reg_len, int *cov)
{
    const int r = blockIdx.x;
    const long long o = off[r], L = off[r + 1] - o, s = st[r] - reg_start;
    const long long j0 = s < 0 ? -s : 0, j1 = min(L, reg_len - s);
    for (long long j = j0 + threadIdx.x; j < j1; j += 128)
        if (!isnan(lv[o + j])) atomicAdd(cov + s + j, 1);
}

__global__ void __launch_bounds__(128)
k_scatter(const double *lv, const long long *off, const long long *st, long long reg_start,
          long long reg_len, const int *map, const long long *csr_off, int *fill, double *vals,
          int *reads)
{
    const int r = blockIdx.x;
    const long long o = off[r], L = off[r + 1] - o, s = st[r] - reg_start;
    const long long j0 = s < 0 ? -s : 0, j1 = min(L, reg_len - s);
    for (long long j = j0 + threadIdx.x; j < j1; j += 128) {
        const double v = lv[o + j];
        const int q = map[s + j];
        if (isnan(v) || q < 0) continue;
        const long long at = csr_off[q] + atomicAdd(fill + q, 1);
        vals[at] = v;
        if (reads) reads[at] = r;
    }
}

// np.diff of [False, cov >= m (both samples), False] -> runs; runs shorter than min_run are
// skipped (:4355).  Position p is kept when it sits in a run of >= min_run ok positions.
__device__ __forceinline__ bool cov_ok(const int *cs, const int *cc, long long p, int m)
{
    return cs[p] >= m && (!cc || cc[p] >= m);
}

__device__ bool keep_at(const int *cs, const int *cc, long long p, long long n, int m, int min_run)
{
    if (min_run > n || p < 0 || p >= n || !cov_ok(cs, cc, p, m)) return false;
    int l = 1, r = 1;
    while (l < min_run && p - l >= 0 && cov_ok(cs, cc, p - l, m)) ++l;
    while (l + r - 1 < min_run && p + r < n && cov_ok(cs, cc, p + r, m)) ++r;
    return l + r - 1 >= min_run;
}

// exclusive scan over a 1024-thread block; `tot` gets the block total.  k_compact keeps this
// two-level form rather than tb2_block_excl_scan (common.cuh): there every thread reads all 32
// warp totals, which for four 64-bit scans per chunk made k_compact ~40 us slower per call.
__device__ __forceinline__ long long block_scan(long long v, long long *ws, long long &tot)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long u = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += u;
    }
    if (lane == 31) ws[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        long long w = ws[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += u;
        }
        ws[lane] = w;
    }
    __syncthreads();
    const long long before = warp ? ws[warp - 1] : 0;
    tot = ws[31];
    __syncthreads();
    return before + inc - v;
}

// idx layout (n = reg_len): pos[n] cov_s[n] cov_c[n] off_s[n+1] off_c[n+1] seg[n+1];
// hdr: n_out, n_seg, tot_s, tot_c
__global__ void __launch_bounds__(1024)
k_compact(const int *cs, const int *cc, long long n, int m, int min_run, int *map, long long *idx,
          long long *hdr)
{
    __shared__ long long ws[32];
    __shared__ long long base[4];
    long long *pos = idx, *ocs = idx + n, *occ = idx + 2 * n, *offs = idx + 3 * n,
              *offc = offs + n + 1, *seg = offc + n + 1;
    if (threadIdx.x < 4) base[threadIdx.x] = 0;
    __syncthreads();
    for (long long c0 = 0; c0 < n; c0 += 1024) {
        const long long p = c0 + threadIdx.x;
        const bool k = keep_at(cs, cc, p, n, m, min_run);
        const bool first = k && !keep_at(cs, cc, p - 1, n, m, min_run);
        const long long vs = k ? cs[p] : 0, vc = (k && cc) ? cc[p] : 0;
        long long t0, t1, t2, t3;
        const long long o = block_scan(k, ws, t0) + base[0];
        const long long g = block_scan(first, ws, t1) + base[1];
        const long long es = block_scan(vs, ws, t2) + base[2];
        const long long ec = block_scan(vc, ws, t3) + base[3];
        if (p < n) map[p] = k ? (int)o : -1;
        if (k) {
            pos[o] = p; ocs[o] = vs; occ[o] = vc; offs[o] = es; offc[o] = ec;
            if (first) seg[g] = o;
        }
        __syncthreads();
        if (threadIdx.x == 0) { base[0] += t0; base[1] += t1; base[2] += t2; base[3] += t3; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        offs[base[0]] = base[2]; offc[base[0]] = base[3]; seg[base[1]] = base[0];
        hdr[0] = base[0]; hdr[1] = base[1]; hdr[2] = base[2]; hdr[3] = base[3];
    }
}

// Block-wide in-place ascending sort of key[0, n) (payload moves along).  Bitonic network
// in the form whose every comparator puts the minimum at the lower index, so entries past
// n act as +inf and never move: any n, no padding.
template <class K, class V>
__device__ void block_sort(K *key, V *pay, int n)
{
    int N = 1;
    while (N < n) N <<= 1;
    for (int k = 2; k <= N; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < (N >> 1); i += blockDim.x) {
                int a, b;
                if (j == (k >> 1)) {               // flip: pair r with k-1-r inside each k-block
                    const int r = i % j;
                    a = (i / j) * k + r; b = (i / j) * k + k - 1 - r;
                } else {
                    const int r = i % j;
                    a = (i / j) * 2 * j + r; b = a + j;
                }
                if (b < n && key[b] < key[a]) {
                    const K t = key[a]; key[a] = key[b]; key[b] = t;
                    if (pay) { const V u = pay[a]; pay[a] = pay[b]; pay[b] = u; }
                }
            }
            __syncthreads();
        }
    }
}

// c_mean_std _c_helper.pyx:22-36: sequential sums in array order, divided by n
__device__ void mean_std(const double *v, int n, double &mean, double &sd)
{
    double m = 0.0;
    for (int i = 0; i < n; ++i) m += v[i];
    m /= (double)n;
    double var = 0.0;
    for (int i = 0; i < n; ++i) { const double d = v[i] - m; var += d * d; }
    mean = m; sd = sqrt(var / (double)n);
}

// get_reads_ref :3644-3656 for one covered position: np.median (or np.mean) and np.std of the
// levels in read order
__global__ void __launch_bounds__(BT)
k_ref_pos(const long long *pos, const long long *off, double *vals, int *reads, double *sqbuf,
          int est_mean, double *means, double *sds)
{
    __shared__ double shv[R_SH], shq[R_SH];
    __shared__ int shr[R_SH];
    __shared__ double mean_s;
    const int o = blockIdx.x, tid = threadIdx.x;
    const int n = (int)(off[o + 1] - off[o]);
    double *v = vals + off[o], *q = sqbuf + off[o];
    int *rd = reads + off[o];
    if (n <= R_SH) {
        for (int i = tid; i < n; i += BT) { shv[i] = v[i]; shr[i] = rd[i]; }
        v = shv; q = shq; rd = shr;
        __syncthreads();
    }
    block_sort<int, double>(rd, v, n);                  // read order
    if (tid == 0) mean_s = tb2_pairwise_sum(v, n) / (double)n;
    __syncthreads();
    const double mean = mean_s;
    for (int i = tid; i < n; i += BT) { const double d = v[i] - mean; q[i] = d * d; }
    __syncthreads();
    double centre = mean;
    if (!est_mean) {
        block_sort<double, double>(v, nullptr, n);
        centre = (n & 1) ? v[n / 2] : (v[n / 2 - 1] + v[n / 2]) / 2.0;
    }
    if (tid == 0) {
        means[pos[o]] = centre;
        sds[pos[o]] = sqrt(tb2_pairwise_sum(q, n) / (double)n);
    }
}

struct Sample { int n; long long total; const double *lv; const long long *off, *st; };

// at most 2^30 - 1 reads per sample: a position's coverage then fits the int counts and the
// bitonic network's power-of-two size, and n_s + n_c fits an int
constexpr long long MAX_READS = (1LL << 30) - 1;

int check_sample(int64_t n, const double *lv, const int64_t *off, const int64_t *st)
{
    if (n < 0 || n > MAX_READS || (n > 0 && (!off || !st))) return TB2_ERR_INVALID_ARG;
    if (n == 0) return TB2_OK;
    if (off[0] != 0) return TB2_ERR_INVALID_ARG;
    for (int64_t r = 0; r < n; ++r)
        if (off[r + 1] < off[r]) return TB2_ERR_INVALID_ARG;
    if (off[n] > 0 && !lv) return TB2_ERR_INVALID_ARG;
    return TB2_OK;
}

// the sample's three arrays go to P[slot], P[slot + 1], P[slot + 2]
int upload_sample(tb2_ctx *ctx, DevBuf *P, int slot, int64_t n, const double *lv, const int64_t *off,
                  const int64_t *st, Sample &s)
{
    cudaStream_t q = ctx->stream;
    s.n = (int)n;
    s.total = n ? off[n] : 0;
    TB2_CUDA_TRY(ctx, P[slot].upload(lv, (size_t)s.total, q));
    TB2_CUDA_TRY(ctx, P[slot + 1].upload(off, n ? (size_t)n + 1 : 0, q));   // off may be null when n == 0
    TB2_CUDA_TRY(ctx, P[slot + 2].upload(st, (size_t)n, q));
    s.lv = P[slot].as<double>(); s.off = P[slot + 1].as<long long>(); s.st = P[slot + 2].as<long long>();
    return TB2_OK;
}

// steps 1-3 for one or two samples; on return hdr holds n_out, n_seg, tot_s, tot_c
int gather(tb2_ctx *ctx, DevBuf *P, long long reg_start, long long reg_len, const Sample &a, const Sample *b,
           int min_reads, int min_run, bool want_reads, long long hdr[4])
{
    cudaStream_t q = ctx->stream;
    const long long n = reg_len;
    TB2_CUDA_TRY(ctx, P[G_INT].reserve((size_t)n * 5 * 4));
    TB2_CUDA_TRY(ctx, P[G_IDX].reserve((size_t)(6 * n + 3) * 8));
    TB2_CUDA_TRY(ctx, P[G_HDR].reserve(64));
    int *cs = P[G_INT].as<int>(), *cc = cs + n, *fs = cs + 2 * n, *fc = cs + 3 * n, *map = cs + 4 * n;
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));          // kernel time: tb2_last_timing
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(cs, 0, (size_t)n * 4 * 4, q));
    if (a.n) { k_count<<<a.n, 128, 0, q>>>(a.lv, a.off, a.st, reg_start, n, cs); TB2_CHECK_LAUNCH(ctx); }
    if (b && b->n) { k_count<<<b->n, 128, 0, q>>>(b->lv, b->off, b->st, reg_start, n, cc); TB2_CHECK_LAUNCH(ctx); }
    long long *idx = P[G_IDX].as<long long>();
    k_compact<<<1, 1024, 0, q>>>(cs, b ? cc : nullptr, n, min_reads, min_run, map, idx, P[G_HDR].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(hdr, P[G_HDR].p, 32, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    const long long tot = hdr[2] + hdr[3];
    TB2_CUDA_TRY(ctx, P[G_VAL].reserve((size_t)tot * 8 + 8));
    if (want_reads) {
        TB2_CUDA_TRY(ctx, P[G_RD].reserve((size_t)tot * 4 + 8));
        TB2_CUDA_TRY(ctx, P[G_SQ].reserve((size_t)tot * 8 + 8));
    }
    const long long *offs = idx + 3 * n, *offc = offs + n + 1;
    double *vals = P[G_VAL].as<double>();
    int *rd = want_reads ? P[G_RD].as<int>() : nullptr;
    if (hdr[0] && a.n) {
        k_scatter<<<a.n, 128, 0, q>>>(a.lv, a.off, a.st, reg_start, n, map, offs, fs, vals, rd);
        TB2_CHECK_LAUNCH(ctx);
    }
    if (hdr[0] && b && b->n) {
        k_scatter<<<b->n, 128, 0, q>>>(b->lv, b->off, b->st, reg_start, n, map, offc, fc, vals + hdr[2], nullptr);
        TB2_CHECK_LAUNCH(ctx);
    }
    return TB2_OK;
}
}  // namespace
