// group_stats.cu -- level_sample_compare and control-sample reference levels on the device.
//
//   tb2_group_reg_stats   compute_group_reg_stats tombo_stats.py:4335-4393 with
//                         compute_ks_tests / compute_u_tests / compute_t_tests :4236-4324,
//                         calc_window_fishers_method / calc_window_means :2252-2287
//   tb2_reads_ref_levels  get_reads_ref :3627-3673 (+ compute_posterior_samp_dists
//                         :3572-3625)
//
// One region per call.  Reads arrive as ragged genome-ordered level arrays (levels, off,
// start).  Steps (DESIGN.md §3 "Level tests"):
//   1. k_count: non-NaN levels per position (samp_cov / ctrl_cov), atomics.
//   2. k_compact (one block): positions inside coverage runs that are at least
//      min_run long, ascending; CSR offsets of their values; run (segment) offsets.
//   3. k_scatter: each kept level goes to its position's CSR slot with its read ordinal.
//   4. k_group_pos / k_ref_pos: one block per position; values sorted in shared memory
//      (bitonic, in place), or in place in the global CSR when the position's coverage
//      exceeds the shared buffer -- same code, exact either way.
//   5. windows over each run: k_fisher (fisher.cuh) for p-values, k_window_mean for the
//      *_stat_test variants; k_ref_final for the posterior and the sd == 0 mask.
#include "batch.h"
#include "kernels.h"
#include "common.cuh"
#include "fisher.cuh"
#include "special.cuh"
#include <cmath>

namespace {
// per-call scratch of tb2_group_reg_stats / tb2_reads_ref_levels; nothing reads it after a
// call returns
enum { G_LV_S = 0, G_OFF_S, G_ST_S, G_LV_C, G_OFF_C, G_ST_C, G_INT, G_IDX, G_VAL, G_RD, G_SQ,
       G_RES, G_PRI_M, G_PRI_S, G_REF, G_HDR, G_COUNT };
}  // namespace
struct GroupState { DevBuf scratch[G_COUNT]; };

namespace {

constexpr int BT = 256;            // threads of the per-position kernels
constexpr int G_SH = 5632;         // doubles of shared memory per position (group tests)
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

// exclusive scan over a 1024-thread block; `tot` gets the block total
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

// ---------------------------------------------------------------------------
// per-position statistics
// ---------------------------------------------------------------------------
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

__device__ __forceinline__ int upper_bound(const double *a, int n, double x)
{
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] <= x) lo = mid + 1; else hi = mid; }
    return lo;
}

__device__ __forceinline__ int lower_bound(const double *a, int n, double x)
{
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
    return lo;
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

// ndtr (scipy.special) as norm.cdf evaluates it
__device__ __forceinline__ double ndtr(double a)
{
    const double x = a * 0.70710678118654752440, z = fabs(x);
    if (z < 0.70710678118654752440) return 0.5 + 0.5 * erf(x);
    const double y = 0.5 * erfc(z);
    return x > 0 ? 1.0 - y : y;
}

__global__ void __launch_bounds__(BT)
k_group_pos(const long long *offs, const long long *offc, long long tot_s, double *vals, int test,
            int return_stat, double *stat)
{
    __shared__ double sh[G_SH];
    __shared__ double red_d[BT / 32];
    __shared__ long long red_l[BT / 32];
    const int o = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ns = (int)(offs[o + 1] - offs[o]), nc = (int)(offc[o + 1] - offc[o]);
    double *s = vals + offs[o], *c = vals + tot_s + offc[o];
    if (ns + nc <= G_SH) {
        for (int i = tid; i < ns; i += BT) sh[i] = s[i];
        for (int i = tid; i < nc; i += BT) sh[ns + i] = c[i];
        s = sh; c = sh + ns;
        __syncthreads();
    }
    block_sort<double, double>(s, nullptr, ns);
    block_sort<double, double>(c, nullptr, nc);
    double res = NAN;
    if (test == 0) {
        // KS :4236-4255: d = max |searchsorted(s, all, 'right')/n_s - searchsorted(c, ..)/n_c|
        double d = 0.0;
        for (int i = tid; i < ns + nc; i += BT) {
            const double x = i < ns ? s[i] : c[i - ns];
            const double e = fabs((double)upper_bound(s, ns, x) / (double)ns -
                                  (double)upper_bound(c, nc, x) / (double)nc);
            d = e > d ? e : d;
        }
        for (int w = 16; w > 0; w >>= 1) { const double u = __shfl_xor_sync(0xffffffffu, d, w); d = u > d ? u : d; }
        if (lane == 0) red_d[warp] = d;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < BT / 32; ++w) d = red_d[w] > d ? red_d[w] : d;
            if (return_stat) res = 1.0 - d;
            else {
                const double en = sqrt((double)((long long)ns * nc) / (double)(ns + nc));
                res = tb2_kolmogorov_sf((en + 0.12 + 0.11 / en) * d);
            }
        }
    } else if (test == 1) {
        // U :4266-4291: rank sum - n_s(n_s+1)/2 = sum_i #{c < s_i} (stable rule: sample first)
        long long cnt = 0;
        for (int i = tid; i < ns; i += BT) cnt += lower_bound(c, nc, s[i]);
        for (int w = 16; w > 0; w >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, w);
        if (lane == 0) red_l[warp] = cnt;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < BT / 32; ++w) cnt += red_l[w];
            const long long half = (long long)ns * (ns + 1) / 2, tot = (long long)ns * nc;
            const double u1 = (double)(cnt + half) - (double)half;
            const double u2 = (double)tot - u1;
            const double u = u2 < u1 ? u2 : u1;
            const double mu = (double)tot / 2.0;
            if (return_stat) res = (u - mu) / mu;
            else {
                const double rhou = sqrt(tb2_div12((unsigned __int128)tot * (unsigned __int128)(tot + 1)));
                res = ndtr((u - mu) / rhou) * 2.0;
            }
        }
    } else if (tid == 0) {
        // t :4302-4324 on the sorted values
        double sm, ssd, cm, csd;
        mean_std(s, ns, sm, ssd);
        mean_std(c, nc, cm, csd);
        if (return_stat) {
            const double den = sqrt(((ssd * ssd) + (csd * csd)) / 2.0);
            res = den > 0.0 ? -fabs(sm - cm) / den : NAN;    // the reference raises here
        } else if (ns + nc > 2) {
            const double sp = sqrt((((double)(ns - 1) * (ssd * ssd)) + (double)(nc - 1) * (csd * csd)) /
                                   (double)(ns + nc - 2));
            if (sp > 0.0) {
                const double t = -fabs(sm - cm) / (sp * sqrt((1.0 / (double)ns) + (1.0 / (double)nc)));
                res = tb2_t_two_sided_p((double)(ns + nc - 2), t);
            }
        }
    }
    if (tid == 0) stat[o] = res;
}

// calc_window_means :2273-2287: np.mean over 2 lag + 1 values (pairwise sum / width)
__global__ void __launch_bounds__(256)
k_window_mean(const double *in, const long long *seg, int lag, double *out)
{
    const long long o = seg[blockIdx.x];
    const int n = (int)(seg[blockIdx.x + 1] - o), width = 2 * lag + 1;
    for (int i = threadIdx.x; i < n; i += 256)
        out[o + i] = (i >= lag && i < n - lag) ? tb2_pairwise_sum(in + o + i - lag, width) / (double)width : NAN;
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

// uncovered -> NaN; compute_posterior_samp_dists :3589-3594; sd == 0 -> NaN (:3668-3671)
__global__ void k_ref_final(const int *map, const int *cov, long long n, const double *pm,
                            const double *ps, double w0, double w1, double *means, double *sds,
                            long long *cov_out)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    double m = map[p] >= 0 ? means[p] : NAN, s = map[p] >= 0 ? sds[p] : NAN;
    const double c = (double)cov[p];
    if (pm) {
        m = ((w0 * pm[p]) + (c * m)) / (w0 + c);
        s = ((w1 * ps[p]) + (c * s)) / (w1 + c);
    }
    if (s == 0.0) { m = NAN; s = NAN; }
    means[p] = m; sds[p] = s; cov_out[p] = cov[p];
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
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

int upload_sample(tb2_ctx *ctx, int slot, int64_t n, const double *lv, const int64_t *off,
                  const int64_t *st, Sample &s)
{
    auto &P = tb2_state(ctx->group).scratch;
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
int gather(tb2_ctx *ctx, long long reg_start, long long reg_len, const Sample &a, const Sample *b,
           int min_reads, int min_run, bool want_reads, long long hdr[4])
{
    auto &P = tb2_state(ctx->group).scratch;
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

extern "C" int tb2_group_reg_stats(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len,
                                   int64_t n_samp, const double *samp_levels, const int64_t *samp_off,
                                   const int64_t *samp_start, int64_t n_ctrl, const double *ctrl_levels,
                                   const int64_t *ctrl_off, const int64_t *ctrl_start, int test,
                                   int return_stat, int64_t min_test_reads, int64_t fm_offset, int64_t cap,
                                   int64_t *pos_out, double *stat_out, int64_t *cov_out,
                                   int64_t *ctrl_cov_out, int64_t *n_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (reg_len < 1 || reg_len > MAX_REG_LEN || test < 0 || test > 2 || min_test_reads < 1 ||
        min_test_reads > (1LL << 31) - 1 || fm_offset < 0 || fm_offset > MAX_REG_LEN || cap < 0 || !n_out ||
        (cap > 0 && (!pos_out || !stat_out || !cov_out || !ctrl_cov_out)))
        return TB2_ERR_INVALID_ARG;
    if ((rc = check_sample(n_samp, samp_levels, samp_off, samp_start))) return rc;
    if ((rc = check_sample(n_ctrl, ctrl_levels, ctrl_off, ctrl_start))) return rc;
    auto &P = tb2_state(ctx->group).scratch;
    cudaStream_t q = ctx->stream;
    Sample a, b;
    if ((rc = upload_sample(ctx, G_LV_S, n_samp, samp_levels, samp_off, samp_start, a))) return rc;
    if ((rc = upload_sample(ctx, G_LV_C, n_ctrl, ctrl_levels, ctrl_off, ctrl_start, b))) return rc;
    long long hdr[4];
    if ((rc = gather(ctx, reg_start, reg_len, a, &b, (int)min_test_reads, (int)(2 * fm_offset + 1), false, hdr)))
        return rc;
    const long long n = reg_len, n_pos = hdr[0], n_seg = hdr[1];
    *n_out = n_pos;
    if (n_pos == 0) return tb2_record_kernel_time(ctx);
    long long *idx = P[G_IDX].as<long long>();
    const long long *offs = idx + 3 * n, *offc = offs + n + 1, *seg = offc + n + 1;
    TB2_CUDA_TRY(ctx, P[G_RES].reserve((size_t)n_pos * 3 * 8));
    double *stat = P[G_RES].as<double>(), *out = stat + n_pos, *logp = out + n_pos;
    k_group_pos<<<(unsigned)n_pos, BT, 0, q>>>(offs, offc, hdr[2], P[G_VAL].as<double>(), test,
                                               return_stat ? 1 : 0, stat);
    TB2_CHECK_LAUNCH(ctx);
    const double *res = stat;
    if (fm_offset > 0) {
        if (!return_stat) {
            FisherArgs fa;
            memset(&fa, 0, sizeof(fa));
            fa.means = stat; fa.off = seg; fa.lag = (int)fm_offset; fa.input_is_p = 1;
            fa.smallest = 1e-50;                              // SMALLEST_PVAL _default_parameters.py:158
            fa.logp = logp; fa.out = out;
            k_fisher<false><<<(unsigned)n_seg, 256, 0, q>>>(fa);
        } else {
            k_window_mean<<<(unsigned)n_seg, 256, 0, q>>>(stat, seg, (int)fm_offset, out);
        }
        TB2_CHECK_LAUNCH(ctx);
        res = out;
    }
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    const size_t m = (size_t)std::min<long long>(n_pos, cap);
    if (m) {
        // positions are relative to reg_start on the device
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(pos_out, idx, m * 8, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cov_out, idx + n, m * 8, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(ctrl_cov_out, idx + 2 * n, m * 8, cudaMemcpyDeviceToHost, q));
        TB2_CUDA_TRY(ctx, cudaMemcpyAsync(stat_out, res, m * 8, cudaMemcpyDeviceToHost, q));
    }
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    for (size_t i = 0; i < m; ++i) pos_out[i] += reg_start;
    return n_pos > cap ? TB2_ERR_CAPACITY : TB2_OK;
}

extern "C" int tb2_reads_ref_levels(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len, int64_t n_reads,
                                    const double *levels, const int64_t *off, const int64_t *start,
                                    int64_t min_test_reads, int est_mean, const double *prior_means,
                                    const double *prior_sds, double mean_prior_weight,
                                    double sd_prior_weight, double *means_out, double *sds_out,
                                    int64_t *cov_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (reg_len < 1 || reg_len > MAX_REG_LEN || min_test_reads < 1 || min_test_reads > (1LL << 31) - 1 ||
        !means_out || !sds_out || !cov_out || (!prior_means != !prior_sds))
        return TB2_ERR_INVALID_ARG;
    if ((rc = check_sample(n_reads, levels, off, start))) return rc;
    auto &P = tb2_state(ctx->group).scratch;
    cudaStream_t q = ctx->stream;
    Sample a;
    if ((rc = upload_sample(ctx, G_LV_S, n_reads, levels, off, start, a))) return rc;
    const long long n = reg_len;
    const double *pm = nullptr, *ps = nullptr;
    if (prior_means) {
        TB2_CUDA_TRY(ctx, P[G_PRI_M].upload(prior_means, (size_t)n, q));
        TB2_CUDA_TRY(ctx, P[G_PRI_S].upload(prior_sds, (size_t)n, q));
        pm = P[G_PRI_M].as<double>(); ps = P[G_PRI_S].as<double>();
    }
    long long hdr[4];
    if ((rc = gather(ctx, reg_start, reg_len, a, nullptr, (int)min_test_reads, 1, true, hdr))) return rc;
    const long long n_pos = hdr[0];
    long long *idx = P[G_IDX].as<long long>();
    TB2_CUDA_TRY(ctx, P[G_REF].reserve((size_t)n * 3 * 8));
    double *means = P[G_REF].as<double>(), *sds = means + n;
    long long *cov = (long long *)(sds + n);
    if (n_pos) {
        k_ref_pos<<<(unsigned)n_pos, BT, 0, q>>>(idx, idx + 3 * n, P[G_VAL].as<double>(), P[G_RD].as<int>(),
                                                 P[G_SQ].as<double>(), est_mean ? 1 : 0, means, sds);
        TB2_CHECK_LAUNCH(ctx);
    }
    const int *map = P[G_INT].as<int>() + 4 * n;
    k_ref_final<<<(unsigned)((n + 255) / 256), 256, 0, q>>>(map, P[G_INT].as<int>(), n, pm, ps, mean_prior_weight,
                                                           sd_prior_weight, means, sds, cov);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(means_out, means, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(sds_out, sds, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cov_out, cov, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}
