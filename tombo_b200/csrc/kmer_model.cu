// kmer_model.cu -- standard and motif k-mer model estimation on the device.
//
//   tb2_kmer_level_summaries  get_region_kmer_levels tombo_stats.py:1263-1280, 1349-1355: per
//                             covered position, calc_med_sd (np.median, np.std) or c_mean_std
//                             of the levels, where coverage > cov_thresh
//   tb2_kmer_medians          tabulate_kmer_levels :1462-1487 / tabulate_mod_kmer_levels
//                             :2116-2144: per key, np.median of the levels and of the sds
//
// Summaries (DESIGN.md §3 "K-mer model estimation"): the batch's regions lie end to end in
// one coordinate range, and the gather of level_gather.cuh runs over it with min_reads =
// cov_thresh + 1 and runs of length 1.  k_ref_pos gives the median and np.std in read order;
// k_mean_std_pos gives c_mean_std in read order.
//
// Medians: the key plays the position's role.  k_key_count counts each key, k_compact (one
// block) keeps the keys that occur and lays out their CSR, k_key_scatter fills it, and
// k_key_median sorts each key's levels and sds in place (shared memory, or the global CSR
// above its capacity) and takes the middle element(s).
#include "level_gather.cuh"
#include <climits>
#include <cmath>

namespace {
// per-call scratch of both entry points (after the gather's slots); nothing reads it after
// a call returns
enum { M_SUM = G_GATHER_COUNT, M_KEY, M_LVL, M_SD, M_OUT, M_COUNT };
}  // namespace
struct KmerModelState { DevBuf buf[M_COUNT]; };

namespace {

constexpr int M_SH = 4096;         // doubles of shared memory per key (k_key_median)

// c_mean_std _c_helper.pyx:22-36 of one covered position's levels in read order
__global__ void __launch_bounds__(BT)
k_mean_std_pos(const long long *pos, const long long *off, double *vals, int *reads, double *means,
               double *sds)
{
    __shared__ double shv[R_SH];
    __shared__ int shr[R_SH];
    const int o = blockIdx.x, tid = threadIdx.x;
    const int n = (int)(off[o + 1] - off[o]);
    double *v = vals + off[o];
    int *rd = reads + off[o];
    if (n <= R_SH) {
        for (int i = tid; i < n; i += BT) { shv[i] = v[i]; shr[i] = rd[i]; }
        v = shv; rd = shr;
        __syncthreads();
    }
    block_sort<int, double>(rd, v, n);                  // read order
    if (tid == 0) mean_std(v, n, means[pos[o]], sds[pos[o]]);
}

// (level, sd, coverage) per position; NaN where coverage <= cov_thresh
__global__ void k_summary_final(const int *map, const int *cov, long long n, const double *means,
                                const double *sds, double *lv_out, double *sd_out, long long *cov_out)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    lv_out[p] = map[p] >= 0 ? means[p] : NAN;
    sd_out[p] = map[p] >= 0 ? sds[p] : NAN;
    cov_out[p] = cov[p];
}

__global__ void k_key_count(const long long *key, long long n_obs, int *cnt)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_obs;
         i += (long long)gridDim.x * blockDim.x)
        atomicAdd(cnt + key[i], 1);
}

// levels to [0, tot), sds to [tot, 2 tot), each in its key's CSR slot
__global__ void k_key_scatter(const long long *key, const double *lv, const double *sd, long long n_obs,
                              const int *map, const long long *csr_off, long long tot, int *fill,
                              double *vals)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_obs;
         i += (long long)gridDim.x * blockDim.x) {
        const int q = map[key[i]];
        const long long at = csr_off[q] + atomicAdd(fill + q, 1);
        vals[at] = lv[i];
        vals[tot + at] = sd[i];
    }
}

// np.median of one key's values, sorted in place: the middle element, or the mean of the
// two middle elements as numpy takes it
__device__ double block_median(double *v, double *sh, int n)
{
    if (n <= M_SH) {
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += BT) sh[i] = v[i];
        v = sh;
        __syncthreads();
    }
    block_sort<double, double>(v, nullptr, n);
    return (n & 1) ? v[n / 2] : (v[n / 2 - 1] + v[n / 2]) / 2.0;
}

__global__ void __launch_bounds__(BT)
k_key_median(const long long *keys, const long long *off, long long tot, double *vals, double *med_lv,
             double *med_sd)
{
    __shared__ double sh[M_SH];
    const int o = blockIdx.x;
    const int n = (int)(off[o + 1] - off[o]);
    const double ml = block_median(vals + off[o], sh, n);
    const double ms = block_median(vals + tot + off[o], sh, n);
    if (threadIdx.x == 0) { med_lv[keys[o]] = ml; med_sd[keys[o]] = ms; }
}

__global__ void k_key_final(const int *cnt, long long n, double *med_lv, double *med_sd, long long *cnt_out)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    cnt_out[p] = cnt[p];
    if (!cnt[p]) { med_lv[p] = NAN; med_sd[p] = NAN; }
}

}  // namespace

extern "C" int tb2_kmer_level_summaries(tb2_ctx *ctx, int64_t n_pos, int64_t n_reads, const double *levels,
                                        const int64_t *off, const int64_t *start, int64_t cov_thresh,
                                        int est_mean, double *level_out, double *sd_out, int64_t *cov_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    if (n_pos < 1 || n_pos > MAX_REG_LEN || cov_thresh < 0 || cov_thresh >= (1LL << 31) - 1 || !level_out ||
        !sd_out || !cov_out)
        return TB2_ERR_INVALID_ARG;
    if ((rc = check_sample(n_reads, levels, off, start))) return rc;
    DevBuf *P = tb2_state(ctx->kmer).buf;
    cudaStream_t q = ctx->stream;
    Sample a;
    if ((rc = upload_sample(ctx, P, G_LV, n_reads, levels, off, start, a))) return rc;
    long long hdr[4];
    if ((rc = gather(ctx, P, 0, n_pos, a, nullptr, (int)cov_thresh + 1, 1, true, hdr))) return rc;
    const long long n = n_pos, n_cov = hdr[0];
    long long *idx = P[G_IDX].as<long long>();
    TB2_CUDA_TRY(ctx, P[M_SUM].reserve((size_t)n * 2 * 8));
    TB2_CUDA_TRY(ctx, P[M_OUT].reserve((size_t)n * 3 * 8));
    double *means = P[M_SUM].as<double>(), *sds = means + n;
    double *lv = P[M_OUT].as<double>(), *sd = lv + n;
    long long *cov = (long long *)(sd + n);
    if (n_cov) {
        if (est_mean)
            k_mean_std_pos<<<(unsigned)n_cov, BT, 0, q>>>(idx, idx + 3 * n, P[G_VAL].as<double>(),
                                                          P[G_RD].as<int>(), means, sds);
        else
            k_ref_pos<<<(unsigned)n_cov, BT, 0, q>>>(idx, idx + 3 * n, P[G_VAL].as<double>(), P[G_RD].as<int>(),
                                                     P[G_SQ].as<double>(), 0, means, sds);
        TB2_CHECK_LAUNCH(ctx);
    }
    const int *cnt = P[G_INT].as<int>();
    k_summary_final<<<(unsigned)((n + 255) / 256), 256, 0, q>>>(cnt + 4 * n, cnt, n, means, sds, lv, sd, cov);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(level_out, lv, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(sd_out, sd, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(cov_out, cov, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}

extern "C" int tb2_kmer_medians(tb2_ctx *ctx, int64_t n_keys, int64_t n_obs, const int64_t *keys,
                                const double *levels, const double *sds, int64_t *count_out,
                                double *level_med_out, double *sd_med_out)
{
    int rc = tb2_use(ctx);
    if (rc) return rc;
    // a key's count fits the int counts and the bitonic network's power-of-two size
    if (n_keys < 1 || n_keys > MAX_REG_LEN || n_obs < 0 || n_obs > (1LL << 30) ||
        (n_obs > 0 && (!keys || !levels || !sds)) || !count_out || !level_med_out || !sd_med_out)
        return TB2_ERR_INVALID_ARG;
    for (int64_t i = 0; i < n_obs; ++i)
        if (keys[i] < 0 || keys[i] >= n_keys || std::isnan(levels[i]) || std::isnan(sds[i]))
            return TB2_ERR_INVALID_ARG;
    DevBuf *P = tb2_state(ctx->kmer).buf;
    cudaStream_t q = ctx->stream;
    const long long n = n_keys;
    TB2_CUDA_TRY(ctx, P[M_KEY].upload(keys, (size_t)n_obs, q));
    TB2_CUDA_TRY(ctx, P[M_LVL].upload(levels, (size_t)n_obs, q));
    TB2_CUDA_TRY(ctx, P[M_SD].upload(sds, (size_t)n_obs, q));
    TB2_CUDA_TRY(ctx, P[G_INT].reserve((size_t)n * 3 * 4));
    TB2_CUDA_TRY(ctx, P[G_IDX].reserve((size_t)(6 * n + 3) * 8));
    TB2_CUDA_TRY(ctx, P[G_HDR].reserve(64));
    TB2_CUDA_TRY(ctx, P[G_VAL].reserve((size_t)n_obs * 2 * 8 + 8));
    TB2_CUDA_TRY(ctx, P[M_OUT].reserve((size_t)n * 3 * 8));
    int *cnt = P[G_INT].as<int>(), *fill = cnt + n, *map = cnt + 2 * n;
    long long *idx = P[G_IDX].as<long long>();
    const long long *key = P[M_KEY].as<long long>();
    double *vals = P[G_VAL].as<double>(), *med_lv = P[M_OUT].as<double>(), *med_sd = med_lv + n;
    long long *cnt_out = (long long *)(med_sd + n);
    const unsigned grid = (unsigned)std::min<long long>((n_obs + 255) / 256 + 1, 4LL * ctx->sm_count);
    TB2_CUDA_TRY(ctx, cudaEventRecord(ctx->ev0, q));          // kernel time: tb2_last_timing
    TB2_CUDA_TRY(ctx, cudaMemsetAsync(cnt, 0, (size_t)n * 2 * 4, q));
    if (n_obs) { k_key_count<<<grid, 256, 0, q>>>(key, n_obs, cnt); TB2_CHECK_LAUNCH(ctx); }
    k_compact<<<1, 1024, 0, q>>>(cnt, nullptr, n, 1, 1, map, idx, P[G_HDR].as<long long>());
    TB2_CHECK_LAUNCH(ctx);
    long long hdr[4];
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(hdr, P[G_HDR].p, 32, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    const long long n_used = hdr[0], *csr = idx + 3 * n;
    if (n_used) {
        k_key_scatter<<<grid, 256, 0, q>>>(key, P[M_LVL].as<double>(), P[M_SD].as<double>(), n_obs, map, csr,
                                           n_obs, fill, vals);
        TB2_CHECK_LAUNCH(ctx);
        k_key_median<<<(unsigned)n_used, BT, 0, q>>>(idx, csr, n_obs, vals, med_lv, med_sd);
        TB2_CHECK_LAUNCH(ctx);
    }
    k_key_final<<<(unsigned)((n + 255) / 256), 256, 0, q>>>(cnt, n, med_lv, med_sd, cnt_out);
    TB2_CHECK_LAUNCH(ctx);
    if ((rc = tb2_record_kernel_time(ctx))) return rc;
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(count_out, cnt_out, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(level_med_out, med_lv, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaMemcpyAsync(sd_med_out, med_sd, (size_t)n * 8, cudaMemcpyDeviceToHost, q));
    TB2_CUDA_TRY(ctx, cudaStreamSynchronize(q));
    return TB2_OK;
}
