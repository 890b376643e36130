// batch.h -- device-resident layout of one batch of reads (host + device view)
#pragma once
#ifdef TB2_EMUL   // host emulation of the device code (tests/emul): no CUDA runtime types
#include <stddef.h>
#include "../../include/tombo_b200.h"
struct tb2_ctx;
#else
#include <climits>
#include "ctx.h"
#endif

// Per-read state.  One resquiggle_read "call" (resquiggle.py:1122-1214) is one
// trip through the stage kernels; the worker policy (resquiggle.py:1492-1504,
// 1578-1588) is driven by `active`, `n_iters`, `attempt`.
struct ReadState {
    int status;        // status of the current attempt (TB2_OK while running)
    int active;        // takes part in the current call
    int done;          // finished (success or final failure)
    int n_iters;       // calls completed in this attempt
    int calls;         // calls over both attempts (keys the Theil-Sen sub-sampling)
    int attempt;       // 0 normal params, 1 save params
    int first_status;  // status of the failed normal attempt
    int use_sv;        // scale values provided (iterations >= 2)
    int num_events;    // compute_num_events for this call
    int n_cpts;        // changepoints after stall removal
    int rsrtr;         // read_start_rel_to_raw
    int n_norm;        // segs[-1]: clipped signal length
    int changed;       // norm_params_changed
    int path;          // 0 static, 1 adaptive
    int mapped_start, clip;
    int n_stalls;
    int pad_;
    double shc, scc;   // shift / scale correction factors of this call
    double score;      // sig_match_score
    tb2_scale_values sv;  // scale values produced by this call
};

// All pointers are device pointers.  Offsets: raw_off (n+1) samples; seq_off (n+1)
// base codes; base_off (n+1) mapped bases; ev_off (n+1) event slots.
struct BatchView {
    int n_reads;
    int kmer_width;
    int max_raw;       // longest raw signal of the batch (samples)
    const long long *raw_off, *seq_off, *base_off, *ev_off;
    const int *order;  // reads by descending raw length (launch order), null = index order
    const unsigned char *seq;
    double *rawf;      // raw signal as fp64 (reversed for RNA)          [sum S]
    double *norm;      // normalised signal of the current call         [sum S]
    double *cs;        // cumulative sums / candidate scores scratch    [sum S + n]
    double *scores;    //                                               [sum S]
    unsigned char *cstate;  // changepoint bit sets (spill)                [2 sum S + 2 n + 8]
    int *cpts;         // changepoints                                  [sum E]
    double *em;        // event means                                   [sum E]
    double *rm, *rs;   // expected levels                               [sum B]
    double *bm;        // per-base means                                [sum B]
    double *tmp_b;     // scratch                                       [sum B + n]
    int *starts;       // band starts / scratch                         [sum B]
    int *read_tb;      // traceback / scratch                           [sum B + n]
    int *segs_dp;      // segs after DP                                 [sum B + n]
    int *segs;         // final segs                                    [sum B + n]
    int *stall_ints;   // RNA stall intervals, 2 * stall_cap per read
    int stall_cap;
    ReadState *st;     //                                               [n]
};

struct StagePolicy {
    double outlier_thresh;       // NaN = None
    long long max_raw_cpts;      // < 0 = None
    double min_event_to_seq_ratio;
    double sig_match_thresh;
    int max_scaling_iters;
    int is_rna;
    int skip_seq_scaling;
    double const_scale;          // NaN = None
    unsigned int subsample_seed;
    int literal_key;             // mirror API: subsample_seed already is the key
    int read_index_base;         // index of the batch's first read in the caller's batch
    int thresh_with_sv;          // mirror API: winsorise supplied scale values by outlier_thresh
};

// launch wrappers (stage_kernels.cu); all enqueue on ctx->stream
int tb2_launch_prep(tb2_ctx *ctx, const BatchView &b, const void *raw_dev, int raw_dtype,
                    int is_rna, long long total_samples, long long total_bases);
int tb2_launch_begin_call(tb2_ctx *ctx, const BatchView &b, const tb2_params &p,
                          const StagePolicy &pol);
int tb2_launch_normalize(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol, int first_call);
int tb2_launch_cpts(tb2_ctx *ctx, const BatchView &b, const tb2_params &p, int on_raw);
int tb2_launch_rna_scale(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol);
int tb2_launch_event_means(tb2_ctx *ctx, const BatchView &b);
int tb2_launch_stalls(tb2_ctx *ctx, const BatchView &b);
int tb2_launch_resolve(tb2_ctx *ctx, const BatchView &b, const tb2_params &p,
                       const StagePolicy &pol, size_t rawdp_cap_doubles);
int tb2_launch_base_means(tb2_ctx *ctx, const BatchView &b);
int tb2_launch_theil_sen(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol, int first_call);
int tb2_launch_finalize(tb2_ctx *ctx, const BatchView &b, const StagePolicy &pol, int first_call,
                        double *norm_mean_out, double *norm_signal_out);
int tb2_launch_count_active(tb2_ctx *ctx, const BatchView &b, int *dev_counter);

// device view of the resident batch's results for the per-read statistics that follow
// the resquiggle (llr.cu, region_stats.cu); valid after tb2_batch_compute
struct BatchResultView {
    int n_reads;
    long long total_bases;
    const double *norm_mean;            // [sum B], offsets base_off
    const long long *base_off, *seq_off;
    const unsigned char *seq;
    const int *status;                  // status[r * stride]
    int stride;
};
int tb2_batch_result_view(tb2_ctx *ctx, BatchResultView *out);
int tb2_region_accumulate_dev(tb2_ctx *ctx, long long n, const double *stats_dev,
                              const long long *pos_dev, double thresh, double lower, int stat_type);

#ifndef TB2_EMUL
// Reads in host arrays (tb2_alt_model_llr_batch, tb2_alt_model_llr_motif_batch,
// tb2_de_novo_read_stats_batch): read r holds nb = mean_off[r + 1] - mean_off[r] means and
// the nb + K - 1 base codes of their k-mers at seq_off[r].  Checks that layout, with
// n_reads and every nb at most INT_MAX (the kernels index reads and bases with int), before
// reading any array past its first entry.  Then uploads the five arrays into buf[0..4] in
// argument order and points the read arrays of `a` (LlrArgs or FisherArgs) at them.
template <class Args>
int tb2_stage_reads(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean, const int64_t *mean_off,
                    const uint8_t *seq, const int64_t *seq_off, const int64_t *read_start,
                    DevBuf buf[5], Args &a)
{
    if (n_reads < 0 || n_reads > INT_MAX || !mean_off || !seq_off || !read_start)
        return TB2_ERR_INVALID_ARG;
    const int n = (int)n_reads;
    if (mean_off[0] < 0 || seq_off[0] < 0) return TB2_ERR_INVALID_ARG;
    for (int r = 0; r < n; ++r) {
        const long long nb = mean_off[r + 1] - mean_off[r];
        if (nb < 0 || nb > INT_MAX || seq_off[r + 1] - seq_off[r] != nb + (ctx->kmer_width - 1))
            return TB2_ERR_INVALID_ARG;
    }
    const size_t tm = (size_t)mean_off[n], ts = (size_t)seq_off[n];
    if ((tm && !norm_mean) || (ts && !seq)) return TB2_ERR_INVALID_ARG;
    cudaStream_t s = ctx->stream;
    TB2_CUDA_TRY(ctx, buf[0].upload(norm_mean, tm, s));
    TB2_CUDA_TRY(ctx, buf[1].upload(mean_off, (size_t)n + 1, s));
    TB2_CUDA_TRY(ctx, buf[2].upload(seq, ts, s));
    TB2_CUDA_TRY(ctx, buf[3].upload(seq_off, (size_t)n + 1, s));
    TB2_CUDA_TRY(ctx, buf[4].upload(read_start, (size_t)n, s));
    a.norm_mean = buf[0].as<double>();
    a.mean_off = buf[1].as<long long>();
    a.seq = buf[2].as<unsigned char>();
    a.seq_off = buf[3].as<long long>();
    a.read_start = buf[4].as<long long>();
    return TB2_OK;
}
#endif
