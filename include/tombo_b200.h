/* tombo_b200.h -- C ABI of the CUDA resquiggle engine (NVIDIA H100, sm_90a).
 *
 * Drop-in boundary for the native layer of nanoporetech/tombo's resquiggle hot
 * path: it replaces the two Cython extension modules
 *   tombo/_c_dynamic_programming.pyx   and   tombo/_c_helper.pyx
 * (built by the reference's setup.py:51-62) plus the per-read numpy glue of
 * tombo/resquiggle.py:345-1214 and tombo/tombo_stats.py:203-573, 2327-2370,
 * 3972-4082 with hand-written CUDA for sm_90a.
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / numpy types.
 *   - all buffers are CALLER allocated host memory (pinned where it matters); the
 *     library never frees caller memory.  Device memory is owned by the opaque
 *     tb2_ctx (one per GPU / host thread); calls on one ctx are serialised by the
 *     caller, different ctxs are independent.
 *   - floating point data is float64, indices int64 (as the reference:
 *     _c_dynamic_programming.pyx:9-13, _c_helper.pyx:6-13).
 *   - every call returns 0 (TB2_OK) or a TB2_ERR_* code; per-read outcomes of
 *     batched calls are reported in a status array with the same codes.  Codes
 *     1..25 map 1:1 onto the reference's TomboError / NotImplementedError message
 *     strings (tb2_status_message); the reference raises, we return.
 *   - there is NO CPU fallback: every entry point runs CUDA kernels and fails with
 *     TB2_ERR_CUDA if no sm_90-class device is usable.
 */
#ifndef TOMBO_B200_H
#define TOMBO_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TB2_ABI_VERSION 1

enum {
    TB2_OK = 0,
    TB2_ERR_FEWER_CPTS = 1,             /* _c_helper.pyx:118,200 */
    TB2_ERR_BEYOND_BANDWIDTH = 2,       /* _c_dynamic_programming.pyx:305 */
    TB2_ERR_ADAPTIVE_BEYOND_SIGNAL = 3, /* _c_dynamic_programming.pyx:354 */
    TB2_ERR_NOT_ENOUGH_DEL_SIGNAL = 4,  /* resquiggle.py:491 */
    TB2_ERR_TOO_MANY_DELS = 5,          /* resquiggle.py:496 */
    TB2_ERR_INVALID_SEG = 6,            /* resquiggle.py:530 */
    TB2_ERR_ZERO_LEN_SEG = 7,           /* resquiggle.py:534 */
    TB2_ERR_NEG_SEG = 8,                /* resquiggle.py:536 */
    TB2_ERR_SEG_PAST_END = 9,           /* resquiggle.py:538 */
    TB2_ERR_START_TOO_FAR = 10,         /* resquiggle.py:612 */
    TB2_ERR_MASKED_TOO_FEW = 11,        /* resquiggle.py:672 */
    TB2_ERR_READ_TOO_SHORT_START = 12,  /* resquiggle.py:704 */
    TB2_ERR_MAP_TOO_SHORT_START = 13,   /* resquiggle.py:706 */
    TB2_ERR_POOR_START_MATCH = 14,      /* resquiggle.py:746 */
    TB2_ERR_DISCORDANT_LEN = 15,        /* resquiggle.py:976 */
    TB2_ERR_OPEN_PORE = 16,             /* resquiggle.py:1010 */
    TB2_ERR_NO_RAW = 17,                /* resquiggle.py:1149 */
    TB2_ERR_TOO_MUCH_SIGNAL = 18,       /* resquiggle.py:1160 */
    TB2_ERR_SEG_COUNT = 19,             /* resquiggle.py:1201 */
    TB2_ERR_THEIL_SEN_ZERO = 20,        /* tombo_stats.py:421 */
    TB2_ERR_INVALID_START_PATH = 21,    /* tombo_stats.py:2356 */
    TB2_ERR_READ_TOO_SHORT_IN_REGION = 22,  /* tombo_stats.py:3944 */
    TB2_ERR_NO_INFO_IN_REGION = 23,     /* tombo_stats.py:3839-3841 */
    TB2_ERR_FISHER_TOO_SHORT = 24,      /* tombo_stats.py:2257-2259 */
    TB2_ERR_NO_VALID_Z = 25,            /* tombo_stats.py:3757-3758 */
    TB2_ERR_UNEXPECTED = 100,  /* the reference would raise a non-Tombo exception */
    /* library level */
    TB2_ERR_CUDA = 200,        /* CUDA runtime failure (see tb2_last_error) */
    TB2_ERR_INVALID_ARG = 201,
    TB2_ERR_CAPACITY = 202,    /* problem exceeds a compiled-in capacity */
    TB2_ERR_INVALID_SEQ = 203  /* non-ACGT base (reference exits: tombo_stats.py:858) */
};

/* mirrors tombo_helper.resquiggleParams (tombo_helper.py:173-198) */
typedef struct tb2_params {
    double match_evalue, skip_pen;
    int64_t bandwidth;
    double max_half_z_score;       /* NaN <=> None (no winsorising) */
    int64_t running_stat_width, min_obs_per_base, raw_min_obs_per_base,
        mean_obs_per_event;
    double z_shift, stay_pen;
    int64_t use_t_test_seg;
    int64_t band_bound_thresh, start_bw, start_save_bw, start_n_bases;
} tb2_params;

/* mirrors tombo_helper.scaleValues (tombo_helper.py:160-171); NaN <=> None */
typedef struct tb2_scale_values {
    double shift, scale, lower_lim, upper_lim, outlier_thresh;
} tb2_scale_values;

/* per-read policy constants (_default_parameters.py) and the worker's
 * iterate / rescue policy (resquiggle.py:1492-1504, 1578-1588) */
typedef struct tb2_policy {
    double outlier_thresh;          /* OUTLIER_THRESH; NaN <=> None */
    int64_t max_raw_cpts;           /* MAX_RAW_CPTS; < 0 <=> None */
    double min_event_to_seq_ratio;  /* MIN_EVENT_TO_SEQ_RATIO */
    double sig_match_thresh;        /* SIG_MATCH_THRESH[sample type] */
    int64_t max_scaling_iters;      /* MAX_SCALING_ITERS */
    int64_t is_rna;                 /* reverse signal + stall masking */
    int64_t skip_seq_scaling;
    double const_scale;             /* NaN <=> None */
    uint32_t subsample_seed;        /* keyed Theil-Sen sub-sampling (>1000 bases) */
    uint32_t rescue;                /* 1: retry failed reads with save params */
} tb2_policy;

typedef struct tb2_ctx tb2_ctx;

/* a TomboMotif (tombo_helper.py:542-640): mask[j] is the IUPAC class of motif base j as a
 * bit set (A = 1, C = 2, G = 4, T = 8; 'N' = 15), 1 <= len <= 32, 1-based
 * 1 <= mod_pos <= len; no mask may be 0 */
typedef struct tb2_motif {
    int32_t len, mod_pos;
    uint8_t mask[32];
} tb2_motif;

/* ---- context ---------------------------------------------------------- */
int tb2_abi_version(void);
int tb2_device_count(void);
int tb2_ctx_create(int device, tb2_ctx **out);
void tb2_ctx_destroy(tb2_ctx *ctx);
const char *tb2_status_message(int status);
/* the message of the last call on this ctx, empty if that call set none: every call that
 * takes a ctx starts from an empty message, except tb2_last_error, tb2_launch_count and
 * tb2_last_timing, which report on the call before them */
const char *tb2_last_error(tb2_ctx *ctx);
/* kernels launched by this ctx since creation (bench.py "gpu_launches") */
int64_t tb2_launch_count(tb2_ctx *ctx);
/* device time (ms, CUDA events on the ctx stream) of the last tb2_batch_compute:
 * out[0] whole compute stage, out[1] sum over launches of the dominant kernel
 * (banded DP, k_align), out[2] number of k_align launches, out[3] reads
 * processed summed over those launches.  After tb2_group_reg_stats / tb2_reads_ref_levels /
 * tb2_kmer_level_summaries / tb2_kmer_medians / tb2_de_novo_read_stats_batch /
 * tb2_de_novo_region_stats / tb2_sample_compare_region_stats / tb2_batch_de_novo_region /
 * tb2_accuracy_label_motif / _truth / _ctrl / tb2_accuracy_curve / tb2_accuracy_rates_ordered:
 * out[0] is the device time from the call's first kernel to its last (upload and download
 * excluded), out[1..3] are 0.  After tb2_kernel_densities: out[0] likewise, out[1] the part
 * of it spent in the per-set setup kernel (std, factor, kernel width), out[2..3] 0 */
int tb2_last_timing(tb2_ctx *ctx, double *out4);

/* page-locked host buffers (optional; any host memory is accepted by all calls) */
void *tb2_host_alloc(size_t bytes);
void tb2_host_free(void *p);

/* ---- k-mer model (TomboModel / AltModel tables) ----------------------- */
/* Dense table indexed by base-4 k-mer code (A=0,C=1,G=2,T=3, first base most
 * significant): replaces the dict lookups of TomboModel.get_exp_levels_from_seq
 * (tombo_stats.py:834-862, tombo_helper.py:526-540). */
int tb2_set_model(tb2_ctx *ctx, const double *means, const double *sds,
                  int kmer_width, int central_pos);
/* alt table: alt_means[code * kmer_width + pos], NaN where (kmer,pos) absent
 * (AltModel.get_exp_level tombo_stats.py:1084-1094) */
int tb2_set_alt_model(tb2_ctx *ctx, const double *alt_means, int kmer_width);

/* ---- single-array kernels mirroring the Cython entry points ----------- */
/* c_new_means _c_helper.pyx:59-71 */
int tb2_new_means(tb2_ctx *ctx, const double *sig, int64_t n_sig,
                  const int64_t *segs, int64_t n_segs, double *means_out);
/* c_new_mean_stds _c_helper.pyx:38-57 */
int tb2_new_mean_stds(tb2_ctx *ctx, const double *sig, int64_t n_sig,
                      const int64_t *segs, int64_t n_segs, double *means_out,
                      double *sds_out);
/* normalize_raw_signal tombo_stats.py:482-573 (+ c_apply_outlier_thresh
 * _c_helper.pyx:73-87).  norm_type 0 'median', 1 'median_const_scale';
 * sv_in may be NULL.  With sv_in and a threshold the limits come from the median
 * and MAD of the normalised signal, as in the reference. */
int tb2_normalize_raw_signal(tb2_ctx *ctx, const double *raw, int64_t n,
                             int norm_type, double outlier_thresh,
                             double const_scale, const tb2_scale_values *sv_in,
                             double *norm_out, tb2_scale_values *sv_out);
/* identify_stalls (mean-window method, MEAN_STALL_PARAMS) tombo_stats.py:269-368;
 * ints_out receives n_out (start, end) pairs (capacity `cap` pairs) */
int tb2_identify_stalls(tb2_ctx *ctx, const double *raw, int64_t n, int64_t *ints_out,
                        int64_t cap, int64_t *n_out);
/* c_valid_cpts_w_cap _c_helper.pyx:89-120 (+ sort, tombo_helper.py:76-82);
 * t_test != 0: c_valid_cpts_w_cap_t_test _c_helper.pyx:144-202.
 * Rank order: score descending, ties -> larger position first. */
int tb2_valid_cpts_w_cap(tb2_ctx *ctx, const double *sig, int64_t n,
                         int64_t min_base_obs, int64_t running_stat_width,
                         int64_t num_cpts, int t_test, int64_t *cpts_out,
                         int *read_status);
/* c_banded_forward_pass _c_dynamic_programming.pyx:240-279.
 * z: n_bases x bw; fwd_out / tb_out: (n_bases+1) x bw (row 0 of tb_out is 0). */
int tb2_banded_forward_pass(tb2_ctx *ctx, const double *z,
                            const int64_t *event_starts, int64_t n_bases,
                            int64_t bw, double skip_pen, double stay_pen,
                            double *fwd_out, int64_t *tb_out);
/* c_banded_traceback _c_dynamic_programming.pyx:281-310 */
int tb2_banded_traceback(tb2_ctx *ctx, const int64_t *tb,
                         const int64_t *event_starts, int64_t n_bases,
                         int64_t bw, int64_t band_pos,
                         int64_t band_boundary_thresh, int64_t *seq_poss_out,
                         int *read_status);
/* c_adaptive_banded_forward_pass _c_dynamic_programming.pyx:314-412: in place on
 * fwd / tb / event_starts from row start_seq_pos (rows <= start_seq_pos and
 * event_starts[:start_seq_pos] are inputs). */
int tb2_adaptive_banded_forward_pass(
    tb2_ctx *ctx, double *fwd, int64_t *tb, int64_t *event_starts,
    int64_t n_bases, int64_t bw, const double *event_means, int64_t n_events,
    const double *ref_means, const double *ref_sds, double z_shift,
    double skip_pen, double stay_pen, int64_t start_seq_pos,
    double mask_fill_z_score, int do_winsorize_z, double max_half_z_score,
    int *read_status);
/* calc_kmer_fitted_shift_scale(method='theil_sen') tombo_stats.py:401-450
 * (+ c_compute_slopes _c_helper.pyx:362-377); out4 = shift, scale,
 * shift_corr_factor, scale_corr_factor */
int tb2_theil_sen(tb2_ctx *ctx, double prev_shift, double prev_scale,
                  const double *event_means, const double *model_means,
                  int64_t n, uint32_t subsample_key, double *out4,
                  int *read_status);

/* ---- event -> sequence assignment ------------------------------------- */
/* find_adaptive_base_assignment resquiggle.py:866-1050 (start_clip_bases=None):
 * start finding, masked start, adaptive band, traceback, raw coordinates.
 * dbg (may be NULL) receives [path(0 static,1 adaptive), mapped_start,
 * events_start_clip]. */
int tb2_find_adaptive_base_assignment(
    tb2_ctx *ctx, const int64_t *valid_cpts, int64_t n_cpts,
    const double *event_means, const tb2_params *params,
    const double *ref_means, const double *ref_sds, int64_t n_bases,
    double sig_match_thresh, int64_t *segs_out, int64_t *read_start_rel_to_raw,
    int64_t *dbg, int *read_status);
/* find_static_base_assignment resquiggle.py:547-600: read_tb_out has n_bases + 1
 * event positions (the th.banded_traceback result) */
int tb2_find_static_base_assignment(tb2_ctx *ctx, const double *event_means,
                                    int64_t n_events, const double *ref_means,
                                    const double *ref_sds, int64_t n_bases,
                                    const tb2_params *params, int64_t *read_tb_out,
                                    int *read_status);
/* find_seq_start_in_events resquiggle.py:685-752; check_score <=> seq_samp_type
 * passed (SIG_MATCH_THRESH test, :742-746) */
int tb2_find_seq_start_in_events(tb2_ctx *ctx, const double *event_means,
                                 int64_t n_events, const double *ref_means,
                                 const double *ref_sds, int64_t n_ref,
                                 const tb2_params *params, int64_t num_bases,
                                 int64_t num_events, int check_score,
                                 double sig_match_thresh, int64_t *start_loc,
                                 double *events_per_base, int *read_status);
/* self-check: blocks x 256 x per_thread random / adversarial (a, b) pairs; counts
 * pairs where the reciprocal-based division of the DP rows differs from a / b */
int tb2_debug_div_check(tb2_ctx *ctx, uint64_t seed, int blocks, int per_thread,
                        uint64_t *mismatches, double *example4);
/* tuning / test counters (device-global, cumulative: compare deltas): [0] Theil-Sen calls,
 * [1] fp32 bracket over every pair, [2] exact histogram path, [3] generic radix-select path,
 * [4] fp32 bracket over sampled pairs, [5] sort-and-sweep finished, [6] sort-and-sweep
 * abandoned (one of [1]-[4] then finishes), [7] sweep phases (TS_DEBUG builds only) */
int tb2_debug_counters(tb2_ctx *ctx, unsigned long long *out8, int reset);
/* resolve_skipped_bases_with_raw resquiggle.py:402-540 */
int tb2_resolve_skipped_bases_with_raw(
    tb2_ctx *ctx, const int64_t *segs, int64_t n_bases, const double *ref_means,
    const double *ref_sds, const double *norm_signal, int64_t n_norm,
    const tb2_params *params, int64_t max_raw_cpts, int64_t *segs_out,
    int *read_status);

/* ---- the batched hot path --------------------------------------------- */
/* Inputs are flat concatenations with int64 offsets (n_reads + 1 entries):
 *   raw      raw signal of all reads; raw_dtype 0 = float64, 1 = int16
 *   seq      base codes (0..3 = ACGT) of each read's genome_seq
 *            (n_bases + kmer_width - 1 codes per read)
 * Outputs (caller allocated):
 *   segs            sum(n_bases + 1) int64 with seg_off = seq based offsets
 *                   computed by the caller as cumsum(n_bases_r + 1)
 *   read_start_rel_to_raw, status, n_iters, flags   [n_reads]
 *   scale_out       [n_reads] tb2_scale_values
 *   sig_match_score [n_reads]
 *   norm_mean       sum(n_bases) float64 per-base means of the final normalised
 *                   signal (the FAST5 Events.norm_mean column,
 *                   tombo_helper.py:2341-2460) with offsets cumsum(n_bases_r)
 *   norm_signal     optional (NULL to skip): clipped, re-normalised signal with
 *                   the raw offsets; read r holds segs_r[-1] valid samples.
 * flags bit0: norm_params_changed after the last iteration, bit1: rescued with
 * save params, bit2: static (short read) path taken (clear for a read that failed
 * before the alignment).
 * A sequence without a k-mer (fewer than kmer_width codes) fails with
 * TB2_ERR_TOO_MUCH_SIGNAL as in resquiggle_read, or TB2_ERR_DISCORDANT_LEN when the read
 * has too few samples for one event.
 * raw_off[0] and seq_off[0] must be 0 and neither may decrease (else
 * TB2_ERR_INVALID_ARG), whether the batch goes as one chunk or is pipelined.
 * Whatever it returns, the call leaves no resident batch: afterwards the calls on the
 * resident batch (tb2_batch_download, tb2_batch_alt_llr, tb2_batch_alt_llr_motif,
 * tb2_batch_de_novo_region) return TB2_ERR_INVALID_ARG until the next tb2_batch_compute. */
int tb2_resquiggle_batch(
    tb2_ctx *ctx, int64_t n_reads, const void *raw, int raw_dtype,
    const int64_t *raw_off, const uint8_t *seq, const int64_t *seq_off,
    const tb2_params *params, const tb2_params *save_params,
    const tb2_policy *policy, int64_t *segs, int64_t *read_start_rel_to_raw,
    tb2_scale_values *scale_out, double *sig_match_score, double *norm_mean,
    double *norm_signal, int32_t *status, int32_t *n_iters, int32_t *flags);

/* Host-only helper: the chunk schedule tb2_resquiggle_batch uses for n_reads on a device
 * with sm_count SMs (chunk k = reads [starts_out[k], starts_out[k+1])).  Returns the
 * number of chunks (1 = unpipelined) or a negated TB2_ERR_* code; needs no device. */
int tb2_pipeline_chunks(int sm_count, int64_t n_reads, int64_t *starts_out, int cap);

/* The same call in three stages, for callers that keep inputs resident in HBM or
 * overlap transfers themselves: upload (H2D of raw / seq, allocation), compute
 * (kernels only, results stay on the device), download (D2H into caller buffers
 * laid out as in tb2_resquiggle_batch).  compute may be repeated on one upload.  A failed
 * upload leaves no batch, a failed compute no results: the calls that need them return
 * TB2_ERR_INVALID_ARG until the next successful upload / compute. */
int tb2_batch_upload(tb2_ctx *ctx, int64_t n_reads, const void *raw, int raw_dtype,
                     const int64_t *raw_off, const uint8_t *seq,
                     const int64_t *seq_off, const tb2_params *params,
                     const tb2_policy *policy);
/* optional, between upload and compute: per-read map_res.scale_values (sv_in[r]
 * with NaN shift = none) and map_res.stall_ints (pairs (start, end), stall_off has
 * n_reads + 1 entries counting pairs, starting at 0 and never decreasing); either may
 * be NULL, and a later call replaces both.  A changepoint c is tested against the first
 * interval of its read, in list order, whose end is >= c (the last interval if none),
 * as remove_stall_cpts does; any int64 interval list is accepted.  Stall inputs on an
 * RNA-policy upload, which detects stalls itself, return TB2_ERR_INVALID_ARG; stall
 * lists with n_reads * (longest list) above 4 * samples + 1024 pairs return
 * TB2_ERR_CAPACITY. */
int tb2_batch_set_read_inputs(tb2_ctx *ctx, const tb2_scale_values *sv_in,
                              const int64_t *stall_ints, const int64_t *stall_off);
int tb2_batch_compute(tb2_ctx *ctx, const tb2_params *params,
                      const tb2_params *save_params, const tb2_policy *policy,
                      int want_norm_signal);
int tb2_batch_download(tb2_ctx *ctx, int64_t *segs, int64_t *read_start_rel_to_raw,
                       tb2_scale_values *scale_out, double *sig_match_score,
                       double *norm_mean, double *norm_signal, int32_t *status,
                       int32_t *n_iters, int32_t *flags);

/* compute_alt_model_read_stats tombo_stats.py:3972-4082 for whole reads
 * (reg_data=None, '+' strand read-centric data), default
 * c_calc_scaled_llh_ratio_const_var (_c_helper.pyx:313-358) or, with
 * use_standard_llhr, c_calc_llh_ratio_const_var (:298-311).
 * Sites are the positions of `alt_base_code` in the motif-searchable part of each
 * read (single-base motif, TomboMotif(alt_base, 1)).  site_off has n_reads+1
 * entries (filled); llr_out / pos_out sized by the caller to site capacity
 * (sum of n_bases is always enough).  Motif models, '-' strand reads and regions:
 * tb2_alt_model_llr_motif_batch. */
int tb2_alt_model_llr_batch(
    tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
    const int64_t *mean_off, const uint8_t *seq, const int64_t *seq_off,
    const int64_t *read_start, int alt_base_code, int use_standard_llhr,
    double scale_factor, double height_factor, double height_power,
    double *llr_out, int64_t *pos_out, int64_t *site_off);

/* The three Cython scorers batched over explicit windows (n_sites x kmer_width,
 * row-major): mode 0 c_calc_scaled_llh_ratio_const_var (_c_helper.pyx:313-358),
 * mode 1 c_calc_llh_ratio_const_var (:298-311), mode 2 c_calc_llh_ratio (:277-296).
 * var_a = const_var[n_sites] (modes 0, 1) or ref_vars[n_sites x K] (mode 2);
 * var_b = alt_vars[n_sites x K] (mode 2 only). */
int tb2_calc_llh_ratio_windows(tb2_ctx *ctx, int mode, int64_t n_sites, int kmer_width,
                               const double *means, const double *ref_means,
                               const double *alt_means, const double *var_a,
                               const double *var_b, double scale_factor,
                               double height_factor, double height_power,
                               double *llr_out);

/* device stopwatch (CUDA events on the context's stream) around any sequence of calls on
 * this context; stop synchronises and returns the elapsed milliseconds */
int tb2_timer_start(tb2_ctx *ctx);
int tb2_timer_stop(tb2_ctx *ctx, double *ms_out);

/* ---- per-read statistics on the RESIDENT batch (after tb2_batch_compute) -------------
 * compute_alt_model_read_stats (tombo_stats.py:3972-4082) for every successfully
 * resquiggled read of the batch without leaving HBM: sequence, per-base means and status
 * are already there.  read_start[n_reads] are the reads' genome start positions.  LLRs and
 * positions stay on the device for tb2_region_stats_add_batch_llr; tb2_batch_llr_download
 * copies them out (site_off has n_reads + 1 entries; llr_out / pos_out sized
 * *n_sites_total).  Single-base motif, whole '+' strand reads; any motif, both strands and
 * a region: tb2_batch_alt_llr_motif.  A failed call of either leaves no LLRs resident:
 * tb2_batch_llr_download and tb2_region_stats_add_batch_llr then return
 * TB2_ERR_INVALID_ARG until the next successful one. */
int tb2_batch_alt_llr(tb2_ctx *ctx, const int64_t *read_start, int alt_base_code,
                      int use_standard_llhr, double scale_factor, double height_factor,
                      double height_power, int64_t *n_sites_total);
int tb2_batch_llr_download(tb2_ctx *ctx, double *llr_out, int64_t *pos_out, int64_t *site_off);

/* ---- alternative-model LLRs for any motif, both strands, one region ------------------
 * compute_alt_model_read_stats (tombo_stats.py:3972-4082) with trim_seq_and_means
 * (:3888-3970) for one alt model with a motif (tombo.DNA.CpG / dam / dcm: CG:1, GATC:2,
 * CCWGG:2), reads mapped to either strand and the region [reg_start, reg_end).  The data
 * are read-centric as the reference stores them: read r's nb trimmed bases S (the reverse
 * complement of the genome for '-' reads) sit at seq[seq_off[r] + cpos ...] inside its
 * nb + K - 1 codes, with the nb per-base means; read_start[r] is the genome's low
 * coordinate on both strands.  Codes outside S are read as 'N' whatever they hold.
 *   - strand[r]: 0 '+', 1 '-', -1 skip the read (no sites, status 0; on the resident
 *     batch a read whose resquiggle failed reports that status whatever its strand).
 *   - max_motif_bb / max_motif_ab: max(mod_pos - 1) and max(len - mod_pos) over every alt
 *     model of the reference's call, so several calls (one per model) reproduce one joint
 *     call; each must be at least this motif's own value.
 *   - reads that reach outside the region are clipped as the reference does; a read with
 *     fewer than K testable levels left gets TB2_ERR_READ_TOO_SHORT_IN_REGION in
 *     read_status (nullable, n_reads entries; 0 otherwise) and no sites.  A region that
 *     contains every read ([min start, max start + nb)) scores whole reads (reg_data=None).
 *   - sites are the leftmost non-overlapping motif matches (re.finditer) in read order;
 *     positions are genome positions, descending for '-' reads, as the reference returns
 *     them.
 *   - the reference's zero-width slice quirks are kept: with central_pos == K - 1 every
 *     read whose 3' end is not clipped is too short, and when clip3 + K - 1 == max_ab
 *     (e.g. CNNNNN:1 with 6-mers on a whole read) the read has no sites.
 * TB2_ERR_INVALID_ARG: malformed motif, max_motif_bb < mod_pos - 1, max_motif_ab <
 * len - mod_pos, a strand outside {-1, 0, 1}, models of different k-mer widths, or reads
 * whose code count is not nb + K - 1.  llr_out / pos_out hold up to sum(nb) sites. */
int tb2_alt_model_llr_motif_batch(
    tb2_ctx *ctx, int64_t n_reads, const double *norm_mean, const int64_t *mean_off,
    const uint8_t *seq, const int64_t *seq_off, const int64_t *read_start, const int8_t *strand,
    const tb2_motif *motif, int64_t max_motif_bb, int64_t max_motif_ab, int64_t reg_start,
    int64_t reg_end, int use_standard_llhr, double scale_factor, double height_factor,
    double height_power, double *llr_out, int64_t *pos_out, int64_t *site_off,
    int32_t *read_status);
/* the same on the RESIDENT batch (after tb2_batch_compute); read_start / strand have
 * n_reads entries.  It replaces the resident LLRs exactly as tb2_batch_alt_llr does, so
 * tb2_batch_llr_download and tb2_region_stats_add_batch_llr read its sites: one call per
 * strand (the other strand's reads at -1) feeds that strand's region counters.  Reads whose
 * resquiggle failed hold no sites and report their resquiggle status in read_status, also
 * when their strand is -1. */
int tb2_batch_alt_llr_motif(tb2_ctx *ctx, const int64_t *read_start, const int8_t *strand,
                            const tb2_motif *motif, int64_t max_motif_bb, int64_t max_motif_ab,
                            int64_t reg_start, int64_t reg_end, int use_standard_llhr,
                            double scale_factor, double height_factor, double height_power,
                            int32_t *read_status, int64_t *n_sites_total);

/* ---- SURVEY 8(f)-1: per-position aggregation of per-read statistics -----------------
 * collate_reg_stats tombo_stats.py:4124-4178 + apply_per_read_thresh :4084-4122 +
 * calc_damp_fraction :2537-2552 for one region [reg_start, reg_start + reg_len) (the
 * reference works in 10 kb blocks, :4591-4595).  begin zeroes three dense int32 counters
 * per position (coverage, valid coverage, stats >= single_read_thresh); add* accumulate
 * (NaN stats are dropped like :4130-4133; lower_thresh NaN <=> None; stat_type 0 =
 * alternative-model LLR, 1 = de novo / sample compare); finalize returns the covered
 * positions in ascending order with reg_frac_standard_base, the dampened fraction
 * (unmod_count / mod_count pseudo counts, NaN unmod_count = skip), reg_cov and valid_cov.
 * Counters are sums: reads of one region sharded over GPUs are combined by adding the
 * arrays returned by tb2_region_counts_get (3 * reg_len int32) -- with NCCL / any
 * all-reduce -- and storing the sum with tb2_region_counts_set before finalize. */
int tb2_region_stats_begin(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len);
int tb2_region_stats_add(tb2_ctx *ctx, int64_t n, const double *stats, const int64_t *pos,
                         double single_read_thresh, double lower_thresh, int stat_type);
int tb2_region_stats_add_batch_llr(tb2_ctx *ctx, double single_read_thresh,
                                   double lower_thresh, int stat_type);
int tb2_region_counts_get(tb2_ctx *ctx, int32_t *counts);
int tb2_region_counts_set(tb2_ctx *ctx, const int32_t *counts);
int tb2_region_stats_finalize(tb2_ctx *ctx, double unmod_count, double mod_count, int64_t cap,
                              int64_t *pos_out, double *frac_out, double *damp_frac_out,
                              int64_t *cov_out, int64_t *valid_cov_out, int64_t *n_out);

/* ---- SURVEY 8(f)-2: de novo / sample-compare per-read tests -------------------------
 * z = |mean - ref| / sd -> two-sided normal p -> windowed Fisher's method
 * (calc_window_fishers_method tombo_stats.py:2252-2271; fm_offset 0 = plain p-values).
 * tb2_window_fisher_pvals works on explicit level arrays cut into segments (seg_off has
 * n_segs + 1 entries): the arithmetic of compute_sample_compare_read_stats (:3675-3769,
 * final_clamp 0) and of compute_de_novo_read_stats (:3771-3873, final_clamp 1:
 * np.maximum(p, SMALLEST_PVAL)).  Outputs have the inputs' length; the first / last
 * fm_offset entries of a segment and entries with NaN inputs are NaN.  With ref_means and
 * ref_sds both NULL, `means` holds p-values already (the bare Fisher window).  Floating point:
 * erfc / log of the device library and tb2_chi2_sf_even (special.cuh: the closed form below
 * y = 700, Loader's saddle-point form above, relative error <= 1e-12 + 16 u y); each p within
 * (4 x^2 + 16) u of the exact value (x = z / sqrt 2, u = 2^-53), each window within the
 * propagated log-sum error plus the chi-square error (tests/stats_cases.py).
 * tb2_de_novo_read_stats_batch runs the de novo test for whole '+' strand reads with
 * the canonical levels looked up on the device (tb2_set_model): stat_off (n_reads + 1,
 * filled) counts n_bases - (kmer_width - 1) positions per read. */
int tb2_window_fisher_pvals(tb2_ctx *ctx, int64_t n_segs, const double *means,
                            const double *ref_means, const double *ref_sds,
                            const int64_t *seg_off, int64_t fm_offset, int final_clamp,
                            double *pvals_out);
int tb2_de_novo_read_stats_batch(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                                 const int64_t *mean_off, const uint8_t *seq,
                                 const int64_t *seq_off, const int64_t *read_start,
                                 int64_t fm_offset, double *pvals_out, int64_t *pos_out,
                                 int64_t *stat_off);

/* ---- de novo / sample-compare tests of one region, both strands ----------------------
 * compute_reg_stats (tombo_stats.py:4180-4229) runs one per-read test per read of a region
 * block; these run it for n_reads reads over [reg_start, reg_end) in one call.  strand[r]:
 * 0 '+', 1 '-', -1 skip the read (no statistics, status 0).  Read data are read-centric as
 * the reference stores them; read_start[r] is the genome's low coordinate on both strands and
 * the read ends at read_start[r] + nb.  Outputs are laid out by stat_off (n_reads + 1,
 * filled); pvals_out / pos_out hold up to sum(nb) entries.  read_status (nullable, n_reads)
 * gets 0 or the code of the TomboError the reference raises for the read; such a read has no
 * statistics.  The statistics also stay on the device for tb2_region_stats_add_tests, until
 * the next call of either function or of tb2_batch_de_novo_region; a failed call of any of
 * the three leaves none, and tb2_region_stats_add_tests returns TB2_ERR_INVALID_ARG until
 * the next successful one.  fm_offset 0 .. 64.
 * tb2_last_timing out[0] is the kernel time.
 *
 * tb2_de_novo_region_stats: compute_de_novo_read_stats (:3771-3873) with the canonical model
 * (tb2_set_model) in the layout of tb2_alt_model_llr_motif_batch (nb + K - 1 codes per read,
 * the read's bases from code cpos).  Per read: the clip by the strand's k-mer lags plus
 * fm_offset, with Python's slicing (a clip longer than the read empties it); k-mers of the
 * clipped bases, reversed for '-' reads; means flipped to genome order and trimmed by the
 * lags; z -> two-sided p -> Fisher window -> max(p, SMALLEST_PVAL).  Positions ascend on
 * both strands; the window's NaN edges are kept.  r_means[begin:-0] is empty when the end
 * lag is 0 (central_pos == K - 1 on '+', 0 on '-'): such a read has no statistics.
 * Statuses: TB2_ERR_NO_INFO_IN_REGION (fewer than K clipped bases), TB2_ERR_INVALID_SEQ
 * (a non-ACGT code or a k-mer absent from the model among the clipped bases' k-mers; codes
 * outside them are never read), TB2_ERR_FISHER_TOO_SHORT.
 *
 * tb2_sample_compare_region_stats: compute_sample_compare_read_stats (:3675-3769) against
 * ctrl_means / ctrl_sds over [reg_start - fm_offset, reg_end + fm_offset) (get_reads_ref).
 * Per read: the clip by fm_offset, flip, z against the control slice, p (no clamp), the
 * Fisher window; only the non-NaN entries are returned, in genome order.  Statuses:
 * TB2_ERR_NO_VALID_Z, TB2_ERR_FISHER_TOO_SHORT.
 *
 * TB2_ERR_INVALID_ARG: a strand outside {-1, 0, 1}, fm_offset outside 0 .. 64,
 * reg_end <= reg_start, NULL ctrl_* (sample compare), a code count that is not nb + K - 1 or
 * no model set (de novo). */
int tb2_de_novo_region_stats(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                             const int64_t *mean_off, const uint8_t *seq, const int64_t *seq_off,
                             const int64_t *read_start, const int8_t *strand, int64_t fm_offset,
                             int64_t reg_start, int64_t reg_end, double *pvals_out,
                             int64_t *pos_out, int64_t *stat_off, int32_t *read_status);
int tb2_sample_compare_region_stats(tb2_ctx *ctx, int64_t n_reads, const double *norm_mean,
                                    const int64_t *mean_off, const int64_t *read_start,
                                    const int8_t *strand, const double *ctrl_means,
                                    const double *ctrl_sds, int64_t fm_offset, int64_t reg_start,
                                    int64_t reg_end, double *pvals_out, int64_t *pos_out,
                                    int64_t *stat_off, int32_t *read_status);
/* the de novo test on the RESIDENT batch (after tb2_batch_compute): read_start / strand have
 * one entry per read of the batch.  Reads whose resquiggle failed report that status (also at
 * strand -1) and feed nothing to the counters; their outputs are NaN.  pvals_out / pos_out /
 * stat_off / read_status may be NULL: the statistics stay on the device for
 * tb2_region_stats_add_tests, so resquiggle -> de novo -> region counts never leaves HBM. */
int tb2_batch_de_novo_region(tb2_ctx *ctx, const int64_t *read_start, const int8_t *strand,
                             int64_t fm_offset, int64_t reg_start, int64_t reg_end,
                             double *pvals_out, int64_t *pos_out, int64_t *stat_off,
                             int32_t *read_status);
/* accumulate the statistics of the last de novo / sample-compare region call into the open
 * region (tb2_region_stats_begin) as stat_type 1; lower_thresh NaN <=> None */
int tb2_region_stats_add_tests(tb2_ctx *ctx, double single_read_thresh, double lower_thresh);

/* ---- level_sample_compare and control-sample reference levels ------------------------
 * One region [reg_start, reg_start + reg_len) per call, already widened by fm_offset
 * (tombo_stats.py:4337-4342, :3639-3641).  Each sample is a set of ragged per-read level
 * arrays in genome order: read r has levels[off[r] .. off[r+1]) at genome positions
 * start[r], start[r] + 1, ... (minus-strand reads reversed by the caller, as
 * get_single_slot_genome_centric does).  Levels outside the region are ignored; NaN is
 * missing.  reg_len is at most 2^24, each sample at most 2^30 - 1 reads.
 *
 * tb2_group_reg_stats: compute_group_reg_stats :4335-4393.  test 0 = KS (:4236-4255),
 * 1 = Mann-Whitney U (:4266-4291), 2 = t (:4302-4324); return_stat selects the
 * *_stat_test variant.  Positions where both samples have >= min_test_reads levels form
 * runs; runs shorter than 2 fm_offset + 1 are dropped (:4355); with fm_offset > 0 the
 * p-values of each run go through Fisher's method (calc_window_fishers_method :2252-2271)
 * and statistics through calc_window_means (:2273-2287), NaN at the first / last fm_offset
 * positions of a run.  Outputs: covered positions ascending, statistic, sample and control
 * coverage; *n_out = number of positions (TB2_ERR_CAPACITY when it exceeds cap; the first
 * cap are written).  U ties: sample levels rank before equal control levels.  Where the
 * reference raises FloatingPointError (zero pooled variance in the t test, a single level
 * in each sample) the statistic is NaN.  min_test_reads < 1, reg_len, fm_offset (0 .. 2^24)
 * or a read count out of range -> TB2_ERR_INVALID_ARG.
 *
 * tb2_reads_ref_levels: get_reads_ref :3627-3673.  Per position with >= min_test_reads
 * levels: np.median (np.mean with est_mean) and np.std of the levels in read order; with
 * prior_means / prior_sds (reg_len each) compute_posterior_samp_dists' weighted means
 * (:3589-3594); positions with sd == 0 and uncovered ones are NaN.  cov_out[reg_len] is
 * the number of levels per position. */
int tb2_group_reg_stats(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len,
                        int64_t n_samp, const double *samp_levels, const int64_t *samp_off,
                        const int64_t *samp_start, int64_t n_ctrl, const double *ctrl_levels,
                        const int64_t *ctrl_off, const int64_t *ctrl_start, int test,
                        int return_stat, int64_t min_test_reads, int64_t fm_offset, int64_t cap,
                        int64_t *pos_out, double *stat_out, int64_t *cov_out,
                        int64_t *ctrl_cov_out, int64_t *n_out);
int tb2_reads_ref_levels(tb2_ctx *ctx, int64_t reg_start, int64_t reg_len, int64_t n_reads,
                         const double *levels, const int64_t *off, const int64_t *start,
                         int64_t min_test_reads, int est_mean, const double *prior_means,
                         const double *prior_sds, double mean_prior_weight,
                         double sd_prior_weight, double *means_out, double *sds_out,
                         int64_t *cov_out);

/* ---- alternative-model estimation: per-k-mer Gaussian kernel densities ----------------
 * est_kernel_density tombo_stats.py:1914-1939 for n_sets ragged sets of levels (set s is
 * levels[off[s] .. off[s+1]), in the order parse_base_levels :1811-1884 collects them):
 * gaussian_kde(levels, bw_method=bw / levels.std(ddof=1)).evaluate(x) on the n_points grid
 * x.  dens_out[s * n_points + j] is the density of set s at x[j]; cho_cov_out[s] is the
 * kernel width (scipy's cho_cov); factor_out (may be NULL) gets bw / std(ddof=1).
 * Arithmetic (DESIGN.md §2 "Kernel densities"): std(ddof=1) and factor in numpy's pairwise
 * order, bit-exact; cho_cov from pairwise sums where np.cov uses a BLAS dot (within
 * gamma_n + 6u of scipy's); each term exp(-(p_i - q_j)^2 / 2) * norm times 1/n as
 * gaussian_kernel_estimate computes it, with the device exp and a different summation
 * order (bound in DESIGN.md).  Where the reference raises -- fewer than 2 levels, a
 * non-finite level, zero or overflowing standard deviation -- the set's row, cho_cov and
 * factor are NaN.  n_sets out of 0 .. 2^31 - 1, a set of more than 2^31 - 1 levels, bad
 * offsets, n_points out of 1 .. 2^20, a NULL grid, or bw <= 0 / non-finite ->
 * TB2_ERR_INVALID_ARG.  tb2_last_timing out[0] is the kernel time, out[1] the setup kernel's
 * share of it. */
int tb2_kernel_densities(tb2_ctx *ctx, int64_t n_sets, const double *levels,
                         const int64_t *off, int64_t n_points, const double *x, double bw,
                         double *dens_out, double *cho_cov_out, double *factor_out);

/* ---- standard and motif k-mer model estimation ------------------------------------------
 * Per-position level summaries of get_region_kmer_levels tombo_stats.py:1263-1280 and
 * 1349-1355 for a batch of regions laid end to end in positions 0 .. n_pos - 1.  Reads are
 * ragged genome-ordered levels (read r is levels[off[r] .. off[r+1]) starting at position
 * start[r]; levels outside 0 .. n_pos - 1 are ignored).  cov_out[p] is the number of
 * non-NaN levels at p.  Where cov_out[p] > cov_thresh: level_out[p], sd_out[p] are
 * calc_med_sd (:1236-1240: np.median, np.std) or, with est_mean, c_mean_std
 * (_c_helper.pyx:22-36) of the levels in read order; elsewhere NaN.  Arithmetic: DESIGN.md
 * §2 "K-mer model estimation".  n_pos out of 1 .. 2^24, more than 2^30 - 1 reads, bad
 * offsets, cov_thresh out of 0 .. 2^31 - 2 or a NULL output -> TB2_ERR_INVALID_ARG.
 * tb2_last_timing out[0] is the kernel time. */
int tb2_kmer_level_summaries(tb2_ctx *ctx, int64_t n_pos, int64_t n_reads, const double *levels,
                             const int64_t *off, const int64_t *start, int64_t cov_thresh,
                             int est_mean, double *level_out, double *sd_out, int64_t *cov_out);
/* Grouped medians of tabulate_kmer_levels :1462-1487 and tabulate_mod_kmer_levels
 * :2116-2144: for each key k in 0 .. n_keys - 1, count_out[k] observations i with
 * keys[i] == k, and np.median of their levels and of their sds (the mean of the two middle
 * values for an even count; NaN for no observation), exact.  The key is the base-4 k-mer
 * code, or code * kmer_width + offset for motif k-mers.  n_keys out of 1 .. 2^24, n_obs out
 * of 0 .. 2^30, a key out of range, a NaN level or sd, or a NULL pointer ->
 * TB2_ERR_INVALID_ARG.  tb2_last_timing out[0] is the kernel time. */
int tb2_kmer_medians(tb2_ctx *ctx, int64_t n_keys, int64_t n_obs, const int64_t *keys,
                     const double *levels, const double *sds, int64_t *count_out,
                     double *level_med_out, double *sd_med_out);

/* ---- accuracy of modified-base calls (tombo plot roc and friends) ------ */
/* Labelling appends (stat, label) entries to slots 0 .. 15 (one per modification name) that
 * stay on the device until tb2_accuracy_reset; tb2_accuracy_curve turns a slot into the
 * sampled rates of prep_accuracy_rates (_plot_commands.py:60-82).
 *
 * One statistics block (chrm, strand, start, end, block_stats) of the stats iterator:
 * its reg_seq as codes seq[seq_off .. seq_off + seq_len) (A C G T = 0..3, anything else 4)
 * starting at genome position seq_start; its statistics (pos, stat)[stat_off .. + n_stat);
 * control statistics [ctrl_off .. + n_ctrl) (tb2_accuracy_label_ctrl); the sorted unique
 * mod / unmod locations of its (chrm, strand) inside [start, end) (tb2_accuracy_label_truth);
 * strand 0 '+', 1 '-'.  Unused ranges are 0.  The calls take the blocks as rows of
 * TB2_ACC_BLOCK_FIELDS int64 values in this field order. */
typedef struct tb2_acc_block {
    int64_t seq_off, seq_len, seq_start;
    int64_t stat_off, n_stat, ctrl_off, n_ctrl;
    int64_t mod_off, n_mod, unmod_off, n_unmod;
    int64_t strand;
} tb2_acc_block;
#define TB2_ACC_BLOCK_FIELDS 12

/* empties every slot */
int tb2_accuracy_reset(tb2_ctx *ctx);
/* entries of a slot */
int tb2_accuracy_count(tb2_ctx *ctx, int slot, int64_t *n_out);
/* a slot's entries in append order (stat, label 0/1) */
int tb2_accuracy_download(tb2_ctx *ctx, int slot, double *stat_out, uint8_t *label_out);
/* replaces a slot's entries (labels 0/1) */
int tb2_accuracy_load(tb2_ctx *ctx, int slot, int64_t n, const double *stat, const uint8_t *label);
/* _compute_motif_stats (tombo_stats.py:2406-2456) of n_blocks blocks: for each statistic
 * and each motif in order whose mod base is window[bb], appends (stat, prefix match) to
 * slot[m].  bb / ab are max(mod_pos) - 1 and max(len - mod_pos) over the motifs (1 .. 8).
 * counts_out[b * n_motifs + m]: entries of block b for motif m.  A window the reference
 * cannot index (IndexError) -> TB2_ERR_UNEXPECTED and nothing appended. */
int tb2_accuracy_label_motif(tb2_ctx *ctx, int64_t n_blocks, const int64_t *blocks,
                             int64_t n_seq, const uint8_t *seq, int64_t n_stat,
                             const uint32_t *pos, const double *stat, int n_motifs,
                             const tb2_motif *motifs, const int32_t *slot, int64_t bb,
                             int64_t ab, int64_t *counts_out);
/* _compute_ground_truth_stats (:2458-2483): statistics at a mod or unmod location, in block
 * order, labelled pos in mod; counts_out[b] */
int tb2_accuracy_label_truth(tb2_ctx *ctx, int64_t n_blocks, const int64_t *blocks,
                             int64_t n_stat, const uint32_t *pos, const double *stat,
                             int64_t n_mod, const int64_t *mod_locs, int64_t n_unmod,
                             const int64_t *unmod_locs, int slot, int64_t *counts_out);
/* _compute_ctrl_motif_stats (:2485-2535): per block and motif, the re.finditer sites of the
 * motif ('+') or its reverse complement ('-') in reg_seq; sample statistics at a site
 * (True), then control statistics at a site (False); counts_out[b * n_motifs + m] */
int tb2_accuracy_label_ctrl(tb2_ctx *ctx, int64_t n_blocks, const int64_t *blocks,
                            int64_t n_seq, const uint8_t *seq, int64_t n_stat,
                            const uint32_t *pos, const double *stat, int64_t n_ctrl,
                            const uint32_t *ctrl_pos, const double *ctrl_stat, int n_motifs,
                            const tb2_motif *motifs, const int32_t *slot, int64_t *counts_out);
/* prep_accuracy_rates of one slot: the labels in Python's (stat, label) tuple order, then
 * compute_accuracy_rates sampled at rate_idx (tp_rate, fp_rate) and prec_idx (precision),
 * n_points each, computed by the caller as numpy's linspace(...).astype(int64).  An empty
 * slot or a NaN statistic -> TB2_ERR_INVALID_ARG; a buffer that does not fit on the device
 * -> TB2_ERR_CAPACITY.  tb2_last_timing out[0] is the kernel time. */
int tb2_accuracy_curve(tb2_ctx *ctx, int slot, int64_t n_points, const int64_t *rate_idx,
                       const int64_t *prec_idx, double *tp_rate, double *fp_rate,
                       double *precision);
/* compute_accuracy_rates (:2384-2404) of n labels already in order */
int tb2_accuracy_rates_ordered(tb2_ctx *ctx, int64_t n, const uint8_t *labels, int64_t n_points,
                               const int64_t *rate_idx, const int64_t *prec_idx,
                               double *tp_rate, double *fp_rate, double *precision);

/* ---- statistics files (aggregate_per_read_stats, ModelStats / LevelStats writers) ---- */
/* One per-read statistics block (chrm, strand, start, end, block_stats) of a PerReadStats
 * iterator: its statistics (pos, stat)[stat_off .. + n_stat), its start, the id of its
 * chromosome in the most-significant table (order of first appearance) and its strand as the
 * byte the table stores ('+' or '-').  The calls take the blocks as rows of
 * TB2_SF_BLOCK_FIELDS int64 values in this field order. */
typedef struct tb2_sf_block {
    int64_t start, stat_off, n_stat, chrm, strand;
} tb2_sf_block;
#define TB2_SF_BLOCK_FIELDS 5

/* _agg_stats_worker (tombo_stats.py:4699-4725, apply_per_read_thresh :4084-4122) and the
 * block table of ModelStats._write_stat_block (:2737-2773, calc_damp_fraction :2537-2552) for
 * n_blocks blocks of region_size positions.  stat_type 0: alternative-model LLRs (|stat| >=
 * thresh is valid when lower_thresh is NaN = None), 1: p-values.  Unlike
 * tb2_region_stats_add, a NaN statistic is not dropped: it counts in cov, in valid_cov only
 * for stat_type 1 without lower_thresh, and never as >= thresh.  Block b's rows are its
 * covered positions in ascending order without those whose damp_frac is NaN; row_off
 * (n_blocks + 1, caller's) receives their offsets.  control_cov is 0 for every row (:2756).
 * The rows stay on the device for tb2_stats_file_aggregate_download and
 * tb2_most_signif_add_aggregate until the next call; a failed call leaves none, and those
 * two return TB2_ERR_INVALID_ARG until the next successful one.  A position outside
 * [start, start + region_size), an invalid block range, region_size outside 1 .. 2^28 or a
 * NaN threshold or pseudo-count -> TB2_ERR_INVALID_ARG; a buffer that does not fit on the
 * device -> TB2_ERR_CAPACITY.  tb2_last_timing out[0] is the kernel time. */
int tb2_stats_file_aggregate(tb2_ctx *ctx, int64_t n_blocks, const int64_t *blocks,
                             int64_t region_size, int64_t n_stat, const uint32_t *pos,
                             const double *stat, double single_read_thresh, double lower_thresh,
                             int stat_type, double unmod_count, double mod_count,
                             int64_t *row_off);
/* the rows of the last aggregation (row_off[n_blocks] each, caller's buffers) */
int tb2_stats_file_aggregate_download(tb2_ctx *ctx, uint32_t *pos_out, double *damp_frac_out,
                                      double *frac_out, uint32_t *cov_out, uint32_t *valid_cov_out);

/* The running most-significant table of ModelStats (kind 0: rows damp_frac, frac, pos, cov,
 * control_cov, valid_cov, chrm, strand) or LevelStats (kind 1: stat, pos, cov, control_cov,
 * chrm, strand), held on the device: after any sequence of adds it is the first
 * num_most_signif rows of one stable sort of every row added, in order of arrival, by numpy's
 * structured-array order (the key field, then the other fields in dtype order, floats as
 * numbers with -0.0 == +0.0) -- what _add_to_most_signif / _update_most_signif
 * (:2714-2735) and the trim of _close_write (:2775-2785) leave, at every
 * most_signif_num_batches.  A context holds one table: begin opens it empty with its kind and
 * size (1 .. 2^31 - 1), and refuses (TB2_ERR_INVALID_ARG) while one is open, so two writers
 * open at once (one per alternative model in test_significance) need a context each; end
 * closes it; reset empties it and keeps it open.  The other calls need an open table. */
int tb2_most_signif_begin(tb2_ctx *ctx, int kind, int64_t num_most_signif);
int tb2_most_signif_end(tb2_ctx *ctx);
int tb2_most_signif_reset(tb2_ctx *ctx);
/* n rows of one block from host arrays (regionStats / groupStats after the NaN filter of
 * _write_stat_block): key is damp_frac or stat; frac and valid_cov are read for kind 0 only.
 * A NaN key -> TB2_ERR_INVALID_ARG. */
int tb2_most_signif_add_rows(tb2_ctx *ctx, int64_t n, const double *key, const double *frac,
                             const uint32_t *pos, const uint32_t *cov, const uint32_t *control_cov,
                             const uint32_t *valid_cov, uint32_t chrm, uint8_t strand);
/* every row of the last tb2_stats_file_aggregate, in block order, without leaving the device
 * (kind 0 only) */
int tb2_most_signif_add_aggregate(tb2_ctx *ctx);
/* rows in the table: min(num_most_signif, rows added) */
int tb2_most_signif_count(tb2_ctx *ctx, int64_t *n_out);
/* the table in order into caller's buffers of tb2_most_signif_count rows; frac_out and
 * valid_cov_out are written for kind 0 only.  tb2_last_timing out[0] after count or get is the
 * time of the sort they ran. */
int tb2_most_signif_get(tb2_ctx *ctx, double *key_out, double *frac_out, uint32_t *pos_out,
                        uint32_t *cov_out, uint32_t *control_cov_out, uint32_t *valid_cov_out,
                        uint32_t *chrm_out, uint8_t *strand_out);

/* ---- read filters (read_filter.cu; DESIGN.md §3 "Read filters") ----
 * np.percentile(lens of read r, pctl[j]) into out[r * n_pctl + j], exactly numpy 2.3.5's
 * default method='linear' (np.percentile in read_is_stuck, _filter_reads.py:61-69).  Read r
 * holds lens[len_off[r] .. len_off[r + 1]) (the Events `length` column widened to int64).
 * TB2_ERR_INVALID_ARG: n_pctl < 1, a percentile outside [0, 100], a negative len_off[0], or a
 * read without lengths (len_off not strictly increasing). */
int tb2_dwell_percentiles(tb2_ctx *ctx, int64_t n_reads, const int64_t *lens,
                          const int64_t *len_off, int n_pctl, const double *pctl, double *out);
/* The reversible filters of _io_and_map_read (resquiggle.py:1437-1453) on the resident batch
 * after a successful tb2_batch_compute, over each read's final segs and sig_match_score.
 * code[r]: -1 failed read, 1 sig_match_score > sig_match_thresh, 2 any
 * np.percentile(np.diff(segs), pctl[j]) > thresh[j] (consulted only when not 1, the
 * reference's elif), 0 kept.  n_pctl == 0: no observations-per-base filter.  pctl_out
 * (nullable) gets the n_pctl percentiles of every successful read, NaN for failed ones.
 * Before any compute, or after a failed one, TB2_ERR_INVALID_ARG. */
int tb2_batch_read_filters(tb2_ctx *ctx, double sig_match_thresh, int n_pctl, const double *pctl,
                           const double *thresh, int8_t *code, double *pctl_out);
/* `tombo filter level_coverage` coverage (_filter_reads.py:112-126): reads of group g (one
 * chromosome and strand) are grp_off[g] .. grp_off[g + 1], grp_off[0] = 0.  Each group's
 * coverage has max(end) positions, every read of the group adds 1 over [start, end), and
 * mid_cov[i] = cov[start + (end - start) / 2].  A read with start < 0 or end <= start is
 * TB2_ERR_INVALID_ARG. */
int tb2_read_mid_coverage(tb2_ctx *ctx, int64_t n_groups, const int64_t *grp_off,
                          const int64_t *start, const int64_t *end, int64_t *mid_cov);

/* ---- genome browser tracks (browser_tracks.cu; DESIGN.md §3 "Genome browser tracks") ----
 * Run-length coverage of `tombo text_output browser_files --file-types coverage`
 * (TomboReads._compute_coverage + iter_coverage_regions, tombo_helper.py:1394-1453): reads of
 * group g (one chromosome and strand) are grp_off[g] .. grp_off[g + 1], grp_off[0] = 0.  Each
 * group's coverage has max(end) positions, every read adds 1 over [start, end), and is
 * written as runs of equal coverage: run k of group g, for run_off[g] <= k < run_off[g + 1],
 * starts at run_start[k] (0-based, within the group) with coverage run_cov[k], and lasts to
 * the next run's start or to the group's max(end).  Zero-coverage runs are included.  A group
 * of n_g reads has at most 2 n_g + 1 runs, so run_start and run_cov sized sum(2 n_g + 1)
 * always suffice; run_off (n_groups + 1 entries) returns the real counts.  A read with
 * start < 0 or end <= start is TB2_ERR_INVALID_ARG. */
int tb2_coverage_runs(tb2_ctx *ctx, int64_t n_groups, const int64_t *grp_off, const int64_t *start,
                      const int64_t *end, int64_t *run_off, int64_t *run_start, int64_t *run_cov);
/* Per-position means of an Events slot over one chromosome and strand
 * (get_mean_slot_genome_centric, tombo_helper.py:1661-1676), accumulated across calls.
 * tb2_slot_sums_begin opens an accumulation of chrm_len positions (0 <= chrm_len <= 2^40),
 * sums +0.0 and counts 0.  Each tb2_slot_sums_add then adds reads in order: read r holds
 * vals[val_off[r] .. val_off[r + 1]), placed at start[r] onwards, reversed when reverse[r]
 * (the - strand).  Every position's sum is the sequential fp64 sum of its values in read
 * order across all calls, as the reference's slice-adds make it; NaN values are added and
 * counted like any other.  start[r] < 0, start[r] + n_r > chrm_len or decreasing offsets are
 * TB2_ERR_INVALID_ARG before anything runs, as is a position covered more than 2^31 - 1
 * times; a failed add invalidates the accumulation.  tb2_slot_sums_means writes
 * sums / (double)counts for all chrm_len positions (0 / 0 is NaN); without a begin, or after a
 * failed add, it is TB2_ERR_INVALID_ARG. */
int tb2_slot_sums_begin(tb2_ctx *ctx, int64_t chrm_len);
int tb2_slot_sums_add(tb2_ctx *ctx, int64_t n_reads, const int64_t *start, const int64_t *val_off,
                      const double *vals, const uint8_t *reverse);
int tb2_slot_sums_means(tb2_ctx *ctx, double *out_mean);

#ifdef __cplusplus
}
#endif
#endif /* TOMBO_B200_H */
