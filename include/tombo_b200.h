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
 *     1..22 map 1:1 onto the reference's TomboError / NotImplementedError message
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
const char *tb2_last_error(tb2_ctx *ctx);
/* kernels launched by this ctx since creation (bench.py "gpu_launches") */
int64_t tb2_launch_count(tb2_ctx *ctx);
/* device time (ms, CUDA events on the ctx stream) of the last tb2_batch_compute:
 * out[0] whole compute stage, out[1] sum over launches of the dominant kernel
 * (banded DP, k_align), out[2] number of k_align launches, out[3] reads
 * processed summed over those launches.  After tb2_group_reg_stats / tb2_reads_ref_levels:
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
 * sv_in may be NULL. */
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
 * save params, bit2: static (short read) path taken. */
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
 * laid out as in tb2_resquiggle_batch).  compute may be repeated on one upload. */
int tb2_batch_upload(tb2_ctx *ctx, int64_t n_reads, const void *raw, int raw_dtype,
                     const int64_t *raw_off, const uint8_t *seq,
                     const int64_t *seq_off, const tb2_params *params,
                     const tb2_policy *policy);
/* optional, between upload and compute: per-read map_res.scale_values (sv_in[r]
 * with NaN shift = none) and map_res.stall_ints (pairs (start, end), stall_off has
 * n_reads + 1 entries counting pairs); either may be NULL */
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
 * a region: tb2_batch_alt_llr_motif. */
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

#ifdef __cplusplus
}
#endif
#endif /* TOMBO_B200_H */
