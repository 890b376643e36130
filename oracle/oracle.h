/* oracle.h -- CPU restatement of the Tombo resquiggle hot path (plain C, fp64/int64).
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference leg may load this.  The product
 * (tombo_b200/) never links, imports or executes anything under oracle/.
 *
 * Parity pinning: the reference holds no golden vectors or value-asserting tests
 * (SURVEY.md section 4).  This restatement is pinned against outputs of the
 * UNMODIFIED reference run in the build container (oracle/_ref, built by
 * oracle/build_ref.py) -- committed as tests/golden/*.npz by
 * tests/golden/make_golden.py -- and, when oracle/_ref is present, against the
 * live reference on fresh seeded inputs (tests/test_oracle_vs_reference.py).
 *
 * Every function cites the reference file:line (relative to /root/reference/tombo)
 * it restates.  Build: gcc -O2 -ffp-contract=off (no FMA contraction: the
 * reference's Cython objects contain no fused multiply-adds, SURVEY.md section 7).
 */
#ifndef TOMBO_ORACLE_H
#define TOMBO_ORACLE_H
#include <stdint.h>

typedef int64_t i64;

/* status codes <-> reference error strings (see orc_status_message) */
enum {
    ORC_OK = 0,
    ORC_ERR_FEWER_CPTS = 1,        /* _c_helper.pyx:118,200 */
    ORC_ERR_BEYOND_BANDWIDTH = 2,  /* _c_dynamic_programming.pyx:305 */
    ORC_ERR_ADAPTIVE_BEYOND_SIGNAL = 3, /* _c_dynamic_programming.pyx:354 */
    ORC_ERR_NOT_ENOUGH_DEL_SIGNAL = 4,  /* resquiggle.py:491 */
    ORC_ERR_TOO_MANY_DELS = 5,     /* resquiggle.py:496 */
    ORC_ERR_INVALID_SEG = 6,       /* resquiggle.py:530 */
    ORC_ERR_ZERO_LEN_SEG = 7,      /* resquiggle.py:534 */
    ORC_ERR_NEG_SEG = 8,           /* resquiggle.py:536 */
    ORC_ERR_SEG_PAST_END = 9,      /* resquiggle.py:538 */
    ORC_ERR_START_TOO_FAR = 10,    /* resquiggle.py:612 */
    ORC_ERR_MASKED_TOO_FEW = 11,   /* resquiggle.py:672 */
    ORC_ERR_READ_TOO_SHORT_START = 12, /* resquiggle.py:704 */
    ORC_ERR_MAP_TOO_SHORT_START = 13,  /* resquiggle.py:706 */
    ORC_ERR_POOR_START_MATCH = 14, /* resquiggle.py:746 */
    ORC_ERR_DISCORDANT_LEN = 15,   /* resquiggle.py:976 */
    ORC_ERR_OPEN_PORE = 16,        /* resquiggle.py:1010 */
    ORC_ERR_NO_RAW = 17,           /* resquiggle.py:1149 */
    ORC_ERR_TOO_MUCH_SIGNAL = 18,  /* resquiggle.py:1160 */
    ORC_ERR_SEG_COUNT = 19,        /* resquiggle.py:1201 */
    ORC_ERR_THEIL_SEN_ZERO = 20,   /* tombo_stats.py:421 */
    ORC_ERR_INVALID_START_PATH = 21, /* tombo_stats.py:2356 */
    ORC_ERR_UNEXPECTED = 100       /* any non-TomboError exception in the reference */
};

typedef struct {
    double match_evalue, skip_pen;
    i64 bandwidth;
    double max_half_z_score;   /* NaN <=> None */
    i64 running_stat_width, min_obs_per_base, raw_min_obs_per_base,
        mean_obs_per_event;
    double z_shift, stay_pen;
    i64 use_t_test_seg;
    i64 band_bound_thresh, start_bw, start_save_bw, start_n_bases;
} orc_params;

typedef struct {
    double shift, scale, lower_lim, upper_lim, outlier_thresh; /* NaN <=> None */
} orc_scale_values;

/* constants of _default_parameters.py needed by the per-read policy */
typedef struct {
    double outlier_thresh;         /* OUTLIER_THRESH 5.0; NaN <=> None */
    i64 max_raw_cpts;              /* MAX_RAW_CPTS 200; <0 <=> None */
    double min_event_to_seq_ratio; /* 1.1 */
    double sig_match_thresh;       /* SIG_MATCH_THRESH[sample type] */
    i64 max_scaling_iters;         /* 3 */
    i64 tie_stable;                /* 0: library argsort order (ties undefined);
                                      1: pinned rule (score desc, position desc) */
    i64 is_rna;
    i64 skip_seq_scaling;
    double const_scale;            /* NaN <=> None */
    uint32_t subsample_seed;       /* keyed Theil-Sen sub-sampling */
} orc_policy;

const char *orc_status_message(int status);

/* ---- _c_helper.pyx ---- */
void orc_new_means(const double *sig, const i64 *segs, i64 n_segs, double *out);
void orc_new_mean_stds(const double *sig, const i64 *segs, i64 n_segs,
                       double *means, double *sds);
void orc_apply_outlier_thresh(const double *sig, i64 n, double lo, double hi,
                              double *out);
int orc_valid_cpts_w_cap(const double *sig, i64 n, i64 min_base_obs,
                         i64 running_stat_width, i64 num_cpts, int tie_stable,
                         i64 *cpts_sorted);
int orc_valid_cpts_w_cap_t_test(const double *sig, i64 n, i64 min_base_obs,
                                i64 running_stat_width, i64 num_cpts,
                                int tie_stable, i64 *cpts_sorted);
void orc_compute_slopes(const double *ev, const double *md, i64 n,
                        double max_slope, double *slopes);
double orc_calc_llh_ratio(const double *m, const double *rm, const double *am,
                          const double *rv, const double *av, i64 n);
double orc_calc_llh_ratio_const_var(const double *m, const double *rm,
                                    const double *am, double cv, i64 n);
double orc_calc_scaled_llh_ratio_const_var(
    const double *m, const double *rm, const double *am, double cv,
    double scale_factor, double height_factor, double height_power, i64 n);

/* ---- numpy restatements ---- */
double orc_median(const double *x, i64 n);         /* np.median */
double orc_pairwise_sum(const double *a, i64 n);   /* np.add.reduce (float64) */
double orc_np_mean(const double *a, i64 n);
void orc_linspace(double start, double stop, i64 num, double *out);

/* ---- _c_dynamic_programming.pyx ---- */
void orc_base_z_scores(const double *sig, i64 n, double ref_mean, double ref_sd,
                       int do_winsorize, double max_half_z, double *out);
void orc_banded_forward_pass(const double *z, const i64 *event_starts,
                             i64 n_bases, i64 bw, double skip_pen,
                             double stay_pen, double *fwd, i64 *tb);
int orc_banded_traceback(const i64 *tb, const i64 *event_starts, i64 n_bases,
                         i64 bw, i64 band_pos, i64 band_boundary_thresh,
                         i64 *seq_poss);
int orc_adaptive_banded_forward_pass(
    double *fwd, i64 *tb, i64 *event_starts, i64 n_bases, i64 bw,
    const double *event_means, i64 n_events, const double *ref_means,
    const double *ref_sds, double z_shift, double skip_pen, double stay_pen,
    i64 start_seq_pos, double mask_fill_z, int do_winsorize, double max_half_z,
    double *all_z /* may be NULL; (n_bases-start_seq_pos) x bw */);

/* ---- tombo_stats.py ---- */
int orc_normalize_raw_signal(const double *raw, i64 n, int norm_type,
                             /* 0 median, 1 median_const_scale */
                             double outlier_thresh, double const_scale,
                             const orc_scale_values *sv_in /* may be NULL */,
                             double *norm, orc_scale_values *sv_out);
int orc_theil_sen(double prev_shift, double prev_scale, const double *ev,
                  const double *md, i64 n, uint32_t subsample_key,
                  double *shift, double *scale, double *shift_corr,
                  double *scale_corr);
double orc_get_read_seg_score(const double *means, const double *ref_means,
                              const double *ref_sds, i64 n);
i64 orc_compute_num_events(i64 sig_len, i64 seq_len, i64 mean_obs_per_event,
                           double min_ratio);
i64 orc_identify_stalls(const double *raw, i64 n, i64 *ints /* 2*cap */, i64 cap);
i64 orc_remove_stall_cpts(const i64 *stall_ints, i64 n_stalls, const i64 *cpts,
                          i64 n_cpts, i64 *out);

/* ---- resquiggle.py ---- */
int orc_find_static_base_assignment(const double *em, i64 n_em,
                                    const double *rm, const double *rs, i64 nb,
                                    const orc_params *p, i64 *read_tb);
int orc_find_seq_start_in_events(const double *em, i64 n_em, const double *rm,
                                 const double *rs, i64 n_ref,
                                 const orc_params *p, i64 num_bases,
                                 i64 num_events, int check_score,
                                 double sig_match_thresh, i64 *start_loc,
                                 double *events_per_base);
int orc_find_adaptive_base_assignment(
    const i64 *cpts, i64 n_cpts, const double *em, const orc_params *p,
    const double *rm, const double *rs, i64 nb, double sig_match_thresh,
    i64 *segs /* nb+1 */, i64 *read_start_rel_to_raw,
    i64 *dbg_path /* may be NULL: [0]=0 static,1 adaptive; [1]=mapped_start;
                     [2]=events_start_clip */,
    double *dbg_epb /* may be NULL */);
void orc_set_debug_buffers(i64 *es, i64 *tb);
int orc_resolve_skipped_bases_with_raw(
    const i64 *segs, i64 nb, const double *rm, const double *rs,
    const double *norm, i64 n_norm, const orc_params *p, i64 max_raw_cpts,
    i64 *out_segs);

typedef struct {
    i64 read_start_rel_to_raw;
    orc_scale_values sv;
    double sig_match_score;
    i64 norm_params_changed;
    i64 n_norm;            /* length of clipped norm signal */
} orc_read_result;

/* resquiggle_read (resquiggle.py:1122-1214).  seq levels are passed already
 * looked up (ref_means/ref_sds, nb = mapped bases).  segs: nb+1.  norm_out may be
 * NULL, else capacity n_raw.  stall_ints may be NULL. */
int orc_resquiggle_read(const double *raw, i64 n_raw, const double *rm,
                        const double *rs, i64 nb, const orc_params *p,
                        const orc_policy *pol, const orc_scale_values *sv_in,
                        int first_call, const i64 *stall_ints, i64 n_stalls,
                        uint32_t subsample_key, i64 *segs, double *norm_out,
                        orc_read_result *res);

/* worker policy: adjust (RNA flip + stalls), iterate, rescue
 * (resquiggle.py:1492-1530, 1575-1595).  info[0]=calls, info[1]=rescued,
 * info[2]=n_iters of the successful run, info[3]=status of the first attempt. */
int orc_run_read(const double *raw, i64 n_raw, const double *rm,
                 const double *rs, i64 nb, const orc_params *p,
                 const orc_params *save_p, const orc_policy *pol,
                 uint32_t read_index, i64 *segs, double *norm_out,
                 orc_read_result *res, i64 *info);
/* orc_run_read with the caller's map_res.scale_values (sv_in, may be NULL) and, for
 * DNA, map_res.stall_ints (n_stalls pairs, may be NULL).  The RNA policy replaces the
 * stalls with identify_stalls, as adjust_map_res does.  orc_run_read is the NULL case. */
int orc_run_read_inputs(const double *raw, i64 n_raw, const double *rm,
                        const double *rs, i64 nb, const orc_params *p,
                        const orc_params *save_p, const orc_policy *pol,
                        uint32_t read_index, i64 *segs, double *norm_out,
                        orc_read_result *res, i64 *info, const orc_scale_values *sv_in,
                        const i64 *stall_ints, i64 n_stalls);

uint32_t orc_subsample_key(uint32_t seed, uint32_t read_index, uint32_t call);
i64 orc_perm_index(i64 i, i64 n, uint32_t key);

#endif
