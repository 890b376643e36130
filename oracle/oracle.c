/* oracle.c -- CPU restatement of the Tombo resquiggle hot path.  See oracle.h.
 * TEST INFRASTRUCTURE ONLY.  Citations are file:line under /root/reference/tombo.
 * Arithmetic: fp64, sequential sums in the reference's order, no FMA contraction.
 */
#include "oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define MASK_BASES 50            /* _default_parameters.py:69 */
#define MASK_FILL_Z_SCORE (-15.0) /* _default_parameters.py:70 */
#define DEL_FIX_WINDOW 2         /* :72 */
#define MAX_DEL_FIX_WINDOW 10    /* :73 */
#define EXTRA_SIG_FACTOR 1.1     /* :67 */
#define SHIFT_CHANGE_THRESH 0.1  /* :169 */
#define SCALE_CHANGE_THRESH 0.1  /* :170 */
#define MAX_POINTS_FOR_THEIL_SEN 1000 /* :178 */
#define RNA_SCALE_NUM_EVENTS 10000     /* :79 */
#define RNA_SCALE_MAX_FRAC_EVENTS 0.75 /* :80 */

static void *xmalloc(size_t n) { void *p = malloc(n ? n : 1); if (!p) abort(); return p; }

const char *orc_status_message(int s)
{
    switch (s) {
    case ORC_OK: return "";
    case ORC_ERR_FEWER_CPTS: return "Fewer changepoints found than requested";
    case ORC_ERR_BEYOND_BANDWIDTH: return "Read event to sequence alignment extends beyond bandwidth";
    case ORC_ERR_ADAPTIVE_BEYOND_SIGNAL: return "Adaptive signal to seqeunce alignment extended beyond raw signal";
    case ORC_ERR_NOT_ENOUGH_DEL_SIGNAL: return "Not enough raw signal around potential genomic deletion(s)";
    case ORC_ERR_TOO_MANY_DELS: return "Read contains too many potential genomic deletions";
    case ORC_ERR_INVALID_SEG: return "Invalid segmentation results.";
    case ORC_ERR_ZERO_LEN_SEG: return "New segments include zero length events";
    case ORC_ERR_NEG_SEG: return "New segments start with negative index";
    case ORC_ERR_SEG_PAST_END: return "New segments end past raw signal values";
    case ORC_ERR_START_TOO_FAR: return "Read sequence to signal matching starts too far into events for full adaptive assignment";
    case ORC_ERR_MASKED_TOO_FEW: return "Masked z-score contains too few events.";
    case ORC_ERR_READ_TOO_SHORT_START: return "Read too short for start/end discovery";
    case ORC_ERR_MAP_TOO_SHORT_START: return "Genomic mapping too short for start/end discovery";
    case ORC_ERR_POOR_START_MATCH: return "Poor raw to expected signal matching in beginning of read.";
    case ORC_ERR_DISCORDANT_LEN: return "Discordant reference and seqeunce lengths.";
    case ORC_ERR_OPEN_PORE: return "Very poor signal quality. Read likely includes open pore.";
    case ORC_ERR_NO_RAW: return "Must have raw signal in order to complete re-squiggle algorithm";
    case ORC_ERR_TOO_MUCH_SIGNAL: return "Too much raw signal for mapped sequence";
    case ORC_ERR_SEG_COUNT: return "Aligned sequence does not match number of segments produced";
    case ORC_ERR_THEIL_SEN_ZERO: return "Read failed sequence-based signal re-scaling parameter estimation.";
    case ORC_ERR_INVALID_START_PATH: return "Invalid path through read start";
    default: return "UNEXPECTED";
    }
}

/* ===================================================================== */
/* numpy restatements                                                     */
/* ===================================================================== */
static int cmp_double(const void *a, const void *b)
{
    double x = *(const double *)a, y = *(const double *)b;
    return (x > y) - (x < y);
}

/* np.median: middle order statistic, or (a+b)/2 of the two middle ones
 * (numpy lib/_function_base_impl.py _median: mean(part[index-1:index+1])). */
double orc_median(const double *x, i64 n)
{
    double *t = (double *)xmalloc(sizeof(double) * (size_t)n), r;
    memcpy(t, x, sizeof(double) * (size_t)n);
    qsort(t, (size_t)n, sizeof(double), cmp_double);
    if (n % 2) r = t[n / 2];
    else r = (t[n / 2 - 1] + t[n / 2]) / 2.0;
    free(t);
    return r;
}

/* numpy DOUBLE_pairwise_sum (umath/loops_utils.h.src), contiguous input */
double orc_pairwise_sum(const double *a, i64 n)
{
    if (n < 8) {
        double res = 0.;
        for (i64 i = 0; i < n; i++) res += a[i];
        return res;
    } else if (n <= 128) {
        double r[8], res;
        i64 i;
        for (i = 0; i < 8; i++) r[i] = a[i];
        for (i = 8; i < n - (n % 8); i += 8)
            for (int k = 0; k < 8; k++) r[k] += a[i + k];
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; i++) res += a[i];
        return res;
    } else {
        i64 n2 = n / 2;
        n2 -= n2 % 8;
        return orc_pairwise_sum(a, n2) + orc_pairwise_sum(a + n2, n - n2);
    }
}

double orc_np_mean(const double *a, i64 n) { return orc_pairwise_sum(a, n) / (double)n; }

/* np.linspace(start, stop, num) (endpoint=True), float64 result
 * (numpy _core/function_base.py: y = arange(num)*step + start; y[-1] = stop) */
void orc_linspace(double start, double stop, i64 num, double *out)
{
    if (num <= 0) return;
    i64 div = num - 1;
    double delta = stop - start;
    if (div > 0) {
        double step = delta / (double)div;
        if (step == 0.0) {
            for (i64 i = 0; i < num; i++) out[i] = ((double)i / (double)div) * delta + start;
        } else {
            for (i64 i = 0; i < num; i++) out[i] = (double)i * step + start;
        }
        out[num - 1] = stop;
    } else {
        out[0] = 0.0 * delta + start;
    }
}

/* ===================================================================== */
/* _c_helper.pyx                                                          */
/* ===================================================================== */
/* c_new_means _c_helper.pyx:59-71 */
void orc_new_means(const double *sig, const i64 *segs, i64 n_segs, double *out)
{
    for (i64 i = 0; i < n_segs; i++) {
        double s = 0;
        for (i64 k = segs[i]; k < segs[i + 1]; k++) s += sig[k];
        out[i] = s / (double)(segs[i + 1] - segs[i]);
    }
}

/* c_new_mean_stds _c_helper.pyx:38-57 */
void orc_new_mean_stds(const double *sig, const i64 *segs, i64 n_segs,
                       double *means, double *sds)
{
    for (i64 i = 0; i < n_segs; i++) {
        i64 len = segs[i + 1] - segs[i];
        double s = 0, v = 0, m;
        for (i64 k = segs[i]; k < segs[i + 1]; k++) s += sig[k];
        m = s / (double)len;
        means[i] = m;
        for (i64 k = segs[i]; k < segs[i + 1]; k++) { double d = sig[k] - m; v += d * d; }
        sds[i] = sqrt(v / (double)len);
    }
}

/* c_apply_outlier_thresh _c_helper.pyx:73-87 */
void orc_apply_outlier_thresh(const double *sig, i64 n, double lo, double hi, double *out)
{
    for (i64 i = 0; i < n; i++) {
        double v = sig[i];
        out[i] = v > hi ? hi : (v < lo ? lo : v);
    }
}

typedef struct { double score; i64 pos; } cand_t;
/* rank order of np.argsort(scores)[::-1]; ties: larger position first (the
 * kind='stable' pin of SURVEY.md 8c-7; unpinned numpy order is undefined) */
static int cmp_cand_desc(const void *a, const void *b)
{
    const cand_t *x = (const cand_t *)a, *y = (const cand_t *)b;
    if (x->score > y->score) return -1;
    if (x->score < y->score) return 1;
    return (x->pos < y->pos) - (x->pos > y->pos);
}
static int cmp_i64(const void *a, const void *b)
{
    i64 x = *(const i64 *)a, y = *(const i64 *)b;
    return (x > y) - (x < y);
}

/* greedy pick shared by both changepoint variants (_c_helper.pyx:100-120 /
 * 184-202), followed by the .sort() of tombo_helper.py:81,89 */
static int greedy_pick(cand_t *cand, i64 n_cand, i64 num_cands_bound,
                       i64 min_base_obs, i64 w, i64 num_cpts, i64 *cpts)
{
    if (n_cand <= 0 || num_cpts <= 0) return ORC_ERR_UNEXPECTED;
    qsort(cand, (size_t)n_cand, sizeof(cand_t), cmp_cand_desc);
    /* blacklist over positions [-min_base_obs, n_cand + min_base_obs) */
    i64 off = min_base_obs;
    char *black = (char *)calloc((size_t)(n_cand + 2 * min_base_obs + 2), 1);
    cpts[0] = cand[0].pos + w;
    for (i64 k = cand[0].pos - min_base_obs + 1; k < cand[0].pos + min_base_obs; k++)
        black[k + off] = 1;
    i64 cand_idx = 1, added = 1;
    int st = ORC_OK;
    while (added < num_cpts) {
        if (cand_idx >= n_cand) { st = ORC_ERR_UNEXPECTED; break; } /* IndexError */
        i64 cp = cand[cand_idx].pos;
        if (!black[cp + off]) {
            cpts[added++] = cp + w;
            for (i64 k = cp - min_base_obs + 1; k < cp + min_base_obs; k++) black[k + off] = 1;
        }
        cand_idx++;
        if (cand_idx >= num_cands_bound) { st = ORC_ERR_FEWER_CPTS; break; }
    }
    free(black);
    if (st == ORC_OK) qsort(cpts, (size_t)num_cpts, sizeof(i64), cmp_i64);
    return st;
}

/* c_valid_cpts_w_cap _c_helper.pyx:89-120 (+ sort, tombo_helper.py:76-82) */
int orc_valid_cpts_w_cap(const double *sig, i64 n, i64 min_base_obs, i64 w,
                         i64 num_cpts, int tie_stable, i64 *cpts)
{
    (void)tie_stable;
    i64 n_cand = n + 1 - 2 * w;
    if (n_cand <= 0) return ORC_ERR_UNEXPECTED;
    double *cs = (double *)xmalloc(sizeof(double) * (size_t)(n + 1));
    cs[0] = 0.0;
    for (i64 i = 0; i < n; i++) cs[i + 1] = cs[i] + sig[i]; /* np.cumsum: sequential */
    cand_t *cand = (cand_t *)xmalloc(sizeof(cand_t) * (size_t)n_cand);
    for (i64 i = 0; i < n_cand; i++) {
        cand[i].score = fabs(((2 * cs[i + w]) - cs[i]) - cs[i + 2 * w]);
        cand[i].pos = i;
    }
    /* num_cands = candidate_poss.shape[0] - 2*w  (:105-106) */
    int st = greedy_pick(cand, n_cand, n_cand - 2 * w, min_base_obs, w, num_cpts, cpts);
    free(cand); free(cs);
    return st;
}

/* c_valid_cpts_w_cap_t_test _c_helper.pyx:144-202 */
int orc_valid_cpts_w_cap_t_test(const double *sig, i64 n, i64 min_base_obs, i64 w,
                                i64 num_cpts, int tie_stable, i64 *cpts)
{
    (void)tie_stable;
    i64 num_cands = n - 2 * w;
    if (num_cands <= 0) return ORC_ERR_UNEXPECTED;
    cand_t *cand = (cand_t *)xmalloc(sizeof(cand_t) * (size_t)num_cands);
    for (i64 pos = 0; pos < num_cands; pos++) {
        double m1 = 0, m2 = 0, var1 = 0, var2 = 0, d;
        for (i64 k = 0; k < w; k++) m1 += sig[pos + k];
        m1 /= (double)w;
        for (i64 k = 0; k < w; k++) m2 += sig[pos + w + k];
        m2 /= (double)w;
        for (i64 k = 0; k < w; k++) { d = sig[pos + k] - m1; var1 += d * d; }
        for (i64 k = 0; k < w; k++) { d = sig[pos + w + k] - m2; var2 += d * d; }
        double t;
        if (var1 + var2 == 0) t = 0.0;
        else if (m1 > m2) t = (m1 - m2) / sqrt(var1 + var2);
        else t = (m2 - m1) / sqrt(var1 + var2);
        cand[pos].score = t;
        cand[pos].pos = pos;
    }
    /* here the bound is num_cands itself (:199) */
    int st = greedy_pick(cand, num_cands, num_cands, min_base_obs, w, num_cpts, cpts);
    free(cand);
    return st;
}

/* c_compute_slopes _c_helper.pyx:362-377 (combinations order i<j) */
void orc_compute_slopes(const double *ev, const double *md, i64 n, double max_slope,
                        double *slopes)
{
    i64 s = 0;
    for (i64 i = 0; i < n; i++)
        for (i64 j = i + 1; j < n; j++, s++)
            slopes[s] = (ev[i] == ev[j]) ? max_slope : (md[i] - md[j]) / (ev[i] - ev[j]);
}

/* c_calc_llh_ratio _c_helper.pyx:277-296 */
double orc_calc_llh_ratio(const double *m, const double *rm, const double *am,
                          const double *rv, const double *av, i64 n)
{
    double rz = 0, rl = 0, az = 0, al = 0;
    for (i64 i = 0; i < n; i++) {
        double rd = m[i] - rm[i];
        rz += (rd * rd) / rv[i];
        rl += log(rv[i]);
        double ad = m[i] - am[i];
        az += (ad * ad) / av[i];
        al += log(av[i]);
    }
    return az + al - rz - rl;
}

/* c_calc_llh_ratio_const_var _c_helper.pyx:298-311 */
double orc_calc_llh_ratio_const_var(const double *m, const double *rm,
                                    const double *am, double cv, i64 n)
{
    double r = 0;
    for (i64 i = 0; i < n; i++) {
        double rd = m[i] - rm[i], ad = m[i] - am[i];
        r += ((ad * ad) - (rd * rd)) / cv;
    }
    return r;
}

/* c_calc_scaled_llh_ratio_const_var _c_helper.pyx:313-358 */
double orc_calc_scaled_llh_ratio_const_var(const double *m, const double *rm,
                                           const double *am, double cv, double sf,
                                           double hf, double hp, i64 n)
{
    double r = 0;
    for (i64 i = 0; i < n; i++) {
        double ref_mean = rm[i], alt_mean = am[i];
        if (ref_mean == alt_mean) continue;
        double obs = m[i];
        double scale_mean = (alt_mean + ref_mean) / 2;
        double ref_diff = obs - ref_mean, alt_diff = obs - alt_mean;
        double scale_diff = obs - scale_mean;
        double means_diff = alt_mean - ref_mean;
        if (means_diff < 0) means_diff = means_diff * -1;
        r += exp(-(scale_diff * scale_diff) / (sf * cv)) *
             ((alt_diff * alt_diff) - (ref_diff * ref_diff)) /
             (cv * pow(means_diff, hp) * hf);
    }
    return r;
}

/* ===================================================================== */
/* _c_dynamic_programming.pyx                                             */
/* ===================================================================== */
/* c_base_z_scores :17-32 */
void orc_base_z_scores(const double *sig, i64 n, double ref_mean, double ref_sd,
                       int do_winsorize, double max_half_z, double *out)
{
    for (i64 i = 0; i < n; i++) {
        double z = (sig[i] - ref_mean) / ref_sd;
        if (z > 0) z = -z;
        if (do_winsorize && z < -max_half_z) z = -max_half_z;
        out[i] = z;
    }
}

/* c_process_band :202-236 */
static void process_band(double *fwd, i64 *tb, const double *z, double stay_pen,
                         double skip_pen, i64 bw, i64 diff, i64 seq_pos)
{
    const double *prev = fwd + seq_pos * bw;
    double *cur = fwd + (seq_pos + 1) * bw;
    i64 *ctb = tb + (seq_pos + 1) * bw;
    for (i64 bp = 1; bp < bw; bp++) {
        double pz = z[bp];
        i64 pb = bp + diff;
        double max_score = cur[bp - 1] - stay_pen + pz;
        i64 from = 0;
        if (pb - 1 < bw) {
            double diag = prev[pb - 1] + pz;
            if (diag > max_score) { max_score = diag; from = 2; }
            if (pb < bw) {
                double skip = prev[pb] - skip_pen;
                if (skip > max_score) { max_score = skip; from = 1; }
            }
        }
        cur[bp] = max_score;
        ctb[bp] = from;
    }
}

/* c_banded_forward_pass :240-279.  fwd, tb: (n_bases+1) x bw */
void orc_banded_forward_pass(const double *z, const i64 *es, i64 n_bases, i64 bw,
                             double skip_pen, double stay_pen, double *fwd, i64 *tb)
{
    for (i64 i = 0; i < bw; i++) { fwd[i] = 0.0; tb[i] = 0; /* row 0 tb unset in ref */ }
    for (i64 sp = 0; sp < n_bases; sp++) {
        if (sp == 0 || es[sp] == es[sp - 1]) {
            fwd[(sp + 1) * bw] = fwd[sp * bw] - skip_pen;
            tb[(sp + 1) * bw] = 1;
        } else {
            fwd[(sp + 1) * bw] = fwd[sp * bw + es[sp] - es[sp - 1] - 1] + z[sp * bw];
            tb[(sp + 1) * bw] = 2;
        }
        i64 diff = sp > 0 ? es[sp] - es[sp - 1] : 0;
        process_band(fwd, tb, z + sp * bw, stay_pen, skip_pen, bw, diff, sp);
    }
}

/* c_banded_traceback :281-310 */
int orc_banded_traceback(const i64 *tb, const i64 *es, i64 n_bases, i64 bw,
                         i64 band_pos, i64 thresh, i64 *seq_poss)
{
    i64 cur_event = band_pos + es[n_bases - 1];
    seq_poss[n_bases] = cur_event + 1;
    for (i64 sp = n_bases; sp > 0; sp--) {
        band_pos = cur_event - es[sp - 1];
        if (band_pos < 0 || band_pos >= bw) return ORC_ERR_UNEXPECTED;
        while (tb[sp * bw + band_pos] == 0) {
            band_pos--;
            if (band_pos < 0) return ORC_ERR_UNEXPECTED;
        }
        if (tb[sp * bw + band_pos] == 2) band_pos--;
        if (thresh >= 0) {
            i64 a = band_pos, b = bw - band_pos - 1;
            if ((a < b ? a : b) < thresh) return ORC_ERR_BEYOND_BANDWIDTH;
        }
        cur_event = es[sp - 1] + band_pos;
        seq_poss[sp - 1] = cur_event + 1;
    }
    return ORC_OK;
}

/* c_argmax :186-197 (first maximum) */
static i64 argmax_first(const double *v, i64 n)
{
    double mv = v[0];
    i64 mp = 0;
    for (i64 i = 1; i < n; i++) if (v[i] > mv) { mv = v[i]; mp = i; }
    return mp;
}

/* c_adaptive_banded_forward_pass :314-412 */
int orc_adaptive_banded_forward_pass(double *fwd, i64 *tb, i64 *es, i64 n_bases, i64 bw,
                                     const double *em, i64 n_events, const double *rm,
                                     const double *rs, double z_shift, double skip_pen,
                                     double stay_pen, i64 start_seq_pos, double mask_fill_z,
                                     int do_winsorize, double max_half_z, double *all_z)
{
    i64 half_bw = bw / 2;
    double *z = (double *)xmalloc(sizeof(double) * (size_t)bw);
    for (i64 sp = start_seq_pos; sp < n_bases; sp++) {
        i64 prev_start = es[sp - 1];
        i64 cur_start = prev_start + argmax_first(fwd + sp * bw, bw) - half_bw + 1;
        if (cur_start < prev_start) cur_start = prev_start;
        if (cur_start >= n_events) {
            if (sp < n_bases - 2) { free(z); return ORC_ERR_ADAPTIVE_BEYOND_SIGNAL; }
            cur_start = n_events - 1;
        }
        es[sp] = cur_start;
        double ref_mean = rm[sp], ref_sd = rs[sp];
        i64 lim = cur_start + bw <= n_events ? cur_start + bw : n_events;
        for (i64 ep = cur_start; ep < lim; ep++) {
            double pz = (em[ep] - ref_mean) / ref_sd;
            if (pz < 0) pz = -pz;
            if (do_winsorize) pz = pz < max_half_z ? pz : max_half_z;
            z[ep - cur_start] = z_shift - pz;
        }
        if (cur_start + bw > n_events)
            for (i64 ep = n_events - cur_start; ep < bw; ep++) z[ep] = mask_fill_z;
        if (all_z) memcpy(all_z + (sp - start_seq_pos) * bw, z, sizeof(double) * (size_t)bw);
        if (cur_start == prev_start) {
            fwd[(sp + 1) * bw] = fwd[sp * bw] - skip_pen;
            tb[(sp + 1) * bw] = 1;
        } else {
            fwd[(sp + 1) * bw] = fwd[sp * bw + cur_start - prev_start - 1] + z[0];
            tb[(sp + 1) * bw] = 2;
        }
        process_band(fwd, tb, z, stay_pen, skip_pen, bw, cur_start - prev_start, sp);
    }
    free(z);
    return ORC_OK;
}

/* ===================================================================== */
/* tombo_stats.py                                                         */
/* ===================================================================== */
/* normalize_raw_signal tombo_stats.py:482-573 ('median', 'median_const_scale',
 * or provided scale_values) */
int orc_normalize_raw_signal(const double *raw, i64 n, int norm_type, double outlier_thresh,
                             double const_scale, const orc_scale_values *sv_in,
                             double *norm, orc_scale_values *sv_out)
{
    double shift, scale, lo = NAN, hi = NAN;
    if (n <= 0) return ORC_ERR_UNEXPECTED;
    if (sv_in == NULL) {
        shift = orc_median(raw, n);                       /* :541 / :545 */
        if (norm_type == 0) {
            double *t = (double *)xmalloc(sizeof(double) * (size_t)n);
            for (i64 i = 0; i < n; i++) t[i] = fabs(raw[i] - shift);
            scale = orc_median(t, n);                     /* :542 */
            free(t);
        } else scale = const_scale;                       /* :546 */
    } else { shift = sv_in->shift; scale = sv_in->scale; }
    if (scale == 0.0) return ORC_ERR_UNEXPECTED; /* FloatingPointError (seterr raise) */
    for (i64 i = 0; i < n; i++) norm[i] = (raw[i] - shift) / scale;   /* :554 */
    if (!isnan(outlier_thresh) || sv_in != NULL) {        /* :558 */
        if (!isnan(outlier_thresh)) {
            double med = orc_median(norm, n);
            double *t = (double *)xmalloc(sizeof(double) * (size_t)n);
            for (i64 i = 0; i < n; i++) t[i] = fabs(norm[i] - med);
            double mad = orc_median(t, n);
            free(t);
            lo = med - (mad * outlier_thresh);
            hi = med + (mad * outlier_thresh);
        } else { lo = sv_in->lower_lim; hi = sv_in->upper_lim; }
        if (!isnan(lo) && !isnan(hi)) orc_apply_outlier_thresh(norm, n, lo, hi, norm);
    }
    sv_out->shift = shift; sv_out->scale = scale;
    sv_out->lower_lim = lo; sv_out->upper_lim = hi;
    sv_out->outlier_thresh = outlier_thresh;
    return ORC_OK;
}

/* keyed sub-sampler (mirror of tombo_b200/synthetic.py; stands in for
 * np.random.choice at tombo_stats.py:413) */
static uint32_t mix32(uint32_t x)
{
    x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
    return x;
}
uint32_t orc_subsample_key(uint32_t seed, uint32_t read_index, uint32_t call)
{
    return mix32(mix32(seed ^ 0x9E3779B9u) + mix32(read_index * 2654435761u + 1u) +
                 call * 0x632BE5ABu);
}
i64 orc_perm_index(i64 i, i64 n, uint32_t key)
{
    int bits = 0;
    for (i64 t = n - 1; t > 0; t >>= 1) bits++;
    if (bits < 2) bits = 2;
    int half = (bits + 1) / 2;
    uint32_t mask = (1u << half) - 1u;
    uint32_t x = (uint32_t)i;
    for (;;) {
        uint32_t l = x >> half, r = x & mask;
        for (uint32_t rnd = 0; rnd < 4; rnd++) {
            uint32_t f = mix32(r ^ key ^ (rnd * 0x9E3779B9u)) & mask;
            uint32_t nl = r, nr = l ^ f;
            l = nl; r = nr;
        }
        x = (l << half) | r;
        if ((i64)x < n) return (i64)x;
    }
}

/* calc_kmer_fitted_shift_scale(method='theil_sen') tombo_stats.py:401-450 */
int orc_theil_sen(double prev_shift, double prev_scale, const double *ev_in,
                  const double *md_in, i64 n, uint32_t key, double *shift, double *scale,
                  double *shift_corr, double *scale_corr)
{
    const double *ev = ev_in, *md = md_in;
    double *sev = NULL, *smd = NULL;
    if (n > MAX_POINTS_FOR_THEIL_SEN) {
        sev = (double *)xmalloc(sizeof(double) * MAX_POINTS_FOR_THEIL_SEN);
        smd = (double *)xmalloc(sizeof(double) * MAX_POINTS_FOR_THEIL_SEN);
        for (i64 i = 0; i < MAX_POINTS_FOR_THEIL_SEN; i++) {
            i64 k = orc_perm_index(i, n, key);
            sev[i] = ev_in[k]; smd[i] = md_in[k];
        }
        ev = sev; md = smd; n = MAX_POINTS_FOR_THEIL_SEN;
    }
    i64 ns = n * (n - 1) / 2;
    if (ns <= 0) { free(sev); free(smd); return ORC_ERR_UNEXPECTED; }
    double *sl = (double *)xmalloc(sizeof(double) * (size_t)ns);
    orc_compute_slopes(ev, md, n, 1000.0, sl);
    double slope = orc_median(sl, ns);
    free(sl);
    double *t = (double *)xmalloc(sizeof(double) * (size_t)n);
    for (i64 i = 0; i < n; i++) t[i] = md[i] - (slope * ev[i]);
    double inter = orc_median(t, n);
    free(t); free(sev); free(smd);
    if (slope == 0) return ORC_ERR_THEIL_SEN_ZERO;
    *scale_corr = 1 / slope;
    *shift_corr = -inter / slope;
    *shift = prev_shift + (*shift_corr * prev_scale);
    *scale = prev_scale * *scale_corr;
    return ORC_OK;
}

/* get_read_seg_score tombo_stats.py:2327-2338 */
double orc_get_read_seg_score(const double *means, const double *rm, const double *rs, i64 n)
{
    double *t = (double *)xmalloc(sizeof(double) * (size_t)n);
    for (i64 i = 0; i < n; i++) t[i] = fabs((means[i] - rm[i]) / rs[i]);
    double r = orc_np_mean(t, n);
    free(t);
    return r;
}

/* score_valid_bases tombo_stats.py:2340-2362 */
static int score_valid_bases(const i64 *tbk, i64 n_tb, const double *em, const double *rm,
                             const double *rs, double *score)
{
    i64 nv = 0;
    double *bm = (double *)xmalloc(sizeof(double) * (size_t)n_tb);
    double *vm = (double *)xmalloc(sizeof(double) * (size_t)n_tb);
    double *vs = (double *)xmalloc(sizeof(double) * (size_t)n_tb);
    for (i64 i = 0; i + 1 < n_tb; i++) {
        if (tbk[i + 1] - tbk[i] != 0) {
            bm[nv] = orc_np_mean(em + tbk[i], tbk[i + 1] - tbk[i]);
            vm[nv] = rm[i]; vs[nv] = rs[i];
            nv++;
        }
    }
    int st = ORC_OK;
    if (nv == 0) st = ORC_ERR_INVALID_START_PATH;
    else *score = orc_get_read_seg_score(bm, vm, vs, nv);
    free(bm); free(vm); free(vs);
    return st;
}

/* compute_num_events tombo_stats.py:1558-1574 */
i64 orc_compute_num_events(i64 sig_len, i64 seq_len, i64 mean_obs_per_event, double min_ratio)
{
    i64 a = sig_len / mean_obs_per_event;
    i64 b = (i64)((double)seq_len * min_ratio);
    return a > b ? a : b;
}

/* identify_stalls (mean-window method) tombo_stats.py:269-368 with
 * MEAN_STALL_PARAMS _default_parameters.py:93-97.  Returns number of intervals. */
i64 orc_identify_stalls(const double *raw, i64 n, i64 *ints, i64 cap)
{
    const i64 window = 350, mini = 50, nwin = 7, min_consec = 200, edge = 100;
    const double thresh = 40;
    if (n < window) return 0;
    /* compute_running_mean_diffs :273-301 */
    double *ma = (double *)xmalloc(sizeof(double) * (size_t)n);
    double *cs = (double *)xmalloc(sizeof(double) * (size_t)n);
    cs[0] = raw[0];
    for (i64 i = 1; i < n; i++) cs[i] = cs[i - 1] + raw[i];
    for (i64 i = 0; i < n; i++) ma[i] = i >= mini ? cs[i] - cs[i - mini] : cs[i];
    i64 n_ma = n - (mini - 1);
    double *mav = (double *)xmalloc(sizeof(double) * (size_t)n_ma);
    for (i64 i = 0; i < n_ma; i++) mav[i] = ma[i + mini - 1] / (double)mini;
    i64 n_off = n_ma - mini * (nwin - 1);
    double *sum = (double *)xmalloc(sizeof(double) * (size_t)n_off);
    i64 n_diffs = nwin * (nwin - 1) / 2;
    /* diff_sums = diffs[0].copy(); for d in diffs: diff_sums += d  (diffs[0] twice) */
    for (i64 p = 0; p < n_off; p++) sum[p] = fabs(mav[p] - mav[p + mini]);
    for (i64 i = 0; i < nwin; i++)
        for (i64 j = i + 1; j < nwin; j++)
            for (i64 p = 0; p < n_off; p++)
                sum[p] += fabs(mav[p + mini * i] - mav[p + mini * j]);
    i64 start_off = (i64)((double)window * 0.5);
    i64 end_off = n - window + start_off + 1;
    /* stall_metric[start_off:end_off] = diff_sums / len(diffs); NaN elsewhere */
    char *below = (char *)calloc((size_t)n + 1, 1);
    for (i64 p = 0; p < n_off && start_off + p < end_off; p++)
        below[start_off + p] = (sum[p] / (double)n_diffs) <= thresh;
    free(ma); free(cs); free(mav); free(sum);
    /* runs of True longer than min_consecutive_obs (:333-340) */
    i64 ni = 0;
    i64 *locs = (i64 *)xmalloc(sizeof(i64) * 2 * (size_t)(n / 2 + 2));
    i64 i = 0;
    while (i < n) {
        if (below[i]) {
            i64 j = i;
            while (j < n && below[j]) j++;
            if (j - i > min_consec) { locs[2 * ni] = i; locs[2 * ni + 1] = j; ni++; }
            i = j;
        } else i++;
    }
    free(below);
    if (ni == 0) { free(locs); return 0; }
    /* expand and merge (:348-364) */
    i64 expand = window / 2 - edge, no = 0;
    if (expand > 0) {
        for (i64 k = 0; k < ni; k++) { locs[2 * k] -= expand; locs[2 * k + 1] += expand; }
        i64 ps = locs[0], pe = locs[1];
        for (i64 k = 0; k < ni; k++) {
            if (locs[2 * k] > pe) {
                if (no < cap) { ints[2 * no] = ps; ints[2 * no + 1] = pe; }
                no++;
                ps = locs[2 * k]; pe = locs[2 * k + 1];
            } else pe = locs[2 * k + 1];
        }
        if (no < cap) { ints[2 * no] = ps; ints[2 * no + 1] = pe; }
        no++;
    } else {
        for (i64 k = 0; k < ni; k++) {
            if (no < cap) { ints[2 * no] = locs[2 * k]; ints[2 * no + 1] = locs[2 * k + 1]; }
            no++;
        }
    }
    free(locs);
    return no;
}

/* remove_stall_cpts tombo_stats.py:1576-1597 */
i64 orc_remove_stall_cpts(const i64 *si, i64 ns, const i64 *cpts, i64 nc, i64 *out)
{
    if (ns == 0) { memcpy(out, cpts, sizeof(i64) * (size_t)nc); return nc; }
    i64 k = 0, no = 0;
    for (i64 i = 0; i < nc; i++) {
        i64 c = cpts[i];
        while (c > si[2 * k + 1]) {
            if (k + 1 >= ns) break;
            k++;
        }
        if (!(si[2 * k] < c && c < si[2 * k + 1])) out[no++] = c;
    }
    return no;
}

/* ===================================================================== */
/* resquiggle.py                                                          */
/* ===================================================================== */
static double shifted_z(double ev, double rm, double rs, const orc_params *p)
{
    /* z_shift - min(max_half_z, |ev - mean| / sd)  resquiggle.py:574-582, 712-720 */
    double a = fabs(ev - rm) / rs;
    if (!isnan(p->max_half_z_score)) a = p->max_half_z_score < a ? p->max_half_z_score : a;
    return p->z_shift - a;
}

/* find_static_base_assignment resquiggle.py:547-600 */
int orc_find_static_base_assignment(const double *em, i64 n_em, const double *rm,
                                    const double *rs, i64 nb, const orc_params *p,
                                    i64 *read_tb)
{
    i64 mask_len = (nb < n_em ? nb : n_em) / 4;
    i64 bw = n_em - mask_len;
    if (bw <= 0 || nb <= 0) return ORC_ERR_UNEXPECTED;
    i64 *es = (i64 *)xmalloc(sizeof(i64) * (size_t)nb);
    i64 n0 = nb - mask_len * 2;
    for (i64 i = 0; i < n0; i++) es[i] = 0;
    if (mask_len > 0) {
        double *ls = (double *)xmalloc(sizeof(double) * (size_t)(mask_len * 2));
        orc_linspace(0, (double)mask_len, mask_len * 2, ls);
        for (i64 i = 0; i < mask_len * 2; i++) es[n0 + i] = (i64)ls[i];
        free(ls);
    }
    double *z = (double *)xmalloc(sizeof(double) * (size_t)(nb * bw));
    for (i64 r = 0; r < nb; r++)
        for (i64 j = 0; j < bw; j++) z[r * bw + j] = shifted_z(em[es[r] + j], rm[r], rs[r], p);
    double *fwd = (double *)xmalloc(sizeof(double) * (size_t)((nb + 1) * bw));
    i64 *tb = (i64 *)xmalloc(sizeof(i64) * (size_t)((nb + 1) * bw));
    orc_banded_forward_pass(z, es, nb, bw, p->skip_pen, p->stay_pen, fwd, tb);
    i64 top = argmax_first(fwd + nb * bw, bw);               /* :589 */
    int st = orc_banded_traceback(tb, es, nb, bw, top, -1, read_tb);
    free(es); free(z); free(fwd); free(tb);
    return st;
}

/* find_seq_start_in_events resquiggle.py:685-752 */
int orc_find_seq_start_in_events(const double *em, i64 n_em, const double *rm,
                                 const double *rs, i64 n_ref, const orc_params *p,
                                 i64 num_bases, i64 num_events, int check_score,
                                 double sig_match_thresh, i64 *start_loc, double *epb)
{
    if (n_em < num_events + num_bases) return ORC_ERR_READ_TOO_SHORT_START;
    if (n_ref < num_bases) return ORC_ERR_MAP_TOO_SHORT_START;
    double *z = (double *)xmalloc(sizeof(double) * (size_t)(num_bases * num_events));
    i64 *es = (i64 *)xmalloc(sizeof(i64) * (size_t)num_bases);
    for (i64 r = 0; r < num_bases; r++) {
        es[r] = r;
        for (i64 j = 0; j < num_events; j++)
            z[r * num_events + j] = shifted_z(em[r + j], rm[r], rs[r], p);
    }
    double *fwd = (double *)xmalloc(sizeof(double) * (size_t)((num_bases + 1) * num_events));
    i64 *tb = (i64 *)xmalloc(sizeof(i64) * (size_t)((num_bases + 1) * num_events));
    i64 *stb = (i64 *)xmalloc(sizeof(i64) * (size_t)(num_bases + 1));
    orc_banded_forward_pass(z, es, num_bases, num_events, p->skip_pen, p->stay_pen, fwd, tb);
    i64 top = argmax_first(fwd + num_bases * num_events, num_events);
    int st = orc_banded_traceback(tb, es, num_bases, num_events, top, -1, stb);
    if (st == ORC_OK && check_score) {
        double sc;
        st = score_valid_bases(stb, num_bases + 1, em, rm, rs, &sc);
        if (st == ORC_OK && sc > sig_match_thresh) st = ORC_ERR_POOR_START_MATCH;
    }
    if (st == ORC_OK) {
        *epb = (double)(stb[num_bases] - stb[0]) / (double)(num_bases + 1);  /* :749 */
        *start_loc = stb[0];
    }
    free(z); free(es); free(fwd); free(tb); free(stb);
    return st;
}

/* _get_masked_start_fwd_pass resquiggle.py:607-683.  Allocates outputs. */
static int masked_start_fwd_pass(const double *em, i64 n_em, const double *rm, const double *rs,
                                 i64 nb, i64 mso, const orc_params *p, double epb,
                                 double **fwd_o, i64 **tb_o, i64 **es_o, i64 *n_rows_o)
{
    i64 bw = p->bandwidth;
    if (n_em - mso < bw) return ORC_ERR_START_TOO_FAR;
    int do_win = !isnan(p->max_half_z_score);
    double mhz = do_win ? p->max_half_z_score : 0.0;
    i64 half_bw = bw / 2;
    i64 bes0 = half_bw <= mso ? 0 : mso - half_bw;                     /* :627-629 */
    i64 t = half_bw > MASK_BASES ? half_bw : MASK_BASES;
    i64 t2 = (i64)((double)(half_bw + 1) / epb);
    i64 tmp_len = (t > t2 ? t : t2) + 1;                               /* :631-632 */
    double *ls = (double *)xmalloc(sizeof(double) * (size_t)tmp_len);
    orc_linspace((double)bes0, (double)bes0 + ((double)tmp_len * epb), tmp_len, ls);
    i64 *es = (i64 *)xmalloc(sizeof(i64) * (size_t)tmp_len);
    for (i64 i = 0; i < tmp_len; i++) es[i] = (i64)ls[i];
    free(ls);
    i64 first = -1;
    for (i64 i = 0; i < tmp_len; i++) if (es[i] >= mso) { first = i; break; }
    if (first < 0) { free(es); return ORC_ERR_UNEXPECTED; }           /* StopIteration */
    i64 mask_seq_len = MASK_BASES > first + 2 ? MASK_BASES : first + 2; /* :637-639 */
    if (mask_seq_len > tmp_len) mask_seq_len = tmp_len;                /* slice clip */
    if (mask_seq_len > nb) { free(es); return ORC_ERR_UNEXPECTED; }    /* IndexError */
    double msp[MASK_BASES];
    orc_linspace((double)(mso + 1), (double)(es[MASK_BASES - 1] + bw), MASK_BASES, msp);
    double *z = (double *)xmalloc(sizeof(double) * (size_t)(mask_seq_len * bw));
    double fill = MASK_FILL_Z_SCORE - p->z_shift;                      /* :666 */
    for (i64 sp = 0; sp < mask_seq_len; sp++) {
        i64 ep = es[sp];
        i64 sml = mso - ep > 0 ? mso - ep : 0;
        i64 eml = sp >= MASK_BASES ? 0 : bw - ((i64)msp[sp] - ep);
        if (ep + bw - eml > n_em) eml = ep + bw - n_em;
        i64 a = ep + sml, b = ep + bw - eml;
        if (b > n_em) b = n_em;
        i64 nv = b - a > 0 ? b - a : 0;
        if (a < 0 || sml < 0 || eml < 0 || sml + nv + eml != bw) {
            free(es); free(z); return ORC_ERR_MASKED_TOO_FEW;
        }
        double *zr = z + sp * bw;
        for (i64 j = 0; j < sml; j++) zr[j] = fill;
        orc_base_z_scores(em + a, nv, rm[sp], rs[sp], do_win, mhz, zr + sml);
        for (i64 j = sml + nv; j < bw; j++) zr[j] = fill;
        for (i64 j = 0; j < bw; j++) zr[j] += p->z_shift;             /* :678 */
    }
    double *fwd = (double *)xmalloc(sizeof(double) * (size_t)((nb + 1) * bw));
    i64 *tb = (i64 *)xmalloc(sizeof(i64) * (size_t)((nb + 1) * bw));
    i64 *es_full = (i64 *)xmalloc(sizeof(i64) * (size_t)nb);
    memcpy(es_full, es, sizeof(i64) * (size_t)mask_seq_len);
    orc_banded_forward_pass(z, es, mask_seq_len, bw, p->skip_pen, p->stay_pen, fwd, tb);
    free(z); free(es);
    *fwd_o = fwd; *tb_o = tb; *es_o = es_full; *n_rows_o = mask_seq_len;
    return ORC_OK;
}

static int short_read_results(const i64 *cpts, const double *em, i64 n_em, const double *rm,
                              const double *rs, i64 nb, const orc_params *p, i64 *segs,
                              i64 *rsrtr)
{
    /* get_short_read_results :886-893 + get_rel_raw_coords :858-864 */
    i64 *tbk = (i64 *)xmalloc(sizeof(i64) * (size_t)(nb + 1));
    int st = orc_find_static_base_assignment(em, n_em, rm, rs, nb, p, tbk);
    if (st == ORC_OK) {
        for (i64 i = 0; i <= nb; i++) {
            if (tbk[i] < 0 || tbk[i] > n_em) { st = ORC_ERR_UNEXPECTED; break; }
            segs[i] = cpts[tbk[i]];
        }
        if (st == ORC_OK) {
            *rsrtr = segs[0];
            for (i64 i = nb; i >= 0; i--) segs[i] -= segs[0];
        }
    }
    free(tbk);
    return st;
}

/* debug taps for parity tests (band starts / event traceback of the last
 * adaptive assignment) */
static i64 *g_dbg_es = NULL, *g_dbg_tb = NULL;
void orc_set_debug_buffers(i64 *es, i64 *tb) { g_dbg_es = es; g_dbg_tb = tb; }

/* find_adaptive_base_assignment resquiggle.py:866-1050 (start_clip_bases=None) */
int orc_find_adaptive_base_assignment(const i64 *cpts, i64 n_cpts, const double *em,
                                      const orc_params *p, const double *rm, const double *rs,
                                      i64 nb, double sig_match_thresh, i64 *segs, i64 *rsrtr,
                                      i64 *dbg_path, double *dbg_epb)
{
    i64 n_em = n_cpts - 1;
    i64 mapped_start = 0;
    double epb = 0;
    if (dbg_path) { dbg_path[0] = 0; dbg_path[1] = -1; dbg_path[2] = -1; }
    if (n_em < p->start_bw + p->start_n_bases || nb < p->start_n_bases)   /* :986-989 */
        return short_read_results(cpts, em, n_em, rm, rs, nb, p, segs, rsrtr);
    int st = orc_find_seq_start_in_events(em, n_em, rm, rs, nb, p, p->start_n_bases,
                                          p->start_bw, 1, sig_match_thresh, &mapped_start,
                                          &epb);
    if (st != ORC_OK && st != ORC_ERR_UNEXPECTED) {                       /* except TomboError */
        if (n_em < p->start_save_bw + p->start_n_bases)
            return short_read_results(cpts, em, n_em, rm, rs, nb, p, segs, rsrtr);
        st = orc_find_seq_start_in_events(em, n_em, rm, rs, nb, p, p->start_n_bases,
                                          p->start_save_bw, 0, 0.0, &mapped_start, &epb);
    }
    if (st != ORC_OK) return st;
    if (dbg_epb) *dbg_epb = epb;
    if (epb == 0) return ORC_ERR_OPEN_PORE;                               /* :1008 */
    i64 bw = p->bandwidth, half_bw = bw / 2, clip, mso;
    if (mapped_start < half_bw) { clip = 0; mso = mapped_start; }
    else { clip = mapped_start - half_bw; mso = half_bw; }
    if (dbg_path) { dbg_path[1] = mapped_start; dbg_path[2] = clip; }
    if ((i64)((double)(half_bw + 1) / epb) >= nb || (n_em - mso - clip < bw))   /* :1024 */
        return short_read_results(cpts, em, n_em, rm, rs, nb, p, segs, rsrtr);
    if (dbg_path) dbg_path[0] = 1;
    /* run_fwd_pass :895-942 */
    double *fwd; i64 *tb, *es, n_rows;
    const double *emc = em + clip;
    i64 n_emc = n_em - clip;
    st = masked_start_fwd_pass(emc, n_emc, rm, rs, nb, mso, p, epb, &fwd, &tb, &es, &n_rows);
    if (st != ORC_OK) return st;
    int do_win = !isnan(p->max_half_z_score);
    st = orc_adaptive_banded_forward_pass(fwd, tb, es, nb, bw, emc, n_emc, rm, rs, p->z_shift,
                                          p->skip_pen, p->stay_pen, n_rows, MASK_FILL_Z_SCORE,
                                          do_win, do_win ? p->max_half_z_score : 0.0, NULL);
    i64 *tbk = (i64 *)xmalloc(sizeof(i64) * (size_t)(nb + 1));
    if (st == ORC_OK) {
        i64 top = argmax_first(fwd + nb * bw, bw);                        /* :1032 */
        st = orc_banded_traceback(tb, es, nb, bw, top, p->band_bound_thresh, tbk);
    }
    if (g_dbg_es) memcpy(g_dbg_es, es, sizeof(i64) * (size_t)nb);
    if (st == ORC_OK && g_dbg_tb) memcpy(g_dbg_tb, tbk, sizeof(i64) * (size_t)(nb + 1));
    if (st == ORC_OK) {
        /* _trim_traceback :754-764 */
        i64 i = 0;
        while (i <= nb && tbk[i] < 0) tbk[i++] = 0;
        i64 e = 1;
        while (e <= nb + 1 && tbk[nb + 1 - e] > n_emc) { tbk[nb + 1 - e] = n_emc; e++; }
        for (i = 0; i <= nb; i++) segs[i] = cpts[clip + tbk[i]];
        *rsrtr = segs[0];
        for (i = nb; i >= 0; i--) segs[i] -= segs[0];
    }
    free(fwd); free(tb); free(es); free(tbk);
    return st;
}

/* ---- raw-signal DP for skipped bases ---- */
typedef struct { double *z; double *fwd; i64 *ld; i64 start, end; } rawrow_t;

/* c_base_forward_pass _c_dynamic_programming.pyx:99-163 */
static int base_forward_pass(rawrow_t *b, const rawrow_t *pv, i64 min_obs)
{
    i64 b_len = b->end - b->start, p_len = pv->end - pv->start;
    double *cs = (double *)xmalloc(sizeof(double) * (size_t)p_len);
    cs[0] = pv->z[0];
    for (i64 i = 1; i < p_len; i++) cs[i] = cs[i - 1] + pv->z[i];
#define CHK(ix, len) if ((ix) < 0 || (ix) >= (len)) { free(cs); return ORC_ERR_UNEXPECTED; }
    CHK(b->start - pv->start - 1, p_len)
    b->fwd[0] = b->z[0] + pv->fwd[b->start - pv->start - 1];
    b->ld[0] = 1;
    for (i64 pos = b->start + 1; pos < pv->end + 1; pos++) {
        i64 lag = 1;
        for (;;) {
            CHK(pos - pv->start - lag, p_len)
            if (pv->ld[pos - pv->start - lag] + lag <= min_obs) lag++; else break;
        }
        double diag = pv->fwd[pos - pv->start - lag];
        if (lag > 1) {
            CHK(pos - pv->start - 1, p_len)
            diag += cs[pos - pv->start - 1] - cs[pos - pv->start - lag];
        }
        CHK(pos - b->start, b_len)
        double stay = b->fwd[pos - b->start - 1], score;
        i64 dv;
        if (diag > stay) { score = diag; dv = 1; }
        else { score = stay; dv = b->ld[pos - b->start - 1] + 1; }
        b->fwd[pos - b->start] = b->z[pos - b->start] + score;
        b->ld[pos - b->start] = dv;
    }
    if (b->end > pv->end + 1) {
        CHK(pv->end - b->start, b_len)
        double fv = b->fwd[pv->end - b->start];
        i64 cl = b->ld[pv->end - b->start];
        i64 left = b->end - pv->end - 1;
        for (i64 i = 0; i < left; i++) {
            fv += b->z[i + pv->end - b->start + 1];
            cl += 1;
            b->fwd[i + pv->end - b->start + 1] = fv;
            b->ld[i + pv->end - b->start + 1] = cl;
        }
    }
#undef CHK
    free(cs);
    return ORC_OK;
}

/* c_base_traceback :165-182; returns -1 for the reference's implicit None */
static i64 base_traceback(const rawrow_t *cur, const rawrow_t *nxt, i64 sig_start, i64 min_obs)
{
    i64 cbs = 1;
    for (i64 sp = sig_start; sp >= 0; sp--) {
        cbs += 1;
        if (cbs <= min_obs || sp - 1 >= nxt->end) continue;
        if (sp <= cur->start) return sp;
        i64 a = sp - nxt->start - 1, b = sp - cur->start - 1;
        if (a < 0 || a >= nxt->end - nxt->start || b < 0 || b >= cur->end - cur->start) return -2;
        if (nxt->fwd[a] > cur->fwd[b]) return sp;
    }
    return -1;
}

/* one deletion window: c_reg_z_scores (:34-97) + raw_forward_pass
 * (resquiggle.py:345-380) + raw_traceback (:382-400) */
static int raw_window(const double *sig, i64 sig_len, const double *rm, const double *rs,
                      i64 n_ev, const orc_params *p, i64 *new_segs /* n_ev-1 */)
{
    i64 min_obs = p->raw_min_obs_per_base;
    double *ls = (double *)xmalloc(sizeof(double) * (size_t)(n_ev + 1));
    i64 *ps = (i64 *)xmalloc(sizeof(i64) * (size_t)(n_ev + 1));
    orc_linspace(0.0, (double)sig_len, n_ev + 1, ls);               /* resquiggle.py:514 */
    for (i64 i = 0; i <= n_ev; i++) ps[i] = (i64)floor(ls[i]);
    free(ls);
    i64 reg_start = 0, reg_end = n_ev, max_shift = n_ev;
    rawrow_t *rows = (rawrow_t *)calloc((size_t)n_ev, sizeof(rawrow_t));
    int st = ORC_OK;
    i64 prev = 0;
    for (i64 idx = 0; idx < n_ev; idx++) {                          /* :56-66 */
        i64 bi = reg_start + idx, k = bi - max_shift > reg_start ? bi - max_shift : reg_start;
        i64 s = ps[k];
        if (idx > 0 && s < prev + min_obs) s = prev + min_obs;
        rows[idx].start = s; prev = s;
    }
    for (i64 idx = 0; idx < n_ev; idx++) {                          /* :71-81 */
        i64 bi = reg_start + (n_ev - idx - 1);
        i64 k = bi + max_shift + 1 < reg_end ? bi + max_shift + 1 : reg_end;
        i64 e = ps[k];
        if (idx > 0 && e > prev - min_obs) e = prev - min_obs;
        rows[n_ev - idx - 1].end = e; prev = e;
    }
    int do_win = !isnan(p->max_half_z_score);
    for (i64 idx = 0; idx < n_ev && st == ORC_OK; idx++) {
        i64 s = rows[idx].start, e = rows[idx].end;
        if (s < 0 || e > sig_len || e <= s) { st = ORC_ERR_UNEXPECTED; break; }
        i64 len = e - s;
        rows[idx].z = (double *)xmalloc(sizeof(double) * (size_t)len);
        rows[idx].fwd = (double *)xmalloc(sizeof(double) * (size_t)len);
        rows[idx].ld = (i64 *)xmalloc(sizeof(i64) * (size_t)len);
        orc_base_z_scores(sig + s, len, rm[idx], rs[idx], do_win,
                          do_win ? p->max_half_z_score : 0.0, rows[idx].z);
        rows[idx].start = s - ps[reg_start]; rows[idx].end = e - ps[reg_start];
    }
    if (st == ORC_OK) {
        /* raw_forward_pass: first row cumsum, last_diag = min_obs */
        i64 len = rows[0].end - rows[0].start;
        rows[0].fwd[0] = rows[0].z[0];
        for (i64 i = 1; i < len; i++) rows[0].fwd[i] = rows[0].fwd[i - 1] + rows[0].z[i];
        for (i64 i = 0; i < len; i++) rows[0].ld[i] = min_obs;
        for (i64 r = 1; r < n_ev && st == ORC_OK; r++)
            st = base_forward_pass(&rows[r], &rows[r - 1], min_obs);
    }
    if (st == ORC_OK) {
        if (n_ev < 2) st = ORC_ERR_UNEXPECTED;
        else {
            i64 v = base_traceback(&rows[n_ev - 1], &rows[n_ev - 2], rows[n_ev - 1].end - 1,
                                   min_obs);
            if (v < 0) st = ORC_ERR_UNEXPECTED; else new_segs[n_ev - 2] = v;
            for (i64 bp = n_ev - 3; bp >= 0 && st == ORC_OK; bp--) {
                v = base_traceback(&rows[bp + 1], &rows[bp], new_segs[bp + 1] - 1, min_obs);
                if (v < 0) st = ORC_ERR_UNEXPECTED; else new_segs[bp] = v;
            }
        }
    }
    for (i64 i = 0; i < n_ev; i++) { free(rows[i].z); free(rows[i].fwd); free(rows[i].ld); }
    free(rows); free(ps);
    return st;
}

/* resolve_skipped_bases_with_raw resquiggle.py:402-540 */
int orc_resolve_skipped_bases_with_raw(const i64 *segs, i64 nb, const double *rm,
                                       const double *rs, const double *norm, i64 n_norm,
                                       const orc_params *p, i64 max_raw_cpts, i64 *out)
{
    i64 n_segs = nb + 1, nw = 0;
    i64 *ws = (i64 *)xmalloc(sizeof(i64) * (size_t)(nb + 2));
    i64 *we = (i64 *)xmalloc(sizeof(i64) * (size_t)(nb + 2));
    memcpy(out, segs, sizeof(i64) * (size_t)n_segs);
    for (i64 d = 0; d < nb; d++) {                                   /* :465-472 */
        if (segs[d + 1] - segs[d] != 0) continue;
        if (nw > 0 && d < we[nw - 1] + DEL_FIX_WINDOW) we[nw - 1] = d + DEL_FIX_WINDOW + 1;
        else { ws[nw] = d - DEL_FIX_WINDOW; we[nw] = d + DEL_FIX_WINDOW + 1; nw++; }
    }
    int st = ORC_OK;
    if (nw == 0) goto done;
#define TOO_SMALL(s, e) ((double)(segs[e] - segs[s]) <= \
        ((double)(((e) - (s) + 1) * p->raw_min_obs_per_base)) * EXTRA_SIG_FACTOR)
#define MERGE_TRIM() do { \
        i64 m = 0; \
        for (i64 k = 0; k < nw; k++) { \
            if (m > 0 && ws[k] < we[m - 1]) we[m - 1] = we[k]; \
            else { ws[m] = ws[k]; we[m] = we[k]; m++; } } \
        nw = m; \
        if (ws[0] < 0) ws[0] = 0; \
        if (we[nw - 1] > n_segs - 1) we[nw - 1] = n_segs - 1; } while (0)
    MERGE_TRIM();
    int expanded = 0;
    for (int it = 0; it < MAX_DEL_FIX_WINDOW - DEL_FIX_WINDOW; it++) {  /* :481-486 */
        expanded = 0;
        for (i64 k = 0; k < nw; k++)
            if (TOO_SMALL(ws[k], we[k])) { expanded = 1; ws[k] -= 1; we[k] += 1; }
        if (!expanded) break;
        MERGE_TRIM();
    }
    if (expanded) {
        for (i64 k = 0; k < nw; k++)
            if (TOO_SMALL(ws[k], we[k])) { st = ORC_ERR_NOT_ENOUGH_DEL_SIGNAL; goto done; }
    }
    if (max_raw_cpts >= 0) {
        i64 mx = 0;
        for (i64 k = 0; k < nw; k++) if (we[k] - ws[k] > mx) mx = we[k] - ws[k];
        if (mx > max_raw_cpts) { st = ORC_ERR_TOO_MANY_DELS; goto done; }
    }
    for (i64 k = 0; k < nw; k++) {                                   /* :506-531 */
        i64 s = ws[k], e = we[k], n_ev = e - s;
        i64 sig_start = segs[s], sig_len = segs[e] - segs[s];
        if (sig_start < 0 || sig_start + sig_len > n_norm) { st = ORC_ERR_UNEXPECTED; goto done; }
        i64 *ns = (i64 *)xmalloc(sizeof(i64) * (size_t)(n_ev));
        st = raw_window(norm + sig_start, sig_len, rm + s, rs + s, n_ev, p, ns);
        if (st == ORC_OK) for (i64 i = 0; i < n_ev - 1; i++) out[s + 1 + i] = ns[i] + sig_start;
        free(ns);
        if (st != ORC_OK) goto done;
    }
    for (i64 i = 0; i < nb; i++) if (out[i + 1] - out[i] < 1) { st = ORC_ERR_ZERO_LEN_SEG; goto done; }
    if (out[0] < 0) { st = ORC_ERR_NEG_SEG; goto done; }
    if (out[nb] > n_norm) { st = ORC_ERR_SEG_PAST_END; goto done; }
done:
    free(ws); free(we);
    return st;
}

/* segment_signal resquiggle.py:1057-1120 */
static int segment_signal(const double *raw, i64 n_raw, i64 num_events, const orc_params *p,
                          const orc_policy *pol, const orc_scale_values *sv_in, int first_call,
                          const i64 *stall_ints, i64 n_stalls, double *norm,
                          orc_scale_values *sv, i64 *cpts, i64 *n_cpts)
{
    int st;
    /* iterations >= 2 are called without const_scale (resquiggle.py:1499-1502) */
    int use_const = first_call && !isnan(pol->const_scale);
    if (p->use_t_test_seg) {
        st = orc_valid_cpts_w_cap_t_test(raw, n_raw, p->min_obs_per_base, p->running_stat_width,
                                         num_events, (int)pol->tie_stable, cpts);
        if (st != ORC_OK) return st;
        *n_cpts = num_events;
        if (stall_ints != NULL) {
            i64 *t = (i64 *)xmalloc(sizeof(i64) * (size_t)num_events);
            *n_cpts = orc_remove_stall_cpts(stall_ints, n_stalls, cpts, num_events, t);
            memcpy(cpts, t, sizeof(i64) * (size_t)*n_cpts);
            free(t);
        }
        if (sv_in != NULL)
            return orc_normalize_raw_signal(raw, n_raw, 0, NAN, NAN, sv_in, norm, sv);
        if (use_const)
            return orc_normalize_raw_signal(raw, n_raw, 1, pol->outlier_thresh, pol->const_scale,
                                            NULL, norm, sv);
        /* get_scale_values_from_events tombo_stats.py:217-233 */
        i64 ne = RNA_SCALE_NUM_EVENTS;
        if ((double)*n_cpts * RNA_SCALE_MAX_FRAC_EVENTS < (double)ne)
            ne = (i64)((double)*n_cpts * RNA_SCALE_MAX_FRAC_EVENTS);
        if (ne < 2) return ORC_ERR_UNEXPECTED;
        double *evm = (double *)xmalloc(sizeof(double) * (size_t)ne);
        orc_new_means(raw, cpts, ne - 1, evm);
        double med = orc_median(evm, ne - 1);
        for (i64 i = 0; i < ne - 1; i++) evm[i] = fabs(evm[i] - med);
        double mad = orc_median(evm, ne - 1);
        free(evm);
        orc_scale_values ev_sv = { med, mad, -pol->outlier_thresh, pol->outlier_thresh, NAN };
        return orc_normalize_raw_signal(raw, n_raw, 0, NAN, NAN, &ev_sv, norm, sv);
    }
    if (sv_in != NULL) st = orc_normalize_raw_signal(raw, n_raw, 0, NAN, NAN, sv_in, norm, sv);
    else if (use_const)
        st = orc_normalize_raw_signal(raw, n_raw, 1, pol->outlier_thresh, pol->const_scale, NULL,
                                      norm, sv);
    else st = orc_normalize_raw_signal(raw, n_raw, 0, pol->outlier_thresh, NAN, NULL, norm, sv);
    if (st != ORC_OK) return st;
    st = orc_valid_cpts_w_cap(norm, n_raw, p->min_obs_per_base, p->running_stat_width,
                              num_events, (int)pol->tie_stable, cpts);
    if (st != ORC_OK) return st;
    *n_cpts = num_events;
    if (stall_ints != NULL) {
        i64 *t = (i64 *)xmalloc(sizeof(i64) * (size_t)num_events);
        *n_cpts = orc_remove_stall_cpts(stall_ints, n_stalls, cpts, num_events, t);
        memcpy(cpts, t, sizeof(i64) * (size_t)*n_cpts);
        free(t);
    }
    return ORC_OK;
}

/* resquiggle_read resquiggle.py:1122-1214 */
int orc_resquiggle_read(const double *raw, i64 n_raw, const double *rm, const double *rs, i64 nb,
                        const orc_params *p, const orc_policy *pol,
                        const orc_scale_values *sv_in, int first_call, const i64 *stall_ints,
                        i64 n_stalls, uint32_t key, i64 *segs, double *norm_out,
                        orc_read_result *res)
{
    if (raw == NULL || n_raw <= 0) return ORC_ERR_NO_RAW;
    i64 num_events = orc_compute_num_events(n_raw, nb, p->mean_obs_per_event,
                                            pol->min_event_to_seq_ratio);
    if ((double)num_events / (double)p->bandwidth > (double)nb) return ORC_ERR_TOO_MUCH_SIGNAL;
    double *norm = (double *)xmalloc(sizeof(double) * (size_t)n_raw);
    i64 *cpts = (i64 *)xmalloc(sizeof(i64) * (size_t)(num_events + 1));
    i64 *dp_segs = (i64 *)xmalloc(sizeof(i64) * (size_t)(nb + 1));
    double *em = NULL, *bm = NULL;
    i64 n_cpts = 0, rsrtr = 0;
    orc_scale_values sv;
    int st = segment_signal(raw, n_raw, num_events, p, pol, sv_in, first_call, stall_ints,
                            n_stalls, norm, &sv, cpts, &n_cpts);
    if (st != ORC_OK) goto done;
    if (n_cpts < 2) { st = ORC_ERR_UNEXPECTED; goto done; }
    em = (double *)xmalloc(sizeof(double) * (size_t)n_cpts);
    orc_new_means(norm, cpts, n_cpts - 1, em);                       /* :1164 */
    st = orc_find_adaptive_base_assignment(cpts, n_cpts, em, p, rm, rs, nb,
                                           pol->sig_match_thresh, dp_segs, &rsrtr, NULL, NULL);
    if (st != ORC_OK) goto done;
    {
        const double *ns = norm + rsrtr;                             /* :1171 */
        i64 n_norm = dp_segs[nb];
        st = orc_resolve_skipped_bases_with_raw(dp_segs, nb, rm, rs, ns, n_norm, p,
                                                pol->max_raw_cpts, segs);
        if (st != ORC_OK) goto done;
        bm = (double *)xmalloc(sizeof(double) * (size_t)nb);
        double *nn = (double *)xmalloc(sizeof(double) * (size_t)(n_norm > 0 ? n_norm : 1));
        memcpy(nn, ns, sizeof(double) * (size_t)n_norm);
        int changed = 0;
        int skip_scaling = first_call && pol->skip_seq_scaling;
        if (!skip_scaling) {
            double shift, scale, shc, scc;
            orc_new_means(nn, segs, nb, bm);
            st = orc_theil_sen(sv.shift, sv.scale, bm, rm, nb, key, &shift, &scale, &shc, &scc);
            if (st != ORC_OK) { free(nn); goto done; }
            sv.shift = shift; sv.scale = scale; sv.outlier_thresh = pol->outlier_thresh;
            for (i64 i = 0; i < n_norm; i++) nn[i] = (nn[i] - shc) / scc;   /* :1190 */
            changed = fabs(shc) > SHIFT_CHANGE_THRESH || fabs(scc - 1) > SCALE_CHANGE_THRESH;
        }
        orc_new_means(nn, segs, nb, bm);
        res->sig_match_score = orc_get_read_seg_score(bm, rm, rs, nb);
        res->read_start_rel_to_raw = rsrtr;
        res->sv = sv;
        res->norm_params_changed = changed;
        res->n_norm = n_norm;
        if (norm_out) memcpy(norm_out, nn, sizeof(double) * (size_t)n_norm);
        free(nn);
    }
done:
    free(norm); free(cpts); free(dp_segs); free(em); free(bm);
    return st;
}

/* worker policy resquiggle.py:1492-1530, 1575-1595 */
int orc_run_read(const double *raw_in, i64 n_raw, const double *rm, const double *rs, i64 nb,
                 const orc_params *p, const orc_params *save_p, const orc_policy *pol,
                 uint32_t read_index, i64 *segs, double *norm_out, orc_read_result *res,
                 i64 *info)
{
    return orc_run_read_inputs(raw_in, n_raw, rm, rs, nb, p, save_p, pol, read_index, segs,
                               norm_out, res, info, NULL, NULL, 0);
}

int orc_run_read_inputs(const double *raw_in, i64 n_raw, const double *rm, const double *rs,
                        i64 nb, const orc_params *p, const orc_params *save_p,
                        const orc_policy *pol, uint32_t read_index, i64 *segs, double *norm_out,
                        orc_read_result *res, i64 *info, const orc_scale_values *sv_in,
                        const i64 *stall_ints_in, i64 n_stalls_in)
{
    double *raw = (double *)xmalloc(sizeof(double) * (size_t)(n_raw > 0 ? n_raw : 1));
    i64 *stalls = NULL, n_stalls = 0;
    const i64 *use_stalls = stall_ints_in;
    if (pol->is_rna) {
        for (i64 i = 0; i < n_raw; i++) raw[i] = raw_in[n_raw - 1 - i];  /* :1516 */
        i64 cap = n_raw / 200 + 4;
        stalls = (i64 *)xmalloc(sizeof(i64) * 2 * (size_t)cap);
        n_stalls = orc_identify_stalls(raw, n_raw, stalls, cap);          /* :1524-1528 */
        use_stalls = stalls;
    } else {
        memcpy(raw, raw_in, sizeof(double) * (size_t)n_raw);
        n_stalls = n_stalls_in;
    }
    uint32_t calls = 0;
    int st = ORC_OK, first_st = ORC_OK;
    i64 rescued = 0, n_iters = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
        const orc_params *prm = attempt == 0 ? p : save_p;
        /* a rescue starts again from the caller's map_res */
        st = orc_resquiggle_read(raw, n_raw, rm, rs, nb, prm, pol, sv_in, 1, use_stalls, n_stalls,
                                 orc_subsample_key(pol->subsample_seed, read_index, calls),
                                 segs, norm_out, res);
        calls++;
        n_iters = 1;
        while (st == ORC_OK && n_iters < pol->max_scaling_iters && res->norm_params_changed) {
            orc_scale_values sv = res->sv;
            st = orc_resquiggle_read(raw, n_raw, rm, rs, nb, prm, pol, &sv, 0, use_stalls, n_stalls,
                                     orc_subsample_key(pol->subsample_seed, read_index, calls),
                                     segs, norm_out, res);
            calls++;
            n_iters++;
        }
        if (st == ORC_OK) break;
        if (attempt == 0) { first_st = st; rescued = 1; }
    }
    if (info) { info[0] = calls; info[1] = rescued; info[2] = n_iters; info[3] = first_st; }
    free(raw); free(stalls);
    return st;
}
