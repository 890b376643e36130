"""Plain restatements of the per-read statistics stage and the error bounds that the device
is held to (helper module of test_stats_cpu.py / test_stats_gpu.py, no pytest here).

- LLRs of compute_alt_model_read_stats for whole '+' strand reads and a single-base motif,
  with the three Cython scorers (c_calc_scaled_llh_ratio_const_var, c_calc_llh_ratio_const_var,
  c_calc_llh_ratio) in the reference's operation order.  They use math.exp / math.pow /
  math.log, i.e. the C library the reference's compiled scorers call; numpy's vectorised
  np.exp / np.power / np.log are not glibc and differ in the last bit for a few per cent of
  inputs, so nothing here that must be bit-exact uses a numpy ufunc.
- z -> two-sided p -> Fisher window, twice: the reference's own path (scipy ndtr,
  np.maximum(p, 1e-50), log, window sum, chi2.sf, the de novo final clamp) and an exact path
  (mpmath at 40 digits, starting from the float64 z that both sides compute identically).
- The region counters: collate_reg_stats / apply_per_read_thresh / calc_damp_fraction.
- Seeded case families, each named for the edge it exercises.

Error bounds are in units of u = 2^-53.  They rest on these documented maximum errors:
  CUDA (Programming Guide, mathematical functions appendix, double precision):
    exp 1 ulp, log 1 ulp, pow 2 ulp, erfc 5 ulp;
  glibc (manual, "Known Maximum Errors in Math Functions", x86_64):
    exp 1 ulp, log 1 ulp, pow 1 ulp;
  scipy's ndtr (Cephes erfc/erf), used only by the reference path: a few ulp.
One ulp of a double is at most 2u relative.  Every basic operation (+ - * /, sqrt) is
correctly rounded on both sides and the library is built with -fmad=false, so device and
restatement take identical bits through every operation except the transcendental calls; the
bounds propagate only those differences."""
import math

import mpmath
import numpy as np

U = 2.0 ** -53
SMALLEST_PVAL = 1e-50                    # SMALLEST_PVAL _default_parameters.py
Y_PER_CLAMPED_P = 115.13                 # -log(1e-50) = 115.1293, the most one p adds to y
TINY = 1e-300                            # below this only "tiny" is asserted


# ---------------------------------------------------------------------------
# chi-square survival function with even degrees of freedom
# ---------------------------------------------------------------------------
def _poisson_cdf(k, y):
    """P(N <= k - 1), N ~ Poisson(y), summed outward from the largest term at 60 digits"""
    with mpmath.workdps(60):
        y = mpmath.mpf(y)
        if y == 0:
            return mpmath.mpf(1)
        jt = min(k - 1, int(mpmath.floor(y)))
        top = mpmath.exp(-y + jt * mpmath.log(y) - mpmath.loggamma(jt + 1))
        s, t, eps = mpmath.mpf(1), mpmath.mpf(1), mpmath.mpf('1e-35')
        for j in range(jt, 0, -1):
            t = t * j / y
            s += t
            if t < s * eps:
                break
        t = mpmath.mpf(1)
        for j in range(jt + 1, k):
            t = t * y / j
            s += t
            if t < s * eps:
                break
        return top * s


def exact_chi2_sf_even(y, k):
    """scipy.stats.chi2.sf(2 y, 2 k) = Q(k, y) = gammainc(k, y, inf, regularized), exactly
    (mpmath; its hypergeometric series gives up for a few large k near y = k, where the
    Poisson sum from the mode takes over)"""
    with mpmath.workdps(40):
        try:
            return mpmath.gammainc(k, mpmath.mpf(y), mpmath.inf, regularized=True)
        except mpmath.libmp.NoConvergence:
            return _poisson_cdf(k, y)


def chi2_bound(y):
    """relative error allowed for tb2_chi2_sf_even(y, k) where Q > 1e-300 (DESIGN §2): the
    large-y branch rounds log p(j; y), of size up to ~y, so exp() carries ~y u; 16 y u covers
    it with the saddle-point terms, and 1e-12 covers the ratio sums"""
    return 1e-12 + 16.0 * U * y


# ---------------------------------------------------------------------------
# LLR scorers (_c_helper.pyx), one site each: (llr, S = sum |term|)
# ---------------------------------------------------------------------------
def scaled_llr(m, r, a, cv, sf, hf, hp):
    acc, s_abs = 0.0, 0.0
    for obs, ref_mean, alt_mean in zip(m, r, a):
        if ref_mean == alt_mean:
            continue
        scale_mean = (alt_mean + ref_mean) / 2
        ref_diff = obs - ref_mean
        alt_diff = obs - alt_mean
        scale_diff = obs - scale_mean
        means_diff = alt_mean - ref_mean
        if means_diff < 0:
            means_diff = means_diff * -1
        t = math.exp(-(scale_diff * scale_diff) / (sf * cv)) * (
            (alt_diff * alt_diff) - (ref_diff * ref_diff)) / (
                cv * math.pow(means_diff, hp) * hf)
        acc += t
        s_abs += abs(t)
    return acc, s_abs


def standard_llr(m, r, a, cv):
    acc, s_abs = 0.0, 0.0
    for obs, ref_mean, alt_mean in zip(m, r, a):
        ref_diff = obs - ref_mean
        alt_diff = obs - alt_mean
        t = ((alt_diff * alt_diff) - (ref_diff * ref_diff)) / cv
        acc += t
        s_abs += abs(t)
    return acc, s_abs


def var_llr(m, r, a, rv, av):
    rz = rl = az = al = 0.0
    s_abs = 0.0
    for i in range(len(m)):
        rd = m[i] - r[i]
        rz += (rd * rd) / rv[i]
        rl += math.log(rv[i])
        ad = m[i] - a[i]
        az += (ad * ad) / av[i]
        al += math.log(av[i])
        s_abs += abs((rd * rd) / rv[i]) + abs(math.log(rv[i])) + abs((ad * ad) / av[i]) + \
            abs(math.log(av[i]))
    return az + al - rz - rl, s_abs


def score_window(mode, m, r, a, va, vb=None, sf=4.0, hf=1.0, hp=0.2):
    """tb2_calc_llh_ratio_windows' three modes: 0 scaled, 1 standard (const var), 2 var"""
    m, r, a = [float(x) for x in m], [float(x) for x in r], [float(x) for x in a]
    if mode == 0:
        return scaled_llr(m, r, a, float(va), sf, hf, hp)
    if mode == 1:
        return standard_llr(m, r, a, float(va))
    return var_llr(m, r, a, [float(x) for x in va], [float(x) for x in vb])


def llr_bound(mode, s_abs, K):
    """|device - restatement| allowed for one site.
    mode 1: no transcendental call, so 0 (bit-exact).
    mode 0, per term: exp differs by <= 1 + 1 ulp (4u), pow by <= 2 + 1 ulp (6u); the four
      roundings that follow them (E * N, cv * P, * hf, /) may each round differently (2u
      each): <= 18u of |term|, taken as 20u.  The running sum over K terms adds <= 2u of the
      partial sum per step, <= 2K u S in all.  Bound (20 + 2K) u S.
    mode 2: only the 2K logs differ, by <= 2 ulp (4u) of |log v| each; with the 4 running
      sums (2u per step) and the final three operations: (8 + 2K) u S."""
    if mode == 1:
        return 0.0
    if mode == 0:
        return (20.0 + 2.0 * K) * U * s_abs
    return (8.0 + 2.0 * K) * U * s_abs


def kmer_codes(bases, K):
    c = np.zeros(bases.shape[0] - K + 1, dtype=np.int64)
    for j in range(K):
        c = c * 4 + (bases[j:j + c.shape[0]] & 3)
    return c


def llr_reads(norm_mean, mean_off, seq, seq_off, read_start, kmeans, ksds, alt, K, cpos,
              alt_code, mode, sf=4.0, hf=1.0, hp=0.2, alt_sds=None):
    """compute_alt_model_read_stats for whole '+' strand reads (TomboMotif(alt, 1)) in the
    library's layout: read r has nb = mean_off[r+1] - mean_off[r] per-base means and
    nb + K - 1 base codes, the sequence running cpos bases ahead of the means.  The trimmed
    read (trim_seq_and_means) keeps means[cpos : nb - (K-1-cpos)] and its k-mers; the testable
    bases are those with a whole K-mer window on both sides, nb - 2 (K-1) of them; a site is a
    testable base equal to alt_code, scored over the K k-mers that contain it with the
    reference variance of the first one (r_ref_vars[alt_pos]).  alt is the (4^K, K) table of
    alternative means by k-mer code and position of the base inside the k-mer.
    Returns (llr, pos, site_off, S)."""
    llr, pos, s_all, off = [], [], [], [0]
    for r in range(mean_off.shape[0] - 1):
        nb = int(mean_off[r + 1] - mean_off[r])
        means = norm_mean[mean_off[r]:mean_off[r + 1]]
        testable = nb - 2 * (K - 1)
        n = 0
        if testable > 0:
            bases = np.asarray(seq[seq_off[r] + cpos:seq_off[r] + cpos + nb], dtype=np.int64)
            codes = kmer_codes(bases, K)               # k-mers of the trimmed read
            for i in range(testable):
                if bases[i + K - 1] != alt_code:
                    continue
                w = codes[i:i + K]
                m = means[cpos + i:cpos + i + K]
                rm = kmeans[w]
                am = alt[w, K - 1 - np.arange(K)]
                if mode == 2:
                    v, s = score_window(2, m, rm, am, ksds[w] * ksds[w],
                                        alt_sds[w, K - 1 - np.arange(K)] ** 2)
                else:
                    sd = float(ksds[w[0]])
                    v, s = score_window(mode, m, rm, am, sd * sd, sf=sf, hf=hf, hp=hp)
                llr.append(v)
                s_all.append(s)
                pos.append(int(read_start[r]) + (K - 1) + i)
                n += 1
        off.append(off[-1] + n)
    return (np.array(llr, dtype=np.float64), np.array(pos, dtype=np.int64),
            np.array(off, dtype=np.int64), np.array(s_all, dtype=np.float64))


def assert_llr(got, want, s_abs, mode, K):
    """standard LLRs bit for bit, the others within llr_bound; returns the largest
    error / bound ratio"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape
    if mode == 1:
        assert np.array_equal(got, want, equal_nan=True)
        return 0.0
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    err = np.abs(got[ok] - want[ok])
    bound = np.array([llr_bound(mode, s, K) for s in s_abs[ok]])
    assert np.all(err <= bound), (np.max(err - bound), np.nonzero(err > bound)[0][:5])
    keep = bound > 0
    return float(np.max(err[keep] / bound[keep])) if keep.any() else 0.0


# ---------------------------------------------------------------------------
# z -> p -> Fisher window
# ---------------------------------------------------------------------------
def z_scores(m, rm, rs):
    """np.abs(r_means - ref) / sds; the device's fabs(m - rm) / rs has the same bits"""
    with np.errstate(all='ignore'):
        return np.abs(np.asarray(m, dtype=np.float64) - rm) / rs


def ref_pvals(z):
    """stats.norm.cdf(-z) * 2.0"""
    from scipy import special
    return special.ndtr(-np.asarray(z)) * 2.0


def ref_window(p, lag, final_clamp):
    """the reference's calc_window_fishers_method (lag > 0) and the de novo clamp"""
    from scipy import stats
    p = np.asarray(p, dtype=np.float64)
    out = p.copy()
    if lag > 0:
        width = 2 * lag + 1
        out = np.full(p.shape, np.nan)
        if p.shape[0] >= width:
            with np.errstate(invalid='ignore'):
                lp = np.log(np.maximum(p, SMALLEST_PVAL))
            ls = np.lib.stride_tricks.sliding_window_view(lp, width).sum(-1)
            with np.errstate(invalid='ignore'):
                out[lag:-lag] = stats.chi2.sf(ls * -2, width * 2)
    if final_clamp:
        with np.errstate(invalid='ignore'):
            out = np.maximum(out, SMALLEST_PVAL)
    return out


def exact_pvals(z):
    """erfc(z / sqrt 2) at 40 digits from the float64 z (mpf values, NaN kept as None)"""
    with mpmath.workdps(40):
        return [None if math.isnan(x) else mpmath.erfc(mpmath.mpf(float(x)) / mpmath.sqrt(2))
                for x in np.asarray(z, dtype=np.float64)]


def exact_given(p):
    """p-values given as input: exact as they stand (None for NaN)"""
    return [None if math.isnan(x) else mpmath.mpf(float(x)) for x in np.asarray(p, np.float64)]


def p_rel_bound(z):
    """relative error of the device's p = erfc(z * 0.7071...) against the exact one: x is
    rounded twice (the constant and the product, <= 1.5 u), and erfc's condition number is
    ~2 x^2, so 3 x^2 u; erfc itself <= 5 ulp (10 u).  Bound (4 x^2 + 16) u, x = z / sqrt 2."""
    x2 = np.asarray(z, dtype=np.float64) ** 2 / 2.0
    return (4.0 * x2 + 16.0) * U


def exact_window(p_exact, p_err, lag, final_clamp):
    """(value, relative bound) per position from exact p-values (mpf or None for NaN) and
    their relative error bounds p_err (0 for p-values given as input).
    A window's y = -sum log max(p, 1e-50) carries, per member, the member's relative error
    (the clamp only shrinks it) and log's 1 + 1 ulp of |log p| (2u|log p| on the device side
    against the exact one), and the sequential sum of `width` terms <= width u y.  Since
    |d log Q / dy| = p(k-1; y) / Q <= 1, those are Q's relative error, to which the
    chi-square evaluation adds chi2_bound(y)."""
    n = len(p_exact)
    vals, bounds = [None] * n, np.zeros(n)
    with mpmath.workdps(40):
        clamp = mpmath.mpf(SMALLEST_PVAL)
        if lag == 0:
            for i, p in enumerate(p_exact):
                if p is None:
                    continue
                vals[i] = max(p, clamp) if final_clamp else p
                bounds[i] = p_err[i]
            return vals, bounds
        width = 2 * lag + 1
        logs = [None if p is None else mpmath.log(max(p, clamp)) for p in p_exact]
        for i in range(lag, n - lag):
            win = logs[i - lag:i + lag + 1]
            if any(v is None for v in win):
                continue
            y = -mpmath.fsum(win)
            q = exact_chi2_sf_even(y, width)
            yf = float(y)
            b = sum(float(p_err[i - lag + j]) + 2.0 * U * abs(float(win[j]))
                    for j in range(width))
            bounds[i] = b + width * U * yf + chi2_bound(yf)
            vals[i] = max(q, clamp) if final_clamp else q
    return vals, bounds


def assert_window(got, vals, bounds):
    """device values against the exact path; returns the largest error / bound ratio"""
    worst = 0.0
    got = np.asarray(got)
    for i, (g, v) in enumerate(zip(got, vals)):
        if v is None:
            assert math.isnan(g), (i, g)
            continue
        assert not math.isnan(g), (i, v)
        fv = float(v)
        if v > TINY:
            err = abs(g - fv) / fv
            r = err / bounds[i] if err else 0.0
            assert r <= 1.0, (i, g, fv, bounds[i])
            worst = max(worst, r)
        else:
            assert g <= TINY * (1.0 + bounds[i]), (i, g, fv)
    return worst


# ---------------------------------------------------------------------------
# region counters
# ---------------------------------------------------------------------------
def region_counters(stats, pos, reg_start, reg_len, thresh, lower, stat_type, unmod=None,
                    mod=0.0):
    """collate_reg_stats + apply_per_read_thresh + calc_damp_fraction over the statistics whose
    position lies in [reg_start, reg_start + reg_len).  lower None (or NaN): no lower
    threshold; stat_type 0 = model_compare (|stat| >= thresh is valid), 1 = anything else.
    Returns dict(pos, frac, damp_frac, cov, valid_cov)."""
    stats, pos = np.asarray(stats, dtype=np.float64), np.asarray(pos, dtype=np.int64)
    if lower is not None and math.isnan(lower):
        lower = None
    keep = ~np.isnan(stats) & (pos >= reg_start) & (pos < reg_start + reg_len)
    stats, pos = stats[keep], pos[keep]
    order = np.argsort(pos, kind='stable')
    stats, pos = stats[order], pos[order]
    up = np.unique(pos)
    split = np.split(stats, np.nonzero(np.diff(pos))[0] + 1) if pos.shape[0] else []
    out = dict(pos=up, frac=[], damp_frac=[], cov=[], valid_cov=[])
    for base_stats in split:
        cov = base_stats.shape[0]
        if lower is not None:
            base_stats = base_stats[(base_stats <= lower) | (base_stats >= thresh)]
        elif stat_type == 0:
            base_stats = base_stats[np.abs(base_stats) >= thresh]
        valid = base_stats.shape[0]
        frac = (int(np.sum(base_stats >= thresh)) / valid) if valid else float('nan')
        out['cov'].append(cov)
        out['valid_cov'].append(valid)
        out['frac'].append(frac)
        if unmod is None or math.isnan(unmod):
            out['damp_frac'].append(float('nan'))
        else:
            with np.errstate(all='ignore'):
                non_mod = np.round(np.float64(frac) * np.float64(valid))
                out['damp_frac'].append(float((non_mod + unmod) / (valid + (unmod + mod))))
    for k in ('frac', 'damp_frac'):
        out[k] = np.array(out[k], dtype=np.float64)
    for k in ('cov', 'valid_cov'):
        out[k] = np.array(out[k], dtype=np.int64)
    return out


# ---------------------------------------------------------------------------
# seeded case families
# ---------------------------------------------------------------------------
def synthetic_tables(K, seed):
    """random canonical (means, sds) and alternative means / sds tables for k-mer width K;
    about one alternative level in eight equals the canonical one (the scaled score skips
    those terms)"""
    rs = np.random.RandomState(seed)
    n = 4 ** K
    means = rs.normal(0.0, 1.0, n)
    sds = rs.uniform(0.05, 0.4, n)
    alt = means[:, None] + rs.normal(0.0, 0.5, (n, K))
    same = rs.uniform(size=(n, K)) < 0.125
    alt[same] = np.broadcast_to(means[:, None], (n, K))[same]
    alt_sds = rs.uniform(0.05, 0.4, (n, K))
    return means, sds, alt, alt_sds


def alt_tables(kmer_ref):
    """(4^K, K) alternative means and sds of the synthetic 5mC model
    (synthetic.make_alt_kmer_ref(kmer_ref, 'C', seed=1)); NaN where a k-mer has no C there"""
    from tombo_b200 import synthetic as syn
    K = len(kmer_ref[0][0])
    alt, alt_sd = np.full((4 ** K, K), np.nan), np.full((4 ** K, K), np.nan)
    for km, pos, m, sd in syn.make_alt_kmer_ref(kmer_ref, 'C', seed=1):
        idx = 0
        for b in km:
            idx = idx * 4 + 'ACGT'.index(b)
        alt[idx, pos], alt_sd[idx, pos] = m, sd
    return alt, alt_sd


def llr_of_genome_read(norm_mean, genome_seq, read_start, kmer_ref, cpos, mode):
    """llr_reads for one resquiggled read given as its per-base means and the bases they
    belong to (the k-mer centres), as compute_alt_model_read_stats receives them"""
    from tombo_b200 import synthetic as syn
    K = len(kmer_ref[0][0])
    means, sds = syn.kmer_table(kmer_ref)
    alt, _ = alt_tables(kmer_ref)
    nb = norm_mean.shape[0]
    codes = np.concatenate([np.zeros(cpos, np.uint8), syn.seq_to_codes(genome_seq),
                            np.zeros(K - 1 - cpos, np.uint8)])
    return llr_reads(np.asarray(norm_mean, np.float64), np.array([0, nb]), codes,
                     np.array([0, codes.shape[0]]), np.array([read_start]), means, sds, alt,
                     K, cpos, 1, mode)


def llr_read_shapes(K, cpos, alt_code, rs):
    """(name, base codes of nb + K - 1 bases, nb) for the read shapes where the site loop
    and the per-read scan can go wrong.  Testable base i of a read is sequence code
    cpos + K - 1 + i."""
    def rand_seq(nb, avoid_alt=False):
        s = rs.randint(0, 4, nb + K - 1).astype(np.uint8)
        if avoid_alt:
            s[s == alt_code] = (alt_code + 1) % 4
        return s

    def with_alt_at(s, idx):
        s = s.copy()
        for i in idx:
            s[cpos + K - 1 + i] = alt_code
        return s
    cases = []
    for nb in sorted({0, 1, K - 1, 2 * (K - 1)}):       # nb <= 2 (K - 1): no site
        if nb <= 2 * (K - 1):
            cases.append(('no_testable_nb%d' % nb, rand_seq(nb), nb))
    nb = 2 * (K - 1) + 1                                   # exactly one testable base
    cases.append(('one_testable_alt', with_alt_at(rand_seq(nb), [0]), nb))
    cases.append(('one_testable_not_alt', rand_seq(nb, avoid_alt=True), nb))
    for tl in (255, 256, 257, 513):
        nb = tl + 2 * (K - 1)
        cases.append(('testable_%d' % tl, rand_seq(nb), nb))
        cases.append(('testable_%d_sites_at_ends' % tl,
                      with_alt_at(rand_seq(nb, avoid_alt=True), [0, tl - 1]), nb))
    nb = 40 + 2 * (K - 1)
    cases.append(('all_alt', np.full(nb + K - 1, alt_code, dtype=np.uint8), nb))
    cases.append(('no_alt', rand_seq(nb, avoid_alt=True), nb))
    return cases


def flatten(reads):
    """[(codes, means)] -> norm_mean, mean_off, seq, seq_off"""
    nm = np.concatenate([m for _, m in reads]) if reads else np.zeros(0)
    mo = np.concatenate([[0], np.cumsum([m.shape[0] for _, m in reads])]).astype(np.int64)
    sq = np.concatenate([c for c, _ in reads]).astype(np.uint8)
    so = np.concatenate([[0], np.cumsum([c.shape[0] for c, _ in reads])]).astype(np.int64)
    return nm, mo, sq, so
