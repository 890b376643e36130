"""Theil-Sen test cases (a plain helper module, imported by test_theil_sen_cpu.py and
test_theil_sen_gpu.py).

* `theil_sen` restates calc_kmer_fitted_shift_scale(method='theil_sen') (tombo_stats.py:401-450
  with c_compute_slopes, _c_helper.pyx:362-377) literally in numpy: every pairwise slope, two
  np.median calls, the zero-slope error and the correction factors.  It shares no code with the
  C oracle or the kernel; only the keyed sub-sample of reads above 1000 points comes from
  `oracle.perm_index`, the draw the library pins in place of np.random.choice.
* Seeded case families that drive k_theil_sen (tombo_b200/csrc/stage_kernels.cuh) down each of
  its selection paths.  A case carries the debug-counter slots (`tb2_debug_counters`) its call
  must move: `expected_path` is the set of slots [1]-[6] that move, or None where the path is not
  fixed by how the case was built.  Paths [1] and [4] are entered after a decision on sampled
  fp32 slopes, and the device's approximate fp32 divide can move a sample into another bin, so
  cases that declare them are pinned on the host emulation only (`emul_only`).
"""
import collections

import numpy as np

import oracle

MAX_POINTS = 1000            # MAX_POINTS_FOR_THEIL_SEN
MAX_SLOPE = 1000.0           # c_compute_slopes' value for a pair of equal event means
OK = 0
ERR_THEIL_SEN_ZERO = 20      # TB2_ERR_THEIL_SEN_ZERO (include/tombo_b200.h)
ZERO_SLOPE_MESSAGE = 'Read failed sequence-based signal re-scaling parameter estimation.'

# g_tb2_counters slots (include/tombo_b200.h)
READS, FP32_ALL, HISTOGRAM, GENERIC, FP32_SAMPLED, SWEEP, SWEEP_ABANDONED = range(7)
PATH_SLOTS = (FP32_ALL, HISTOGRAM, GENERIC, FP32_SAMPLED, SWEEP, SWEEP_ABANDONED)

Case = collections.namedtuple(
    'Case', 'ev md prev_shift prev_scale key expected_path name emul_only')


# ------------------------------------------------------------------ the restatement
def subsample(ev, md, key):
    """the 1000 points a longer read keeps (tombo_stats.py:411-416, keyed draw)"""
    n = ev.shape[0]
    if n <= MAX_POINTS:
        return ev, md
    idx = np.array([oracle.perm_index(i, n, key) for i in range(MAX_POINTS)], dtype=np.int64)
    return ev[idx], md[idx]


def slopes(ev, md):
    """c_compute_slopes: pairs in combinations(range(n), 2) order (np.triu_indices is that
    order), (md_i - md_j) / (ev_i - ev_j), and 1000.0 where ev_i == ev_j"""
    i, j = np.triu_indices(ev.shape[0], 1)
    with np.errstate(divide='ignore', invalid='ignore'):
        q = (md[i] - md[j]) / (ev[i] - ev[j])
    return np.where(ev[i] == ev[j], MAX_SLOPE, q)


def theil_sen(prev_shift, prev_scale, ev, md, key=0):
    """-> (status, (shift, scale, shift_corr, scale_corr)); the outputs are None on error"""
    ev = np.ascontiguousarray(ev, dtype=np.float64)
    md = np.ascontiguousarray(md, dtype=np.float64)
    ev, md = subsample(ev, md, key)
    # the reference runs under np.seterr(all='raise') (tombo_helper.py:18)
    with np.errstate(all='raise'):
        slope = np.median(slopes(ev, md))
        inter = np.median(md - (slope * ev))
        if slope == 0:
            return ERR_THEIL_SEN_ZERO, None
        scale_corr = 1 / slope
        shift_corr = -inter / slope
        shift = prev_shift + (shift_corr * prev_scale)
        scale = prev_scale * scale_corr
    return OK, (float(shift), float(scale), float(shift_corr), float(scale_corr))


def middle_slopes(ev, md, key=0):
    """the order statistics np.median averages: (rank k1, rank k1 + 1) for an even number of
    slopes, (rank k1, None) for an odd one"""
    ev, md = subsample(np.asarray(ev, np.float64), np.asarray(md, np.float64), key)
    s = np.sort(slopes(ev, md))
    k1 = (s.shape[0] - 1) // 2
    return (float(s[k1]), float(s[k1 + 1])) if s.shape[0] % 2 == 0 else (float(s[k1]), None)


# ------------------------------------------------------------------ input families
# Each family is f(rs, n) -> (ev, md, expected_path); the path only where the construction
# fixes it.  n is the number of points before sub-sampling.
def _small_n_path(n):
    # fewer than 16 bracket samples (n < 32): generic select; below 128 points no sort-and-sweep
    return (GENERIC,) if n < 32 else (HISTOGRAM,) if n < 128 else None


def smooth(rs, n):
    """the rescaling's usual input: model levels against a noisy affine image of them"""
    md = rs.normal(0, 1.4826, n)
    ev = (md - 0.07) / 1.06 + rs.normal(0, 0.15, n)
    return ev, md, _small_n_path(n) or (SWEEP,)


def near_collinear(rs, n):
    """md = ev + 1e-9 noise: every gap is inside the sort-and-sweep guard and the fp32 screen,
    so both give up and the exact histogram finishes"""
    ev = rs.normal(0, 1.5, n)
    md = ev + 1e-9 * rs.normal(0, 1, n)
    return ev, md, _small_n_path(n) or (SWEEP_ABANDONED, HISTOGRAM)


def cauchy(rs, n):
    """Cauchy-distributed event means: slopes all over the place, any path may finish"""
    md = rs.normal(0, 1.4826, n)
    ev = rs.standard_cauchy(n)
    return ev, md, _small_n_path(n)


def _exact_line(rs, n):
    # distinct points on a binary grid on the line md = 1.5 ev + 0.25: every slope between
    # two of them is exactly 1.5
    ev = (rs.permutation(8 * n)[:n] - 4 * n) * 0.25
    return ev, ev * 1.5 + 0.25


def outliers(rs, n):
    """30 % outliers on exactly linear points: half of all slopes tie at 1.5, the median among
    them -- too many for the pair list and for the histogram's median bins"""
    ev, md = _exact_line(rs, n)
    k = max(1, (3 * n) // 10)
    idx = rs.choice(n, k, replace=False)
    md[idx] = rs.normal(0, 0.5 * n, k)
    # below 128 points every decision is on fp64 values: the tie block holds the 30th and 70th
    # percentile bracket samples (hi == lo).  From 200 points on the tied pairs overflow the
    # pair list, the fp32 bracket buffer and the histogram's median bins
    return ev, md, (GENERIC,) if n < 128 else (SWEEP_ABANDONED, GENERIC) if n >= 200 else None


def steep(rs, n):
    """true slopes near 5000, event means on a 1/64 grid: the equal-ev value 1000.0 sits below
    the median, sort-and-sweep is skipped (hi >= 1000) and the fp32 queue overflows"""
    ev = np.round(rs.normal(0, 1, n) * 64) / 64
    md = 5000.0 * ev + rs.normal(0, 1, n)
    return ev, md, _small_n_path(n) or (HISTOGRAM,)


def tie_groups(rs, n):
    """many groups of equal event means (slope 1000.0 inside each group)"""
    ev = rs.randint(0, max(2, n // 6), size=n) * 0.125
    md = 0.9 * ev + rs.normal(0, 0.3, n)
    return ev, md, _small_n_path(n)


def all_equal_ev(rs, n):
    """every event mean equal: every slope is exactly 1000.0"""
    ev = np.full(n, 0.6180339887)
    md = rs.normal(0, 1, n)
    return ev, md, (GENERIC,)


def int16_levels(rs, n):
    """means of 5-12 integer samples, then an affine map (the int16 DAC dtype): exact ties"""
    md = rs.normal(0, 1.0, n)
    cnt = rs.randint(5, 13, size=n)
    tot = np.round((md * 80 + 400) * cnt + rs.normal(0, 12, n) * np.sqrt(cnt))
    ev = ((tot / cnt) - 400.0) / 80.0
    ev[rs.randint(0, n, size=n // 10)] = ev[rs.randint(0, n, size=n // 10)]
    return ev, md, _small_n_path(n) or (SWEEP,)


def duplicate_points(rs, n):
    """smooth data with a tenth of the points repeated exactly (equal ev and equal md): such a
    pair has slope 1000.0 and a zero Q gap at every threshold, which sort-and-sweep must exempt
    from its guard rather than abandon"""
    ev, md, path = smooth(rs, n)
    k = max(1, n // 10)
    src, dst = rs.randint(0, n, size=k), rs.randint(0, n, size=k)
    ev[dst], md[dst] = ev[src], md[src]
    return ev, md, path


def coarse_grid(rs, n):
    """a 6 x 5 integer grid: thousands of slopes tie exactly at the median"""
    ev = rs.randint(0, 6, size=n).astype(np.float64)
    md = ev + rs.randint(-2, 3, size=n)
    return ev, md, (SWEEP_ABANDONED, GENERIC) if n >= 200 else None


def constant_md(rs, n):
    """md constant: the median slope is 0, the reference raises"""
    ev = rs.normal(0, 1.5, n)
    md = np.full(n, 0.75)
    return ev, md, (GENERIC,)


FAMILIES = collections.OrderedDict([
    ('smooth', smooth), ('near_collinear', near_collinear), ('cauchy', cauchy),
    ('outliers', outliers), ('steep', steep), ('tie_groups', tie_groups),
    ('all_equal_ev', all_equal_ev), ('int16_levels', int16_levels),
    ('duplicate_points', duplicate_points),
    ('coarse_grid', coarse_grid), ('constant_md', constant_md)])

SIZES = (2, 3, 17, 31, 32, 33, 127, 128, 129, 181, 182, 183, 720, 721, 999, 1000)
SUBSAMPLED_SIZES = (1001, 1024, 1025, 4097, 65536, 65537, 200003)
RESCALE_EXPONENTS = (-140, -60, -20, 20, 60, 130)


def _case(name, fam, rs, n, key=0, prev=(0.1, 1.2)):
    ev, md, path = fam(rs, n)
    return Case(ev, md, prev[0], prev[1], key, path, name, False)


def size_cases():
    """every size boundary of the kernel, smooth data; at each size the outlier mixture too,
    whose two middle slopes (when the count is even) tie"""
    out = []
    for n in SIZES:
        out.append(_case('smooth_n%d' % n, smooth, np.random.RandomState(n), n))
        if n >= 3:
            out.append(_case('tied_middle_n%d' % n, outliers, np.random.RandomState(10000 + n), n))
    return out


def family_cases():
    out = []
    for fname, fam in FAMILIES.items():
        for q, n in enumerate((40, 300, 1000)):
            out.append(_case('family_%s_n%d' % (fname, n), fam, np.random.RandomState(100 * q + len(fname)), n,
                             key=q, prev=(0.3 * q, 1.0 + 0.25 * q)))
    return out


def rescaled_cases():
    """exact power-of-two rescalings of one smooth read: the fp32 images of the points overflow
    or go subnormal, the slopes stay the same doubles.  prev_shift is 0, so every output of
    exponent k is the k = 0 output times 2^k (shift, shift_corr) or unchanged (scale,
    scale_corr) -- see `rescale_expectation`."""
    base = _case('rescaled_base', smooth, np.random.RandomState(77), 500, prev=(0.0, 1.0))
    out = [base]
    for k in RESCALE_EXPONENTS:
        # 2^20, 2^60: the same path as the base read.  2^-60, 2^-140: every gap is inside the
        # guards (both floor M at 1); 2^130: no fp32 image is finite.  2^-20 abandons sort-and-
        # sweep on a sampled decision: pinned on the emulation only
        path = (SWEEP,) if k > 0 and k != 130 else (SWEEP_ABANDONED, HISTOGRAM)
        out.append(base._replace(ev=np.ldexp(base.ev, k), md=np.ldexp(base.md, k),
                                 expected_path=path, name='rescaled_2^%d' % k, emul_only=k == -20))
    return out


def rescale_expectation(base_out, k):
    """outputs of the 2^k-rescaled read from the base read's outputs (prev_shift 0, scale 1)"""
    shift, scale, shc, scc = base_out
    return (float(np.ldexp(shift, k)), scale, float(np.ldexp(shc, k)), scc)


def subsampled_cases():
    out = []
    for n in SUBSAMPLED_SIZES:
        rs = np.random.RandomState(n % 100003)
        ev, md, _ = smooth(rs, n)
        for key in (0, 12345, 0xDEADBEEF):
            out.append(Case(ev, md, 0.2, 1.1, key, (SWEEP,), 'subsampled_n%d_key%d' % (n, key), False))
    return out


def fp32_cases():
    """heavy-tailed reads that, on the host emulation, abandon sort-and-sweep and finish on
    the fp32 bracket: over sampled pairs [4] (n <= 720) and over every pair [1] (n >= 721).
    Found by a seeded search; the device may finish them on another path."""
    out = []
    for name, n, seed, path in FP32_FINDS:
        ev, md, _ = cauchy(np.random.RandomState(seed), n)
        out.append(Case(ev, md, 0.0, 1.0, 0, path, name, True))
    return out


# (name, n, seed of `cauchy`, path on the emulation)
FP32_FINDS = (('fp32_sampled_n600', 600, 272, (FP32_SAMPLED, SWEEP_ABANDONED)),
              ('fp32_sampled_n700', 700, 174, (FP32_SAMPLED, SWEEP_ABANDONED)),
              ('fp32_sampled_n720', 720, 211, (FP32_SAMPLED, SWEEP_ABANDONED)),
              ('fp32_retry_n600', 600, 245, (FP32_ALL, SWEEP_ABANDONED)),   # sampled bracket missed
              ('fp32_all_n721', 721, 203, (FP32_ALL, SWEEP_ABANDONED)),
              ('fp32_all_n1000', 1000, 170, (FP32_ALL, SWEEP_ABANDONED)))


def all_cases():
    return size_cases() + family_cases() + rescaled_cases() + subsampled_cases() + fp32_cases()


def random_case(rs):
    """one case of the seeded sweep: a random family, size and key; no declared path.  A third
    of the cases are Cauchy reads of 182-1000 points, the only family that reaches the fp32
    paths [1] and [4] (and those only now and then)"""
    fam = list(FAMILIES.values())[rs.randint(len(FAMILIES))]
    u = rs.rand()
    if rs.rand() < 0.3:
        fam, n = cauchy, int(rs.randint(182, 1001))
    elif u < 0.1:
        n = int(rs.randint(2, 128))
    elif u < 0.9:
        n = int(rs.randint(128, 1001))
    else:
        n = int(rs.randint(1001, 5000))
    key = int(rs.randint(0, 1 << 32, dtype=np.uint64))
    ev, md, _ = fam(rs, n)
    if rs.rand() < 0.1:
        k = int(rs.choice(RESCALE_EXPONENTS))
        ev, md = np.ldexp(ev, k), np.ldexp(md, k)
    return Case(ev, md, float(rs.normal(0, 1)), float(rs.uniform(0.5, 2)), key, None,
                '%s_n%d' % (fam.__name__, n), False)
