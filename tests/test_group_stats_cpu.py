"""The numpy / scipy restatement that the level-test GPU sweeps compare against reproduces
the unmodified reference's goldens (tests/golden/group_stats.npz) without a GPU."""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_group_stats_gpu as g  # noqa: E402


def test_restatement_matches_reference_goldens():
    gold = np.load(g.GOLD)
    cases = [('A', (0, 1, 2, 4), (1, 5, 20)), ('B', (0, 1), (20,)), ('C', (1,), (20,))]
    n_cmp = 0
    for tag, fms, mins in cases:
        start = int(gold['%s_reg' % tag][0])
        for fm in fms:
            samp, ctrl = gold['%s_fm%d_samp' % (tag, fm)], gold['%s_fm%d_ctrl' % (tag, fm)]
            for mn in mins:
                for st in g.STATS:
                    key = '%s_%s_fm%d_m%d' % (tag, st, fm, mn)
                    want = g.restate_group(samp, ctrl, start - fm, fm, mn, st)
                    assert (want is not None) == bool(int(gold[key + '_n'])), key
                    if want is None:
                        continue
                    np.testing.assert_array_equal(want[1], gold[key + '_pos'])
                    np.testing.assert_array_equal(want[2], gold[key + '_cov'])
                    np.testing.assert_array_equal(want[3], gold[key + '_ccov'])
                    g.assert_stats(want[0], gold[key + '_stats'], st)
                    n_cmp += 1
    assert n_cmp > 50


def test_reads_ref_restatement_matches_reference_goldens():
    gold = np.load(g.GOLD)
    for fm in (0, 1):
        for mn in (1, 5):
            for e in (0, 1):
                key = 'ref_fm%d_m%d_e%d_p0' % (fm, mn, e)
                means, sds, cov = g.restate_ref(gold['ref_fm%d_levels' % fm], mn, bool(e))
                np.testing.assert_array_equal(means, gold[key + '_means'])
                np.testing.assert_array_equal(sds, gold[key + '_sds'])
                np.testing.assert_array_equal(cov, gold[key + '_cov'])


# ---------------------------------------------------------------------------
# special.cuh (built for the host from the same source) against scipy
# ---------------------------------------------------------------------------
def _special_lib():
    import ctypes as C
    path = os.path.join(os.path.dirname(g.REPO + '/'), 'tombo_b200', 'libtb2_special_host.so')
    lib = C.CDLL(path)
    for name, args in (('tb2_host_kolmogorov_sf', [C.c_double]),
                       ('tb2_host_t_two_sided_p', [C.c_double, C.c_double]),
                       ('tb2_host_chi2_sf_even', [C.c_double, C.c_int]),
                       ('tb2_host_div12', [C.c_uint64, C.c_uint64])):
        getattr(lib, name).restype = C.c_double
        getattr(lib, name).argtypes = args
    return lib


def _rel_err(got, want):
    keep = want > 1e-290
    return np.max(np.abs(got[keep] - want[keep]) / want[keep])


def test_kolmogorov_sf_matches_scipy_on_a_dense_grid():
    from scipy import special
    lib = _special_lib()
    ys = np.concatenate([np.linspace(1e-3, 30.0, 60001), [0.82, np.nextafter(0.82, 1.0)]])
    # and the arguments the KS p-value forms for n_s, n_c in 1..1e4 and every d = k / n_s
    ns = np.unique(np.round(np.logspace(0, 4, 40)).astype(int))
    for a in ns:
        for b in ns[::3]:
            en = np.sqrt(a * b / float(a + b))
            d = np.arange(1, a + 1, max(1, a // 50)) / a
            ys = np.concatenate([ys, (en + 0.12 + 0.11 / en) * d])
    got = np.array([lib.tb2_host_kolmogorov_sf(float(y)) for y in ys])
    assert _rel_err(got, special.kolmogorov(ys)) <= 1e-9


def test_student_t_matches_scipy_on_a_dense_grid():
    from scipy import special
    lib = _special_lib()
    dfs = np.unique(np.concatenate([np.arange(1, 40), np.round(np.logspace(1.6, np.log10(2e4), 50)),
                                    [2e4]]))
    ts = -np.concatenate([np.linspace(0.0, 40.0, 801), np.logspace(-8, -1, 15)])
    worst = 0.0
    for df in dfs:
        got = np.array([lib.tb2_host_t_two_sided_p(float(df), float(t)) for t in ts])
        want = 2.0 * special.stdtr(df, ts)
        for i in np.nonzero(np.abs(got - want) > 1e-9 * want)[0]:
            # scipy's stdtr loses digits for tiny |t| at df 1 (3e-9 at t = -1e-8); settle
            # those points with the exact regularised incomplete beta
            import mpmath
            mpmath.mp.dps = 40
            x = mpmath.mpf(df) / (df + mpmath.mpf(float(ts[i])) ** 2)
            want[i] = float(mpmath.betainc(mpmath.mpf(df) / 2, 0.5, 0, x, regularized=True))
        worst = max(worst, _rel_err(got, want))
    assert worst <= 1e-9, worst


def _old_chi2_sf_even(y, k):
    """the closed form exactly as the kernels evaluated it before the large-y branch"""
    term, s = 1.0, 1.0
    for i in range(1, k):
        term *= y / float(i)
        s += term
    return math.exp(-y) * s


def test_chi2_sf_even_matches_mpmath_on_every_window_width():
    """Q(k, y) = chi2.sf(2 y, 2 k) for every de novo / sample-compare width k = 1..129 and
    the widths of fm_offset up to 2^24, with y up to the width's maximum (every p at the
    1e-50 clamp, y = 115.13 k) and dense where the closed form hands over (700..750)."""
    import stats_cases as sc
    lib = _special_lib()
    ks = list(range(1, 130)) + [681, 701, 721, 801, 2001, 2 ** 15 + 1, 2 ** 20 + 1, 2 ** 25 + 1]
    worst, n_tiny, n_close = 0.0, 0, 0
    for k in ks:
        ymax = sc.Y_PER_CLAMPED_P * k
        ys = np.concatenate([np.linspace(0.0, ymax, 25), np.linspace(700.0, 750.0, 26),
                             [k - 1.0, float(k), k + 0.5, np.nextafter(700.0, 0.0)]])
        for y in np.unique(ys[ys <= ymax]):
            y = float(y)
            got = lib.tb2_host_chi2_sf_even(y, k)
            assert not math.isnan(got), (k, y)
            if y < 700.0 and k <= 2001:
                # unchanged below 700: same operations, same bits
                assert got == _old_chi2_sf_even(y, k), (k, y)
            want = sc.exact_chi2_sf_even(y, k)
            if want > 1e-300:
                err = abs(got - float(want)) / float(want)
                worst = max(worst, err / sc.chi2_bound(y))
                n_close += 1
            else:
                assert got <= 1e-300, (k, y, got)
                n_tiny += 1
    assert worst <= 1.0, worst
    assert n_close > 2000 and n_tiny > 1000


def test_div12_rounds_like_python():
    lib = _special_lib()
    rs = np.random.RandomState(5)
    tots = list(range(1, 20001)) + [int(x) for x in rs.randint(1, 2 ** 62, 20000, dtype=np.int64)]
    tots += [2 ** 26, 94906265, 94906266, 2 ** 31 - 1, 2 ** 40 + 7]
    for tot in tots:
        p = tot * (tot + 1)
        assert lib.tb2_host_div12(p >> 64, p & (2 ** 64 - 1)) == p / 12, tot
