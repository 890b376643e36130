"""level_sample_compare (KS / U / t) and get_reads_ref on the device against the unmodified
reference's results (tests/golden/group_stats.npz, make_group_golden.py) and against an
in-file numpy / scipy restatement on seeded sweeps."""
import os
import sys

import numpy as np
import pytest
from scipy import special, stats

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from tombo_b200 import _lib, tombo_stats as ts, tombo_helper as th  # noqa: E402
from tombo_b200 import synthetic as syn  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(REPO, 'tests', 'golden', 'group_stats.npz')
STATS = ('ks_test', 'u_test', 't_test', 'ks_stat_test', 'u_stat_test', 't_stat_test')
P_RTOL = 1e-7


class Region(object):
    """intervalData stand-in: get_base_levels serves a stored positions x reads matrix for
    the widened region, or builds one from genome-ordered reads"""

    def __init__(self, start, end, levels=None, reads=None, seq=None, strand=None):
        self.chrm, self.strand, self.start, self.end = 'chr', strand, start, end
        self.levels, self.reads, self.seq_src = levels, reads, seq

    def copy(self):
        return Region(self.start, self.end, self.levels, self.reads, self.seq_src, self.strand)

    def update(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)
        return self

    def add_seq(self):
        self.seq = self.seq_src[self.start:self.end]
        return self

    def get_base_levels(self):
        if self.levels is not None:
            return self.levels[(self.start, self.end)]
        m = np.full((self.end - self.start, len(self.reads)), np.nan)
        for j, (a, lv) in enumerate(self.reads):
            lo, hi = max(a, self.start), min(a + lv.shape[0], self.end)
            if hi > lo:
                m[lo - self.start:hi - self.start, j] = lv[lo - a:hi - a]
        return m


# ---------------------------------------------------------------------------
# restatement of tombo_stats.py:2252-2287, 4236-4393 (tie rule: sample before control)
# ---------------------------------------------------------------------------
def pos_stat(s, c, stat_type):
    s, c = np.sort(s), np.sort(c)
    ns, nc = s.shape[0], c.shape[0]
    if stat_type.startswith('ks'):
        al = np.concatenate([s, c])
        d = np.max(np.abs(np.searchsorted(s, al, 'right') / ns -
                          np.searchsorted(c, al, 'right') / nc))
        if stat_type == 'ks_stat_test':
            return 1 - d
        en = np.sqrt(ns * nc / float(ns + nc))
        return special.kolmogorov((en + 0.12 + 0.11 / en) * d)
    if stat_type.startswith('u'):
        tot = ns * nc
        ranks = np.empty(ns + nc, int)
        ranks[np.concatenate([s, c]).argsort(kind='stable')] = np.arange(1, ns + nc + 1)
        u1 = ranks[:ns].sum() - (ns * (ns + 1)) / 2
        u = min(u1, tot - u1)
        mu = tot / 2
        if stat_type == 'u_stat_test':
            return (u - mu) / mu
        return special.ndtr((u - mu) / np.sqrt(tot * (tot + 1) / 12)) * 2.0

    def mean_sd(v):
        m = 0.0
        for x in v:
            m += x
        m /= v.shape[0]
        var = 0.0
        for x in v:
            var += (x - m) ** 2
        return m, np.sqrt(var / v.shape[0])
    sm, ssd = mean_sd(s)
    cm, csd = mean_sd(c)
    with np.errstate(all='ignore'):
        if stat_type == 't_stat_test':
            den = np.sqrt(((ssd ** 2) + (csd ** 2)) / 2)
            return -np.abs(sm - cm) / den if den > 0 else np.nan
        if ns + nc <= 2:
            return np.nan
        sp = np.sqrt((((ns - 1) * (ssd ** 2)) + (nc - 1) * (csd ** 2)) / (ns + nc - 2))
        if not sp > 0:
            return np.nan
        t = -np.abs(sm - cm) / (sp * np.sqrt((1 / ns) + (1 / nc)))
        return special.stdtr(ns + nc - 2, t) * 2.0


def windowed(v, lag, pvals):
    out = np.full(v.shape, np.nan)
    win = np.lib.stride_tricks.sliding_window_view
    with np.errstate(all='ignore'):
        if pvals:
            ls = win(np.log(np.maximum(v, 1e-50)), 2 * lag + 1).sum(-1)
            out[lag:-lag] = stats.chi2.sf(ls * -2, (2 * lag + 1) * 2)
        else:
            out[lag:-lag] = np.mean(win(v, 2 * lag + 1), -1)
    return out


def restate_group(samp, ctrl, start, fm, mn, stat_type):
    vs, vc = ~np.isnan(samp), ~np.isnan(ctrl)
    cs, cc = vs.sum(1), vc.sum(1)
    ok = np.concatenate([[False], (cs >= mn) & (cc >= mn), [False]])
    edges = np.nonzero(np.diff(ok))[0]
    res = [[], [], [], []]
    for a, b in zip(edges[::2], edges[1::2]):
        if b - a < 2 * fm + 1:
            continue
        v = np.array([pos_stat(samp[i][vs[i]], ctrl[i][vc[i]], stat_type) for i in range(a, b)])
        if fm > 0:
            v = windowed(v, fm, not stat_type.endswith('stat_test'))
        for lst, x in zip(res, (v, np.arange(start + a, start + b), cs[a:b], cc[a:b])):
            lst.append(x)
    if not res[0]:
        return None
    return [np.concatenate(x) for x in res]


# The reference squares standard deviations with C pow(x, 2.0) (c_mean_std, and
# `samp_sd ** 2` on Python floats); glibc's pow is not correctly rounded and differs from
# x * x by one ulp for about 0.1 % of inputs.  The device squares with x * x, so
# t_stat_test values may differ from the reference in the last bit (rtol 2e-15).
T_STAT_RTOL = 2e-15


def stats_equal(got, want, stat_type):
    if stat_type == 't_stat_test':
        return np.allclose(got, want, rtol=T_STAT_RTOL, atol=0, equal_nan=True)
    if stat_type.endswith('stat_test'):
        return np.array_equal(got, want, equal_nan=True)
    return np.allclose(got, want, rtol=P_RTOL, atol=0, equal_nan=True)


def assert_stats(got, want, stat_type):
    if stat_type == 't_stat_test':
        np.testing.assert_allclose(got, want, rtol=T_STAT_RTOL, atol=0)
    elif stat_type.endswith('stat_test'):
        np.testing.assert_array_equal(got, want)
    else:
        np.testing.assert_allclose(got, want, rtol=P_RTOL, atol=0)
        assert np.array_equal(np.isnan(got), np.isnan(want))


def restate_ref(levels, mn, est_mean):
    """get_reads_ref :3644-3656 without the posterior (levels in column order)"""
    valid = ~np.isnan(levels)
    cov = valid.sum(1)
    means, sds = np.full(cov.shape[0], np.nan), np.full(cov.shape[0], np.nan)
    for i in np.nonzero(cov >= mn)[0]:
        b = levels[i][valid[i]]
        means[i] = np.mean(b) if est_mean else np.median(b)
        sds[i] = np.std(b)
    z = sds == 0
    means[z] = sds[z] = np.nan
    return means, sds, cov


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


# ---------------------------------------------------------------------------
def test_group_reg_stats_match_reference_goldens(gold):
    cases = [('A', (0, 1, 2, 4), (1, 5, 20)), ('B', (0, 1), (20,)), ('C', (1,), (20,))]
    n_cmp = 0
    for tag, fms, mins in cases:
        start, end = (int(x) for x in gold['%s_reg' % tag])
        for fm in fms:
            lv = {(start - fm, end + fm): gold['%s_fm%d_samp' % (tag, fm)]}
            lc = {(start - fm, end + fm): gold['%s_fm%d_ctrl' % (tag, fm)]}
            reg, creg = Region(start, end, lv), Region(start, end, lc)
            for mn in mins:
                for st in STATS:
                    key = '%s_%s_fm%d_m%d' % (tag, st, fm, mn)
                    res = ts.compute_group_reg_stats(reg, creg, fm, mn, st)
                    assert len(res) == int(gold[key + '_n']), key
                    if not res:
                        continue
                    name, g = res[0]
                    assert name == st and isinstance(g, th.groupStats)
                    assert (g.chrm, g.strand, g.start) == ('chr', None, start)
                    np.testing.assert_array_equal(g.reg_poss, gold[key + '_pos'], err_msg=key)
                    np.testing.assert_array_equal(g.reg_cov, gold[key + '_cov'], err_msg=key)
                    np.testing.assert_array_equal(g.ctrl_cov, gold[key + '_ccov'], err_msg=key)
                    assert_stats(g.reg_stats, gold[key + '_stats'], st)
                    n_cmp += 1
    assert n_cmp > 50
    # the extreme tails are covered
    assert np.nanmin(gold['B_ks_test_fm0_m20_stats']) < 1e-100
    assert np.nanmin(gold['B_t_test_fm0_m20_stats']) < 1e-100


def test_reads_ref_matches_reference_goldens(gold):
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    genome = str(gold['genome'])
    for fm in (0, 1):
        levels = {(1000 - fm, 1200 + fm): gold['ref_fm%d_levels' % fm]}
        for mn in (1, 5):
            for e in (0, 1):
                for p in (0, 1):
                    key = 'ref_fm%d_m%d_e%d_p%d' % (fm, mn, e, p)
                    reg = Region(1000, 1200, levels, seq=genome)
                    means, sds, cov = ts.get_reads_ref(reg, mn, fm, std_ref if p else None,
                                                       None, bool(e))
                    np.testing.assert_array_equal(means, gold[key + '_means'], err_msg=key)
                    np.testing.assert_array_equal(sds, gold[key + '_sds'], err_msg=key)
                    np.testing.assert_array_equal(sorted(cov), gold[key + '_covpos'])
                    np.testing.assert_array_equal([cov[k] for k in sorted(cov)], gold[key + '_cov'])


def test_reads_ref_posterior_on_both_strands_matches_reference(gold):
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    genome = str(gold['genome'])
    assert 'NN' in genome[1000:1200]                 # the expected-level gap branch is hit
    for strand, name in (('+', 'plus'), ('-', 'minus')):
        for fm in (0, 1):
            key = 'refs_%s_fm%d' % (name, fm)
            levels = {(1000 - fm, 1200 + fm): gold[key + '_levels']}
            reg = Region(1000, 1200, levels, seq=genome, strand=strand)
            means, sds, cov = ts.get_reads_ref(reg, 1, fm, std_ref)
            np.testing.assert_array_equal(means, gold[key + '_means'], err_msg=key)
            np.testing.assert_array_equal(sds, gold[key + '_sds'], err_msg=key)
            np.testing.assert_array_equal([cov[k] for k in sorted(cov)], gold[key + '_cov'])
            assert np.isnan(gold[key + '_means']).any()


def random_region(rs, n_pos, n_reads, start, shift=0.0, integer=False):
    reads = []
    for _ in range(n_reads):
        a = int(rs.randint(start - 10, start + n_pos - 5))
        ln = int(rs.randint(5, n_pos + 20))
        lv = rs.normal(shift, 1.0, ln)
        if integer:
            lv = np.round(lv * 2.0)
        lv[rs.uniform(size=ln) < 0.05] = np.nan
        reads.append((a, lv))
    return Region(start, start + n_pos, reads=reads)


def test_sweep_matches_restatement():
    rs = np.random.RandomState(20261015)
    for k in range(64):
        n_pos = int(rs.randint(20, 80))
        start = int(rs.randint(0, 10 ** 6))
        reg = random_region(rs, n_pos, int(rs.randint(3, 40)), start, rs.uniform(0, 1))
        creg = random_region(rs, n_pos, int(rs.randint(3, 40)), start)
        mn = int(rs.randint(1, 6))
        for fm in (0, 1, 2):
            samp = reg.copy().update(start=start - fm, end=start + n_pos + fm).get_base_levels()
            ctrl = creg.copy().update(start=start - fm, end=start + n_pos + fm).get_base_levels()
            for st in STATS:
                want = restate_group(samp, ctrl, start - fm, fm, mn, st)
                res = ts.compute_group_reg_stats(reg, creg, fm, mn, st)
                if want is None:
                    assert res == [], (k, fm, st)
                    continue
                g = res[0][1]
                np.testing.assert_array_equal(g.reg_poss, want[1])
                np.testing.assert_array_equal(g.reg_cov, want[2])
                np.testing.assert_array_equal(g.ctrl_cov, want[3])
                assert_stats(g.reg_stats, want[0], st)


def test_u_ties_follow_the_stable_rule():
    rs = np.random.RandomState(7)
    samp = np.round(rs.normal(0.3, 1.0, (50, 30)) * 2.0)
    ctrl = np.round(rs.normal(0.0, 1.0, (50, 25)) * 2.0)
    for rstat in (False, True):
        got = ts.compute_u_tests(samp, ctrl, rstat)
        st = 'u_stat_test' if rstat else 'u_test'
        want = np.array([pos_stat(samp[i], ctrl[i], st) for i in range(50)])
        assert_stats(got, want, st)


def test_coverage_beyond_shared_memory():
    rs = np.random.RandomState(11)
    n = 4000                            # 8000 levels at one position: the global-memory path
    samp = np.vstack([rs.normal(0.05, 1.0, n), rs.normal(0.0, 1.0, n)])
    ctrl = np.vstack([rs.normal(0.0, 1.0, n), rs.normal(0.0, 1.0, n)])
    for st in STATS:
        fn = {'ks': ts.compute_ks_tests, 'u_': ts.compute_u_tests, 't_': ts.compute_t_tests}[st[:2]]
        got = fn(samp, ctrl, st.endswith('stat_test'))
        want = np.array([pos_stat(samp[i], ctrl[i], st) for i in range(2)])
        assert_stats(got, want, st)
    # get_reads_ref with more reads than the shared buffer holds
    lv = rs.normal(0.0, 1.0, (3, 2500))
    reg = Region(0, 3, {(0, 3): lv})
    means, sds, _ = ts.get_reads_ref(reg, 1, 0)
    wm, ws, _ = restate_ref(lv, 1, False)
    np.testing.assert_array_equal(means, wm)
    np.testing.assert_array_equal(sds, ws)


def test_p_values_at_large_coverage_match_scipy():
    # 10 000 reads per sample (t with 19 998 degrees of freedom, KS with en ~ 70): the device's
    # Kolmogorov and Student-t functions against scipy at rtol 1e-9
    rs = np.random.RandomState(21)
    shifts = np.array([0.0, 0.005, 0.01, 0.02, 0.03, 0.05, 0.08, 0.12, 0.2, 0.3, 0.4, 0.5])
    samp = rs.normal(0.0, 1.0, (shifts.shape[0], 10000)) + shifts[:, None]
    ctrl = rs.normal(0.0, 1.0, (shifts.shape[0], 10000))
    for fn, st in ((ts.compute_t_tests, 't_test'), (ts.compute_ks_tests, 'ks_test')):
        got = fn(samp, ctrl, False)
        want = np.array([pos_stat(samp[i], ctrl[i], st) for i in range(shifts.shape[0])])
        assert want.min() < 1e-100
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=0)


def test_reads_ref_follows_read_order():
    rs = np.random.RandomState(3)
    lv = rs.normal(0.0, 1.0, (40, 300))
    lv[rs.uniform(size=lv.shape) < 0.1] = np.nan
    for perm in (np.arange(300), rs.permutation(300), rs.permutation(300)):
        m = lv[:, perm]
        for est_mean in (False, True):
            means, sds, cov = ts.get_reads_ref(Region(0, 40, {(0, 40): m}), 3, 0,
                                               est_mean=est_mean)
            wm, ws, wc = restate_ref(m, 3, est_mean)
            np.testing.assert_array_equal(means, wm)
            np.testing.assert_array_equal(sds, ws)
            assert [cov[k] for k in range(40)] == list(wc)


def test_zero_variance_and_empty_positions_are_nan():
    samp = np.array([[1.0, 1.0, 1.0], [np.nan, np.nan, np.nan], [1.0, 2.0, 3.0], [5.0, np.nan, np.nan]])
    ctrl = np.array([[1.0, 1.0, np.nan], [0.0, 1.0, 2.0], [np.nan] * 3, [4.0, np.nan, np.nan]])
    for rstat in (False, True):
        t = ts.compute_t_tests(samp, ctrl, rstat)
        assert np.isnan(t).all()                     # zero variance, empty, empty, 1 + 1 levels
        for fn in (ts.compute_ks_tests, ts.compute_u_tests):
            v = fn(samp, ctrl, rstat)
            assert np.isnan(v[1]) and np.isnan(v[2]) and not np.isnan(v[0])
    lv = np.array([[2.0, 2.0, 2.0], [1.0, 2.0, np.nan], [np.nan] * 3])
    means, sds, cov = ts.get_reads_ref(Region(0, 3, {(0, 3): lv}), 1, 0)
    assert np.isnan(means[0]) and np.isnan(sds[0])    # sd == 0
    assert means[1] == 1.5 and sds[1] == 0.5
    assert np.isnan(means[2]) and cov == {0: 3, 1: 2, 2: 0}


def test_invalid_arguments_are_rejected():
    ctx = _lib.get_context()
    r = (np.zeros(3), np.array([0, 3]), np.array([0]))
    for kw in (dict(min_test_reads=0, reg_len=10), dict(min_test_reads=1, reg_len=(1 << 24) + 1),
               dict(min_test_reads=1, reg_len=0)):
        with pytest.raises(_lib.TomboB200Error, match=r'\(201\)'):
            ctx.group_reg_stats(0, kw['reg_len'], r, r, 0, False, kw['min_test_reads'], 0)
    with pytest.raises(_lib.TomboB200Error, match=r'\(201\)'):
        ctx.reads_ref_levels(0, 10, r, 0)
    with pytest.raises(_lib.TomboB200Error, match=r'\(201\)'):
        ctx.reads_ref_levels(0, (1 << 24) + 1, r, 1)
