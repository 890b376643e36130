"""GPU parity of the non-DP stage kernels (through the C ABI) against the C oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _sig(seed, n, int16=False):
    rs = np.random.RandomState(seed)
    nb = max(4, n // 9)
    lev = np.repeat(rs.normal(0, 1.4826, nb), 3 + rs.geometric(1 / 6.0, nb))[:n]
    if lev.shape[0] < n:
        lev = np.concatenate([lev, np.zeros(n - lev.shape[0])])
    raw = (lev + 0.2 * rs.normal(0, 1, n)) * 60.0 + 480.0
    if int16:
        raw = np.round(raw)
    return raw


@pytest.mark.parametrize('seed,n', [(1, 4301), (2, 4000), (3, 257), (4, 20011), (5, 50)])
def test_normalize_bit_exact(ctx, orc, seed, n):
    raw = _sig(seed, n, int16=(seed % 2 == 0))
    s0, n0, sv0 = orc.normalize_raw_signal(raw, outlier_thresh=5.0)
    s1, n1, sv1 = ctx.normalize_raw_signal(raw, outlier_thresh=5.0)
    assert s0 == s1 == 0
    assert np.array_equal(n0, n1)
    assert sv0[:4] == sv1[:4]
    # provided scale values (iterations >= 2)
    sv_in = (sv0[0] + 1.5, sv0[1] * 1.07, sv0[2], sv0[3], 5.0)
    s0, n0, sv0b = orc.normalize_raw_signal(raw, scale_values=sv_in)
    s1, n1, sv1b = ctx.normalize_raw_signal(raw, scale_values=sv_in)
    assert s0 == s1 == 0
    assert np.array_equal(n0, n1)
    assert sv0b[:4] == sv1b[:4]
    # no winsorising
    s0, n0, _ = orc.normalize_raw_signal(raw)
    s1, n1, _ = ctx.normalize_raw_signal(raw)
    assert np.array_equal(n0, n1)
    # constant scale
    s0, n0, sv0c = orc.normalize_raw_signal(raw, outlier_thresh=5.0, const_scale=55.0)
    s1, n1, sv1c = ctx.normalize_raw_signal(raw, outlier_thresh=5.0, const_scale=55.0)
    assert np.array_equal(n0, n1) and sv0c[:4] == sv1c[:4]


def test_normalize_constant_signal_fails_like_reference(ctx, orc):
    raw = np.full(300, 480.0)
    s0, _, _ = orc.normalize_raw_signal(raw, outlier_thresh=5.0)
    s1, _, _ = ctx.normalize_raw_signal(raw, outlier_thresh=5.0)
    assert s0 == s1 == 100


@pytest.mark.parametrize('seed,n,int16', [(1, 4301, False), (2, 4000, True), (3, 400, False),
                                          (4, 20011, False), (5, 9000, True)])
def test_valid_cpts_w_cap_bit_exact(ctx, orc, seed, n, int16):
    raw = _sig(seed, n, int16)
    _, norm, _ = orc.normalize_raw_signal(raw, outlier_thresh=5.0)
    for num in (n // 5, max(2, n // 9), 1):
        s0, c0 = orc.valid_cpts_w_cap(norm, 3, 5, num)
        s1, c1 = ctx.valid_cpts_w_cap(norm, 3, 5, num)
        assert s0 == s1, (s0, s1, num)
        if s0 == 0:
            assert np.array_equal(c0, c1)
    # too many requested -> same failure
    s0, _ = orc.valid_cpts_w_cap(norm, 3, 5, n // 3)
    s1, _ = ctx.valid_cpts_w_cap(norm, 3, 5, n // 3)
    assert s0 == s1 != 0


@pytest.mark.parametrize('seed,n', [(11, 8000), (12, 3000)])
def test_valid_cpts_t_test_bit_exact(ctx, orc, seed, n):
    raw = _sig(seed, n)
    for num in (n // 15, n // 40):
        s0, c0 = orc.valid_cpts_w_cap(raw, 6, 12, num, t_test=True)
        s1, c1 = ctx.valid_cpts_w_cap(raw, 6, 12, num, t_test=True)
        assert s0 == s1
        if s0 == 0:
            assert np.array_equal(c0, c1)


def test_valid_cpts_plateau_ties(ctx, orc):
    # clamped plateaus give exact score ties: pinned rule (score desc, position desc)
    rs = np.random.RandomState(3)
    sig = np.concatenate([rs.normal(0, 1, 500), np.full(300, 2.5), rs.normal(0, 1, 400),
                          np.full(120, -2.5), rs.normal(0, 1, 300)])
    for num in (100, 300, 330):
        s0, c0 = orc.valid_cpts_w_cap(sig, 3, 5, num)
        s1, c1 = ctx.valid_cpts_w_cap(sig, 3, 5, num)
        assert s0 == s1
        if s0 == 0:
            assert np.array_equal(c0, c1)


def test_new_means_and_stds(ctx, orc):
    rs = np.random.RandomState(0)
    sig = rs.normal(0, 1, 5000)
    segs = np.sort(rs.choice(np.arange(1, 5000), 600, replace=False))
    assert np.array_equal(orc.new_means(sig, segs), ctx.new_means(sig, segs))
    m0, s0 = orc.new_mean_stds(sig, segs)
    m1, s1 = ctx.new_mean_stds(sig, segs)
    assert np.array_equal(m0, m1) and np.array_equal(s0, s1)


@pytest.mark.parametrize('n,seed', [(444, 1), (445, 2), (1000, 3), (1500, 4), (30, 5), (2, 6),
                                    (17, 7)])
def test_theil_sen_bit_exact(ctx, orc, n, seed):
    rs = np.random.RandomState(seed)
    md = rs.normal(0, 1.4826, n)
    ev = (md - 0.07) / 1.06 + rs.normal(0, 0.15, n)
    if seed == 7:
        ev[3] = ev[9]          # equal event means -> slope 1000.0
    key = 12345 + seed
    s0, o0 = orc.theil_sen(480.0, 60.0, ev, md, key)
    s1, o1 = ctx.theil_sen(480.0, 60.0, ev, md, key)
    assert s0 == s1 == 0
    assert o0 == o1


def test_theil_sen_heavy_tail_uses_exact_fallback(ctx, orc):
    from test_theil_sen_gpu import debug_counters
    import theil_sen_cases as tc
    rs = np.random.RandomState(9)
    n = 300
    md = rs.normal(0, 1.4826, n)
    ev = rs.standard_cauchy(n)        # slopes all over the place: sort-and-sweep still copes
    s0, o0 = orc.theil_sen(0.0, 1.0, ev, md, 0)
    s1, o1 = ctx.theil_sen(0.0, 1.0, ev, md, 0)
    assert s0 == s1 == 0 and o0 == o1
    # Cauchy event means on a line to 1e-9: every gap is inside the guards, so sort-and-sweep
    # is abandoned and the exact 2048-bin histogram over all pairs finishes
    md = ev + 1e-9 * rs.normal(0, 1, n)
    before = debug_counters(ctx)
    s1, o1 = ctx.theil_sen(0.0, 1.0, ev, md, 0)
    delta = debug_counters(ctx) - before
    s0, o0 = orc.theil_sen(0.0, 1.0, ev, md, 0)
    assert s0 == s1 == 0 and o0 == o1
    assert delta[tc.READS] == 1 and delta[tc.SWEEP_ABANDONED] == 1 and delta[tc.HISTOGRAM] == 1, delta
    assert delta[tc.SWEEP] == delta[tc.FP32_ALL] == delta[tc.FP32_SAMPLED] == delta[tc.GENERIC] == 0, delta


def test_resolve_skipped_bases_bit_exact(ctx, orc, RPcls):
    rp = RPcls()
    for seed in range(6):
        rs = np.random.RandomState(100 + seed)
        nb = 300
        dwell = 3 + rs.geometric(1 / 6.0, nb)
        # plant deletions: zero-length bases
        dels = rs.choice(np.arange(5, nb - 5), 12, replace=False)
        dwell[dels] = 0
        if seed == 5:
            dwell[40:47] = 0    # a run of deletions
        segs = np.concatenate([[0], np.cumsum(dwell)]).astype(np.int64)
        rm = rs.normal(0, 1.4826, nb)
        rsd = np.full(nb, 0.2)
        norm = np.repeat(rm, dwell) + 0.2 * rs.normal(0, 1, segs[-1])
        s0, o0 = orc.resolve_skipped_bases_with_raw(segs, rm, rsd, norm, rp)
        s1, o1 = ctx.resolve_skipped_bases_with_raw(segs, rm, rsd, norm, rp)
        assert s0 == s1, (s0, s1)
        if s0 == 0:
            assert np.array_equal(o0, o1)
    # RNA-like raw_min_obs_per_base = 2
    rp2 = RPcls(seg=(12, 6, 2, 15))
    rs = np.random.RandomState(77)
    nb = 200
    dwell = 6 + rs.geometric(1 / 20.0, nb)
    dwell[rs.choice(np.arange(5, nb - 5), 8, replace=False)] = 0
    segs = np.concatenate([[0], np.cumsum(dwell)]).astype(np.int64)
    rm = rs.normal(0, 1.4826, nb)
    rsd = np.full(nb, 0.25)
    norm = np.repeat(rm, dwell) + 0.25 * rs.normal(0, 1, segs[-1])
    s0, o0 = orc.resolve_skipped_bases_with_raw(segs, rm, rsd, norm, rp2)
    s1, o1 = ctx.resolve_skipped_bases_with_raw(segs, rm, rsd, norm, rp2)
    assert s0 == s1
    if s0 == 0:
        assert np.array_equal(o0, o1)
