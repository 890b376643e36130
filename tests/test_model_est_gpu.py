"""tb2_kernel_densities (per-k-mer Gaussian kernel densities) and est_kernel_density ->
isolate_alt_density on the device, held to the restatement and bounds of tests/kde_cases.py
and to the unmodified reference's goldens (tests/golden/model_est.npz)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import kde_cases as kc  # noqa: E402
import test_model_est_cpu as cpu  # noqa: E402
from tombo_b200 import _lib, synthetic as syn, tombo_stats as ts  # noqa: E402

pytestmark = pytest.mark.gpu


def ragged(sets):
    off = np.concatenate([[0], np.cumsum([s.shape[0] for s in sets])]).astype(np.int64)
    return (np.concatenate(sets) if sets else np.zeros(0)), off


def check_set(x, grid, bw, dens, c, factor):
    """one device row against scipy at the device's c, c against scipy's, factor exact"""
    assert factor == kc.factor_of(x, bw)
    assert c == kc.cho_cov_pairwise(x, factor)
    want, c_ref = kc.scipy_kde(x, grid, bw)
    assert abs(c - c_ref) <= kc.c_bound(x.shape[0]) * c_ref
    at_c = kc.scipy_kde_at(x, grid, c)
    err = np.abs(dens - at_c)
    assert (err <= kc.density_bound(x, grid, c, at_c)).all(), err.max()
    widened = kc.density_bound(x, grid, c, at_c) + kc.c_widening(x, grid, c, c_ref)
    assert (np.abs(dens - want) <= widened).all()


def test_fresh_seed_sets_within_bound(ctx):
    rs = np.random.RandomState(1939)
    grid = np.linspace(-5, 5, 200)
    sets, bws = [], []
    for n in (2, 3, 8, 9, 129, 1000, 2048, 2049, 5000):
        for bw in (0.01, 0.05, 0.5):
            sets.append(rs.normal(rs.uniform(-4.5, 4.5), rs.uniform(0.05, 1.5), n))
            bws.append(bw)
    for bw in (0.01, 0.05, 0.5):
        sub = [s for s, b in zip(sets, bws) if b == bw]
        lv, off = ragged(sub)
        dens, cho, factor = ctx.kernel_densities(lv, off, grid, bw)
        total, setup = ctx.last_timing()[:2]
        assert 0 < setup < total
        for i, x in enumerate(sub):
            check_set(x, grid, bw, dens[i], cho[i], factor[i])


def test_goldens_end_to_end(monkeypatch):
    """est_kernel_density on the device -> isolate_alt_density: the reference's levels,
    densities within the widened bound of scipy's, the same decisions, alt means within the
    tolerance the density bound implies"""
    g = cpu.golden()
    cfg = lambda k: cpu.cfg_of(g, k)   # noqa: E731
    save_x = np.linspace(-5, 5, cfg('n_points'))
    dens, bounds = {}, {}
    for tag in ('alt', 'ctrl'):
        index, kmer_ref = cpu.serve(monkeypatch, g, tag)
        std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cfg('central_pos'))
        captured = {}
        parse = ts.parse_base_levels

        def keep(*a, **k):
            captured['levels'] = parse(*a, **k)
            return captured['levels']
        monkeypatch.setattr(ts, 'parse_base_levels', keep)
        np.random.seed(cfg('shuffle_' + tag))
        d = ts.est_kernel_density(index, std_ref, cfg('kmer_obs_thresh'), None, save_x, cfg('bw'), 1,
                                  tag, cfg('batch'), cfg('max_kmer_obs'), cfg('min_kmer_obs_to_est'))
        monkeypatch.setattr(ts, 'parse_base_levels', parse)
        np.testing.assert_array_equal(cpu.digests(captured['levels']), g[tag + '_sha'])
        lv, off = ragged(list(captured['levels'].values()))
        _, cho, _ = _lib.get_context().kernel_densities(lv, off, save_x[:1], cfg('bw'))
        b = []
        for i, (k, x) in enumerate(captured['levels'].items()):
            ref = g[tag + '_dens'][i]
            c_ref = g[tag + '_cho_cov'][i]
            assert abs(cho[i] - c_ref) <= kc.c_bound(x.shape[0]) * c_ref
            bd = kc.density_bound(x, save_x, cho[i], ref) + kc.c_widening(x, save_x, cho[i], c_ref)
            assert (np.abs(d[k] - ref) <= bd).all(), k
            b.append(bd)
        dens[tag], bounds[tag] = d, np.array(b)
    alt_ref, dec = ts._isolate_alt_density(dens['alt'], dens['ctrl'], 'C', cfg('alt_pctl'),
                                           std_ref, save_x)
    np.testing.assert_array_equal(list(dec['offsets'].values()), g['dec_offsets'])
    np.testing.assert_array_equal(list(dec['peaks'].values()), g['dec_peaks'])
    # tolerance: the ratio at each peak moves by at most its two relative density errors, so
    # std_frac by at most the largest such move; diff_dens_j by the shifted alt error plus
    # std_frac^k times the control error plus the control times the std_frac^k change; the
    # weighted mean over save_x (width 10) by 10 sum_j |diff change| / sum_j diff
    kmers = list(dens['alt'])
    ea = dict(zip(kmers, bounds['alt']))
    es = dict(zip(kmers, bounds['ctrl']))
    gold_alt = dict(zip(kmers, g['alt_dens']))
    gold_ctrl = dict(zip(kmers, g['ctrl_dens']))

    def shift(v, off):
        return (np.concatenate([np.zeros(-off), v[:off]]) if off < 0 else
                np.concatenate([v[off:], np.zeros(off)]))
    d_ratio = 0.0
    for k, (cp, ap) in dec['peaks'].items():
        a, s = shift(gold_alt[k], dec['offsets'][k]), gold_ctrl[k]
        ra = shift(ea[k], dec['offsets'][k])[ap] / a[ap] + es[k][cp] / s[cp]
        d_ratio = max(d_ratio, a[ap] / s[cp] * ra * 1.01)
    _, gdec = ts._isolate_alt_density(gold_alt, gold_ctrl, 'C', cfg('alt_pctl'), std_ref, save_x)
    ratios = [shift(gold_alt[k], dec['offsets'][k])[ap] / gold_ctrl[k][cp]
              for k, (cp, ap) in gdec['peaks'].items()]
    std_frac = np.percentile(ratios, cfg('alt_pctl'))
    got = dict(((k, p), v) for (k, p), v in alt_ref.means.items())
    for k, p, want in zip(g['alt_kmers'], g['alt_pos'], g['alt_means']):
        n_alt = k.count('C')
        f = std_frac ** n_alt
        df = n_alt * (std_frac + d_ratio) ** (n_alt - 1) * d_ratio
        diff = np.maximum(shift(gold_alt[k], dec['offsets'][k]) - gold_ctrl[k] * f, 0)
        change = shift(ea[k], dec['offsets'][k]) + f * es[k] + gold_ctrl[k] * df
        tol = 10 * change.sum() / diff.sum() * 1.01 + 1e-12
        assert abs(got[(str(k), int(p))] - want) <= tol, (k, p)


def test_default_shape_sweep(ctx):
    """4 096 sets of 1 000 to 12 000 levels on 500 points at bandwidth 0.05; 16 seeded sets
    compared with scipy"""
    rs = np.random.RandomState(4096)
    grid = np.linspace(-5, 5, 500)
    ns = rs.randint(1000, 12001, 4096)
    centres = rs.normal(0, 1, 4096)
    sets = [rs.normal(c, 0.25, n) for c, n in zip(centres, ns)]
    lv, off = ragged(sets)
    dens, cho, factor = ctx.kernel_densities(lv, off, grid, 0.05)
    assert np.isfinite(dens).all() and (dens >= 0).all()
    for i in rs.choice(4096, 16, replace=False):
        check_set(sets[i], grid, 0.05, dens[i], cho[i], factor[i])


def test_large_set_and_single_point(ctx):
    rs = np.random.RandomState(10 ** 6)
    x = rs.normal(0.3, 0.7, 10 ** 6)
    grid = np.linspace(-5, 5, 40)
    dens, cho, factor = ctx.kernel_densities(x, np.array([0, x.shape[0]]), grid, 0.05)
    check_set(x, grid, 0.05, dens[0], cho[0], factor[0])
    small = rs.normal(0, 1, 300)
    dens, cho, factor = ctx.kernel_densities(small, np.array([0, 300]), np.array([0.25]), 0.2)
    assert dens.shape == (1, 1)
    check_set(small, np.array([0.25]), 0.2, dens[0], cho[0], factor[0])


def test_sets_the_reference_cannot_fit_are_nan(ctx):
    rs = np.random.RandomState(5)
    good = rs.normal(0, 1, 50)
    bad_nan, bad_inf = good.copy(), good.copy()
    bad_nan[10], bad_inf[3] = np.nan, np.inf
    sets = [good, np.zeros(0), good[:1], np.full(20, 0.5), bad_nan, bad_inf, good[:2]]
    grid = np.linspace(-5, 5, 70)
    dens, cho, factor = ctx.kernel_densities(*ragged(sets), grid, 0.05)
    for i in (1, 2, 3, 4, 5):
        assert np.isnan(dens[i]).all() and np.isnan(cho[i]) and np.isnan(factor[i]), i
    for i in (0, 6):
        check_set(sets[i], grid, 0.05, dens[i], cho[i], factor[i])


def test_invalid_arguments(ctx):
    lib, h = ctx.lib, ctx.handle
    f64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))        # noqa: E731
    i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))         # noqa: E731
    lv = np.arange(10, dtype=np.float64)
    off = np.array([0, 4, 10], dtype=np.int64)
    x = np.linspace(-5, 5, 8)
    dens, cho, fac = np.empty(16), np.empty(2), np.empty(2)

    def call(n=2, levels=lv, o=off, m=8, grid=x, bw=0.05, d=dens, c=cho):
        return lib.tb2_kernel_densities(
            h, n, None if levels is None else f64p(levels), None if o is None else i64p(o), m,
            None if grid is None else f64p(grid), bw, None if d is None else f64p(d),
            None if c is None else f64p(c), f64p(fac))
    assert call() == 0
    bad = [dict(n=-1), dict(n=2 ** 31), dict(m=0), dict(m=2 ** 20 + 1), dict(grid=None),
           dict(bw=0.0), dict(bw=-0.1), dict(bw=float('nan')), dict(bw=float('inf')),
           dict(o=None), dict(d=None), dict(c=None), dict(levels=None),
           dict(o=np.array([1, 4, 10], dtype=np.int64)), dict(o=np.array([0, 5, 4], dtype=np.int64))]
    for kw in bad:
        assert call(**kw) == 201, kw
    assert call(n=0, o=None, d=None, c=None, levels=None) == 0


def test_call_leaves_resident_batch_intact(ctx, RPcls):
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    means, sds = syn.kmer_table(kmer_ref)
    alt = np.full((4 ** 6, 6), np.nan)
    for km, pos, m, _ in syn.make_alt_kmer_ref(kmer_ref, 'C', seed=1):
        alt[ts._kmer_code(km), pos] = m
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 60, 400, 77)
    read_start = 1000 + np.arange(60, dtype=np.int64) * 50
    rp, sp = RPcls(), RPcls(save=True)
    pol = _lib.make_policy('DNA')
    c = _lib.Context(0)
    try:
        c.set_model(means, sds, 6, cpos)
        c.set_alt_model(alt, 6)
        c.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
        c.batch_compute(rp, sp, pol)
        base = {k: v.copy() for k, v in c.batch_download().items()}
        assert (base['status'] == 0).sum() > 40
        c.batch_alt_llr(read_start, 1)
        llr = [a.copy() for a in c.batch_llr_download()]
        c.region_stats_begin(1000, 4000)
        c.region_stats_add_batch_llr(2.5, -1.5, 0)
        counts = c.region_counts_get().copy()
        rs = np.random.RandomState(3)
        big = rs.normal(0, 1, 2 * raw.shape[0])
        c.kernel_densities(big, np.array([0, raw.shape[0], big.shape[0]]), np.linspace(-5, 5, 500), 0.05)
        got = c.batch_download()
        for k in base:
            assert np.asarray(got[k]).tobytes() == np.asarray(base[k]).tobytes(), k
        for a, b in zip(c.batch_llr_download(), llr):
            assert a.tobytes() == b.tobytes()
        assert c.region_counts_get().tobytes() == counts.tobytes()
    finally:
        c.close()
