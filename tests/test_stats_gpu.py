"""GPU: the per-read statistics stage (llr.cu, fisher.cuh, region_stats.cu and the Fisher window
of group_stats.cu) against the plain restatements of stats_cases.py: standard LLRs, positions,
site offsets and region counters bit for bit; scaled and variable-SD LLRs, p-values and Fisher
windows within the bounds derived there.  Each family's largest error / bound ratio is printed
at the end of the module (pytest -s)."""
import ctypes as C
import math
import os
import sys
from unittest import mock

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import stats_cases as sc  # noqa: E402
import test_group_stats_gpu as gs  # noqa: E402

pytestmark = pytest.mark.gpu
WORST = {}


def _note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print('largest error / bound  %-34s %.3g' % (k, WORST[k]))


# ---------------------------------------------------------------------------
# tables
# ---------------------------------------------------------------------------
def _model_tables(kind):
    """canonical tables and the 5mC alternative tables of the synthetic DNA / RNA models"""
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    K = len(kmer_ref[0][0])
    means, sds = syn.kmer_table(kmer_ref)
    rows = syn.make_alt_kmer_ref(kmer_ref, 'C', seed=1)
    alt, alt_sd = sc.alt_tables(kmer_ref)
    return kmer_ref, rows, K, cpos, means, sds, alt, alt_sd


TABLES = ['dna6', 'rna5', 'K1', 'K2', 'K3', 'K7']


def _tables(name):
    if name in ('dna6', 'rna5'):
        _, _, K, cpos, means, sds, alt, _ = _model_tables('DNA' if name == 'dna6' else 'RNA')
        return K, cpos, means, sds, alt
    K = int(name[1:])
    means, sds, alt, _ = sc.synthetic_tables(K, seed=100 + K)
    return K, K // 2, means, sds, alt


# ---------------------------------------------------------------------------
# tb2_alt_model_llr_batch
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('tables', TABLES)
def test_llr_batch_read_shapes_match_restatement(ctx, tables):
    K, cpos, means, sds, alt = _tables(tables)
    ctx.set_model(means, sds, K, cpos)
    ctx.set_alt_model(alt, K)
    rs = np.random.RandomState(7000 + K + 13 * TABLES.index(tables))
    alt_code = 1
    reads, names = [], []
    for name, codes, nb in sc.llr_read_shapes(K, cpos, alt_code, rs):
        kc = sc.kmer_codes(codes.astype(np.int64), K)
        reads.append((codes, means[kc] + rs.normal(0.0, 0.3, nb)))
        names.append(name)
    nm, mo, sq, so = sc.flatten(reads)
    start = rs.randint(0, 10 ** 6, len(reads)).astype(np.int64)
    for mode in (0, 1):
        llr, pos, off = ctx.alt_model_llr_batch(nm, mo, sq, so, start, alt_code,
                                                use_standard_llhr=(mode == 1))
        w_llr, w_pos, w_off, s_abs = sc.llr_reads(nm, mo, sq, so, start, means, sds, alt, K,
                                                  cpos, alt_code, mode)
        assert np.array_equal(off, w_off), [(n, int(a), int(b)) for n, a, b in
                                            zip(names, np.diff(off), np.diff(w_off)) if a != b]
        assert np.array_equal(pos, w_pos)
        _note('llr_batch mode %d' % mode, sc.assert_llr(llr, w_llr, s_abs, mode, K))
    # the shapes that must and must not carry sites
    n_sites = dict(zip(names, np.diff(w_off)))
    assert all(n_sites[n] == 0 for n in names if n.startswith('no_'))
    assert n_sites['one_testable_alt'] == 1 and n_sites['all_alt'] == 40
    assert all(n_sites['testable_%d_sites_at_ends' % t] == 2 for t in (255, 256, 257, 513))
    # no alternative base anywhere: no sites, total 0
    keep = [i for i, n in enumerate(names) if n.startswith('no_')]
    nm, mo, sq, so = sc.flatten([reads[i] for i in keep])
    llr, pos, off = ctx.alt_model_llr_batch(nm, mo, sq, so, start[keep], alt_code)
    assert off.shape[0] == len(keep) + 1 and not off.any() and llr.shape[0] == 0


def test_llr_batch_rejects_a_sequence_longer_than_its_means(ctx):
    """each read must carry exactly nb + K - 1 base codes; one extra code (which reads nothing
    out of bounds) is an invalid argument"""
    from tombo_b200 import _lib
    K, cpos, means, sds, alt = _tables('dna6')
    ctx.set_model(means, sds, K, cpos)
    ctx.set_alt_model(alt, K)
    rs = np.random.RandomState(3)
    nb = 60
    reads = [(rs.randint(0, 4, nb + K - 1).astype(np.uint8), rs.normal(0, 1, nb)) for _ in range(3)]
    nm, mo, sq, so = sc.flatten(reads)
    ctx.alt_model_llr_batch(nm, mo, sq, so, np.zeros(3, np.int64), 1)
    sq_long = np.concatenate([sq[:so[2]], [0], sq[so[2]:]]).astype(np.uint8)
    so_long = so.copy()
    so_long[2:] += 1
    with pytest.raises(_lib.TomboB200Error):
        ctx.alt_model_llr_batch(nm, mo, sq_long, so_long, np.zeros(3, np.int64), 1)


@pytest.mark.parametrize('call', ['llr', 'motif', 'de_novo'])
def test_host_array_calls_reject_counts_past_int_max(ctx, call):
    """the kernels index reads and bases with int: 2^31 reads, or one read of 2^31 bases, is an
    invalid argument, found before any array is read past its first entries (the arrays here
    hold two)"""
    from tombo_b200 import _lib
    K, cpos, means, sds, alt = _tables('dna6')
    ctx.set_model(means, sds, K, cpos)
    ctx.set_alt_model(alt, K)
    p64, pf = (lambda a: _lib.ptr(a, _lib.i64)), (lambda a: _lib.ptr(a, _lib.f64))
    nm, llr, start = np.zeros(2), np.zeros(2), np.zeros(2, np.int64)
    pos, site_off = np.zeros(2, np.int64), np.zeros(2, np.int64)
    sq, strand, status = np.zeros(2, np.uint8), np.zeros(2, np.int8), np.zeros(2, np.int32)
    motif = _lib.Motif(1, 1)
    motif.mask[0] = 2
    big = 2 ** 31
    for n_reads, mo, so in ((big, np.zeros(2, np.int64), np.zeros(2, np.int64)),
                            (1, np.array([0, big], np.int64), np.array([0, big + K - 1], np.int64))):
        head = (ctx.handle, n_reads, pf(nm), p64(mo), _lib.ptr(sq, C.c_uint8), p64(so), p64(start))
        if call == 'llr':
            rc = ctx.lib.tb2_alt_model_llr_batch(*head, 1, 0, 4.0, 1.0, 0.2, pf(llr), p64(pos),
                                                 p64(site_off))
        elif call == 'motif':
            rc = ctx.lib.tb2_alt_model_llr_motif_batch(
                *head, _lib.ptr(strand, C.c_int8), C.byref(motif), 0, 0, 0, 10 ** 6, 0, 4.0, 1.0,
                0.2, pf(llr), p64(pos), p64(site_off), _lib.ptr(status, C.c_int32))
        else:
            rc = ctx.lib.tb2_de_novo_read_stats_batch(*head, 1, pf(llr), p64(pos), p64(site_off))
        assert rc == 201, (call, n_reads, rc)                # TB2_ERR_INVALID_ARG


# ---------------------------------------------------------------------------
# tb2_batch_alt_llr on a resident batch of >= 2 500 reads (three k_scan_sites chunks)
# ---------------------------------------------------------------------------
def test_resident_llr_over_three_scan_chunks(ctx, RPcls):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, _, K, cpos, means, sds, alt, _ = _model_tables('DNA')
    ctx.set_model(means, sds, K, cpos)
    ctx.set_alt_model(alt, K)
    n = 2600
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, n, 200, 20261016)
    failed = (7, 1100, 2500)
    for r in failed:                                     # hopeless reads carry no sites
        raw[raw_off[r]:raw_off[r + 1]] = 480.0
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    pol = _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    res = ctx.batch_download()
    ok = res['status'] == 0
    assert not ok[list(failed)].any() and ok.sum() >= n - 30
    start = (np.arange(n, dtype=np.int64) * 53) % 7919 + 10 ** 6
    for mode in (0, 1):
        tot = ctx.batch_alt_llr(start, 1, use_standard_llhr=(mode == 1))
        llr, pos, off = ctx.batch_llr_download()
        w_llr, w_pos, w_off, s_abs = sc.llr_reads(res['norm_mean'], res['base_off'], seq,
                                                  seq_off, start, means, sds, alt, K, cpos, 1,
                                                  mode)
        keep = np.repeat(ok, np.diff(w_off))
        w_cnt = np.where(ok, np.diff(w_off), 0)
        assert tot == keep.sum() and np.array_equal(off, np.concatenate([[0], np.cumsum(w_cnt)]))
        assert np.array_equal(pos, w_pos[keep])
        _note('resident llr mode %d' % mode, sc.assert_llr(llr, w_llr[keep], s_abs[keep], mode, K))


# ---------------------------------------------------------------------------
# tb2_calc_llh_ratio_windows, modes 0 / 1 / 2
# ---------------------------------------------------------------------------
def _windows_case(K, rs, n):
    m = rs.normal(0.0, 1.0, (n, K))
    r = m + rs.normal(0.0, 0.3, (n, K))
    a = r + rs.normal(0.0, 0.4, (n, K))
    cv = rs.uniform(0.01, 0.2, n)
    rv, av = rs.uniform(0.01, 0.2, (n, K)), rs.uniform(0.01, 0.2, (n, K))
    e = 0
    a[e, 0] = r[e, 0]                                    # ref == alt: mode 0 skips the term
    a[e + 1, :] = r[e + 1, :]
    m[e + 1, 0] = np.inf                                 # ... so only mode 1 sees inf - inf
    r[e + 2, K - 1], a[e + 2, K - 1] = 0.0, 1e-300       # tiny means_diff
    a[e + 3, 0] = np.nextafter(r[e + 3, 0], np.inf)
    m[e + 4, :] = 1e3                                    # exp underflows to 0
    m[e + 5, 0] = r[e + 5, 0] + 30.0
    a[e + 6, K // 2] = np.nan                            # NaN alternative level
    m[e + 7, 0] = np.nan
    return m, r, a, cv, rv, av


@pytest.mark.parametrize('K', range(1, 9))
def test_llh_ratio_windows_match_restatement(ctx, K):
    rs = np.random.RandomState(500 + K)
    n = 1000 + 37 * K                                    # never a multiple of 128
    m, r, a, cv, rv, av = _windows_case(K, rs, n)
    for mode, hp in ((0, 0.2), (0, 0.0), (1, 0.2), (2, 0.2)):
        if mode == 2:
            got = ctx.calc_llh_ratio_windows(2, m, r, a, rv, av)
            want = [sc.score_window(2, m[i], r[i], a[i], rv[i], av[i]) for i in range(n)]
        else:
            got = ctx.calc_llh_ratio_windows(mode, m, r, a, cv, None, 4.0, 1.0, hp)
            want = [sc.score_window(mode, m[i], r[i], a[i], cv[i], sf=4.0, hf=1.0, hp=hp)
                    for i in range(n)]
        w = np.array([x[0] for x in want])
        s_abs = np.array([x[1] for x in want])
        _note('llh windows mode %d' % mode, sc.assert_llr(got, w, s_abs, mode, K))
        if mode == 0:
            assert got[1] == 0.0 and got[4] == 0.0 and math.isnan(got[6])
        if mode == 1:
            assert math.isnan(got[1])


def test_variable_sd_mirror_matches_restatement(ctx, monkeypatch):
    """compute_alt_model_read_stats with CONST_SD_MODEL False scores with c_calc_llh_ratio
    (mode 2: per-k-mer reference and alternative variances)"""
    from tombo_b200 import tombo_helper as th, tombo_stats as ts
    kmer_ref, rows, K, cpos, means, sds, alt, alt_sd = _model_tables('DNA')
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    alt_ref = ts.AltModel(kmer_ref=rows, central_pos=cpos, alt_base='C', name='5mC')
    rs = np.random.RandomState(99)
    nb = 300
    codes = rs.randint(0, 4, nb + K - 1).astype(np.uint8)
    kc = sc.kmer_codes(codes.astype(np.int64), K)
    norm_mean = means[kc] + rs.normal(0, 0.3, nb)
    genome = ''.join('ACGT'[c] for c in codes)
    bases = np.array(list(genome[cpos:cpos + nb]), dtype='S1')
    r_data = th.readData(start=5000, end=5000 + nb, filtered=False, read_start_rel_to_raw=0,
                         strand='+', fn='x', corr_group='g', rna=False)
    monkeypatch.setattr(ts, 'CONST_SD_MODEL', False)
    with mock.patch.object(th, 'get_multiple_slots_read_centric', lambda *a, **k: (norm_mean, bases)):
        llr, pos, _ = ts.compute_alt_model_read_stats(r_data, std_ref, [('5mC', alt_ref)],
                                                      use_standard_llhr=True)
    w_llr, w_pos, _, s_abs = sc.llr_reads(norm_mean, np.array([0, nb]), codes, np.array([0, nb + K - 1]),
                                          np.array([5000]), means, sds, alt, K, cpos, 1, 2,
                                          alt_sds=alt_sd)
    assert w_llr.shape[0] > 20
    assert np.array_equal(pos['5mC'], w_pos)
    _note('mirror mode 2', sc.assert_llr(llr['5mC'], w_llr, s_abs, 2, K))


# ---------------------------------------------------------------------------
# z -> p -> Fisher window: tb2_window_fisher_pvals and tb2_de_novo_read_stats_batch
# ---------------------------------------------------------------------------
def _levels(rs, n):
    """levels, reference levels and sds whose z-scores cover p = 1 down to p = 0"""
    rm = rs.normal(0.0, 1.0, n)
    rsd = rs.uniform(0.05, 0.3, n)
    z = np.abs(rs.standard_t(3, n)) * 2.0
    z[rs.uniform(size=n) < 0.03] = 15.0                  # p ~ 1e-50: at the clamp
    z[rs.uniform(size=n) < 0.02] = 40.0                  # p underflows below the clamp
    m = rm + z * rsd
    return m, rm, rsd


def _edges(m, rm, rsd):
    m, rm, rsd = m.copy(), rm.copy(), rsd.copy()
    m[3] = rm[3]                                         # z = 0, p = 1
    rsd[11], m[12], rsd[12] = 0.0, rm[12], 0.0           # z = inf (p = 0), and 0 / 0
    m[20] = np.nan
    m[40] = rm[40] + 1e3 * rsd[40]                       # erfc underflows to 0
    return m, rm, rsd


def _seg_lengths(lag):
    w = 2 * lag + 1
    return [max(w - 1, 1), w, (255, 256, 257, 513)[lag % 4]]


def _check_windows(got, vals, bounds, ref, final_clamp, family):
    clamp = sc.mpmath.mpf(sc.SMALLEST_PVAL)
    if final_clamp:
        vals = [None if v is None else max(v, clamp) for v in vals]
    _note(family, sc.assert_window(got, vals, bounds))
    at = ref == sc.SMALLEST_PVAL
    assert np.all(got[at] == sc.SMALLEST_PVAL)


@pytest.mark.parametrize('lag', range(0, 65))
def test_window_fisher_pvals_match_exact_path(ctx, lag):
    rs = np.random.RandomState(300 + lag)
    lens = _seg_lengths(lag)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    m, rm, rsd = _levels(rs, int(off[-1]))
    m, rm, rsd = _edges(m, rm, rsd)
    z = sc.z_scores(m, rm, rsd)
    pe, perr = sc.exact_pvals(z), sc.p_rel_bound(z)
    perr[np.isinf(z)] = 0.0
    p_in = rs.uniform(0.0, 1.0, int(off[-1]))
    p_in[[0, 5, 9, 30]] = [0.0, 1e-60, sc.SMALLEST_PVAL, 1.0]
    p_in[17] = np.nan
    p_in[rs.uniform(size=p_in.shape[0]) < 0.05] = 1e-80
    pg = sc.exact_given(p_in)
    for a, b in zip(off[:-1], off[1:]):
        ex_l = sc.exact_window(pe[a:b], perr[a:b], lag, False)
        ex_p = sc.exact_window(pg[a:b], np.zeros(b - a), lag, False)
        for final_clamp in (0, 1):
            got = ctx.window_fisher_pvals(m[a:b], rm[a:b], rsd[a:b], [0, b - a], lag, final_clamp)
            ref = sc.ref_window(sc.ref_pvals(z[a:b]), lag, final_clamp)
            _check_windows(got, ex_l[0], ex_l[1], ref, final_clamp, 'fisher levels')
            if lag == 0:
                continue                                 # p-value input is for windows only
            got = ctx.window_fisher_pvals(p_in[a:b], None, None, [0, b - a], lag, final_clamp)
            ref = sc.ref_window(p_in[a:b], lag, final_clamp)
            _check_windows(got, ex_p[0], ex_p[1], ref, final_clamp, 'fisher p-values')
    # all segments in one call: the same values
    got = ctx.window_fisher_pvals(m, rm, rsd, off, lag, 1)
    for a, b in zip(off[:-1], off[1:]):
        one = ctx.window_fisher_pvals(m[a:b], rm[a:b], rsd[a:b], [0, b - a], lag, 1)
        assert np.array_equal(got[a:b], one, equal_nan=True)


@pytest.mark.parametrize('lag', range(0, 65))
def test_de_novo_batch_matches_exact_path(ctx, lag):
    _, _, K, cpos, means, sds, _, _ = _model_tables('DNA')
    ctx.set_model(means, sds, K, cpos)
    rs = np.random.RandomState(900 + lag)
    reads, zs = [], []
    for n in _seg_lengths(lag):
        nb = n + K - 1
        codes = rs.randint(0, 4, nb + K - 1).astype(np.uint8)
        kc = sc.kmer_codes(codes[cpos:cpos + nb].astype(np.int64), K)   # k-mers of the stats
        z = np.abs(rs.standard_t(3, n)) * 2.0
        z[rs.uniform(size=n) < 0.03] = 15.0
        z[rs.uniform(size=n) < 0.02] = 40.0
        mm = rs.normal(0, 1, nb)
        mm[cpos:cpos + n] = means[kc] + z * sds[kc]
        mm[cpos + min(2, n - 1)] = means[kc[min(2, n - 1)]]              # m == rm
        if n > 10:
            mm[cpos + 10] = np.nan
        reads.append((codes, mm))
        zs.append(sc.z_scores(mm[cpos:cpos + n], means[kc], sds[kc]))
    nm, mo, sq, so = sc.flatten(reads)
    start = np.array([1000, 50000, 900000], dtype=np.int64)
    pv, pos, off = ctx.de_novo_read_stats_batch(nm, mo, sq, so, start, lag)
    for r, z in enumerate(zs):
        a, b = off[r], off[r + 1]
        assert b - a == z.shape[0]
        assert np.array_equal(pos[a:b], start[r] + cpos + np.arange(z.shape[0]))
        vals, bounds = sc.exact_window(sc.exact_pvals(z), sc.p_rel_bound(z), lag, False)
        ref = sc.ref_window(sc.ref_pvals(z), lag, True)
        _check_windows(pv[a:b], vals, bounds, ref, True, 'de novo')


# ---------------------------------------------------------------------------
# compute_group_reg_stats: Fisher windows far beyond the per-read widths
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('fm', [5, 62, 64, 340, 400, 1000])
def test_group_fisher_windows_at_large_fm_offset(fm):
    from tombo_b200 import tombo_stats as ts
    rs = np.random.RandomState(40 + fm)
    n_pos, start = 2 * fm + 1 + 150, 200000
    lo = start - fm - 3

    def region():
        reads = [(lo, rs.normal(0.0, 1.0, n_pos + 2 * fm + 6)) for _ in range(12)]
        return gs.Region(start, start + n_pos, reads=reads)
    reg, creg = region(), region()
    for st in ('ks_test', 'u_test', 't_test'):
        samp = reg.copy().update(start=start - fm, end=start + n_pos + fm).get_base_levels()
        ctrl = creg.copy().update(start=start - fm, end=start + n_pos + fm).get_base_levels()
        want = gs.restate_group(samp, ctrl, start - fm, fm, 5, st)
        g = ts.compute_group_reg_stats(reg, creg, fm, 5, st)[0][1]
        np.testing.assert_array_equal(g.reg_poss, want[1])
        gs.assert_stats(g.reg_stats, want[0], st)
        fin = ~np.isnan(want[0])
        assert fin.sum() >= 150 and not np.isnan(g.reg_stats[fin]).any()


# ---------------------------------------------------------------------------
# region counters
# ---------------------------------------------------------------------------
PARAMS = [(2.5, -1.5, 0), (2.5, None, 0), (0.5, None, 1), (0.0, 0.0, 1), (1.0, float('nan'), 0)]


def _counter_case(rs, reg_start, reg_len, thresh, lower):
    n = int(min(3 * reg_len + 50, 200000))
    pos = rs.randint(reg_start - 3, reg_start + reg_len + 3, n).astype(np.int64)
    pos[:4] = [reg_start, reg_start + reg_len - 1, reg_start - 1, reg_start + reg_len]
    stats = rs.normal(0.0, 2.0, n)
    pick = rs.uniform(size=n)
    specials = [np.nan, np.inf, -np.inf, thresh, -thresh] + \
        ([] if lower is None or np.isnan(lower) else [lower])
    for i, v in enumerate(specials):
        sel = (pick >= 0.02 * i) & (pick < 0.02 * (i + 1))
        stats[sel] = v
    return stats, pos


@pytest.mark.parametrize('reg_len', [1, 1023, 1024, 1025, 10000, 70001])
def test_region_counters_match_restatement(ctx, reg_len):
    rs = np.random.RandomState(reg_len)
    reg_start = 123456
    for thresh, lower, stat_type in PARAMS:
        stats, pos = _counter_case(rs, reg_start, reg_len, thresh, lower)
        for unmod in (2.0, float('nan')):
            ctx.region_stats_begin(reg_start, reg_len)
            ctx.region_stats_add(stats, pos, thresh, lower, stat_type)
            got = ctx.region_stats_finalize(unmod, 1.0)
            want = sc.region_counters(stats, pos, reg_start, reg_len, thresh, lower, stat_type,
                                      unmod=unmod, mod=1.0)
            for k in want:
                assert np.array_equal(got[k], want[k], equal_nan=True), (k, thresh, lower)
            inside = (pos >= reg_start) & (pos < reg_start + reg_len) & ~np.isnan(stats)
            assert got['cov'].sum() == inside.sum()


def test_region_finalize_reports_capacity(ctx):
    from tombo_b200 import _lib
    rs = np.random.RandomState(11)
    reg_start, reg_len = 777, 5000
    stats, pos = _counter_case(rs, reg_start, reg_len, 2.5, -1.5)
    ctx.region_stats_begin(reg_start, reg_len)
    ctx.region_stats_add(stats, pos, 2.5, -1.5, 0)
    want = sc.region_counters(stats, pos, reg_start, reg_len, 2.5, -1.5, 0, unmod=2.0, mod=0.0)
    n_cov = want['pos'].shape[0]
    cap = n_cov - 37
    out = dict(pos=np.full(cap, -1, np.int64), frac=np.full(cap, -1.0),
               damp_frac=np.full(cap, -1.0), cov=np.full(cap, -1, np.int64),
               valid_cov=np.full(cap, -1, np.int64))
    n = C.c_int64(0)
    rc = ctx.lib.tb2_region_stats_finalize(
        ctx.handle, C.c_double(2.0), C.c_double(0.0), C.c_int64(cap),
        _lib.ptr(out['pos'], _lib.i64), _lib.ptr(out['frac'], _lib.f64),
        _lib.ptr(out['damp_frac'], _lib.f64), _lib.ptr(out['cov'], _lib.i64),
        _lib.ptr(out['valid_cov'], _lib.i64), C.byref(n))
    assert rc == 202                                     # TB2_ERR_CAPACITY
    assert n.value == n_cov
    for k in out:
        assert np.array_equal(out[k], want[k][:cap], equal_nan=True), k
