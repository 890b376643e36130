"""GPU: de novo and sample-compare testing of whole regions (tb2_de_novo_region_stats,
tb2_sample_compare_region_stats, tb2_batch_de_novo_region, tb2_region_stats_add_tests) and
tombo_stats.compute_reg_stats.

1. compute_reg_stats against the unmodified reference (tests/golden/reg_stats.npz) for all
   three statistic types: regionStats and per-read blocks.
2. The batched functions against the single-read mirrors, bit for bit, on the golden's reads
   and on fresh-seed reads over many regions, both strands and fm_offset 0 .. 64.
3. Fused counters against region_stats_add of the downloaded statistics; split calls sum.
4. The resident de novo test against the host-array route.
5. Invalid arguments, and the other modules' device results survive the new calls."""
import os
import queue
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import reg_stats_cases as rc  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, 'golden', 'reg_stats.npz')


@pytest.fixture(scope='module')
def g():
    return dict(np.load(GOLDEN))


def _models():
    from tombo_b200 import synthetic as syn, tombo_helper as th, tombo_stats as ts
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    alt_ref = ts.AltModel(kmer_ref=syn.make_alt_kmer_ref(kmer_ref, 'C', seed=1), central_pos=cpos,
                          alt_base='C', name='CpG', motif=th.TomboMotif('CG', 1))
    return std_ref, alt_ref


@pytest.fixture
def served(monkeypatch):
    """reads served at the FAST5 seam, keyed by r_data.fn"""
    from tombo_b200 import tombo_helper as th
    store = {}

    def slots(r_data, names, corr_grp=None):
        r = store[r_data.fn]
        vals = {'norm_mean': r['means'],
                'base': np.array([('ACGT'[c] if c < 4 else 'N') for c in r['bases']], dtype='S1')}
        return [vals[n] for n in names]

    monkeypatch.setattr(th, 'get_multiple_slots_read_centric', slots)
    monkeypatch.setattr(th, 'get_raw_read_slot', lambda r_data: types.SimpleNamespace(
        attrs={'read_id': ('read_' + r_data.fn).encode()}))
    return store


def _r_data(fn, r):
    return types.SimpleNamespace(start=int(r['start']), end=int(r['end']), strand=r['strand'],
                                 fn=fn, corr_group='g')


class _CtrlReg(object):
    """control region: base levels as the reference's get_base_levels returned them"""

    def __init__(self, start, end, levels, genome):
        self.start, self.end, self.strand, self.chrm = start, end, None, 'chr'
        self._levels, self._genome = levels, genome

    def copy(self):
        return _CtrlReg(self.start, self.end, self._levels, self._genome)

    def update(self, start=None, end=None, seq=None):
        self.start, self.end = start, end
        return self

    def get_base_levels(self):
        return self._levels

    def add_seq(self):
        self.seq = self._genome[self.start:self.end]
        return self


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


# 1. compute_reg_stats against the reference
def _serve_golden(g, served):
    for i in range(g['reads_start'].shape[0]):
        served['s%d' % i] = rc.golden_read(g, i)


def test_compute_reg_stats_matches_reference(g, served):
    from tombo_b200 import tombo_stats as ts
    std_ref, alt_ref = _models()
    _serve_golden(g, served)
    for k in range(int(g['n_calls'])):
        st, reg, fm, mtr, thresh, lower, prior = rc.golden_settings(g, k)
        start, end = [int(x) for x in g['g%d_region' % reg]]
        reads = [_r_data('s%d' % i, served['s%d' % i]) for i in g['q%d_reads' % k]]
        reg_data = types.SimpleNamespace(chrm='chr', strand=None, start=start, end=end, reads=reads)
        ctrl = None
        if st == 'sample_compare':
            ctrl = _CtrlReg(start, end, g['g%d_fm%d_ctrl_levels' % (reg, fm)], str(g['genome']))
        q = queue.Queue()
        want_err = str(g['q%d_error' % k])
        try:
            res = ts.compute_reg_stats(reg_data, fm, mtr, thresh, lower, ctrl,
                                       std_ref if (prior or st != 'sample_compare') else None,
                                       [('CpG', alt_ref)], False, q, st, None)
            err = ''
        except Exception as e:      # TomboError carries the reference's message
            err, res = str(e), []
        assert err == want_err, (k, err, want_err)
        assert len(res) == int(g['q%d_n_stats' % k])
        for n, (name, s) in enumerate(res):
            p = 'q%d_s%d_' % (k, n)
            assert name == str(g[p + 'name'])
            assert np.array_equal(s.reg_poss, g[p + 'poss'])
            assert np.array_equal(s.reg_cov, g[p + 'cov'])
            assert np.array_equal(s.valid_cov, g[p + 'valid_cov'])
            assert np.array_equal(np.asarray(s.ctrl_cov, dtype=np.int64), g[p + 'ctrl_cov'])
            assert np.array_equal(s.reg_frac_standard_base, g[p + 'frac'], equal_nan=True)
        blocks = []
        while not q.empty():
            blocks.append(q.get())
        assert len(blocks) == int(g['q%d_n_blocks' % k])
        for b, (name, (block, lookup, chrm, strand, bstart)) in enumerate(blocks):
            p = 'q%d_b%d_' % (k, b)
            assert name == str(g[p + 'name']) and bstart == int(g[p + 'start'])
            if st == 'model_compare':
                w_pos, w_stat, w_read = g[p + 'pos'], g[p + 'stat'], g[p + 'read']
            else:
                w_pos, w_stat, w_read = rc.golden_block(g, k)
            inv = dict((v, key) for key, v in lookup.items())
            got_ids = np.array([inv[v] for v in block['read_id']])
            want_ids = np.array(['read_s%d' % i for i in w_read])
            assert sorted(set(got_ids)) == sorted(set(want_ids))
            for rid in set(want_ids):
                a, w = got_ids == rid, want_ids == rid
                assert np.array_equal(block['pos'][a], w_pos[w])
                np.testing.assert_allclose(block['stat'][a], w_stat[w], rtol=1e-7, atol=1e-12)


def test_batched_reads_match_reference_results(g, served):
    from tombo_b200 import tombo_stats as ts
    std_ref, _ = _models()
    _serve_golden(g, served)
    for k in range(int(g['n_calls'])):
        st, reg, fm = rc.golden_settings(g, k)[:3]
        if st == 'model_compare':
            continue
        start, end = [int(x) for x in g['g%d_region' % reg]]
        reg_data = types.SimpleNamespace(start=start, end=end)
        reads = [_r_data('s%d' % i, served['s%d' % i]) for i in g['q%d_reads' % k]]
        if st == 'de_novo':
            got = ts.compute_de_novo_reads_stats(reads, std_ref, fm, reg_data)
        else:
            got = ts.compute_sample_compare_reads_stats(
                reads, g['q%d_ctrl_means' % k], g['q%d_ctrl_sds' % k], fm, reg_data)
        for j, (r, (msg, w_pv, w_pos)) in enumerate(zip(got, rc.golden_results(g, k))):
            if msg:
                assert isinstance(r, Exception) and str(r) == msg, (k, j, r, msg)
                continue
            assert not isinstance(r, Exception), (k, j, r)
            assert np.array_equal(r[1][st], w_pos)
            np.testing.assert_allclose(r[0][st], w_pv, rtol=1e-7, atol=0)


# 2. batched == single-read mirrors, bit for bit
def _fresh_reads(rs, n, reg_start, reg_end, K):
    reads = []
    for _ in range(n):
        a = int(rs.randint(reg_start - 150, reg_end + 20))
        b = a + int(rs.randint(1, 220))
        if b <= reg_start or a >= reg_end:                   # region reads overlap the region
            a = reg_start - int(rs.randint(0, 30))
            b = reg_start + int(rs.randint(1, 30))
        nb = b - a
        bases = rs.randint(0, 4, nb)
        if rs.uniform() < 0.05:
            bases[rs.randint(nb)] = 4                          # a non-ACGT base
        means = rs.normal(0.0, 1.0, nb)
        means[rs.uniform(size=nb) < 0.01] = np.nan
        reads.append(dict(start=a, end=b, strand='+-'[rs.randint(2)], means=means, bases=bases))
    return reads


def _assert_same_result(got, want):
    if isinstance(want, Exception):
        assert isinstance(got, Exception) and str(got) == str(want), (got, want)
        return
    assert not isinstance(got, Exception), (got, want)
    for d in (0, 1):
        (name, a), = got[d].items()
        assert _same(a, want[d][name]), (name, a, want[d][name])
    assert got[2] == want[2]


def _single(fn, *args):
    from tombo_b200 import tombo_helper as th
    try:
        return fn(*args)
    except th.TomboError as e:
        return e


def test_batched_equal_single_read_mirrors(served):
    from tombo_b200 import tombo_stats as ts
    std_ref, _ = _models()
    K = std_ref.kmer_width
    rs = np.random.RandomState(20261017)
    total = 0
    for it in range(24):
        reg_start = int(rs.randint(0, 10 ** 6))
        reg_end = reg_start + int(rs.randint(1, 400))
        fm = int(rs.choice([0, 1, 2, 3, 10, 33, 64])) if it else 64
        reads = _fresh_reads(rs, 90, reg_start, reg_end, K)
        rds = []
        for i, r in enumerate(reads):
            served['f%d_%d' % (it, i)] = r
            rds.append(_r_data('f%d_%d' % (it, i), r))
        reg = types.SimpleNamespace(start=reg_start, end=reg_end)
        got = ts.compute_de_novo_reads_stats(rds, std_ref, fm, reg)
        for r, o in zip(rds, got):
            _assert_same_result(o, _single(ts.compute_de_novo_read_stats, r, std_ref, fm, reg))
        n_ctrl = reg_end - reg_start + 2 * fm
        cm = rs.normal(0.0, 1.0, n_ctrl)
        cs = rs.uniform(0.5, 2.0, n_ctrl)
        cm[rs.uniform(size=n_ctrl) < 0.1] = np.nan
        if it % 6 == 5:
            cm[:] = np.nan                                       # no valid z-scores anywhere
        got = ts.compute_sample_compare_reads_stats(rds, cm, cs, fm, reg)
        for r, o in zip(rds, got):
            _assert_same_result(o, _single(ts.compute_sample_compare_read_stats, r, cm, cs, fm, reg))
        total += len(rds)
    assert total >= 2000


# 3. fused counters
def test_fused_counters_equal_downloaded_statistics(served):
    from tombo_b200 import _lib, tombo_stats as ts
    std_ref, _ = _models()
    rs = np.random.RandomState(7)
    reg = types.SimpleNamespace(start=5000, end=5300)
    reads = _fresh_reads(rs, 200, reg.start, reg.end, std_ref.kmer_width)
    rds = []
    for i, r in enumerate(reads):
        served['u%d' % i] = r
        rds.append(_r_data('u%d' % i, r))
    ctx = _lib.get_context()
    for lower in (None, 0.01):
        res = ts.compute_de_novo_reads_stats(rds, std_ref, 2, reg)
        ctx.region_stats_begin(reg.start, reg.end - reg.start)
        ctx.region_stats_add_tests(0.05, lower)
        fused = ctx.region_counts_get()
        ok = [r for r in res if not isinstance(r, Exception)]
        st = np.concatenate([r[0]['de_novo'] for r in ok])
        pos = np.concatenate([r[1]['de_novo'] for r in ok])
        ctx.region_stats_begin(reg.start, reg.end - reg.start)
        ctx.region_stats_add(st, pos, 0.05, lower, 1)
        assert np.array_equal(fused, ctx.region_counts_get())
        # reads split over two calls sum to the same counters
        ctx.region_stats_begin(reg.start, reg.end - reg.start)
        ts.compute_de_novo_reads_stats(rds[:77], std_ref, 2, reg)
        ctx.region_stats_add_tests(0.05, lower)
        ts.compute_de_novo_reads_stats(rds[77:], std_ref, 2, reg)
        ctx.region_stats_add_tests(0.05, lower)
        assert np.array_equal(fused, ctx.region_counts_get())
    cm, cs = rs.normal(0, 1, 302), rs.uniform(0.5, 2, 302)
    res = ts.compute_sample_compare_reads_stats(rds, cm, cs, 1, reg)
    ctx.region_stats_begin(reg.start, reg.end - reg.start)
    ctx.region_stats_add_tests(0.05)
    fused = ctx.region_counts_get()
    ok = [r for r in res if not isinstance(r, Exception)]
    ctx.region_stats_begin(reg.start, reg.end - reg.start)
    ctx.region_stats_add(np.concatenate([r[0]['sample_compare'] for r in ok]),
                         np.concatenate([r[1]['sample_compare'] for r in ok]), 0.05, None, 1)
    assert np.array_equal(fused, ctx.region_counts_get())


# 4. resident de novo
def test_resident_de_novo_equals_host_arrays(ctx, RPcls):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    kmeans, ksds = syn.kmer_table(kmer_ref)
    K = len(kmer_ref[0][0])
    ctx.set_model(kmeans, ksds, K, cpos)
    n = 600
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, n, 200, 20261018)
    failed = (3, 301)
    for r in failed:
        raw[raw_off[r]:raw_off[r + 1]] = 480.0
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    pol = _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    res = ctx.batch_download()
    ok = res['status'] == 0
    assert not ok[list(failed)].any()
    start = (np.arange(n, dtype=np.int64) * 37) % 3001
    strand = (np.arange(n) % 3 - 1).astype(np.int8)
    nm, mo = res['norm_mean'], res['base_off']
    for fm, reg in ((1, (800, 2600)), (0, (0, 10 ** 6)), (10, (1500, 1510))):
        pv, pos, off, st = ctx.batch_de_novo_region(start, strand, fm, *reg)
        host = ctx.de_novo_region_stats(nm, mo, seq, seq_off, start, np.where(ok, strand, -1),
                                        fm, *reg)
        assert np.array_equal(st[~ok], res['status'][~ok])
        assert np.array_equal(np.where(ok, st, 0), host[3])
        for r in np.nonzero(ok)[0]:
            a, b = off[r], off[r + 1]
            ha, hb = host[2][r], host[2][r + 1]
            assert _same(pv[a:b], host[0][ha:hb]) and _same(pos[a:b], host[1][ha:hb])
        for r in np.nonzero(~ok)[0]:
            assert np.isnan(pv[off[r]:off[r + 1]]).all()
        # resident statistics feed the counters as the host-array call's do
        ctx.batch_de_novo_region(start, strand, fm, *reg, download=False)
        ctx.region_stats_begin(reg[0], min(reg[1] - reg[0], 10 ** 4))
        ctx.region_stats_add_tests(0.05)
        fused = ctx.region_counts_get()
        ctx.de_novo_region_stats(nm, mo, seq, seq_off, start, np.where(ok, strand, -1), fm, *reg)
        ctx.region_stats_begin(reg[0], min(reg[1] - reg[0], 10 ** 4))
        ctx.region_stats_add_tests(0.05)
        assert np.array_equal(fused, ctx.region_counts_get())
    t = ctx.last_timing()
    assert t[0] > 0


# 5. invalid arguments and buffer isolation
def test_invalid_arguments(ctx):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    kmeans, ksds = syn.kmer_table(kmer_ref)
    K = len(kmer_ref[0][0])
    fresh = _lib.Context(ctx.device)
    nm = np.zeros(20)
    mo = np.array([0, 20], dtype=np.int64)
    sq = np.zeros(20 + K - 1, dtype=np.uint8)
    so = np.array([0, 20 + K - 1], dtype=np.int64)
    st = np.array([0], dtype=np.int64)
    with pytest.raises(_lib.TomboB200Error):          # no model set
        fresh.de_novo_region_stats(nm, mo, sq, so, st, [0], 1, 0, 100)
    with pytest.raises(_lib.TomboB200Error):          # no region call yet
        fresh.region_stats_begin(0, 10)
        fresh.region_stats_add_tests(0.05)
    fresh.close()
    ctx.set_model(kmeans, ksds, K, cpos)
    ok = ctx.de_novo_region_stats(nm, mo, sq, so, st, [0], 1, 0, 100)
    assert ok[3][0] == 0
    bad = [dict(strand=[2]), dict(strand=[-2]), dict(fm_offset=65), dict(fm_offset=-1),
           dict(reg_end=0), dict(reg_end=-5), dict(seq_off=np.array([0, 20 + K], dtype=np.int64))]
    for b in bad:
        kw = dict(strand=[0], fm_offset=1, reg_start=0, reg_end=100, seq_off=so)
        kw.update(b)
        with pytest.raises(_lib.TomboB200Error):
            ctx.de_novo_region_stats(nm, mo, sq, kw['seq_off'], st, kw['strand'], kw['fm_offset'],
                                     kw['reg_start'], kw['reg_end'])
    cm = np.zeros(102)
    for b in (dict(strand=[3]), dict(fm=65), dict(reg_end=0)):
        kw = dict(strand=[0], fm=1, reg_end=100)
        kw.update(b)
        with pytest.raises((_lib.TomboB200Error, ValueError)):
            ctx.sample_compare_region_stats(nm, mo, st, kw['strand'], cm, cm, kw['fm'], 0,
                                            kw['reg_end'])
    rc_ = ctx.lib.tb2_sample_compare_region_stats(
        ctx.handle, 1, _lib.ptr(nm, _lib.f64), _lib.ptr(mo, _lib.i64), _lib.ptr(st, _lib.i64),
        _lib.ptr(np.zeros(1, np.int8), _lib.C.c_int8), None, None, 1, 0, 100, None, None,
        _lib.ptr(np.zeros(2, np.int64), _lib.i64), None)
    assert rc_ == 201


def test_other_device_results_survive(ctx, RPcls):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    kmeans, ksds = syn.kmer_table(kmer_ref)
    K = len(kmer_ref[0][0])
    ctx.set_model(kmeans, ksds, K, cpos)
    ctx.set_alt_model(np.full((4 ** K, K), 1.0), K)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 64, 200, 99)
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    pol = _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    before = {k: v.copy() for k, v in ctx.batch_download().items() if isinstance(v, np.ndarray)}
    start = np.arange(64, dtype=np.int64) * 11
    ctx.batch_alt_llr(start, 1)
    llr_before = [a.copy() for a in ctx.batch_llr_download()]
    ctx.region_stats_begin(0, 2000)
    ctx.region_stats_add(np.array([0.5, 0.01]), np.array([3, 4]), 0.05, None, 1)
    cnt_before = ctx.region_counts_get()
    lv = np.random.RandomState(1).normal(0, 1, 300)
    kde_before = ctx.kernel_densities(lv, np.array([0, 300]), np.linspace(-3, 3, 50), 0.3)
    med_before = ctx.kmer_medians(8, np.arange(300) % 8, lv, np.abs(lv))
    # the new calls
    res = ctx.batch_download()
    strand = (np.arange(64) % 2).astype(np.int8)
    ctx.de_novo_region_stats(res['norm_mean'], res['base_off'], seq, seq_off, start, strand, 2, 0, 900)
    ctx.sample_compare_region_stats(res['norm_mean'], res['base_off'], start, strand,
                                    np.zeros(904), np.ones(904), 2, 0, 900)
    ctx.batch_de_novo_region(start, strand, 2, 0, 900, download=False)
    # open counters untouched until add_tests
    assert np.array_equal(ctx.region_counts_get(), cnt_before)
    after = ctx.batch_download()
    for k, v in before.items():
        assert np.array_equal(after[k], v, equal_nan=True), k
    for a, b in zip(ctx.batch_llr_download(), llr_before):
        assert np.array_equal(a, b, equal_nan=True)
    kde_after = ctx.kernel_densities(lv, np.array([0, 300]), np.linspace(-3, 3, 50), 0.3)
    for a, b in zip(kde_after, kde_before):
        assert np.array_equal(a, b, equal_nan=True)
    for a, b in zip(ctx.kmer_medians(8, np.arange(300) % 8, lv, np.abs(lv)), med_before):
        assert np.array_equal(a, b, equal_nan=True)
