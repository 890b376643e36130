"""tb2_kmer_level_summaries / tb2_kmer_medians on the device against their numpy
restatement (model_ref_cases.py), bit for bit, and the estimation mirrors end to end."""
import itertools

import numpy as np
import pytest

from tombo_b200 import _lib
from tombo_b200 import synthetic as syn
from tombo_b200 import tombo_helper as th
from tombo_b200 import tombo_stats as ts

import model_ref_cases as mc
from test_model_ref_cpu import run_case
from test_ctx_buffers_gpu import ALN, REG_LEN, REG_START, _context, batch, model  # noqa: F401

pytestmark = pytest.mark.gpu


def same(a, b):
    return np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize('name,kw', mc.extraction_cases(), ids=[c[0] for c in mc.extraction_cases()])
def test_extraction_bit_exact_vs_restatement(monkeypatch, name, kw):
    _, genome, reads, served = mc.make_inputs()
    dev, _ = run_case(name, kw, genome, reads, served)
    monkeypatch.setattr(_lib, 'get_context', lambda device=0: mc.RestatedContext())
    host, _ = run_case(name, kw, genome, reads, served)
    dc, dr = mc.flatten(dev)
    hc, hr = mc.flatten(host)
    assert np.array_equal(dc, hc) and same(dr, hr)


@pytest.mark.parametrize('seed', range(4))
@pytest.mark.parametrize('est_mean', [False, True])
def test_summaries_sweep(seed, est_mean):
    rs = np.random.RandomState(seed)
    n_pos, n_reads = 3000, int(rs.randint(1, 400))
    lens = rs.randint(0, 600, n_reads)
    st = rs.randint(-200, n_pos, n_reads).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    lv = np.round(rs.normal(0, 1, off[-1]), int(rs.randint(1, 4)))      # ties
    lv[rs.uniform(size=lv.shape[0]) < 0.02] = np.nan
    thr = int(rs.randint(0, 5))
    got = _lib.get_context().kmer_level_summaries(n_pos, (lv, off, st), thr, est_mean)
    want = mc.summaries(n_pos, (lv, off, st), thr, est_mean)
    for g, w in zip(got, want):
        assert same(g, w)


def test_summaries_above_shared_capacity():
    # 2500 reads over one position: the global-CSR path of k_ref_pos / k_mean_std_pos
    rs = np.random.RandomState(7)
    n = 2500
    lv = rs.normal(0, 1, n)
    reads = (lv, np.arange(n + 1, dtype=np.int64), np.zeros(n, dtype=np.int64))
    for est_mean in (False, True):
        got = _lib.get_context().kmer_level_summaries(2, reads, 0, est_mean)
        want = mc.summaries(2, reads, 0, est_mean)
        for g, w in zip(got, want):
            assert same(g, w)


@pytest.mark.parametrize('n_obs,n_keys', [(1, 1), (2, 1), (7, 3), (5000, 64), (9000, 2), (10 ** 6, 1)])
def test_medians_exact(n_obs, n_keys):
    rs = np.random.RandomState(n_obs)
    keys = rs.randint(0, n_keys, n_obs).astype(np.int64)
    lv, sd = np.round(rs.normal(0, 1, n_obs), 3), rs.uniform(0, 1, n_obs)
    got = _lib.get_context().kmer_medians(n_keys + 2, keys, lv, sd)
    if n_obs == 10 ** 6:
        cnt = np.bincount(keys, minlength=n_keys + 2)
        want = (cnt, np.array([np.median(lv)] + [np.nan] * 2), np.array([np.median(sd)] + [np.nan] * 2))
    else:
        want = mc.medians(n_keys + 2, keys, lv, sd)
    for g, w in zip(got, want):
        assert same(g, w)


def test_invalid_arguments():
    ctx = _lib.get_context()
    reads = (np.zeros(3), np.array([0, 3]), np.array([0]))
    for n_pos, thr in ((0, 1), (1 << 25, 1), (10, -1)):
        with pytest.raises(_lib.TomboB200Error, match='201'):
            ctx.kmer_level_summaries(n_pos, reads, thr)
    with pytest.raises(_lib.TomboB200Error, match='201'):
        ctx.kmer_level_summaries(10, (np.zeros(3), np.array([1, 3]), np.array([0])), 1)
    for keys, lv in (([5], [0.0]), ([-1], [0.0]), ([0], [np.nan])):
        with pytest.raises(_lib.TomboB200Error, match='201'):
            ctx.kmer_medians(5, keys, lv, [0.0])
    with pytest.raises(_lib.TomboB200Error, match='201'):
        ctx.kmer_medians(0, [], [], [])


def test_resident_state_survives(model, batch, RPcls):
    """a resident resquiggle batch, its LLRs, the region counters and KdeState's results are
    the same after both calls as before them"""
    raw, raw_off, seq, seq_off, read_start = batch
    rp, sp = RPcls(ALN), RPcls(ALN, save=True)
    pol = _lib.make_policy('DNA')
    ctx = _context(model)
    try:
        ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
        ctx.batch_compute(rp, sp, pol)
        base = {k: v.copy() for k, v in ctx.batch_download().items()}
        ctx.batch_alt_llr(read_start, 1)
        llr_base = [a.copy() for a in ctx.batch_llr_download()]
        ctx.region_stats_begin(REG_START, REG_LEN)
        ctx.region_stats_add_batch_llr(2.5, -1.5, 0)
        counts_ref = ctx.region_counts_get()
        rs = np.random.RandomState(3)
        lv = rs.normal(0, 1, 400)
        off, x = np.array([0, 200, 400]), np.linspace(-3, 3, 50)
        kde = ctx.kernel_densities(lv, off, x, 0.1)

        ctx.kmer_level_summaries(400, (lv, off, np.array([0, 100])), 0)
        ctx.kmer_medians(8, rs.randint(0, 8, 400), lv, lv)

        assert same(ctx.region_counts_get(), counts_ref)
        got = ctx.batch_download()
        for k in base:
            assert same(got[k], base[k]), k
        ctx.batch_alt_llr(read_start, 1)
        for a, b in zip(ctx.batch_llr_download(), llr_base):
            assert same(a, b)
        for a, b in zip(ctx.kernel_densities(lv, off, x, 0.1), kde):
            assert same(a, b)
    finally:
        ctx.close()


G = np.load(mc.__file__.replace('model_ref_cases.py', 'golden/model_ref.npz'))


def _kmers():
    return [''.join(k) for k in itertools.product('ACGT', repeat=mc.CFG['kmer_width'])]


def _model_arrays(ref):
    return np.stack([np.array([ref.means[k] for k in _kmers()]),
                     np.array([ref.sds[k] for k in _kmers()])])


def _sd_tol():
    """the median-mode sds' order bound (the model's sds are medians of them)"""
    return mc.order_tol(G['median_order'], G['median_rows'][:, 1]).max()


@pytest.fixture
def factors(monkeypatch):
    got = []
    orig = ts.calc_kmer_fitted_shift_scale

    def fit(*a, **k):
        res = orig(*a, **k)
        got.append(res[2:4])
        return res
    monkeypatch.setattr(ts, 'calc_kmer_fitted_shift_scale', fit)
    return got


def _check_centering(tag, ref, got_factors, stderr, const_sd=True):
    assert np.array_equal(np.array(got_factors).reshape(-1, 2), G[tag + '_factors'])
    after = _model_arrays(ref)
    want = G[tag + ('_after_const_sd' if const_sd else '_after')]
    assert np.array_equal(after[0], want[0])
    assert np.all(np.abs(after[1] - want[1]) <= _sd_tol())
    assert np.array_equal(np.random.get_state()[1], G[tag + '_rng_after'])
    assert np.random.get_state()[2] == G[tag + '_rng_pos']
    want_err = str(G[tag + '_stderr'])
    assert (mc.message(want_err) in stderr) if want_err else ('WARNING' not in stderr)


@pytest.mark.parametrize('kmer_specific_sd', [False, True])
def test_estimate_kmer_model_matches_reference(factors, capsys, kmer_specific_sd):
    """extraction, tabulation, the RNG hand-off to the centering shuffle, the per-read
    factors (60 reads, fewer than NUM_READS_TO_ADJUST_MODEL succeed: the warning) and the
    centered model with and without a constant sd"""
    cfg = mc.CFG
    _, _, reads, served = mc.make_inputs()
    up, dn = cfg['central_pos'], cfg['kmer_width'] - cfg['central_pos'] - 1
    np.random.seed(cfg['shuffle_seed'])
    with mc.serve(served):
        ref = ts.estimate_kmer_model(mc.Index(reads), cfg['cov_thresh'], up, dn, cfg['min_kmer_obs'],
                                     kmer_specific_sd, None, False, cfg['region_size'])
    _check_centering('center_dna_all', ref, factors, capsys.readouterr().err, not kmer_specific_sd)


@pytest.mark.parametrize('tag,rna', [('center_dna', False), ('center_rna', True)])
def test_center_model_to_median_norm_matches_reference(factors, capsys, tag, rna):
    """max_reads reads from the reference's starting model: DNA after the extraction's
    shuffles, RNA (event scaling with stall removal) from a fresh seed"""
    cfg = mc.CFG
    _, _, reads, served = mc.make_inputs(rna=rna)
    before = G[tag + '_before']
    init = ts.TomboModel(kmer_ref=list(zip(_kmers(), before[0], before[1])), central_pos=cfg['central_pos'])
    np.random.seed(cfg['shuffle_seed'])
    with mc.serve(served):
        if not rna:
            kw = dict(mc.extraction_cases()[0][1])
            ts.extract_kmer_levels(mc.Index(reads), **kw)
        ref = ts.center_model_to_median_norm(mc.Index(reads), init, cfg['center_reads'])
    _check_centering(tag, ref, factors, capsys.readouterr().err, const_sd=False)


def test_center_model_without_readable_reads_raises():
    cfg = mc.CFG
    _, _, reads, served = mc.make_inputs()
    before = G['center_none_before']
    init = ts.TomboModel(kmer_ref=list(zip(_kmers(), before[0], before[1])), central_pos=cfg['central_pos'])
    np.random.seed(cfg['shuffle_seed'])
    with mc.serve(served), pytest.raises(th.TomboError) as e:
        ts.center_model_to_median_norm(mc.Index(mc.unreadable(reads)), init, cfg['center_reads'])
    assert str(e.value) == mc.message(G['center_none_stderr'])
    assert np.array_equal(np.random.get_state()[1], G['center_none_rng_after'])


def test_estimate_motif_alt_model_matches_reference():
    cfg = mc.CFG
    _, _, reads, served = mc.make_inputs()
    up, dn = cfg['central_pos'], cfg['kmer_width'] - cfg['central_pos'] - 1
    with mc.serve(served):
        alt = ts.estimate_motif_alt_model(mc.Index(reads), 'CG:1', up, dn, None, cfg['min_kmer_obs'],
                                          cfg['cov_thresh'], None, cfg['region_size'])
    motif = th.TomboMotif('CG', 1)
    keys = [(k, o - 1) for k in _kmers() for o in motif.find_mod_poss(k)]
    tab = G['motif0_tab']
    assert alt.alt_base == 'C'
    assert np.array_equal(np.array([alt.means[k] for k in keys]), tab[:, 0])
    # _make_constant_sd: the median of the tabulated sds
    assert len(set(alt.sds.values())) == 1
    assert abs(next(iter(alt.sds.values())) - np.median(tab[:, 1])) <= _sd_tol()
