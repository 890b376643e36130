"""GPU: resquiggle at caller-chosen parameters.  Every parameter point of
tests/golden/rsqgl_params.npz (outputs of the unmodified reference) through the pipelined
batch (tb2_resquiggle_batch), the staged batch (upload / compute / download) and, for a few
points, the Python API; fresh-seed sweeps of every point against the C oracle; and the
capacity edges of the adaptive and static bands (DESIGN.md section 5: a band wider than 8192
cells is reported as TB2_ERR_CAPACITY for that read, never answered differently).

The file takes about 3.2 minutes on one H100 80GB HBM3 (700 W power limit) with 8 host
cores, most of it the oracle's CPU time for the sweeps."""
import numpy as np
import pytest

import params_cases as pc

pytestmark = pytest.mark.gpu

POINTS = [p['name'] for p in pc.points()]
CAPACITY = 202


@pytest.fixture(scope='module')
def golden():
    g = pc.golden()
    assert list(g['p_name']) == POINTS
    return g


def _flatten(reads):
    from tombo_b200 import synthetic as syn
    raws = [np.asarray(r.raw) for r in reads]
    raw_off = np.concatenate([[0], np.cumsum([x.shape[0] for x in raws])]).astype(np.int64)
    codes = [syn.seq_to_codes(r.genome_seq) for r in reads]
    seq_off = np.concatenate([[0], np.cumsum([c.shape[0] for c in codes])]).astype(np.int64)
    return np.concatenate(raws), raw_off, np.concatenate(codes), seq_off


def _same(a, b):
    return a == b or (np.isnan(a) and np.isnan(b))


def _check_batch(res, g, j):
    from tombo_b200 import _lib
    a0 = int(g['p_read_off'][j])
    for k in range(int(g['p_read_off'][j + 1]) - a0):
        e = pc.expected(g, a0 + k)
        assert _lib.status_message(res['status'][k]) == e['message'], (k, res['status'][k])
        assert bool(res['flags'][k] & 2) == e['rescued'], k
        if e['message']:
            continue
        a, b = res['seg_off'][k], res['seg_off'][k + 1]
        assert np.array_equal(res['segs'][a:b], e['segs']), k
        assert res['read_start_rel_to_raw'][k] == e['read_start_rel_to_raw'], k
        for c, key in enumerate(('shift', 'scale', 'lower_lim', 'upper_lim')):
            assert _same(res['scale_values'][k, c], e[key]), (k, key)
        assert res['sig_match_score'][k] == e['sig_match_score'], k
        assert res['n_iters'][k] == e['n_iters'], k
        assert bool(res['flags'][k] & 1) == e['norm_params_changed'], k


@pytest.mark.parametrize('name', POINTS)
def test_golden_point_pipelined_and_staged(ctx, RPcls, golden, name):
    """the reference's result at every point: the pipelined batch and the staged batch"""
    from tombo_b200 import _lib, synthetic as syn
    g = golden
    j = POINTS.index(name)
    pt = pc.point_of(g, j, RPcls)
    kmer_ref, cpos, reads = pc.reads_of_point(g, j)
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, len(kmer_ref[0][0]), cpos)
    raw, raw_off, seq, seq_off = _flatten(reads)
    pol = _lib.make_policy(pt['kind'], **pt['pol'])
    _check_batch(ctx.resquiggle_batch(raw, raw_off, seq, seq_off, pt['rp'], pt['sp'], pol), g, j)
    ctx.batch_upload(raw, raw_off, seq, seq_off, pt['rp'], pol)
    ctx.batch_compute(pt['rp'], pt['sp'], pol)
    _check_batch(ctx.batch_download(), g, j)


API_POINTS = ['mhz_none', 'bw_2049', 'start_bw_lt_n_bases', 'outlier_none', 'const_scale_dna',
              'model_sd_rna', 'save_bw_2100']


@pytest.mark.parametrize('name', API_POINTS)
def test_golden_point_python_api(RPcls, golden, name):
    """resquiggle_reads (the worker policy) with load_resquiggle_parameters of the point and a
    TomboModel, against the reference's result"""
    from tombo_b200 import resquiggle, tombo_helper as th, tombo_stats as ts
    g = golden
    j = POINTS.index(name)
    pt = pc.point_of(g, j, RPcls)
    kmer_ref, cpos, reads = pc.reads_of_point(g, j)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    sst = th.seqSampleType(pt['kind'], pt['kind'] == 'RNA')
    p = ts.load_resquiggle_parameters(sst, pt['aln'], pt['seg'])
    sp = ts.load_resquiggle_parameters(sst, pt['aln'], pt['seg'], use_save_bandwidth=True)
    mrs = [th.resquiggleResults(
        align_info=th.alignInfo('r%d' % k, 'BaseCalled_template', 0, 0, 0, 0, len(r.genome_seq), 0),
        genome_loc=th.genomeLocation(0, '+', 'chr'), genome_seq=r.genome_seq, mean_q_score=10.0,
        raw_signal=r.raw) for k, r in enumerate(reads)]
    kw = dict(pt['pol'])
    out = resquiggle.resquiggle_reads(mrs, std_ref, p, sp, seq_samp_type=sst, **kw)
    a0 = int(g['p_read_off'][j])
    for k, res in enumerate(out):
        e = pc.expected(g, a0 + k)
        if e['message']:
            assert isinstance(res, th.TomboError) and str(res) == e['message'], (k, res)
            continue
        assert not isinstance(res, Exception), (k, res)
        assert np.array_equal(res.segs, e['segs']), k
        assert res.read_start_rel_to_raw == e['read_start_rel_to_raw'], k
        sv = res.scale_values
        assert sv.shift == e['shift'] and sv.scale == e['scale'], k
        for key in ('lower_lim', 'upper_lim'):
            v = getattr(sv, key)
            assert (v is None and np.isnan(e[key])) or v == e[key], (k, key, v, e[key])
        assert res.sig_match_score == e['sig_match_score'], k
        assert res.norm_params_changed == e['norm_params_changed'], k


def test_golden_iters_1_single_calls(RPcls, golden):
    """max_scaling_iters 1 without a rescue is one resquiggle_read call: read by read.  Reads
    of more than 1000 bases are left out: their Theil-Sen sub-sample is keyed by the read's
    position in the batch, and a single call is read 0"""
    from tombo_b200 import resquiggle, tombo_helper as th, tombo_stats as ts
    g = golden
    j = POINTS.index('iters_1')
    pt = pc.point_of(g, j, RPcls)
    kmer_ref, cpos, reads = pc.reads_of_point(g, j)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    p = ts.load_resquiggle_parameters(th.seqSampleType('DNA', False), pt['aln'], pt['seg'])
    n = 0
    for k, r in enumerate(reads):
        e = pc.expected(g, int(g['p_read_off'][j]) + k)
        if e['message'] or e['rescued'] or len(r.genome_seq) - 5 > 1000:
            continue
        mr = th.resquiggleResults(
            align_info=th.alignInfo('r', 'BaseCalled_template', 0, 0, 0, 0, len(r.genome_seq), 0),
            genome_loc=th.genomeLocation(0, '+', 'chr'), genome_seq=r.genome_seq,
            mean_q_score=10.0, raw_signal=r.raw)
        res = resquiggle.resquiggle_read(mr, std_ref, p, outlier_thresh=5.0)
        assert np.array_equal(res.segs, e['segs']), k
        assert res.scale_values.shift == e['shift'] and res.sig_match_score == e['sig_match_score']
        n += 1
    assert n >= 3


# ---------------------------------------------------------------- fresh-seed sweeps
def _sweep_batch(pt, n_reads, seed):
    """n_reads fresh reads for point pt: lengths uniform over the point's range (so short
    reads take the static band and long ones the adaptive band), stalls where the point
    plants them"""
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref(pt['kind'], 0, sd_range=pt['sd_range'])
    lo, hi = min(pt['nbases']), max(pt['nbases'])
    rs = np.random.RandomState(seed)
    nbs = rs.randint(lo, hi + 1, n_reads)
    if pt['name'].startswith('bw_'):
        # every other read long enough for the adaptive band the point is about
        nbs[1::2] = rs.randint(pc.adaptive_nbases(pt['aln'][2]), hi + 1, n_reads // 2)
    kw = {}
    if pt['stall']:
        kw = dict(stall_every=2, stall_extra=max(s[1] for s in pt['stall'].values()))
    batch = syn.make_read_batch(kmer_ref, n_reads, nbs, seed, kind=pt['kind'], int16=pt['int16'],
                                **kw)
    return kmer_ref, cpos, batch


def _n_reads(pt):
    """128 reads per point; at the lane-chunk bandwidths (2048 and up) the oracle runs on at
    most 8 threads, since each thread holds a (bases x band) move table of up to ~0.7 GB"""
    return 128


def _sweep(ctx, orc, RPcls, pt, seed):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos, (raw, raw_off, seq, seq_off) = _sweep_batch(pt, _n_reads(pt), seed)
    k = len(kmer_ref[0][0])
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, k, cpos)
    rna = pt['kind'] == 'RNA'
    rp, sp = RPcls(pt['aln'], pt['seg'], rna=rna), RPcls(pt['aln'], pt['seg'], rna=rna, save=True)
    res = ctx.resquiggle_batch(raw, raw_off, seq, seq_off, rp, sp,
                               _lib.make_policy(pt['kind'], subsample_seed=seed, **pt['pol']))
    out = orc.run_batch(raw, raw_off, seq, seq_off, means, sds, k, rp, sp,
                        orc.policy(pt['kind'], subsample_seed=seed, **pt['pol']),
                        threads=8 if pt['aln'][2] >= 2048 else None)
    bad = orc.compare_batch(res, out)
    assert not bad, (pt['name'], bad[:10])
    return res


# every read fails: more events requested than changepoints of at least min_obs samples exist
ALL_FAIL = {'min_obs_6', 'min_obs_10', 'mean_obs_1', 'mean_obs_3'}


@pytest.mark.parametrize('name', POINTS)
def test_sweep_point_against_oracle(ctx, orc, RPcls, name):
    """fresh seeds at every point, bit for bit against the oracle, and what the point is for:
    the adaptive share and the engine side at a boundary bandwidth, rescues at the save
    bandwidth, failures where the parameter causes them"""
    pt = [p for p in pc.points() if p['name'] == name][0]
    res = _sweep(ctx, orc, RPcls, pt, 50000 + POINTS.index(name))
    ok = res['status'] == 0
    if name.startswith('bw_'):
        W = pt['aln'][2]
        eng = pc.engine_of(W)
        assert eng[0] != 'capacity'
        if W in pc.BOUNDARY_BWS:
            # the boundaries: W on the wider side of W - 1 or the narrower side of W + 1
            assert pc.engine_of(W - 1) != eng or pc.engine_of(W + 1) != eng, W
        adaptive = ok & (res['flags'] & 4 == 0)
        assert adaptive.mean() > 0.3, (W, adaptive.mean())
    if name == 'save_bw_2100':
        assert (ok & (res['flags'] & 2 != 0) & (res['flags'] & 4 == 0)).any(), \
            'no adaptive rescue at the save bandwidth'
    if name == 'bbt_half_bw_m1':
        # a traceback within 149 cells of the band edge fails: rescued with the save band
        assert (res['flags'] & 2 != 0).any(), name
    if name in ALL_FAIL:
        assert not ok.any(), (name, ok.sum())
    else:
        assert ok.mean() > 0.5, (name, ok.mean())


# ---------------------------------------------------------------- capacity edges
def _capacity_batch(ctx, orc, RPcls, aln, nbs, seed, oracle_reads=None):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, 6, cpos)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, len(nbs), np.asarray(nbs), seed)
    rp, sp = RPcls(aln, pc.DNA_SEG), RPcls(aln, pc.DNA_SEG, save=True)
    res = ctx.resquiggle_batch(raw, raw_off, seq, seq_off, rp, sp,
                               _lib.make_policy('DNA', subsample_seed=seed))
    out = orc.run_batch(raw, raw_off, seq, seq_off, means, sds, 6, rp, sp,
                        orc.policy('DNA', subsample_seed=seed), indices=oracle_reads, threads=4)
    return res, out


@pytest.mark.parametrize('W', [8192, 8193])
def test_adaptive_band_capacity_edge(ctx, orc, RPcls, W):
    """an adaptive band of 8192 cells equals the oracle; at 8193 the reads that take the
    adaptive band report TB2_ERR_CAPACITY (final, not rescued) and the short reads of the
    same batch (static band) equal the oracle"""
    aln = (4.2, 4.2, W, 1500, 20.0, 40, 750, 2500, 250)
    nb_long = pc.adaptive_nbases(W)
    nbs = [nb_long, 444, nb_long + 200, 600, nb_long + 100, 300]
    res, out = _capacity_batch(ctx, orc, RPcls, aln, nbs, 51000 + W)
    cap = res['status'] == CAPACITY
    if W == 8192:
        assert not cap.any()
        assert not orc.compare_batch(res, out)
        assert (res['flags'][::2] & 4 == 0).all() and (res['status'] == 0).all()
    else:
        assert cap[::2].all(), res['status']
        assert all(out[i]['status'] == 0 for i in range(0, len(nbs), 2))
        assert not (res['flags'][cap] & 2).any(), 'a capacity overrun was rescued'
        rest = {i: o for i, o in out.items() if not cap[i]}
        assert len(rest) == 3 and not orc.compare_batch(res, rest)
        assert (res['status'][1::2] == 0).all() and (res['flags'][1::2] & 4 != 0).all()


def test_static_band_over_capacity(ctx, orc, RPcls):
    """a read too short for the start search of a very wide start window takes the static
    band over all its events; above 8192 cells that is TB2_ERR_CAPACITY on the device while
    the smaller reads of the batch equal the oracle"""
    aln = (4.2, 4.2, 300, 1500, 20.0, 40, 20000, 25000, 250)
    nbs = [6000, 444, 900]          # ~10800 events, a static band of ~9300 cells
    res, out = _capacity_batch(ctx, orc, RPcls, aln, nbs, 52000, oracle_reads=[1, 2])
    assert res['status'][0] == CAPACITY, res['status']
    assert not orc.compare_batch(res, out)
    assert (res['status'][1:] == 0).all() and (res['flags'][1:] & 4 != 0).all()
