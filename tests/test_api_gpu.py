"""GPU: the drop-in Python API (tombo_b200.resquiggle / tombo_stats / tombo_helper)
used the way the reference's own API example uses it (tombo/__init__.py:66-83)."""
import numpy as np
import pytest

import golden_util as gu
import stats_cases as sc

pytestmark = pytest.mark.gpu


def _setup(kind='DNA', aln=None):
    from tombo_b200 import tombo_helper as th, tombo_stats as ts, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    sst = th.seqSampleType(kind, kind == 'RNA')
    p = ts.load_resquiggle_parameters(sst, aln)
    sp = ts.load_resquiggle_parameters(sst, aln, use_save_bandwidth=True)
    return th, ts, syn, kmer_ref, cpos, std_ref, sst, p, sp


def _map_res(th, raw, seq, **kw):
    return th.resquiggleResults(
        align_info=th.alignInfo('r', 'BaseCalled_template', 0, 0, 0, 0, len(seq), 0),
        genome_loc=th.genomeLocation(0, '+', 'chr'), genome_seq=seq, mean_q_score=10.0,
        raw_signal=raw, **kw)


@pytest.mark.parametrize('name', ['dna_adapt4k', 'dna_rescue', 'rna_8k'])
def test_resquiggle_reads_matches_reference_goldens(name):
    from tombo_b200 import resquiggle
    g = gu.load(name)
    kind, kmer_ref, cpos, reads = gu.reads_of(g)
    aln = tuple(g['aln']) if g['aln'].shape[0] else None
    if aln is not None:
        aln = tuple(float(a) if i in (0, 1, 4) else int(a) for i, a in enumerate(aln))
    th, ts, syn, _, _, std_ref, sst, p, sp = _setup(kind, aln)
    mrs = [_map_res(th, r.raw, r.genome_seq) for r in reads]
    out = resquiggle.resquiggle_reads(mrs, std_ref, p, sp, outlier_thresh=5.0,
                                      seq_samp_type=sst)
    for i, res in enumerate(out):
        e = gu.expected(g, i)
        if e['message']:
            assert isinstance(res, th.TomboError) and str(res) == e['message']
            continue
        assert np.array_equal(res.segs, e['segs'])
        assert res.read_start_rel_to_raw == e['read_start_rel_to_raw']
        assert res.scale_values.shift == e['shift'] and res.scale_values.scale == e['scale']
        assert res.sig_match_score == e['sig_match_score']
        assert res.norm_params_changed == e['norm_params_changed']
        assert len(res.genome_seq) == res.segs.shape[0] - 1
        assert res.raw_signal.shape[0] == res.segs[-1]


def test_resquiggle_read_single_call_and_iteration(orc, RPcls):
    from tombo_b200 import resquiggle
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 300, 2500, 100)
    th, ts, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup('DNA', aln)
    pol = orc.policy('DNA')
    for seed in (21000, 21001, 21002):
        r = syn.make_read(kmer_ref, cpos, 500, seed)
        rm, rsd = gu.levels(r.genome_seq, kmer_ref)
        mr = _map_res(th, r.raw, r.genome_seq)
        res = resquiggle.resquiggle_read(mr, std_ref, p, outlier_thresh=5.0, seq_samp_type=sst)
        o = orc.resquiggle_read(r.raw, rm, rsd, p, pol)
        assert o['status'] == 0
        assert np.array_equal(res.segs, o['segs'])
        assert res.read_start_rel_to_raw == o['read_start_rel_to_raw']
        assert res.scale_values[:4] == tuple(o['scale_values'][:4])
        assert res.sig_match_score == o['sig_match_score']
        assert np.array_equal(res.raw_signal, o['norm_signal'])
        assert res.norm_params_changed == o['norm_params_changed']
        # second call as the worker does it (resquiggle.py:1499-1502)
        res2 = resquiggle.resquiggle_read(
            mr._replace(scale_values=res.scale_values), std_ref, p, 5.0, all_raw_signal=r.raw,
            seq_samp_type=sst)
        o2 = orc.resquiggle_read(r.raw, rm, rsd, p, pol, scale_values=o['scale_values'],
                                 first_call=False)
        assert np.array_equal(res2.segs, o2['segs'])
        assert res2.scale_values[:4] == tuple(o2['scale_values'][:4])
        assert np.array_equal(res2.raw_signal, o2['norm_signal'])


def test_individual_steps_like_reference_api_example():
    """tombo/__init__.py:66-83: segment_signal -> compute_base_means ->
    find_adaptive_base_assignment -> resolve_skipped_bases_with_raw"""
    from tombo_b200 import resquiggle
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 300, 2500, 100)
    th, ts, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup('DNA', aln)
    r = syn.make_read(kmer_ref, cpos, 500, 22000)
    mr = _map_res(th, r.raw, r.genome_seq)
    full = resquiggle.resquiggle_read(mr, std_ref, p, outlier_thresh=5.0, skip_seq_scaling=True)
    num_events = ts.compute_num_events(r.raw.shape[0], len(r.genome_seq) - std_ref.kmer_width + 1,
                                       p.mean_obs_per_event)
    valid_cpts, norm_signal, scale_values = resquiggle.segment_signal(mr, num_events, p, 5.0)
    event_means = ts.compute_base_means(norm_signal, valid_cpts)
    dp = resquiggle.find_adaptive_base_assignment(valid_cpts, event_means, p, std_ref,
                                                  r.genome_seq)
    ns = norm_signal[dp.read_start_rel_to_raw:dp.read_start_rel_to_raw + dp.segs[-1]]
    segs = resquiggle.resolve_skipped_bases_with_raw(dp, ns, p)
    assert np.array_equal(segs, full.segs)
    assert dp.read_start_rel_to_raw == full.read_start_rel_to_raw
    assert np.array_equal(ns, full.raw_signal)
    assert scale_values.shift == full.scale_values.shift
    score = ts.get_read_seg_score(ts.compute_base_means(ns, segs), dp.ref_means, dp.ref_sds)
    assert score == full.sig_match_score
    # Theil-Sen rescaling step on its own
    sh, sc, shc, scc = ts.calc_kmer_fitted_shift_scale(
        scale_values.shift, scale_values.scale, ts.compute_base_means(ns, segs), dp.ref_means)
    full2 = resquiggle.resquiggle_read(mr, std_ref, p, outlier_thresh=5.0)
    assert (sh, sc) == (full2.scale_values.shift, full2.scale_values.scale)


def test_static_and_start_find_mirrors(orc):
    from tombo_b200 import resquiggle
    th, ts, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup('DNA')
    r = syn.make_read(kmer_ref, cpos, 1500, 23000)
    rm, rsd = gu.levels(r.genome_seq, kmer_ref)
    _, norm, _ = orc.normalize_raw_signal(r.raw, outlier_thresh=5.0)
    ne = ts.compute_num_events(r.raw.shape[0], 1500, 5)
    _, cpts = orc.valid_cpts_w_cap(norm, 3, 5, ne)
    em = orc.new_means(norm, cpts)
    s0, loc0, epb0 = orc.find_seq_start_in_events(em, rm, rsd, p, 250, 750, 1.1)
    loc1, epb1 = resquiggle.find_seq_start_in_events(em, rm, rsd, p, 250, 750, sst)
    assert s0 == 0 and (loc0, epb0) == (loc1, epb1)
    # static band over a short stretch
    em_s, rm_s, rs_s = em[:700], rm[:330], rsd[:330]
    s0, tb0 = orc.find_static_base_assignment(em_s, rm_s, rs_s, p)
    tb1 = resquiggle.find_static_base_assignment(em_s, rm_s, rs_s, p)
    assert s0 == 0 and np.array_equal(tb0, tb1)


def test_errors_are_tombo_errors_with_reference_messages():
    from tombo_b200 import resquiggle
    th, ts, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup('DNA')
    r = syn.make_read(kmer_ref, cpos, 2000, 24000)
    mr = _map_res(th, r.raw, r.genome_seq[:12])
    with pytest.raises(th.TomboError, match='Too much raw signal for mapped sequence'):
        resquiggle.resquiggle_read(mr, std_ref, p, outlier_thresh=5.0)
    with pytest.raises(th.TomboError, match='Must have raw signal'):
        resquiggle.resquiggle_read(mr._replace(raw_signal=None), std_ref, p)
    with pytest.raises(th.TomboError, match='Fewer changepoints found than requested'):
        th.valid_cpts_w_cap(np.random.RandomState(0).normal(0, 1, 300), 3, 5, 100)
    bad = _map_res(th, r.raw, 'ACGTNACGTACGTACGTACGTAAAAC' * 20)
    out = resquiggle.resquiggle_reads([bad], std_ref, p, sp)
    assert isinstance(out[0], th.TomboError)
    assert 'Invalid sequence' in str(out[0])


def test_compute_alt_model_read_stats_matches_reference():
    from unittest import mock
    from tombo_b200 import resquiggle
    g = gu.load('llr_5mc')
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    th, ts, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup('DNA', aln)
    alt_ref = ts.AltModel(kmer_ref=syn.make_alt_kmer_ref(kmer_ref, 'C', seed=1),
                          central_pos=cpos, alt_base='C', name='5mC')
    reads = [syn.make_read(kmer_ref, cpos, int(g['nbases']), int(g['seed0']) + i)
             for i in range(int(g['nreads']))]
    out = resquiggle.resquiggle_reads([_map_res(th, r.raw, r.genome_seq) for r in reads],
                                      std_ref, p, sp)
    for i, res in enumerate(out):
        norm_mean = ts.compute_base_means(res.raw_signal, res.segs)
        bases = np.array(list(res.genome_seq), dtype='S1')
        r_data = th.readData(start=1000 * i, end=1000 * i + len(res.genome_seq), filtered=False,
                             read_start_rel_to_raw=0, strand='+', fn='x', corr_group='g',
                             rna=False)
        with mock.patch.object(th, 'get_multiple_slots_read_centric',
                               lambda *a, **k: (norm_mean, bases)):
            llr, pos, _ = ts.compute_alt_model_read_stats(r_data, std_ref, [('5mC', alt_ref)])
            llr_s, _, _ = ts.compute_alt_model_read_stats(r_data, std_ref, [('5mC', alt_ref)],
                                                          use_standard_llhr=True)
        a, b = int(g['site_off'][i]), int(g['site_off'][i + 1])
        assert np.array_equal(pos['5mC'], g['pos'][a:b])
        assert np.array_equal(llr_s['5mC'], g['llr_standard'][a:b])
        _, _, _, s_abs = sc.llr_of_genome_read(norm_mean, res.genome_seq, 1000 * i, kmer_ref,
                                               cpos, 0)
        sc.assert_llr(llr['5mC'], g['llr_scaled'][a:b], s_abs, 0, len(kmer_ref[0][0]))


def test_identify_stalls_matches_oracle(orc):
    from tombo_b200 import tombo_stats as ts, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('RNA', 0)
    r = syn.make_read(kmer_ref, cpos, 270, 25000, kind='RNA')
    raw = r.raw[::-1].copy()
    raw[3000:3600] = raw[3000] + np.random.RandomState(1).normal(0, 3, 600)  # planted stall
    got = ts.identify_stalls(raw)
    exp = orc.identify_stalls(raw)
    assert len(exp) >= 1
    assert np.array_equal(np.array(got).reshape(-1, 2), exp)


def test_read_batcher_streams_the_golden_reads_in_order():
    """tombo_b200.worker (SURVEY 8(f)-4) over the real backend: small batches, results in
    submission order, failures as the reference's wire messages"""
    from tombo_b200 import worker
    g = gu.load('dna_rescue')
    kind, kmer_ref, cpos, reads = gu.reads_of(g)
    aln = tuple(float(a) if i in (0, 1, 4) else int(a) for i, a in enumerate(tuple(g['aln'])))
    th, ts, syn, _, _, std_ref, sst, p, sp = _setup(kind, aln)
    stream = ((_map_res(th, r.raw, r.genome_seq), 'read%d.fast5' % i) for i, r in enumerate(reads))
    fs = worker.FailureSummary()
    out = list(worker.resquiggle_stream(stream, std_ref, p, sp, max_reads=3,
                                        outlier_thresh=5.0, seq_samp_type=sst))
    assert [fn for fn, _ in out] == ['read%d.fast5' % i for i in range(len(reads))]
    for i, (fn, msg) in enumerate(out):
        fs.record(msg)
        e = gu.expected(g, i)
        if e['message']:
            assert msg == [True, [e['message'], fn, True]]
        else:
            assert msg[0] is False and np.array_equal(msg[1].segs, e['segs'])
    assert fs.num_processed == len(reads)
