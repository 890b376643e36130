"""GPU: the CUDA path against the golden vectors produced by the unmodified
reference (tests/golden/*.npz): bit-exact segmentation / scale values / score,
standard LLRs bit for bit, scaled LLRs within the bound of tests/stats_cases.py (device and
C library exp / pow differ in the last ulp)."""
import numpy as np
import pytest

import golden_util as gu
import stats_cases as sc

pytestmark = pytest.mark.gpu


def _flatten(reads):
    from tombo_b200 import synthetic as syn
    raws = [np.asarray(r.raw) for r in reads]
    raw = np.concatenate(raws)
    raw_off = np.concatenate([[0], np.cumsum([x.shape[0] for x in raws])]).astype(np.int64)
    codes = [syn.seq_to_codes(r.genome_seq) for r in reads]
    seq = np.concatenate(codes)
    seq_off = np.concatenate([[0], np.cumsum([c.shape[0] for c in codes])]).astype(np.int64)
    return raw, raw_off, seq, seq_off


@pytest.mark.parametrize('name', gu.READ_CONFIGS)
def test_batch_reproduces_reference(ctx, RPcls, name):
    from tombo_b200 import _lib, synthetic as syn
    g = gu.load(name)
    kind, kmer_ref, cpos, reads = gu.reads_of(g)
    rp, sp = gu.params_of(g, RPcls)
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, len(kmer_ref[0][0]), cpos)
    raw, raw_off, seq, seq_off = _flatten(reads)
    res = ctx.resquiggle_batch(raw, raw_off, seq, seq_off, rp, sp,
                               _lib.make_policy(kind, const_scale=gu.const_scale_of(g)))
    for i in range(len(reads)):
        e = gu.expected(g, i)
        assert _lib.status_message(res['status'][i]) == e['message'], i
        if e['message']:
            continue
        a, b = res['seg_off'][i], res['seg_off'][i + 1]
        assert np.array_equal(res['segs'][a:b], e['segs']), i
        assert res['read_start_rel_to_raw'][i] == e['read_start_rel_to_raw']
        assert res['scale_values'][i, 0] == e['shift']
        assert res['scale_values'][i, 1] == e['scale']
        assert res['scale_values'][i, 2] == e['lower_lim']
        assert res['scale_values'][i, 3] == e['upper_lim']
        assert res['sig_match_score'][i] == e['sig_match_score']
        assert res['n_iters'][i] == e['n_iters']
        assert bool(res['flags'][i] & 2) == e['rescued']
        assert bool(res['flags'][i] & 1) == e['norm_params_changed']


def test_kernel_known_answers(ctx):
    k = gu.load('kernel_kats')
    fwd, tb = ctx.banded_forward_pass(k['bfp_z'], k['bfp_es'], 4.2, 4.2)
    assert np.array_equal(fwd, k['bfp_fwd'])
    assert np.array_equal(tb[1:], k['bfp_tb'])
    st, tbk = ctx.banded_traceback(tb, k['bfp_es'], int(np.argmax(fwd[-1])), -1)
    assert st == 0 and np.array_equal(tbk, k['bfp_traceback'])
    f, t, e = k['ad_seed_fwd'].copy(), k['ad_seed_tb'].copy(), k['ad_seed_es'].copy()
    st = ctx.adaptive_banded_forward_pass(f, t, e, k['ad_em'], k['ad_rm'], k['ad_rs'], 5.0, 4.2,
                                          4.2, int(k['ad_ssp']), -15.0, True, 20.0)
    assert (st == 0) == bool(k['ad_ok'])
    if st == 0:
        ssp = int(k['ad_ssp'])
        assert np.array_equal(e, k['ad_es'])
        assert np.array_equal(f[ssp + 1:], k['ad_fwd'][ssp + 1:])
        assert np.array_equal(t[ssp + 1:], k['ad_tb'][ssp + 1:])
    assert np.array_equal(ctx.new_means(k['h_sig'], k['h_segs']), k['h_means'])
    m, s = ctx.new_mean_stds(k['h_sig'], k['h_segs'])
    assert np.array_equal(m, k['h_mean_stds_m']) and np.array_equal(s, k['h_mean_stds_s'])
    st, cp = ctx.valid_cpts_w_cap(k['h_sig'], 3, 5, 500)
    assert st == 0 and np.array_equal(cp, k['h_cpts'])
    st, cp = ctx.valid_cpts_w_cap(k['h_sig'], 6, 12, 150, t_test=True)
    assert st == 0 and np.array_equal(cp, k['h_cpts_t'])


@pytest.mark.parametrize('gname', ['llr_5mc', 'llr_rna_5mc'])
def test_alt_model_llr_matches_reference(ctx, RPcls, gname):
    """per-read 5mC LLRs of resquiggled reads == compute_alt_model_read_stats of the
    reference (tombo_stats.py:3972-4082); DNA 6-mer and direct-RNA 5-mer models."""
    from tombo_b200 import _lib, synthetic as syn
    g = gu.load(gname)
    kind = str(g['kind']) if 'kind' in g.files else 'DNA'
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    K = len(kmer_ref[0][0])
    alt_rows = syn.make_alt_kmer_ref(kmer_ref, 'C', seed=1)
    means, sds = syn.kmer_table(kmer_ref)
    alt = np.full((4 ** K, K), np.nan)
    code = {'A': 0, 'C': 1, 'G': 2, 'T': 3}
    for km, pos, m, sd in alt_rows:
        idx = 0
        for b in km:
            idx = idx * 4 + code[b]
        alt[idx, pos] = m
    ctx.set_model(means, sds, K, cpos)
    ctx.set_alt_model(alt, K)
    if kind == 'DNA':
        aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
        rp, sp = RPcls(aln), RPcls(aln, save=True)
    else:
        rp = RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True)
        sp = RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True, save=True)
    reads = [syn.make_read(kmer_ref, cpos, int(g['nbases']), int(g['seed0']) + i, kind=kind)
             for i in range(int(g['nreads']))]
    raw, raw_off, seq, seq_off = _flatten(reads)
    res = ctx.resquiggle_batch(raw, raw_off, seq, seq_off, rp, sp, _lib.make_policy(kind))
    assert (res['status'] == 0).all()
    read_start = np.arange(len(reads), dtype=np.int64) * 1000
    for std, key in ((False, 'llr_scaled'), (True, 'llr_standard')):
        llr, pos, site_off = ctx.alt_model_llr_batch(res['norm_mean'], res['base_off'], seq,
                                                     seq_off, read_start, 1,
                                                     use_standard_llhr=std)
        assert np.array_equal(site_off, g['site_off'])
        assert np.array_equal(pos, g['pos'])
        # standard LLRs bit for bit; scaled ones within the exp / pow bound of stats_cases
        _, _, _, s_abs = sc.llr_reads(res['norm_mean'], res['base_off'], seq, seq_off,
                                      read_start, means, sds, alt, K, cpos, 1, int(std))
        sc.assert_llr(llr, g[key], s_abs, int(std), K)
