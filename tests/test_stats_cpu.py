"""The restatements in stats_cases.py reproduce the unmodified reference's goldens bit for bit
(LLRs, de novo p-values and Fisher windows, region counters), and the exact z -> p -> Fisher
path agrees with them within the documented bounds.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import golden_util as gu  # noqa: E402
import stats_cases as sc  # noqa: E402


@pytest.mark.parametrize('gname', ['llr_5mc', 'llr_rna_5mc'])
def test_llr_restatement_matches_reference_bit_for_bit(orc, RPcls, gname):
    """compute_alt_model_read_stats of the reference on resquiggled reads == the restatement
    on the oracle's per-base means, both scores, every bit"""
    from tombo_b200 import synthetic as syn
    g = gu.load(gname)
    kind = str(g['kind']) if 'kind' in g.files else 'DNA'
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    K = len(kmer_ref[0][0])
    means, sds = syn.kmer_table(kmer_ref)
    alt, _ = sc.alt_tables(kmer_ref)
    if kind == 'DNA':
        aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
        rp, sp = RPcls(aln), RPcls(aln, save=True)
    else:
        rp = RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True)
        sp = RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True, save=True)
    pol = orc.policy(kind)
    reads = []
    for i in range(int(g['nreads'])):
        r = syn.make_read(kmer_ref, cpos, int(g['nbases']), int(g['seed0']) + i, kind=kind)
        rm, rsd = gu.levels(r.genome_seq, kmer_ref)
        o = orc.run_read(np.asarray(r.raw, dtype=np.float64), rm, rsd, rp, sp, pol,
                         read_index=i, want_norm=True)
        assert o['status'] == 0
        reads.append((syn.seq_to_codes(r.genome_seq), orc.new_means(o['norm_signal'], o['segs'])))
    nm, mo, sq, so = sc.flatten(reads)
    start = np.arange(len(reads), dtype=np.int64) * 1000
    for mode, key in ((0, 'llr_scaled'), (1, 'llr_standard')):
        llr, pos, off, s_abs = sc.llr_reads(nm, mo, sq, so, start, means, sds, alt, K, cpos, 1,
                                            mode)
        assert np.array_equal(off, g['site_off'])
        assert np.array_equal(pos, g['pos'])
        assert np.array_equal(llr, g[key]), np.max(np.abs(llr - g[key]))
        assert np.all(s_abs > 0)


def _de_novo_inputs(g, i, kmer_ref, cpos, K):
    """z-scores of stored read i exactly as compute_de_novo_read_stats forms them"""
    from tombo_b200 import synthetic as syn
    means, sds = syn.kmer_table(kmer_ref)
    a, b = int(g['dn_off'][i]), int(g['dn_off'][i + 1])
    codes = syn.seq_to_codes(str(g['dn_seq'][i]))
    kc = sc.kmer_codes(codes.astype(np.int64), K)
    m = g['dn_means'][a:b][cpos:cpos + kc.shape[0]]
    return sc.z_scores(m, means[kc], sds[kc]), int(g['dn_start'][i]) + cpos


def test_reference_p_path_matches_goldens_and_exact_path_agrees():
    from tombo_b200 import synthetic as syn
    g = gu.load('region_stats')
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    K = 6
    worst, n_cmp = 0.0, 0
    # Fisher windows over given p-values
    for lag in (1, 2, 4):
        ref = sc.ref_window(g['fw_p'], lag, False)
        assert np.array_equal(ref, g['fw_lag%d' % lag], equal_nan=True)
        vals, bounds = sc.exact_window(sc.exact_given(g['fw_p']), np.zeros(g['fw_p'].shape[0]),
                                       lag, False)
        worst = max(worst, sc.assert_window(ref, vals, bounds))
        n_cmp += 1
    # de novo p-values of whole '+' strand reads
    for i in range(int(g['dn_n'])):
        if str(g['dn_strand'][i]) != '+':
            continue
        z, first = _de_novo_inputs(g, i, kmer_ref, cpos, K)
        pe = sc.exact_pvals(z)
        perr = sc.p_rel_bound(z)
        for fm in (0, 1, 2):
            key = 'dn_r%d_fm%d_whole' % (i, fm)
            ref = sc.ref_window(sc.ref_pvals(z), fm, True)
            assert np.array_equal(ref, g[key + '_p'], equal_nan=True), key
            assert np.array_equal(first + np.arange(z.shape[0]), g[key + '_pos'])
            vals, bounds = sc.exact_window(pe, perr, fm, True)
            worst = max(worst, sc.assert_window(ref, vals, bounds))
            n_cmp += 1
    assert n_cmp >= 9
    print('largest error / bound, reference path against exact: %.3g' % worst)


@pytest.mark.parametrize('name,stat_type', [('alt_lower', 0), ('alt_abs', 0), ('denovo', 1)])
def test_counter_restatement_matches_reference_goldens(name, stat_type):
    g = gu.load('region_stats')
    thr, lower = g['rg_%s_params' % name]
    got = sc.region_counters(g['rg_stats'], g['rg_locs'], 5000, 1000, float(thr), float(lower),
                             stat_type, unmod=2.0, mod=0.0)
    assert np.array_equal(got['pos'], g['rg_%s_pos' % name])
    assert np.array_equal(got['cov'], g['rg_%s_cov' % name])
    assert np.array_equal(got['valid_cov'], g['rg_%s_valid' % name])
    assert np.array_equal(got['frac'], g['rg_%s_frac' % name], equal_nan=True)
    assert np.array_equal(got['damp_frac'], g['rg_%s_damp' % name], equal_nan=True)


def test_counter_restatement_drops_positions_outside_the_region():
    got = sc.region_counters([1.0, 2.0, 3.0, np.nan, 4.0], [9, 10, 19, 12, 20], 10, 10, 2.0,
                             None, 1)
    assert np.array_equal(got['pos'], [10, 19])
    assert np.array_equal(got['cov'], [1, 1])
    assert np.array_equal(got['frac'], [1.0, 1.0])
