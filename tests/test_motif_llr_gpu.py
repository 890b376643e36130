"""GPU: motif alternative-model LLRs (tb2_alt_model_llr_motif_batch, tb2_batch_alt_llr_motif,
tombo_stats.compute_alt_model_reads_stats) against the reference's golden and the restatement
of motif_cases.py: positions, site offsets and statuses exactly, standard LLRs bit for bit,
scaled LLRs within stats_cases.llr_bound."""
import os
import sys
from unittest import mock

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import motif_cases as mc  # noqa: E402
import stats_cases as sc  # noqa: E402
from test_motif_llr_cpu import golden_calls, models, whole_region  # noqa: E402

alt_table = mc.alt_table

pytestmark = pytest.mark.gpu


def _motif(raw, mod_pos):
    from tombo_b200 import _lib, tombo_helper as th
    return _lib.motif_struct(th.TomboMotif(raw, mod_pos))


def _check(got, want, mode, K):
    llr, pos, off, st = got
    w_llr, w_pos, w_off, s_abs, w_st = want
    assert np.array_equal(st, w_st)
    assert np.array_equal(off, w_off)
    assert np.array_equal(pos, w_pos)
    sc.assert_llr(llr, w_llr, s_abs, mode, K)


def _set(ctx, kind, base):
    kmer_ref, K, cpos, kmeans, ksds = models(kind)
    alt = alt_table(kmer_ref, base)
    ctx.set_model(kmeans, ksds, K, cpos)
    ctx.set_alt_model(alt, K)
    return kmer_ref, K, cpos, kmeans, ksds, alt


# 1. the golden, through the host-array entry and through the Python API
def test_golden_through_host_array_entry(ctx):
    for arrays, kind, motifs, reg, outs in golden_calls():
        bb, ab = mc.motif_bounds([m[:2] for m in motifs])
        reg = reg if reg is not None else whole_region(arrays)
        for (raw, mp, base), o in zip(motifs, outs):
            _, K, cpos, kmeans, ksds, alt = _set(ctx, kind, base)
            for mode, key in ((0, 'llr_scaled'), (1, 'llr_standard')):
                got = ctx.alt_model_llr_motif_batch(*arrays, _motif(raw, mp), bb, ab, reg[0],
                                                    reg[1], use_standard_llhr=(mode == 1))
                want = mc.motif_llr_reads(*arrays, raw, mp, bb, ab, reg[0], reg[1], kmeans,
                                          ksds, alt, K, cpos, mode)
                assert np.array_equal(got[1], o['pos']) and np.array_equal(got[3], o['status'])
                assert np.array_equal(got[2], o['site_off'])
                _check(got, want, mode, K)
                if mode == 1:
                    assert np.array_equal(got[0], o[key], equal_nan=True)


def test_golden_through_compute_alt_model_reads_stats(ctx):
    from tombo_b200 import tombo_helper as th, tombo_stats as ts
    for arrays, kind, motifs, reg, outs in golden_calls():
        kmer_ref, K, cpos, kmeans, ksds = models(kind)
        from tombo_b200 import synthetic as syn
        std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
        alt_refs = [('%s_%d' % (raw, mp), ts.AltModel(
            kmer_ref=syn.make_alt_kmer_ref(kmer_ref, base, seed=1), central_pos=cpos,
            alt_base=base, motif=th.TomboMotif(raw, mp))) for raw, mp, base in motifs]
        nm, mo, sq, so, st, sd = arrays
        r_datas, slots = [], {}
        for r in range(mo.shape[0] - 1):
            nb = int(mo[r + 1] - mo[r])
            S = ''.join('ACGT'[c] for c in sq[so[r] + cpos:so[r] + cpos + nb])
            rd = th.readData(start=int(st[r]), end=int(st[r]) + nb, filtered=False,
                             read_start_rel_to_raw=0, strand='+-'[sd[r]], fn='r%d' % r,
                             corr_group='g', rna=False)
            slots[rd.fn] = (nm[mo[r]:mo[r + 1]], np.array(list(S), dtype='S1'))
            r_datas.append(rd)
        reg_data = None if reg is None else mock.MagicMock(start=reg[0], end=reg[1])
        with mock.patch.object(th, 'get_multiple_slots_read_centric',
                               lambda r_data, names, grp=None: slots[r_data.fn]), \
                mock.patch.object(th, 'get_raw_read_slot',
                                  lambda r_data: mock.MagicMock(attrs={'read_id': r_data.fn})):
            bb, ab = mc.motif_bounds([m[:2] for m in motifs])
            creg = reg if reg is not None else whole_region(arrays)
            for std, key in ((False, 'llr_scaled'), (True, 'llr_standard')):
                res = ts.compute_alt_model_reads_stats(r_datas, std_ref, alt_refs,
                                                       use_standard_llhr=std, reg_data=reg_data)
                for (name, _), (raw, mp, base), o in zip(alt_refs, motifs, outs):
                    # |term| sums of the restatement bound the scaled LLRs (stats_cases)
                    s_abs = mc.motif_llr_reads(*arrays, raw, mp, bb, ab, creg[0], creg[1],
                                               kmeans, ksds, alt_table(kmer_ref, base), K,
                                               cpos, int(std))[3]
                    for r, x in enumerate(res):
                        if o['status'][r]:
                            assert isinstance(x, th.TomboError)
                            assert str(x) == mc.TOO_SHORT_MSG
                            continue
                        a, b = o['site_off'][r], o['site_off'][r + 1]
                        assert x[2] == 'r%d' % r
                        assert np.array_equal(np.asarray(x[1][name], np.int64), o['pos'][a:b])
                        sc.assert_llr(np.asarray(x[0][name], np.float64), o[key][a:b],
                                      s_abs[a:b], int(std), K)


# 2. a single-base motif on whole '+' reads is the existing call, bit for bit
@pytest.mark.parametrize('kind', ['DNA', 'RNA'])
def test_single_base_motif_matches_existing_entry(ctx, kind):
    kmer_ref, K, cpos, kmeans, ksds, alt = _set(ctx, kind, 'C')
    assert cpos < K - 1
    arrays = mc.sweep_reads(400, K, cpos, kmeans, seed=77 if kind == 'DNA' else 78, nb_lo=1,
                            nb_hi=700)
    nm, mo, sq, so, st, _ = arrays
    plus = np.zeros(st.shape[0], np.int8)
    reg = whole_region(arrays)
    for mode in (0, 1):
        old = ctx.alt_model_llr_batch(nm, mo, sq, so, st, 1, use_standard_llhr=(mode == 1))
        new = ctx.alt_model_llr_motif_batch(nm, mo, sq, so, st, plus, _motif('C', 1), 0, 0,
                                            reg[0], reg[1], use_standard_llhr=(mode == 1))
        # reads with fewer than K testable levels raise in the reference; the old entry
        # gives them no sites
        short = new[3] != 0
        assert (new[3][short] == mc.TOO_SHORT).all()
        assert (np.diff(mo)[short] < 2 * K - 1).all() and not np.diff(old[2])[short].any()
        assert np.array_equal(new[2], old[2]) and np.array_equal(new[1], old[1])
        assert np.array_equal(new[0], old[0], equal_nan=True)


@pytest.mark.parametrize('gname', ['llr_5mc', 'llr_rna_5mc'])
def test_single_base_motif_matches_existing_entry_on_llr_goldens(ctx, RPcls, gname):
    """the resquiggled reads of the 5mC goldens (as test_golden_gpu builds them)"""
    import golden_util as gu
    from test_golden_gpu import _flatten
    from tombo_b200 import _lib, synthetic as syn
    g = gu.load(gname)
    kind = str(g['kind']) if 'kind' in g.files else 'DNA'
    kmer_ref, K, cpos, kmeans, ksds, alt = _set(ctx, kind, 'C')
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
    start = np.arange(len(reads), dtype=np.int64) * 1000
    nb = np.diff(res['base_off'])
    for std, key in ((False, 'llr_scaled'), (True, 'llr_standard')):
        old = ctx.alt_model_llr_batch(res['norm_mean'], res['base_off'], seq, seq_off, start, 1,
                                      use_standard_llhr=std)
        new = ctx.alt_model_llr_motif_batch(res['norm_mean'], res['base_off'], seq, seq_off,
                                            start, np.zeros(len(reads), np.int8), _motif('C', 1),
                                            0, 0, 0, int((start + nb).max()),
                                            use_standard_llhr=std)
        assert np.array_equal(new[2], g['site_off']) and np.array_equal(new[1], g['pos'])
        assert np.array_equal(new[0], old[0], equal_nan=True)
        if std:
            assert np.array_equal(new[0], g[key])


# 3. seeded sweep over more than one k_scan_sites chunk
@pytest.mark.parametrize('raw,mod_pos,base', mc.MOTIFS)
def test_seeded_sweep_matches_restatement(ctx, raw, mod_pos, base):
    kmer_ref, K, cpos, kmeans, ksds, alt = _set(ctx, 'DNA', base)
    arrays = mc.sweep_reads(3000, K, cpos, kmeans, seed=900 + len(raw) * 7 + mod_pos,
                            nb_lo=1, nb_hi=300, motif=raw)
    rs = np.random.RandomState(len(raw))
    bb, ab = mc.motif_bounds([(raw, mod_pos), ('GATC', 2), ('CCWGG', 2)])
    for reg in ((-10 ** 9, 10 ** 9),) + tuple(
            (int(a), int(a + rs.randint(1, 3000))) for a in rs.randint(0, 5000, 3)):
        for mode in (0, 1):
            got = ctx.alt_model_llr_motif_batch(*arrays, _motif(raw, mod_pos), bb, ab, reg[0],
                                                reg[1], use_standard_llhr=(mode == 1))
            want = mc.motif_llr_reads(*arrays, raw, mod_pos, bb, ab, reg[0], reg[1], kmeans,
                                      ksds, alt, K, cpos, mode)
            _check(got, want, mode, K)


# 4. homopolymer runs and the greedy non-overlap choice
def test_homopolymers_with_self_overlapping_motifs(ctx):
    kmer_ref, K, cpos, kmeans, ksds, alt = _set(ctx, 'DNA', 'A')
    rs = np.random.RandomState(11)
    reads = []
    for run in list(range(1, 120)) + [255, 256, 257, 300, 700]:
        b = np.concatenate([rs.randint(1, 4, rs.randint(0, 9)), np.zeros(run, np.int64),
                            rs.randint(1, 4, rs.randint(0, 9))]).astype(np.uint8)
        reads.append((b, mc.level_means(b, kmeans, K, cpos, rs), 1000 * run, run % 2))
    arrays = mc.layout(reads, K, cpos, rs)
    for raw, mp in (('AA', 1), ('AA', 2), ('AAA', 2), ('AAAAAAA', 4), ('AWA', 1)):
        bb, ab = mc.motif_bounds([(raw, mp)])
        got = ctx.alt_model_llr_motif_batch(*arrays, _motif(raw, mp), bb, ab, -10 ** 9, 10 ** 9,
                                            use_standard_llhr=True)
        want = mc.motif_llr_reads(*arrays, raw, mp, bb, ab, -10 ** 9, 10 ** 9, kmeans, ksds,
                                  alt, K, cpos, 1)
        _check(got, want, 1, K)
    # re.finditer on AAAA: matches at 0 and 2 only (3-mers, read bases 2.. searched)
    assert mc.motif_sites('CCAAAA' + 'C' * 10, 100, '+', 0, 10 ** 6, 3, 1, 'AA', 1, 0, 1) \
        == (0, [102, 104])


# 5. region edges stepped through every offset near both read ends, both strands
@pytest.mark.parametrize('raw,mod_pos,base', [('CG', 1, 'C'), ('GATC', 2, 'A'),
                                              ('NNNNNNCG', 7, 'C'), ('CNNNNN', 1, 'C')])
def test_region_edge_sweeps(ctx, raw, mod_pos, base):
    kmer_ref, K, cpos, kmeans, ksds, alt = _set(ctx, 'DNA', base)
    rs = np.random.RandomState(5 + mod_pos)
    reads = []
    for i, nb in enumerate((1, K, 2 * K - 1, 2 * K, 2 * K + 1, 3 * K, 25, 40, 64)):
        for strand in (0, 1):
            b = mc.rand_bases(rs, nb, mc.concrete(raw, rs))
            reads.append((b, mc.level_means(b, kmeans, K, cpos, rs), 100, strand))
    arrays = mc.layout(reads, K, cpos, rs)
    bb, ab = mc.motif_bounds([(raw, mod_pos)])
    span = 2 * K + len(raw)
    lo_edges = range(100 - span, 100 + span + 1)
    hi_edges = range(100 + 1 - span, 100 + 64 + span + 1)
    for reg_start in lo_edges:
        for reg_end in (reg_start + 1, 10 ** 6):
            got = ctx.alt_model_llr_motif_batch(*arrays, _motif(raw, mod_pos), bb, ab, reg_start,
                                                reg_end, use_standard_llhr=True)
            want = mc.motif_llr_reads(*arrays, raw, mod_pos, bb, ab, reg_start, reg_end, kmeans,
                                      ksds, alt, K, cpos, 1)
            _check(got, want, 1, K)
    for reg_end in hi_edges:
        got = ctx.alt_model_llr_motif_batch(*arrays, _motif(raw, mod_pos), bb, ab, -10 ** 6,
                                            reg_end, use_standard_llhr=True)
        want = mc.motif_llr_reads(*arrays, raw, mod_pos, bb, ab, -10 ** 6, reg_end, kmeans, ksds,
                                  alt, K, cpos, 1)
        _check(got, want, 1, K)


# 6. the resident path
def test_resident_motif_llr_and_two_strand_region_counters(ctx, RPcls):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, K, cpos, kmeans, ksds, alt = _set(ctx, 'DNA', 'C')
    n = 2600
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, n, 200, 20261017)
    failed = (5, 1300, 2599)
    for r in failed:
        raw[raw_off[r]:raw_off[r + 1]] = 480.0
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    pol = _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    res = ctx.batch_download()
    before = {k: v.copy() for k, v in res.items() if isinstance(v, np.ndarray)}
    ok = res['status'] == 0
    assert not ok[list(failed)].any()
    start = (np.arange(n, dtype=np.int64) * 37) % 3001
    strand = (np.arange(n) % 2).astype(np.int8)
    old = ctx.batch_alt_llr(start, 1), ctx.batch_llr_download()
    nm, mo = res['norm_mean'], res['base_off']
    bb, ab = mc.motif_bounds([('CG', 1), ('GATC', 2), ('CCWGG', 2)])
    reg = (800, 2600)
    for raw_m, mp in (('CG', 1), ('CCWGG', 2)):
        for mode in (0, 1):
            tot, st = ctx.batch_alt_llr_motif(start, strand, _motif(raw_m, mp), bb, ab, *reg,
                                              use_standard_llhr=(mode == 1))
            llr, pos, off = ctx.batch_llr_download()
            host = ctx.alt_model_llr_motif_batch(nm, mo, seq, seq_off, start,
                                                 np.where(ok, strand, -1), _motif(raw_m, mp),
                                                 bb, ab, *reg, use_standard_llhr=(mode == 1))
            assert tot == host[2][-1]
            assert np.array_equal(off, host[2]) and np.array_equal(pos, host[1])
            assert np.array_equal(llr, host[0], equal_nan=True)
            assert np.array_equal(np.where(ok, st, 0), host[3])
            assert np.array_equal(st[~ok], res['status'][~ok])
    # '+' then '-' into their own region counters
    for s in (0, 1):
        only = np.where(strand == s, strand, -1).astype(np.int8)
        ctx.batch_alt_llr_motif(start, only, _motif('CG', 1), bb, ab, *reg)
        llr, pos, _ = ctx.batch_llr_download()
        ctx.region_stats_begin(reg[0], reg[1] - reg[0])
        ctx.region_stats_add_batch_llr(0.0, None, 0)
        got = ctx.region_stats_finalize()
        want = sc.region_counters(llr, pos, reg[0], reg[1] - reg[0], 0.0, None, 0)
        assert np.array_equal(got['pos'], want['pos'])
        for k in ('cov', 'valid_cov'):
            assert np.array_equal(got[k], want[k])
        assert np.array_equal(got['frac'], want['frac'], equal_nan=True)
    # the single-base call and the resident batch are unchanged
    again = ctx.batch_alt_llr(start, 1), ctx.batch_llr_download()
    assert again[0] == old[0]
    for a, b in zip(again[1], old[1]):
        assert np.array_equal(a, b, equal_nan=True)
    after = ctx.batch_download()
    for k, v in before.items():
        assert np.array_equal(after[k], v, equal_nan=True), k


# 7. invalid arguments
def test_invalid_arguments(ctx, RPcls):
    from tombo_b200 import _lib
    kmer_ref, K, cpos, kmeans, ksds, alt = _set(ctx, 'DNA', 'C')
    arrays = mc.sweep_reads(5, K, cpos, kmeans, seed=3, nb_lo=20, nb_hi=40)
    nm, mo, sq, so, st, sd = arrays

    def call(motif, bb=1, ab=1, strand=sd, so_=so, sq_=sq):
        return ctx.alt_model_llr_motif_batch(nm, mo, sq_, so_, st, strand, motif, bb, ab, 0, 10 ** 6)
    call(_motif('CG', 1))
    bad = []
    m = _motif('CG', 1); m.len = 0; bad.append(m)
    m = _motif('CG', 1); m.len = 33; bad.append(m)
    m = _motif('CG', 1); m.mod_pos = 0; bad.append(m)
    m = _motif('CG', 1); m.mod_pos = 3; bad.append(m)
    m = _motif('CG', 1); m.mask[1] = 0; bad.append(m)
    m = _motif('CG', 1); m.mask[0] = 16; bad.append(m)
    for m in bad:
        with pytest.raises(_lib.TomboB200Error):
            call(m)
    with pytest.raises(_lib.TomboB200Error):
        call(_motif('GATC', 2), bb=0, ab=2)          # max_motif_bb < mod_pos - 1
    with pytest.raises(_lib.TomboB200Error):
        call(_motif('GATC', 2), bb=1, ab=1)          # max_motif_ab < len - mod_pos
    with pytest.raises(_lib.TomboB200Error):
        call(_motif('CG', 1), strand=np.array([0, 1, 2, 0, 0], np.int8))
    with pytest.raises(_lib.TomboB200Error):
        call(_motif('CG', 1), strand=np.array([0, -2, 1, 0, 0], np.int8))
    sq_long = np.concatenate([sq[:so[2]], [0], sq[so[2]:]]).astype(np.uint8)
    so_long = so.copy()
    so_long[2:] += 1
    with pytest.raises(_lib.TomboB200Error):
        call(_motif('CG', 1), so_=so_long, sq_=sq_long)
    # the resident entry checks the same, on a small resident batch of its own
    from tombo_b200 import synthetic as syn
    raw, raw_off, rseq, rseq_off = syn.make_read_batch(kmer_ref, 8, 200, 4242)
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    pol = _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, rseq, rseq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    r_start, r_strand = np.arange(8, dtype=np.int64) * 1000, np.zeros(8, np.int8)
    ctx.batch_alt_llr_motif(r_start, r_strand, _motif('CG', 1), 1, 1, 0, 10 ** 6)
    for m in bad:
        with pytest.raises(_lib.TomboB200Error):
            ctx.batch_alt_llr_motif(r_start, r_strand, m, 1, 1, 0, 10 ** 6)
    with pytest.raises(_lib.TomboB200Error):
        ctx.batch_alt_llr_motif(r_start, r_strand, _motif('GATC', 2), 1, 1, 0, 10 ** 6)
    with pytest.raises(_lib.TomboB200Error):
        ctx.batch_alt_llr_motif(r_start, np.full(8, 3, np.int8), _motif('CG', 1), 1, 1, 0, 10 ** 6)
    # read_start / strand shorter than the batch would be read past their end
    with pytest.raises(ValueError):
        ctx.batch_alt_llr_motif(r_start[:5], r_strand[:5], _motif('CG', 1), 1, 1, 0, 10 ** 6)
    # models of different k-mer widths
    _, _, _, _, _, alt5 = _set(ctx, 'RNA', 'C')
    ctx.set_model(kmeans, ksds, K, cpos)
    with pytest.raises(_lib.TomboB200Error):
        call(_motif('CG', 1))


# the process-wide context: testing with another model must not leave resquiggle's cached
# model stale
def test_reads_stats_with_another_model_leaves_resquiggle_unchanged():
    from test_api_gpu import _map_res, _setup
    from tombo_b200 import resquiggle, synthetic as syn, tombo_helper as th, tombo_stats as ts
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    _, _, _, kmer_ref, cpos, std_ref, sst, p, sp = _setup('DNA', aln)
    reads = [syn.make_read(kmer_ref, cpos, 300, 31000 + i) for i in range(6)]
    mrs = [_map_res(th, r.raw, r.genome_seq) for r in reads]

    def rsq():
        out = resquiggle.resquiggle_reads(mrs, std_ref, p, sp, outlier_thresh=5.0,
                                          seq_samp_type=sst)
        assert all(not isinstance(o, th.TomboError) for o in out)
        return [(o.segs.copy(), o.read_start_rel_to_raw, o.scale_values.shift,
                 o.scale_values.scale, o.sig_match_score) for o in out]
    first = rsq()
    # direct-RNA 5-mer model: other tables, another k-mer width and central position
    rna_ref, rna_cpos = syn.make_kmer_ref('RNA', 0)
    rna_std = ts.TomboModel(kmer_ref=rna_ref, central_pos=rna_cpos)
    rna_alt = ts.AltModel(kmer_ref=syn.make_alt_kmer_ref(rna_ref, 'C', seed=1),
                          central_pos=rna_cpos, alt_base='C', motif=th.TomboMotif('CG', 1))
    rs = np.random.RandomState(2)
    bases = mc.rand_bases(rs, 80, 'CG')
    r_data = th.readData(start=0, end=80, filtered=False, read_start_rel_to_raw=0, strand='+',
                         fn='x', corr_group='g', rna=True)
    with mock.patch.object(th, 'get_multiple_slots_read_centric',
                           lambda *a, **k: (rs.normal(0, 1, 80),
                                            np.array(list(''.join('ACGT'[c] for c in bases)),
                                                     dtype='S1'))), \
            mock.patch.object(th, 'get_raw_read_slot', lambda *a, **k: mock.MagicMock()):
        res = ts.compute_alt_model_reads_stats([r_data], rna_std, [('CpG', rna_alt)])
    assert not isinstance(res[0], th.TomboError) and len(res[0][1]['CpG']) > 0
    again = rsq()
    for a, b in zip(first, again):
        assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]
