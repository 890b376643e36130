"""CPU checks of the motif alternative-model LLRs: the restatement (motif_cases) against the
reference's golden, the emulated device site finder against the restatement, the motif
conversion and the new status message."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, 'emul')):
    if p not in sys.path:
        sys.path.insert(0, p)
import motif_cases as mc     # noqa: E402
import stats_cases as sc     # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'llr_motif.npz')


def models(kind):
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    K = len(kmer_ref[0][0])
    kmeans, ksds = syn.kmer_table(kmer_ref)
    return kmer_ref, K, cpos, kmeans, ksds


alt_table = mc.alt_table


def golden_calls():
    """(case arrays, kind, motifs, region, per-model golden dicts) of every golden call"""
    g = np.load(GOLDEN)
    for ci in range(int(g['ncases'])):
        arrays = [g['c%d_%s' % (ci, k)] for k in
                  ('norm_mean', 'mean_off', 'seq', 'seq_off', 'read_start', 'strand')]
        kind = str(g['c%d_kind' % ci])
        for q in range(int(g['c%d_ncalls' % ci])):
            motifs = [(m.split(':')[0], int(m.split(':')[1]), m.split(':')[2])
                      for m in str(g['c%d_q%d_motifs' % (ci, q)]).split(',')]
            has, rs, re_ = (int(x) for x in g['c%d_q%d_reg' % (ci, q)])
            outs = [dict((k, g['c%d_q%d_m%d_%s' % (ci, q, k_i, k)]) for k in
                         ('llr_scaled', 'llr_standard', 'pos', 'site_off', 'status'))
                    for k_i in range(len(motifs))]
            yield arrays, kind, motifs, (rs, re_) if has else None, outs


def whole_region(arrays):
    nm, mo, _, _, st, _ = arrays
    nb = np.diff(mo)
    return int(st.min()), int((st + nb).max())


def test_golden_covers_the_issue_families():
    seen = set()
    regions = set()
    for arrays, kind, motifs, reg, outs in golden_calls():
        seen.update((kind, m[0], m[1]) for m in motifs)
        regions.add(reg is not None)
        if len(motifs) > 1:
            seen.add('joint')
        for o in outs:
            if (o['status'] == mc.TOO_SHORT).any():
                seen.add('too_short')
        assert set(arrays[5].tolist()) == {0, 1}
    for fam in [('DNA', m, p) for m, p, _ in mc.MOTIFS] + [('RNA', 'C', 1), 'joint', 'too_short']:
        assert fam in seen, fam
    assert regions == {True, False}


def test_restatement_reproduces_golden():
    n_sites = 0
    for arrays, kind, motifs, reg, outs in golden_calls():
        kmer_ref, K, cpos, kmeans, ksds = models(kind)
        bb, ab = mc.motif_bounds([m[:2] for m in motifs])
        reg = reg if reg is not None else whole_region(arrays)
        for (raw, mp, base), o in zip(motifs, outs):
            alt = alt_table(kmer_ref, base)
            for mode, key in ((0, 'llr_scaled'), (1, 'llr_standard')):
                llr, pos, off, s_abs, st = mc.motif_llr_reads(
                    *arrays, raw, mp, bb, ab, reg[0], reg[1], kmeans, ksds, alt, K, cpos, mode)
                assert np.array_equal(st, o['status'])
                assert np.array_equal(off, o['site_off'])
                assert np.array_equal(pos, o['pos'])
                # the restatement calls the same C library the reference's scorers do
                assert np.array_equal(llr, o[key], equal_nan=True), (raw, reg, mode)
            n_sites += pos.shape[0]
    assert n_sites > 5000


def test_emulated_site_finder_reproduces_golden():
    em = pytest.importorskip('emul_motif')
    for arrays, kind, motifs, reg, outs in golden_calls():
        kmer_ref, K, cpos, kmeans, ksds = models(kind)
        bb, ab = mc.motif_bounds([m[:2] for m in motifs])
        reg = reg if reg is not None else whole_region(arrays)
        for (raw, mp, base), o in zip(motifs, outs):
            llr, pos, off, st = em.llr_motif(*arrays, K, cpos, kmeans, ksds, alt_table(kmer_ref, base),
                                             mc.iupac_mask(raw), mp, ab, reg[0], reg[1], mode=1)
            assert np.array_equal(st, o['status'])
            assert np.array_equal(off, o['site_off'])
            assert np.array_equal(pos, o['pos'])
            assert np.array_equal(llr, o['llr_standard'], equal_nan=True)


@pytest.mark.parametrize('raw,mod_pos,_base', mc.MOTIFS + [('AAA', 2, 'A'), ('ACA', 1, 'A'),
                                                         ('RGR', 2, 'G'), ('W', 1, 'A')])
def test_emulated_site_finder_matches_restatement_on_seeded_reads(raw, mod_pos, _base):
    em = pytest.importorskip('emul_motif')
    kmer_ref, K, cpos, kmeans, ksds = models('DNA')
    alt = alt_table(kmer_ref, 'C')
    arrays = mc.sweep_reads(60, K, cpos, kmeans, seed=sum(map(ord, raw)) + mod_pos, nb_lo=1,
                            nb_hi=90, motif=raw)
    # a second model with wider context widens the search window, as in a joint call
    for bb, ab in (mc.motif_bounds([(raw, mod_pos)]),
                   mc.motif_bounds([(raw, mod_pos), ('NNNNNNNCG', 8), ('CNNNNNNN', 1)])):
        for reg in ((-10 ** 9, 10 ** 9), (1000, 1100), (2500, 2530), (0, 4000), (3000, 3001)):
            want_llr, want_pos, want_off, _, want_st = mc.motif_llr_reads(
                *arrays, raw, mod_pos, bb, ab, reg[0], reg[1], kmeans, ksds, alt, K, cpos, 1)
            llr, pos, off, st = em.llr_motif(*arrays, K, cpos, kmeans, ksds, alt,
                                             mc.iupac_mask(raw), mod_pos, ab, reg[0], reg[1])
            assert np.array_equal(st, want_st), (bb, ab, reg)
            assert np.array_equal(off, want_off), (bb, ab, reg)
            assert np.array_equal(pos, want_pos)
            assert np.array_equal(llr, want_llr, equal_nan=True)


def test_emulated_site_finder_on_homopolymers_with_self_overlapping_motifs():
    em = pytest.importorskip('emul_motif')
    kmer_ref, K, cpos, kmeans, ksds = models('DNA')
    alt = alt_table(kmer_ref, 'A')
    rs = np.random.RandomState(5)
    reads = []
    for run in range(1, 80):
        b = np.concatenate([rs.randint(1, 4, rs.randint(0, 7)), np.zeros(run, np.int64),
                            rs.randint(1, 4, rs.randint(0, 7))]).astype(np.uint8)
        reads.append((b, mc.level_means(b, kmeans, K, cpos, rs), 100 * run, run % 2))
    arrays = mc.layout(reads, K, cpos, rs)
    for raw, mp in (('AA', 1), ('AA', 2), ('AAA', 2), ('AAAAAAA', 4)):
        bb, ab = mc.motif_bounds([(raw, mp)])
        want = mc.motif_llr_reads(*arrays, raw, mp, bb, ab, -10 ** 9, 10 ** 9, kmeans, ksds,
                                  alt, K, cpos, 1)
        got = em.llr_motif(*arrays, K, cpos, kmeans, ksds, alt, mc.iupac_mask(raw), mp, ab,
                           -10 ** 9, 10 ** 9)
        assert np.array_equal(got[2], want[2]) and np.array_equal(got[1], want[1]), raw
        assert np.array_equal(got[0], want[0], equal_nan=True)


def test_motif_conversion_and_overlap_flag():
    """tb2_motif from a TomboMotif, and the library's overlap rule (motif_can_overlap in
    motif_llr.cuh, run through the host emulation)"""
    em = pytest.importorskip('emul_motif')
    from tombo_b200 import _lib, tombo_helper as th
    cases = {('CG', 1): False, ('GATC', 2): False, ('CCWGG', 2): False, ('AA', 1): True,
             ('C', 1): False, ('NNNNNNCG', 7): True, ('CNNNNN', 1): True, ('GCGC', 2): True}
    for (raw, mp), overlap in cases.items():
        m = _lib.motif_struct(th.TomboMotif(raw, mp))
        assert (m.len, m.mod_pos) == (len(raw), mp)
        assert list(m.mask)[:m.len] == mc.iupac_mask(raw)
        assert all(v == 0 for v in list(m.mask)[m.len:])
        assert em.can_overlap(list(m.mask)[:m.len]) is overlap, raw
    # the rule is exact: a motif can overlap itself iff two matches at distance < len exist
    import itertools
    import re
    for raw in ('AT', 'ATA', 'CGC', 'ACGT', 'TTAT', 'AWW', 'CRY', 'CNG'):
        pat = re.compile('(?=(%s))' % ''.join(mc.SINGLE_LETTER_CODE[c] for c in raw))
        close = False
        for s in map(''.join, itertools.product('ACGT', repeat=2 * len(raw))):
            starts = [x.start() for x in pat.finditer(s)]
            close = close or any(b - a < len(raw) for a, b in zip(starts, starts[1:]))
        assert em.can_overlap(mc.iupac_mask(raw)) is close, raw


def test_too_short_status_message_is_the_reference_string():
    from tombo_b200 import _lib
    assert _lib.status_message(mc.TOO_SHORT) == mc.TOO_SHORT_MSG


def test_header_declares_the_motif_entry_points():
    src = open(os.path.join(os.path.dirname(HERE), 'include', 'tombo_b200.h')).read()
    for name in ('tb2_alt_model_llr_motif_batch', 'tb2_batch_alt_llr_motif', 'tb2_motif',
                 'TB2_ERR_READ_TOO_SHORT_IN_REGION = 22'):
        assert name in src
    from tombo_b200 import _lib
    lib = _lib.load()
    assert hasattr(lib, 'tb2_alt_model_llr_motif_batch') and hasattr(lib, 'tb2_batch_alt_llr_motif')


def test_batched_api_is_exported():
    from tombo_b200 import tombo_stats as ts
    assert 'compute_alt_model_reads_stats' in ts.__all__
    assert callable(ts.compute_alt_model_reads_stats)
