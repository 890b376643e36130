#!/usr/bin/env python
"""Goldens for the level tests from the UNMODIFIED reference (oracle/_ref):
compute_group_reg_stats (KS / U / t, p-values and *_stat_test, Fisher window and window
means) and get_reads_ref (median / mean, std, posterior with the model's levels).

Reads are served at the reference's own seam: get_single_slot_read_centric returns each
read's in-memory levels, so intervalData.get_base_levels (and its strand reversal in
get_single_slot_genome_centric) runs unmodified.  The dense base-level matrices it builds
are stored too, so the tests can feed the mirrors the same matrices.

    python oracle/build_ref.py && python tests/golden/make_group_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'oracle'))

import ref_harness as rh  # noqa: E402
from tombo_b200 import synthetic as syn  # noqa: E402

STATS = ('ks_test', 'u_test', 't_test', 'ks_stat_test', 'u_stat_test', 't_stat_test')


def make_reads(rs, n, lo, hi, shift, hole=None, min_len=40):
    """n reads inside [lo, hi) with continuous levels; shift(pos) is added to the level"""
    reads = []
    for i in range(n):
        a = int(rs.randint(lo, hi - min_len))
        b = int(rs.randint(a + min_len, hi + 1))
        pos = np.arange(a, b)
        lv = rs.normal(0.0, 1.0, b - a) + shift(pos)
        lv[rs.uniform(size=b - a) < 0.03] = np.nan            # scattered missing levels
        if hole is not None:
            lv[(pos >= hole[0]) & (pos < hole[1])] = np.nan
        reads.append((a, b, '+' if i % 2 else '-', lv))
    return reads


def main():
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    rs = np.random.RandomState(4236)
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    std_ref, _ = rh.make_models(kmer_ref, cpos)
    out = {}
    served = {}

    def slot(r_data, slot_name):
        lv = served[r_data.fn]
        # read-centric: minus-strand reads are stored 3' -> 5' in genome terms
        return lv[::-1].copy() if r_data.strand == '-' else lv.copy()
    th.get_single_slot_read_centric = slot

    genome = ''.join(rs.choice(list('ACGT'), 4000))
    genome = genome[:1100] + 'NN' + genome[1102:]           # a gap inside the get_reads_ref region

    def add_seq(self, genome_index=None, error_end=True):
        return self.update(seq=genome[self.start:self.end])
    th.intervalData.add_seq = add_seq

    def interval(tag, reads, start, end, strand=None):
        rd = []
        for i, (a, b, r_strand, lv) in enumerate(reads):
            if b <= start or a >= end:        # region reads overlap the region (as indexed)
                continue
            fn = '%s%d' % (tag, i)
            served[fn] = lv
            rd.append(th.readData(a, b, False, 0, r_strand, fn, 'g', False))
        return th.intervalData('chr', start, end, strand, reads=rd)

    # dataset A: region [1000, 1200); both strands, partial reads, a sample-only hole that
    # splits the runs at min_test_reads 5, a 3-position run between two holes (shorter
    # than the width-5 / width-9 windows)
    eff = lambda p: np.where((p >= 1100) & (p < 1120), 1.2, 0.0)   # noqa: E731
    samp = make_reads(rs, 14, 940, 1260, eff, hole=(1050, 1056))
    samp += make_reads(rs, 2, 940, 1260, eff)
    ctrl = make_reads(rs, 14, 940, 1260, lambda p: 0.0 * p, hole=(1059, 1066))
    ctrl += make_reads(rs, 2, 940, 1260, lambda p: 0.0 * p)
    # dataset B: 400 reads per sample fully covering [2000, 2040), a 4 sd shift -> KS and
    # t p-values far below 1e-100
    big_s = make_reads(rs, 400, 1990, 2050, lambda p: 4.0 + 0.0 * p, min_len=59)
    big_c = make_reads(rs, 400, 1990, 2050, lambda p: 0.0 * p, min_len=59)
    # dataset C: too few reads for any run at min_test_reads 20
    few_s = make_reads(rs, 4, 2990, 3100, lambda p: 0.0 * p)
    few_c = make_reads(rs, 4, 2990, 3100, lambda p: 0.0 * p)
    cases = [('A', samp, ctrl, 1000, 1200, (0, 1, 2, 4), (1, 5, 20)),
             ('B', big_s, big_c, 2000, 2040, (0, 1), (20,)),
             ('C', few_s, few_c, 3000, 3080, (1,), (20,))]
    with rh.ref_errstate():
        for tag, s_reads, c_reads, start, end, fms, mins in cases:
            reg = interval(tag + 's', s_reads, start, end)
            creg = interval(tag + 'c', c_reads, start, end)
            out['%s_reg' % tag] = np.array([start, end], dtype=np.int64)
            for fm in fms:
                out['%s_fm%d_samp' % (tag, fm)] = reg.copy().update(
                    start=start - fm, end=end + fm).get_base_levels()
                out['%s_fm%d_ctrl' % (tag, fm)] = creg.copy().update(
                    start=start - fm, end=end + fm).get_base_levels()
                for mn in mins:
                    for st in STATS:
                        key = '%s_%s_fm%d_m%d' % (tag, st, fm, mn)
                        res = ts.compute_group_reg_stats(reg, creg, fm, mn, st)
                        out[key + '_n'] = np.array(len(res))
                        if res:
                            g = res[0][1]
                            out[key + '_stats'] = np.asarray(g.reg_stats, dtype=np.float64)
                            out[key + '_pos'] = np.asarray(g.reg_poss, dtype=np.int64)
                            out[key + '_cov'] = np.asarray(g.reg_cov, dtype=np.int64)
                            out[key + '_ccov'] = np.asarray(g.ctrl_cov, dtype=np.int64)

        # get_reads_ref on the control of A (12-16 reads per position: > 8, pairwise order)
        creg = interval('Rc', ctrl, 1000, 1200)
        for fm in (0, 1):
            for mn in (1, 5):
                for est_mean in (False, True):
                    for prior in (False, True):
                        key = 'ref_fm%d_m%d_e%d_p%d' % (fm, mn, int(est_mean), int(prior))
                        means, sds, cov = ts.get_reads_ref(
                            creg, mn, fm, std_ref if prior else None, None, est_mean)
                        out[key + '_means'], out[key + '_sds'] = means, sds
                        ks = sorted(cov)
                        out[key + '_covpos'] = np.array(ks, dtype=np.int64)
                        out[key + '_cov'] = np.array([cov[k] for k in ks], dtype=np.int64)
            out['ref_fm%d_levels' % fm] = creg.copy().update(
                start=1000 - fm, end=1200 + fm).get_base_levels()
        # stranded control regions: the '+' / '-' k-mer lags of the posterior's expected levels
        # (and the reverse complement on '-'); get_base_levels keeps that strand's reads only
        for strand, name in (('+', 'plus'), ('-', 'minus')):
            sreg = interval('R' + name, ctrl, 1000, 1200, strand)
            for fm in (0, 1):
                key = 'refs_%s_fm%d' % (name, fm)
                means, sds, cov = ts.get_reads_ref(sreg, 1, fm, std_ref, None, False)
                out[key + '_means'], out[key + '_sds'] = means, sds
                out[key + '_cov'] = np.array([cov[k] for k in sorted(cov)], dtype=np.int64)
                out[key + '_levels'] = sreg.copy().update(
                    start=1000 - fm, end=1200 + fm).get_base_levels()
    out['genome'] = np.array(genome)
    np.savez_compressed(os.path.join(HERE, 'group_stats.npz'), **out)
    print('group_stats.npz:', len(out), 'arrays')


if __name__ == '__main__':
    main()
