#!/usr/bin/env python
"""Writes tests/golden/llr_motif.npz: compute_alt_model_read_stats of the UNMODIFIED
reference (oracle/ref_harness) for motif alt models (AltModel(kmer_ref=...,
motif=TomboMotif(...))), reads on both strands, whole reads and regions clipping either end.

Reads are synthetic per-base levels near the model (the statistic needs no resquiggle), in
the library's layout (motif_cases.layout).  Every call is run with the scaled and with the
standard score.  Key scheme: c<i>_* holds case i's reads; c<i>_q<j>_* one call of that
case: `motifs` ('CG:1:C,GATC:2:A' = raw:mod_pos:alt_base per model), `reg` ([0, 0, 0] for
reg_data=None, else [1, start, end]); c<i>_q<j>_m<k>_* model k's llr_scaled,
llr_standard, pos, site_off and status (22 = 'Read sequence too short in this region.')."""
import os
import sys
import types
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
for p in (REPO, os.path.join(REPO, 'oracle'), os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)
import ref_harness as rh                      # noqa: E402
import motif_cases as mc                      # noqa: E402
from tombo_b200 import synthetic as syn       # noqa: E402

DNA_CALLS = [[m] for m in mc.MOTIFS] + [[('CG', 1, 'C'), ('GATC', 2, 'A'), ('CCWGG', 2, 'C')]]


def make_reads(kind, n, seed, plant):
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    K = len(kmer_ref[0][0])
    kmeans, _ = syn.kmer_table(kmer_ref)
    rs = np.random.RandomState(seed)
    reads = []
    for i in range(n):
        nb = int(rs.randint(3, 160)) if i % 8 else int(rs.randint(1, 2 * K + 2))
        b = mc.rand_bases(rs, nb, plant[i % len(plant)])
        reads.append((b, mc.level_means(b, kmeans, K, cpos, rs), int(rs.randint(0, 400)),
                      int(i % 2)))
    return kmer_ref, cpos, mc.layout(reads, K, cpos, rs)


def run_call(m, kmer_ref, cpos, arrays, motifs, reg):
    th, ts = m['th'], m['ts']
    nm, mo, sq, so, st, sd = arrays
    K = len(kmer_ref[0][0])
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    alt_refs = [('%s_%d' % (raw, mp), ts.AltModel(
        kmer_ref=syn.make_alt_kmer_ref(kmer_ref, base, seed=1), central_pos=cpos,
        alt_base=base, name='%s_%d' % (raw, mp), motif=th.TomboMotif(raw, mp)))
        for raw, mp, base in motifs]
    reg_data = None if reg is None else types.SimpleNamespace(start=reg[0], end=reg[1])
    out = [dict(llr_scaled=[], llr_standard=[], pos=[], site_off=[0], status=[])
           for _ in motifs]
    orig = (th.get_multiple_slots_read_centric, th.get_raw_read_slot)
    try:
        for r in range(mo.shape[0] - 1):
            nb = int(mo[r + 1] - mo[r])
            S = ''.join('ACGT'[c] for c in sq[so[r] + cpos:so[r] + cpos + nb])
            norm_mean = nm[mo[r]:mo[r + 1]].copy()
            bases = np.array(list(S), dtype='S1')
            th.get_multiple_slots_read_centric = lambda *a, **k: (norm_mean, bases)
            th.get_raw_read_slot = lambda *a, **k: mock.MagicMock()
            r_data = th.readData(start=int(st[r]), end=int(st[r]) + nb, filtered=False,
                                 read_start_rel_to_raw=0, strand='+-'[sd[r]], fn='x',
                                 corr_group='g', rna=False)
            res = []
            for std in (False, True):
                try:
                    with rh.ref_errstate():
                        res.append(ts.compute_alt_model_read_stats(
                            r_data, std_ref, alt_refs, use_standard_llhr=std, reg_data=reg_data))
                except th.TomboError as e:
                    assert str(e) == mc.TOO_SHORT_MSG, str(e)
                    res.append(None)
            for k, (name, _) in enumerate(alt_refs):
                o = out[k]
                if res[0] is None:
                    o['status'].append(mc.TOO_SHORT)
                    o['site_off'].append(o['site_off'][-1])
                    continue
                o['status'].append(0)
                o['llr_scaled'].append(np.asarray(res[0][0][name], dtype=np.float64))
                o['llr_standard'].append(np.asarray(res[1][0][name], dtype=np.float64))
                o['pos'].append(np.asarray(res[0][1][name], dtype=np.int64))
                o['site_off'].append(o['site_off'][-1] + len(res[0][1][name]))
    finally:
        th.get_multiple_slots_read_centric, th.get_raw_read_slot = orig
    for o in out:
        for key in ('llr_scaled', 'llr_standard'):
            o[key] = np.concatenate(o[key]) if o[key] else np.zeros(0)
        o['pos'] = np.concatenate(o['pos']).astype(np.int64) if o['pos'] else np.zeros(0, np.int64)
        o['site_off'] = np.array(o['site_off'], dtype=np.int64)
        o['status'] = np.array(o['status'], dtype=np.int32)
    return out


def main():
    m = rh.load_reference()
    plant = [None, 'CG', 'GATC', 'CCAGG', 'CCTGG', 'AAAA', 'CGCG']
    cases = [('DNA', 48, 41000, DNA_CALLS), ('RNA', 32, 42000, [[('C', 1, 'C')]])]
    regions = [None, (150, 300), (0, 120), (300, 10000), (200, 201)]
    store = {}
    for ci, (kind, n, seed, calls) in enumerate(cases):
        kmer_ref, cpos, arrays = make_reads(kind, n, seed, plant)
        for key, a in zip(('norm_mean', 'mean_off', 'seq', 'seq_off', 'read_start', 'strand'),
                          arrays):
            store['c%d_%s' % (ci, key)] = a
        store['c%d_kind' % ci] = np.array(kind)
        q = 0
        for motifs in calls:
            for reg in regions:
                out = run_call(m, kmer_ref, cpos, arrays, motifs, reg)
                store['c%d_q%d_motifs' % (ci, q)] = np.array(
                    ','.join('%s:%d:%s' % t for t in motifs))
                store['c%d_q%d_reg' % (ci, q)] = np.array(
                    [0, 0, 0] if reg is None else [1, reg[0], reg[1]], dtype=np.int64)
                for k, o in enumerate(out):
                    for key, v in o.items():
                        store['c%d_q%d_m%d_%s' % (ci, q, k, key)] = v
                print(kind, ','.join('%s:%d' % t[:2] for t in motifs), reg,
                      [int(o['site_off'][-1]) for o in out],
                      [int((o['status'] != 0).sum()) for o in out])
                q += 1
        store['c%d_ncalls' % ci] = np.array(q)
    store['ncases'] = np.array(len(cases))
    np.savez_compressed(os.path.join(HERE, 'llr_motif.npz'), **store)


if __name__ == '__main__':
    main()
