"""De novo and sample-compare testing of region blocks on the device: one JSON line.

Workload: a seeded two-strand synthetic genome at ~100x coverage (6-mer model, 5 kb reads,
syn.make_mapped_reads as bench_model_ref.py builds it), cut into 10 kb blocks per strand, a
few hundred reads per block.  Per block it times the batched region calls
(compute_de_novo_reads_stats, compute_sample_compare_reads_stats: kernel time from
tb2_last_timing and whole-call host time around the synchronised call) and, in the same run
and alternated with them, today's per-read mirror loop (compute_de_novo_read_stats /
compute_sample_compare_read_stats once per read).  Where the unmodified reference is built
(oracle/_ref) its compute_reg_stats runs on the host for the first blocks; the per-genome
figure scales that mean to every block and is labelled as extrapolated.  A parity sample
holds the batched de novo p-values to the numpy restatement (tests/reg_stats_cases.py).  The
whole measurement runs twice after a warm-up, and the GPU's name, power limit and maximum SM
clock are read in the same run.

    python bench_reg_stats.py [--genome 300000] [--coverage 100]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [REPO, os.path.join(REPO, 'tests')]

from tombo_b200 import _lib, synthetic as syn, tombo_helper as th, tombo_stats as ts  # noqa: E402
import reg_stats_cases as rc  # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
            text=True).strip()
    except Exception as e:
        return 'unavailable: %r' % (e,)


@contextlib.contextmanager
def serve(served):
    orig = th.get_multiple_slots_read_centric, th.get_raw_read_slot
    th.get_multiple_slots_read_centric = lambda r, names, cg=None: [served[r.fn][n] for n in names]
    th.get_raw_read_slot = lambda r: types.SimpleNamespace(attrs={'read_id': r.fn.encode()})
    try:
        yield
    finally:
        th.get_multiple_slots_read_centric, th.get_raw_read_slot = orig


def blocks(reads, genome_len, size):
    for strand in '+-':
        for start in range(0, genome_len, size):
            rds = [r for r in reads if r.strand == strand and r.end > start and r.start < start + size]
            if rds:
                yield types.SimpleNamespace(chrm='chr', strand=strand, start=start,
                                            end=min(start + size, genome_len), reads=rds)


def timed(ctx, fn, *args):
    t0 = time.perf_counter()
    out = fn(*args)
    return out, time.perf_counter() - t0, ctx.last_timing()[0]


def reference_block_seconds(regs, served, std_ref_rows, cpos, fm, n_blocks):
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import ref_harness as rh
    if not rh.available():
        return None
    m = rh.load_reference()
    rth, rts = m['th'], m['ts']

    class Handle(object):
        def __init__(self, fn):
            self.fn = fn

    @contextlib.contextmanager
    def h5_file(fn, mode='r'):
        yield Handle(fn)
    rts.h5py.File = h5_file
    rth.get_multiple_slots_read_centric = lambda f, names, cg=None: [served[f.fn][n] for n in names]
    rth.get_raw_read_slot = lambda f: types.SimpleNamespace(attrs={'read_id': f.fn.encode()})
    std_ref = rts.TomboModel(kmer_ref=std_ref_rows, central_pos=cpos)
    out = []
    with rh.ref_errstate():
        for reg in regs[:n_blocks]:
            rd = [rth.readData(r.start, r.end, False, 0, r.strand, r.fn, 'g', False) for r in reg.reads]
            rreg = rth.intervalData('chr', reg.start, reg.end, reg.strand, reads=rd)
            t0 = time.perf_counter()
            rts.compute_reg_stats(rreg, fm, 1, 0.05, None, None, std_ref, None, False, None,
                                  'de_novo', None)
            out.append(time.perf_counter() - t0)
    return out


def one_pass(ctx, regs, std_ref, fm, rs):
    rec = dict(dn_kernel=[], dn_call=[], dn_loop=[], sc_kernel=[], sc_call=[], sc_loop=[],
               reads=[])
    for reg in regs:
        n_ctrl = reg.end - reg.start + 2 * fm
        cm, cs = rs.normal(90.0, 5.0, n_ctrl), rs.uniform(1.0, 3.0, n_ctrl)
        # new path, then the per-read loop, block by block
        _, t, k = timed(ctx, ts.compute_de_novo_reads_stats, reg.reads, std_ref, fm, reg)
        rec['dn_call'].append(t)
        rec['dn_kernel'].append(k)
        t0 = time.perf_counter()
        for r in reg.reads:
            try:
                ts.compute_de_novo_read_stats(r, std_ref, fm, reg)
            except th.TomboError:
                pass
        rec['dn_loop'].append(time.perf_counter() - t0)
        _, t, k = timed(ctx, ts.compute_sample_compare_reads_stats, reg.reads, cm, cs, fm, reg)
        rec['sc_call'].append(t)
        rec['sc_kernel'].append(k)
        t0 = time.perf_counter()
        for r in reg.reads:
            try:
                ts.compute_sample_compare_read_stats(r, cm, cs, fm, reg)
            except th.TomboError:
                pass
        rec['sc_loop'].append(time.perf_counter() - t0)
        rec['reads'].append(len(reg.reads))
    return rec


def summary(rec):
    out = {}
    for k, v in rec.items():
        v = np.asarray(v, dtype=np.float64)
        scale = 1.0 if k == 'reads' else 1e3 if k.endswith('_call') or k.endswith('_loop') else 1.0
        out[k + ('' if k == 'reads' else '_ms')] = dict(
            median=float(np.median(v) * scale), total=float(v.sum() * scale))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--genome', type=int, default=300000)
    ap.add_argument('--coverage', type=int, default=100)
    ap.add_argument('--read-len', type=int, default=5000)
    ap.add_argument('--region-size', type=int, default=10000)
    ap.add_argument('--fm-offset', type=int, default=1)
    ap.add_argument('--ref-blocks', type=int, default=2)
    a = ap.parse_args()
    kmer_ref = syn.make_event_model(6, 11)
    cpos = 2
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    n_reads = a.genome * a.coverage // a.read_len
    _, reads, served = syn.make_mapped_reads(kmer_ref, cpos, a.genome, n_reads, a.read_len, 17)
    regs = list(blocks(reads, a.genome, a.region_size))
    ctx = _lib.get_context()
    rs = np.random.RandomState(3)
    out = dict(workload=dict(genome=a.genome, coverage=a.coverage, read_len=a.read_len,
                             region_size=a.region_size, fm_offset=a.fm_offset, blocks=len(regs),
                             reads=len(reads)),
               gpu=gpu_info())
    with serve(served):
        one_pass(ctx, regs[:2], std_ref, a.fm_offset, rs)                   # warm-up
        out['runs'] = [summary(one_pass(ctx, regs, std_ref, a.fm_offset, rs)) for _ in range(2)]
        # parity sample: the first block against the restatement
        reg = regs[0]
        got = ts.compute_de_novo_reads_stats(reg.reads, std_ref, a.fm_offset, reg)
        km, ks = syn.kmer_table(kmer_ref)
        worst, n = 0.0, 0
        for r, o in zip(reg.reads, got):
            bases = np.array(['ACGT'.index(b.decode()) for b in served[r.fn]['base']])
            try:
                pv, pos = rc.de_novo(served[r.fn]['norm_mean'], bases, r.start, r.end, r.strand,
                                     km, ks, 6, cpos, a.fm_offset, reg.start, reg.end)
            except rc.CaseError as e:
                assert str(o) == str(e)
                continue
            assert np.array_equal(o[1]['de_novo'], pos)
            d = np.abs(o[0]['de_novo'] - pv) / np.abs(pv)
            worst = max(worst, float(np.nanmax(d)) if d.size else 0.0)
            n += 1
        out['parity'] = dict(reads=n, max_rel_err=worst)
    secs = reference_block_seconds(regs, served, kmer_ref, cpos, a.fm_offset, a.ref_blocks)
    if secs is not None:
        out['reference_host'] = dict(blocks_measured=len(secs), mean_block_s=float(np.mean(secs)),
                                     all_blocks_s_extrapolated=float(np.mean(secs) * len(regs)))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
