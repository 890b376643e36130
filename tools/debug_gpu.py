"""ad-hoc GPU debug script (not a test): Theil-Sen path counters on the bench workloads.

For each bench.py workload, one resident batch_compute of the configuration's default batch
(the inputs bench.py times) and the tb2_debug_counters slots it moved, by name.

usage: python tools/debug_gpu.py [--workloads c1,mixed,rna,c5]"""
import argparse
import ctypes as C
import os
import sys
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench
from tombo_b200 import _lib, synthetic as syn

# tb2_debug_counters slots (include/tombo_b200.h)
SLOTS = ('theil-sen calls', 'fp32 bracket, every pair', 'exact histogram', 'generic select',
         'fp32 bracket, sampled pairs', 'sort-and-sweep finished', 'sort-and-sweep abandoned',
         'sweep phases (TS_DEBUG)')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='c1,mixed,rna,c5')
    args = ap.parse_args()
    for name in args.workloads.split(','):
        cfg = bench.CONFIGS[name]
        rna = cfg['kind'] == 'RNA'
        kmer_ref, cpos, raw, raw_off, seq, seq_off = bench.make_workload(cfg, cfg['reads'], 1)
        means, sds = syn.kmer_table(kmer_ref)
        ctx = _lib.Context(0)
        ctx.set_model(means, sds, len(kmer_ref[0][0]), cpos)
        rp = bench.RP(cfg['aln'], cfg['seg'], rna=rna)
        sp = bench.RP(cfg['aln'], cfg['seg'], save=True, rna=rna)
        pol = _lib.make_policy(cfg['kind'], subsample_seed=0)
        ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
        out = (C.c_ulonglong * 8)()
        ctx.check(ctx.lib.tb2_debug_counters(ctx.handle, out, 1))
        ctx.batch_compute(rp, sp, pol)
        ctx.check(ctx.lib.tb2_debug_counters(ctx.handle, out, 1))
        res = ctx.batch_download()
        print('%s: %s' % (name, '  '.join('[%d] %s %d' % (i, s, out[i]) for i, s in enumerate(SLOTS))))
        print('%s: status ok %d of %d' % (name, int((res['status'] == 0).sum()), len(res['status'])))
        ctx.close()


if __name__ == '__main__':
    main()
