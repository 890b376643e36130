"""ad-hoc GPU debug script (not a test): Theil-Sen path counters on the bench workloads"""
import ctypes as C
import os
import sys
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np
import bench
from tombo_b200 import _lib, synthetic as syn
for mixed in (False, True):
    kmer_ref, cpos, raw, raw_off, seq, seq_off = bench.make_workload(6000, 3, mixed=mixed)
    means, sds = syn.kmer_table(kmer_ref)
    ctx = _lib.Context(0)
    ctx.set_model(means, sds, 6, cpos)
    aln = bench.ALN_MIXED if mixed else bench.ALN_DNA
    rp, sp = bench.RP(aln), bench.RP(aln, save=True)
    pol = _lib.make_policy('DNA')
    fn = ctx.lib.tb2_debug_counters
    out = (C.c_ulonglong * 8)()
    fn(ctx.handle, out, C.c_int(1))
    res = ctx.resquiggle_batch(raw, raw_off, seq, seq_off, rp, sp, pol)
    fn(ctx.handle, out, C.c_int(1))
    print('mixed' if mixed else 'c1', 'theil-sen calls %d  sampled-fast %d  full-fast %d  exact-hist %d  generic %d' % (
        out[0], out[4], out[1], out[2], out[3]))
    print('status ok', int((res['status'] == 0).sum()), 'of', len(res['status']))
    del ctx
