#!/usr/bin/env python
"""Standard k-mer model estimation on the device: one JSON line.

Workload: a seeded 1 Mb two-strand synthetic genome at ~100x coverage (6-mer model, 5 kb
reads), 10 kb regions, calc_med_sd summaries (extract_kmer_levels) and the per-k-mer
medians (tabulate_kmer_levels).  Reports kernel and whole-call time of both steps, a parity
sample of the device summaries against the numpy restatement, and the GPU's name and power
limit read in the same run.  Where the unmodified reference is built (oracle/_ref), its own
get_region_kmer_levels runs on the host for the first few regions of the same reads; the
per-genome figure scales that mean to every region and is labelled as extrapolated.

    python bench_model_ref.py [--genome 1000000] [--coverage 100]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [REPO, os.path.join(REPO, 'tests')]

from tombo_b200 import _lib, synthetic as syn, tombo_stats as ts  # noqa: E402
import model_ref_cases as mc  # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except Exception as e:
        return 'unavailable: %r' % (e,)


def reference_region_seconds(reads, served, region_size, cov_thresh, n_regions):
    """host seconds of the unmodified reference's get_region_kmer_levels for each of the first
    n_regions regions, or None where the reference is not built"""
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import ref_harness as rh
    if not rh.available():
        return None
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    ts.VERBOSE = th.VERBOSE = False
    th.get_single_slot_read_centric = lambda r, slot, corr_grp=None: served[r.fn].get(slot)
    index = object.__new__(th.TomboReads)
    index.reads_index = mc.Index(reads).reads_index
    index.coverage = None
    out = []
    for chrm, strand, reg_start in index.iter_cov_regs(cov_thresh, region_size):
        reg = th.intervalData(chrm=chrm, start=reg_start, end=reg_start + region_size,
                              strand=strand).add_reads(index)
        t0 = time.perf_counter()
        ts.get_region_kmer_levels(reg, cov_thresh, 2, 3, None, False, region_size)
        out.append(time.perf_counter() - t0)
        if len(out) == n_regions:
            break
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--genome', type=int, default=1000000)
    ap.add_argument('--coverage', type=int, default=100)
    ap.add_argument('--read-len', type=int, default=5000)
    ap.add_argument('--region-size', type=int, default=10000)
    a = ap.parse_args()
    kmer_ref = syn.make_event_model(6, 11)
    n_reads = a.genome * a.coverage // a.read_len
    _, reads, served = syn.make_mapped_reads(kmer_ref, 2, a.genome, n_reads, a.read_len, 17)
    index = mc.Index(reads)
    ctx = _lib.get_context()
    calls = {'sum': [], 'med': []}
    orig_sum, orig_med = ctx.kmer_level_summaries, ctx.kmer_medians

    def timed(key, fn):
        def run(*args, **kw):
            t0 = time.perf_counter()
            out = fn(*args, **kw)
            calls[key].append((time.perf_counter() - t0, ctx.last_timing()[0], args))
            return out
        return run
    ctx.kmer_level_summaries, ctx.kmer_medians = timed('sum', orig_sum), timed('med', orig_med)
    with mc.serve(served):
        ts.extract_kmer_levels(index, a.region_size, 10, 2, 3, None)        # warm-up
        for k in calls:
            del calls[k][:]
        t0 = time.perf_counter()
        regs = ts.extract_kmer_levels(index, a.region_size, 10, 2, 3, None)
        t_ext = time.perf_counter() - t0
        t0 = time.perf_counter()
        ts.tabulate_kmer_levels(regs, 5)
        t_tab = time.perf_counter() - t0
    # parity sample: the first 20 kb of the first summaries call against the numpy
    # restatement (reads starting there; the restatement ignores later positions)
    n_pos, rd, thr = calls['sum'][0][2][:3]
    dev = orig_sum(n_pos, rd, thr)
    m = min(n_pos, 20000)
    lv, off, st = rd
    keep = np.nonzero(st < m)[0]
    sub = (np.concatenate([lv[off[r]:off[r + 1]] for r in keep]),
           np.concatenate([[0], np.cumsum(off[keep + 1] - off[keep])]), st[keep])
    want = mc.summaries(m, sub, thr)
    parity = all(np.array_equal(d[:m], w, equal_nan=True) for d, w in zip(dev, want))
    ref_s = reference_region_seconds(reads, served, a.region_size, 10, 3)
    ref = (dict(reference_host_s_per_region=float(np.mean(ref_s)), reference_regions_timed=len(ref_s),
                reference_host_s_per_genome_extrapolated=float(np.mean(ref_s)) * len(regs))
           if ref_s else dict(reference_host='not built'))
    print(json.dumps(dict(ref, **dict(
        workload='estimate_reference 1 Mb x2 strands, %dx, %d kb regions' % (a.coverage, a.region_size // 1000),
        gpu=gpu_info(), n_reads=n_reads, n_regions=len(regs),
        summaries_calls=len(calls['sum']),
        summaries_kernel_ms=sum(c[1] for c in calls['sum']),
        summaries_call_ms=1e3 * sum(c[0] for c in calls['sum']),
        medians_kernel_ms=sum(c[1] for c in calls['med']),
        medians_call_ms=1e3 * sum(c[0] for c in calls['med']),
        extract_kmer_levels_s=t_ext, tabulate_kmer_levels_s=t_tab,
        parity_first_batch_bit_exact=bool(parity)))))


if __name__ == '__main__':
    main()
