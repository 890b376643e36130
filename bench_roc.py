"""Accuracy of modified-base calls on the device: one JSON line.

Workload: a seeded two-strand synthetic genome (two chromosomes, --genome bases each) with
per-read statistics at ~--coverage reads per position in 10 kb blocks (about 5*10^7
statistics at the defaults), the motifs CG:1:cpg::GATC:2:dam, and tombo plot roc's default
limit of 5*10^6 statistics.  It reports:
  - the labelling and curve kernel times of tb2_last_timing for the whole run, and the host
    time of the synchronised calls;
  - accuracy_curves end to end, over every statistic and at the default limit;
  - the drop-in composition (_compute_motif_stats + prep_accuracy_rates, which builds the
    reference's tuples) at the default limit;
  - where the unmodified reference is built (oracle/_ref), its _compute_motif_stats +
    sorted/compute_accuracy_rates on the host for the first --ref-stats statistics, scaled
    to the default limit and labelled as extrapolated;
  - a parity check of the fused curves against tests/roc_cases.py (bit-exact mismatches);
  - the GPU's name, power limit and maximum SM clock, read in the same run.
Nothing is written to the tree.

    python bench_roc.py [--genome 500000] [--coverage 25]
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

from tombo_b200 import _lib, tombo_helper as th, tombo_stats as ts  # noqa: E402
import roc_cases as rc  # noqa: E402

DESCS = 'CG:1:cpg::GATC:2:dam'
CLI_LIMIT = 5000000


def gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
            text=True).strip()
    except Exception as e:
        return 'unavailable: %r' % (e,)


def workload(genome_len, coverage, seed=20261017, block=10000):
    rs = np.random.RandomState(seed)
    seqs = [(c, ''.join(rs.choice(list('ACGT'), genome_len))) for c in ('chr1', 'chr2')]
    blocks = []
    for chrm, _ in seqs:
        for strand in '+-':
            for start in range(0, genome_len, block):
                end = min(genome_len, start + block)
                poss = np.arange(max(start, 8), min(end, genome_len - 8))
                pos = np.repeat(poss, rs.poisson(coverage, poss.shape[0]))
                b = np.zeros(pos.shape[0], dtype=rc.PER_READ_DT)
                b['pos'] = pos
                b['stat'] = rs.beta(0.5, 0.5, pos.shape[0])   # per-read p-value-like fractions
                b['read_id'] = rs.randint(0, 1 << 20, pos.shape[0])
                blocks.append((chrm, strand, start, end, b))
    return rc.Genome(seqs), blocks


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t) * 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--genome', type=int, default=500000)
    ap.add_argument('--coverage', type=float, default=25.0)
    ap.add_argument('--ref-stats', type=int, default=200000)
    args = ap.parse_args()
    genome, blocks = workload(args.genome, args.coverage)
    n_stats = int(sum(b[4].shape[0] for b in blocks))
    descs = th.parse_motif_descs(DESCS)
    ctx = _lib.get_context(0)

    def stats():
        return rc.Stats(blocks, 'stat')
    ts.accuracy_curves(rc.Stats(blocks[:4], 'stat'), descs, genome)          # warm-up
    runs = []
    for _ in range(2):
        _, label_ms = timed(lambda: ts._label_motif(ctx, stats(), descs, genome, None, None))
        label_kernel = ctx.last_timing()[0]
        curve_kernel, curve_host = 0.0, 0.0
        for k in range(2):
            n = ctx.accuracy_count(k)
            idx = ts._sample_idx(n, rc.ROC_PLOT_POINTS)
            _, ms = timed(lambda: ctx.accuracy_curve(k, *idx))
            curve_host += ms
            curve_kernel += ctx.last_timing()[0]
        fused, fused_ms = timed(lambda: ts.accuracy_curves(stats(), descs, genome))
        _, fused_lim_ms = timed(lambda: ts.accuracy_curves(stats(), descs, genome,
                                                           total_stats_limit=CLI_LIMIT))
        runs.append(dict(label_kernel_ms=label_kernel, label_call_ms=label_ms,
                         curve_kernel_ms=curve_kernel, curve_call_ms=curve_host,
                         fused_all_ms=fused_ms, fused_limit_ms=fused_lim_ms))
    n_labelled = {k: ctx.accuracy_count(i) for i, k in enumerate(('cpg', 'dam'))}

    def dropins():
        res = ts._compute_motif_stats(stats(), descs, genome, None, CLI_LIMIT)
        return ts.prep_accuracy_rates(res)
    _, dropin_ms = timed(dropins)
    # parity: the fused curves against the numpy restatement
    want, _ = rc.motif_stats(stats(), descs, genome)
    mismatches = 0
    for name, (st, lab) in want.items():
        for a, b in zip(fused[name], rc.curve(st, lab)):
            a, b = np.atleast_1d(a), np.atleast_1d(b)
            mismatches += int(np.sum(~((a == b) | (np.isnan(a) & np.isnan(b)))))
    out = dict(bench='roc', gpu=gpu_info(), n_stats=n_stats, n_blocks=len(blocks),
               n_labelled=n_labelled, runs=runs, dropin_limit_ms=dropin_ms,
               parity_mismatches=mismatches)
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import ref_harness as rh
    if rh.available():
        import warnings
        m = rh.load_reference()
        rdescs = m['th'].parse_motif_descs(DESCS)
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')

            def ref():
                res = m['ts']._compute_motif_stats(rc.Stats(blocks, 'stat'), rdescs, genome, None,
                                                   args.ref_stats)
                for v in res.values():
                    m['ts'].compute_accuracy_rates(list(zip(*sorted(v)))[1])
            _, ref_ms = timed(ref)
        out['reference_ms_at_%d' % args.ref_stats] = ref_ms
        out['reference_ms_at_limit_extrapolated'] = ref_ms * CLI_LIMIT / args.ref_stats
    print(json.dumps(out))


if __name__ == '__main__':
    main()
