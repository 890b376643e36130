"""Statistics file on the device (aggregate_per_read_stats): one JSON line.

Workload: a synthetic genome-scale per-read statistics file, --blocks blocks of 10 kb over
two chromosomes x both strands, about --entries per-read p-values in all (~110 per covered
position at the defaults: 1e8 entries over 900 blocks), quantised to 1/64 so damp_frac ties
are common, and a most-significant table of N = 100 000 rows.  All blocks go to the device in
one call.  Reported, as the median of --reps runs after a warm-up:
  * agg_kernel_ms   tb2_stats_file_aggregate's kernels (CUDA events, tb2_last_timing);
  * topn_device_ms  CUDA events around tb2_most_signif_add_aggregate's kernel and around the
                    sort of tb2_most_signif_count; the sort's window also holds its one host
                    round trip (the digit histograms to the host to plan the passes);
  * end_to_end_ms   host arrays in, block tables and table out: upload, kernels, downloads
                    (host clock around synchronised calls);
  * numpy_restatement_ms  the same result from tests/stats_file_cases.py on the host, once,
                    for context.
The table is checked against the restatement.  The GPU's name, power limit and maximum SM
clock are read in the same run.

    python bench_stats_file.py [--blocks 900] [--entries 100000000] [--reps 3]
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

from tombo_b200 import _lib  # noqa: E402
import stats_file_cases as sc  # noqa: E402

REGION, N, THRESH, DAMP = 10000, 100000, 0.25, (2.0, 0.0)


def gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
            text=True).strip()
    except Exception as e:
        return 'unavailable: %r' % (e,)


def workload(n_blocks, n_entries, seed=5):
    rng = np.random.default_rng(seed)
    per = n_entries // n_blocks
    rows = np.zeros((n_blocks, 5), dtype=np.int64)
    groups = [(c, s) for c in (0, 1) for s in (b'+', b'-')]
    for b in range(n_blocks):
        c, s = groups[b % 4]
        rows[b] = ((b // 4) * REGION, b * per, per, c, s[0])
    pos = (rng.integers(0, REGION, size=(n_blocks, per), dtype=np.int64)
           + rows[:, :1]).astype(np.uint32).ravel()
    stat = np.floor(rng.random(n_blocks * per) * 64) / 64
    return rows, pos, stat


def run(ctx, rows, pos, stat):
    t0 = time.perf_counter()
    off = ctx.stats_file_aggregate(rows, REGION, pos, stat, THRESH, None, 1, *DAMP)
    agg_ms = ctx.last_timing()[0]
    cols = ctx.stats_file_download(int(off[-1]))
    ctx.most_signif_begin(False, N)
    ctx.most_signif_add_aggregate()
    topn_ms = ctx.last_timing()[0]
    ctx.most_signif_count()
    topn_ms += ctx.last_timing()[0]
    table = ctx.most_signif_get()
    ctx.most_signif_end()
    return (time.perf_counter() - t0) * 1e3, agg_ms, topn_ms, off, cols, table


def restate(rows, pos, stat):
    t0 = time.perf_counter()
    parts = []
    for start, s0, n, c, s in rows:
        tab = sc.restate_block(pos[s0:s0 + n], stat[s0:s0 + n], THRESH, None, False, *DAMP)
        parts.append(sc.with_chrm_strand(tab, c, bytes([s])))
    ms = sc.restate_most_signif(np.concatenate(parts), N)
    return (time.perf_counter() - t0) * 1e3, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--blocks', type=int, default=900)
    ap.add_argument('--entries', type=int, default=100000000)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    rows, pos, stat = workload(a.blocks, a.entries)
    ctx = _lib.Context(0)
    run(ctx, rows, pos, stat)                                  # warm-up: modules, buffers
    res = [run(ctx, rows, pos, stat) for _ in range(a.reps)]
    np_ms, ms = restate(rows, pos, stat)
    t = res[-1][5]
    ok = (np.array_equal(t['key'].view(np.uint64), ms['damp_frac'].view(np.uint64)) and
          all(np.array_equal(t[k], ms[k]) for k in ('pos', 'cov', 'valid_cov', 'chrm', 'strand')) and
          np.array_equal(t['frac'].view(np.uint64), ms['frac'].view(np.uint64)))
    med = lambda i: float(np.median([r[i] for r in res]))
    out = dict(bench='stats_file', gpu=gpu_info(), blocks=a.blocks, entries=int(pos.shape[0]),
               rows=int(res[-1][3][-1]), num_most_signif=N, reps=a.reps,
               agg_kernel_ms=med(1), topn_device_ms=med(2), end_to_end_ms=med(0),
               end_to_end_all_ms=[r[0] for r in res], numpy_restatement_ms=np_ms,
               table_matches_restatement=bool(ok))
    ctx.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
