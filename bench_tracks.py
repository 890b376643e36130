"""Genome browser tracks on the device: one JSON line.

Workloads:
  * coverage: tb2_coverage_runs on --reads reads of ~450 bases over a 5 Mb genome, both strands
    (two groups): kernel ms (tb2_last_timing) and host arrays in to runs out;
  * slot means: tb2_slot_sums_* over the same reads, one accumulation per strand, values fed in
    batches of 2^24: kernel ms summed over the calls, and host arrays in to means out;
  * browser files: text_output.write_all_browser_files(coverage, signal) for --file-reads reads
    whose Events are served from memory (the FakeFile stand-in of the tests), split into Events
    reading, device work, and formatting and writing;
  * the reference's slice-add loop (get_mean_slot_genome_centric) on the host for a sample of
    the reads, scaled to --reads, for context.
Parity with the numpy restatement is checked after the timed regions.  The GPU's name, power
limit and maximum SM clock are read in the same run.

    python bench_tracks.py [--reads 1000000] [--file-reads 100000] [--reps 5]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [REPO, os.path.join(REPO, 'tests')]

from tombo_b200 import _lib, formats, text_output, tombo_helper as th  # noqa: E402

GLEN = 5000000
BATCH = 1 << 24


def gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
            text=True).strip()
    except Exception as e:
        return 'unavailable: %r' % (e,)


def make_reads(rng, n):
    start = rng.randint(0, GLEN - 700, size=n).astype(np.int64)
    nv = rng.randint(300, 600, size=n).astype(np.int64)
    minus = rng.rand(n) < 0.5
    return start, nv, minus


def coverage(ctx, start, nv, minus, reps):
    order = np.concatenate([np.flatnonzero(~minus), np.flatnonzero(minus)])
    s, e = start[order], (start + nv)[order]
    grp_off = np.array([0, int((~minus).sum()), start.shape[0]])
    kern, wall = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = ctx.coverage_runs(grp_off, s, e)
        wall.append((time.perf_counter() - t0) * 1e3)
        kern.append(ctx.last_timing()[0])
    ok = True
    for g in range(2):
        a, b = grp_off[g], grp_off[g + 1]
        diff = np.zeros(e[a:b].max() + 1, dtype=np.int64)
        np.add.at(diff, s[a:b], 1)
        np.add.at(diff, e[a:b], -1)
        cov = np.cumsum(diff)[:-1]
        st = np.concatenate([[0], np.where(np.diff(cov))[0] + 1])
        ok &= np.array_equal(res[1][res[0][g]:res[0][g + 1]], st)
        ok &= np.array_equal(res[2][res[0][g]:res[0][g + 1]], cov[st])
    return float(np.median(kern)), float(np.median(wall)), int(res[0][-1]), bool(ok)


def strand_batches(start, nv, minus, strand, pool):
    sel = np.flatnonzero(minus == strand)
    out, a = [], 0
    cum = np.concatenate([[0], np.cumsum(nv[sel])])
    while a < sel.shape[0]:
        b = int(np.searchsorted(cum, cum[a] + BATCH, side='right')) - 1
        b = max(b, a + 1)
        off = cum[a:b + 1] - cum[a]
        out.append((start[sel[a:b]], off, pool[:off[-1]], np.full(b - a, strand)))
        a = b
    return out


def slot_means(ctx, start, nv, minus, pool, reps):
    batches = [strand_batches(start, nv, minus, s, pool) for s in (False, True)]
    kern, wall = [], []
    for _ in range(reps):
        k = 0.0
        t0 = time.perf_counter()

        def timed(bs):
            nonlocal k
            for b in bs:
                yield b
                k += ctx.last_timing()[0]
        for bs in batches:
            ctx.slot_means(GLEN, timed(bs))
            k += ctx.last_timing()[0]
        wall.append((time.perf_counter() - t0) * 1e3)
        kern.append(k)
    return float(np.median(kern)), float(np.median(wall)), len(batches[0]) + len(batches[1])


def slot_parity(ctx, rng, n):
    import tracks_cases as tc
    start, nv, minus = make_reads(rng, n)
    ok = True
    for strand in (False, True):
        sel = minus == strand
        off = np.concatenate([[0], np.cumsum(nv[sel])])
        vals = rng.normal(0, 1, off[-1]) * 10.0 ** rng.uniform(-3, 3, off[-1])
        cuts = [0, sel.sum() // 3, sel.sum()]
        bs = [(start[sel][a:b], off[a:b + 1] - off[a], vals[off[a]:off[b]], np.full(b - a, strand))
              for a, b in zip(cuts[:-1], cuts[1:])]
        ok &= ctx.slot_means(GLEN, bs).tobytes() == tc.HostContext().slot_means(GLEN, bs).tobytes()
    return bool(ok)


def reference_loop_ms(rng, n_sample, n_total):
    start, nv, minus = make_reads(rng, n_sample)
    vals = [rng.normal(0, 1, k) for k in nv]
    base_sums, base_cov = np.zeros(GLEN), np.zeros(GLEN, dtype=np.int64)
    t0 = time.perf_counter()
    for r in range(n_sample):
        v = vals[r][::-1] if minus[r] else vals[r]
        base_sums[start[r]:start[r] + nv[r]] += v
        base_cov[start[r]:start[r] + nv[r]] += 1
    with np.errstate(invalid='ignore', divide='ignore'):
        base_sums / base_cov
    return (time.perf_counter() - t0) * 1e3 * n_total / n_sample


def browser_files(ctx, rng, n):
    import filters_cases as fc
    import tracks_cases as tc
    start, nv, minus = make_reads(rng, n)
    tmp = tempfile.mkdtemp(prefix='bench_tracks_')
    try:
        d = os.path.join(tmp, 'reads') + '/'
        os.makedirs(d)
        groups, store = {}, {}
        mean_pool, nan_pool, one_pool = rng.normal(0, 1, 1 << 20), np.full(1000, np.nan), np.ones(1000, np.uint32)
        for r in range(n):
            fn = 'r%07d.fast5' % r
            cs = ('chr1', '-' if minus[r] else '+')
            groups.setdefault(cs, []).append([fn, int(start[r]), int(start[r] + nv[r]), 0, tc.CORR_GRP,
                                              tc.SUBGRP, False, False, None, None, 'id%d' % r])
            k = int(nv[r])
            o = int(rng.randint(0, (1 << 20) - k))
            store[d + fn] = dict(events=dict(norm_mean=mean_pool[o:o + k], norm_stdev=nan_pool[:k],
                                             length=one_pool[:k]))
        fc.write_index(d, [[list(k), v] for k, v in groups.items()])
        ev_ms, dev_ms = [0.0], [0.0]
        read_slot, cov_runs, means = th.get_single_slot_read_centric, ctx.coverage_runs, ctx.slot_means

        def timed_read(*a, **k):
            t0 = time.perf_counter()
            try:
                return read_slot(*a, **k)
            finally:
                ev_ms[0] += (time.perf_counter() - t0) * 1e3

        def timed_cov(*a):
            t0 = time.perf_counter()
            try:
                return cov_runs(*a)
            finally:
                dev_ms[0] += (time.perf_counter() - t0) * 1e3

        def timed_means(*a):
            t0, e0 = time.perf_counter(), ev_ms[0]
            try:
                return means(*a)
            finally:
                dev_ms[0] += (time.perf_counter() - t0) * 1e3 - (ev_ms[0] - e0)
        th.get_single_slot_read_centric = timed_read
        ctx.coverage_runs, ctx.slot_means = timed_cov, timed_means
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            with tc.events_h5py(store):
                t0 = time.perf_counter()
                text_output.write_all_browser_files([d], None, tc.CORR_GRP, None, None, 'bench',
                                                    ['coverage', 'signal'], ctx=ctx)
                total = (time.perf_counter() - t0) * 1e3
        finally:
            os.chdir(cwd)
            th.get_single_slot_read_centric = read_slot
            del ctx.coverage_runs, ctx.slot_means
        size = sum(os.path.getsize(os.path.join(tmp, f)) for f in os.listdir(tmp) if f.startswith('bench.'))
        return dict(reads=n, total_ms=round(total, 1), events_ms=round(ev_ms[0], 1),
                    device_ms=round(dev_ms[0], 1), format_write_ms=round(total - ev_ms[0] - dev_ms[0], 1),
                    bytes_written=size)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reads', type=int, default=1000000)
    ap.add_argument('--file-reads', type=int, default=100000)
    ap.add_argument('--ref-sample', type=int, default=20000)
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    ctx = _lib.Context(0)
    rng = np.random.RandomState(5)
    start, nv, minus = make_reads(rng, a.reads)
    pool = rng.normal(0, 1, BATCH)
    cov_k, cov_w, n_runs, cov_ok = coverage(ctx, start, nv, minus, a.reps)
    sm_k, sm_w, n_calls = slot_means(ctx, start, nv, minus, pool, a.reps)
    files = browser_files(ctx, rng, a.file_reads)
    ref_ms = reference_loop_ms(rng, a.ref_sample, a.reads)
    parity = cov_ok and slot_parity(ctx, rng, 20000)
    out = dict(bench='browser_tracks', gpu=gpu_info(), reads=a.reads, genome=GLEN, strands=2,
               values=int(nv.sum()),
               coverage_runs=dict(kernel_ms=round(cov_k, 3), host_to_results_ms=round(cov_w, 2), runs=n_runs),
               slot_means=dict(kernel_ms=round(sm_k, 2), host_to_results_ms=round(sm_w, 1), add_calls=n_calls),
               browser_files=files, reference_slice_add_ms=round(ref_ms, 1), parity=parity)
    ctx.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
