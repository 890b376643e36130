#!/usr/bin/env python
"""Level tests on the device: one 10 kb region (the reference's default
--multiprocess-region-size) of seeded synthetic reads at 20 / 200 / 2000 reads per sample,
each of the six level statistics with fm_offset = 1, and get_reads_ref at 200 reads.

Prints one JSON line, per workload (after warm-up, averaged over at least a second of work):
  kernel_ms   device time from the call's first kernel to its last (tb2_last_timing), and
              kernel_positions_per_s from it;
  device_ms   tb2_timer_start / _stop around the whole call: upload of the levels, kernels,
              download (positions_per_s from it);
  e2e_ms      host clock around the call (ctypes, host checks, the pageable copies).
Also the GPU's name and power limit (queried in the same run), parity mismatches against
the numpy / scipy restatement in tests/test_group_stats_gpu.py on a sample of positions,
and, where oracle/_ref holds a build of the reference, the reference's own
compute_group_reg_stats on the host (positions/s on a 1 000-position region, 200 reads per
sample; "not measured" otherwise)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))

from tombo_b200 import _lib, tombo_stats as ts  # noqa: E402

REG = 10000
TESTS = [(st,) + ts._LEVEL_TESTS[st] for st in ts.LEVEL_STATS_TXTS]


def make_sample(rs, n_reads, shift):
    """n_reads reads of 1-12 kb around the region, genome-ordered, ~2 % missing levels"""
    starts = rs.randint(-2000, REG, n_reads).astype(np.int64)
    lens = rs.randint(1000, 12000, n_reads).astype(np.int64)
    lv = rs.normal(0.0, 1.0, int(lens.sum())) + shift
    lv[rs.uniform(size=lv.shape[0]) < 0.02] = np.nan
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return lv, off, starts


def dense(sample):
    lv, off, st = sample
    m = np.full((REG + 2, off.shape[0] - 1), np.nan)
    for r in range(off.shape[0] - 1):
        a, b = max(st[r], -1), min(st[r] + off[r + 1] - off[r], REG + 1)
        if b > a:
            m[a + 1:b + 1, r] = lv[off[r] + a - st[r]:off[r] + b - st[r]]
    return m


def timed(ctx, fn, min_s=1.0):
    fn()                                      # warm-up (pools, modules)
    reps, t_kern, t_dev, t_e2e = 0, 0.0, 0.0, 0.0
    while t_e2e < min_s:
        t0 = time.perf_counter()
        ctx.timer_start()
        fn()
        t_dev += ctx.timer_stop()
        t_e2e += time.perf_counter() - t0
        t_kern += ctx.last_timing()[0]
        reps += 1
    return t_kern / reps, t_dev / reps, 1e3 * t_e2e / reps


def row(name, n, n_pos, kern_ms, dev_ms, e2e_ms):
    return dict(stat=name, reads=n, kernel_ms=round(kern_ms, 3),
                kernel_positions_per_s=round(n_pos / kern_ms * 1e3), device_ms=round(dev_ms, 3),
                positions_per_s=round(n_pos / dev_ms * 1e3), e2e_ms=round(e2e_ms, 3))


def reference_arm(rs, n_reads=200, n_pos=1000):
    """the unmodified reference's compute_group_reg_stats on the host, reads served at its
    get_single_slot_read_centric seam"""
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import ref_harness as rh
    if not rh.available():
        return 'not measured'
    m = rh.load_reference()
    th = m['th']
    served = {}
    th.get_single_slot_read_centric = lambda r, slot: served[r.fn].copy()

    def interval(tag):
        reads = []
        for i in range(n_reads):
            a = int(rs.randint(-150, n_pos - 100))          # every read overlaps the region
            b = int(min(n_pos + 500, a + rs.randint(200, 1500)))
            served['%s%d' % (tag, i)] = rs.normal(0.0, 1.0, b - a)
            reads.append(th.readData(a, b, False, 0, '+', '%s%d' % (tag, i), 'g', False))
        return th.intervalData('chr', 0, n_pos, None, reads=reads)
    reg, creg = interval('s'), interval('c')
    out = {}
    with rh.ref_errstate():
        for name in ts.LEVEL_STATS_TXTS:
            t0 = time.perf_counter()
            res = m['ts'].compute_group_reg_stats(reg, creg, 1, 1, name)
            dt = time.perf_counter() - t0
            out[name] = round(res[0][1].reg_poss.shape[0] / dt)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reads', default='20,200,2000')
    ap.add_argument('--parity-positions', type=int, default=40)
    args = ap.parse_args()
    import test_group_stats_gpu as chk
    ctx = _lib.Context(0)
    rs = np.random.RandomState(12345)
    out = {'workload': 'one %d-position region, fm_offset 1' % REG, 'results': [],
           'parity_checked': 0, 'parity_mismatches': 0}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        out['gpu'] = q[0] if q else 'unknown'
    except Exception as e:                   # noqa: BLE001
        out['gpu'] = 'unknown (%s)' % e
    for n in [int(x) for x in args.reads.split(',')]:
        samp, ctrl = make_sample(rs, n, 0.1), make_sample(rs, n, 0.0)
        ds, dc = dense(samp), dense(ctrl)
        pick = rs.choice(REG, args.parity_positions, replace=False)
        for name, test, rstat in TESTS:
            call = lambda: ctx.group_reg_stats(-1, REG + 2, samp, ctrl, test, rstat, 1, 1)  # noqa
            kern_ms, dev_ms, e2e_ms = timed(ctx, call)
            r = call()
            out['results'].append(row(name, n, r['pos'].shape[0], kern_ms, dev_ms, e2e_ms))
            # parity: the raw per-position statistic (fm_offset 0) at sampled positions
            r0 = ctx.group_reg_stats(-1, REG + 2, samp, ctrl, test, rstat, 1, 0)
            at = dict(zip(r0['pos'].tolist(), r0['stat']))
            for p in pick:
                s, c = ds[p + 1], dc[p + 1]
                s, c = s[~np.isnan(s)], c[~np.isnan(c)]
                if s.shape[0] == 0 or c.shape[0] == 0:
                    continue
                want = chk.pos_stat(s, c, name)
                got = at[int(p)]
                ok = chk.stats_equal(np.array([got]), np.array([want]), name)
                out['parity_checked'] += 1
                out['parity_mismatches'] += int(not ok)
        if n == 200:
            call = lambda: ctx.reads_ref_levels(-1, REG + 2, ctrl, 1)  # noqa: E731
            kern_ms, dev_ms, e2e_ms = timed(ctx, call)
            out['results'].append(row('get_reads_ref', n, REG + 2, kern_ms, dev_ms, e2e_ms))
    ctx.close()
    out['parity_against'] = 'numpy / scipy restatement (tests/test_group_stats_gpu.py)'
    out['reference_positions_per_s'] = reference_arm(rs)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
