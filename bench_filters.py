"""Read filters on the device: one JSON line.

Workloads:
  * resident: a configs[1] batch (--reads synthetic DNA reads of 444 bases, ~4k samples,
    bandwidth 200) resquiggled once; tb2_batch_compute's kernel time and then
    tb2_batch_read_filters' (signal matching and the obs filter 90:10, 50:5) on the same
    batch, both on CUDA events (tb2_last_timing), median of --reps filter calls;
  * stuck: tb2_dwell_percentiles on --pctl-reads host reads of 1 to 600 Events lengths
    (mean ~60), percentiles 50 and 90: kernel ms and host arrays in to results out;
  * coverage: tb2_read_mid_coverage on --cov-reads reads over a 5 Mb genome, both strands:
    kernel ms and end to end;
  * the numpy / reference time of the same work on the host (np.percentile per read for
    sampled reads scaled up; the slice-add coverage loop of _filter_reads.py) for context.
Device results are checked against the host.  The GPU's name, power limit and maximum SM
clock are read in the same run.

    python bench_filters.py [--reads 100000] [--pctl-reads 1000000] [--cov-reads 1000000]
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

from tombo_b200 import _lib, synthetic as syn  # noqa: E402

ALN_DNA = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
OBS = [[90, 10], [50, 5]]


def gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
            text=True).strip()
    except Exception as e:
        return 'unavailable: %r' % (e,)


class RP(object):
    def __init__(self, save=False):
        (self.match_evalue, self.skip_pen, bw, sbw, self.max_half_z_score, self.band_bound_thresh,
         self.start_bw, self.start_save_bw, self.start_n_bases) = ALN_DNA
        self.bandwidth = sbw if save else bw
        (self.running_stat_width, self.min_obs_per_base, self.raw_min_obs_per_base,
         self.mean_obs_per_event) = (5, 3, 1, 5)
        self.z_shift = float(np.sqrt(2.0 / np.pi)) + self.match_evalue
        self.stay_pen = self.match_evalue
        self.use_t_test_seg = False


def resident(ctx, n_reads, reps):
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, 6, cpos)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, n_reads, 444, 2024)
    rp, sp, pol = RP(), RP(True), _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    compute_ms = ctx.last_timing()[0]
    ms = []
    for _ in range(reps + 1):
        code = ctx.batch_read_filters(1.1, OBS)
        ms.append(ctx.last_timing()[0])
    res = ctx.batch_download()
    segs = [res['segs'][a:b] for a, b in zip(res['seg_off'][:-1], res['seg_off'][1:])]
    ok = res['status'] == 0
    # check, and time the host restatement on a sample of reads
    idx = np.random.RandomState(0).choice(n_reads, size=min(n_reads, 5000), replace=False)
    t0 = time.perf_counter()
    for i in idx:
        if not ok[i]:
            want = -1
        elif res['sig_match_score'][i] > 1.1:
            want = 1
        else:
            d = np.diff(segs[i])
            want = 2 if any(np.percentile(d, p) > t for p, t in OBS) else 0
        assert code[i] == want, (i, code[i], want)
    host_ms = (time.perf_counter() - t0) * 1e3 * n_reads / len(idx)
    return dict(reads=n_reads, compute_kernel_ms=compute_ms, filter_kernel_ms=float(np.median(ms[1:])),
                filter_share_of_compute=float(np.median(ms[1:])) / compute_ms,
                codes=dict((str(c), int((code == c).sum())) for c in (-1, 0, 1, 2)),
                host_numpy_ms_est=host_ms)


def stuck(ctx, n, reps):
    rng = np.random.RandomState(1)
    sizes = np.minimum(rng.geometric(1 / 60.0, size=n), 600)
    lens = rng.choice([1, 2, 3, 4, 6, 10, 30], size=int(sizes.sum())).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    pctl = [p for p, _ in OBS]
    ctx.dwell_percentiles(lens[:off[100]], off[:101], pctl)
    kern, e2e = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = ctx.dwell_percentiles(lens, off, pctl)
        e2e.append((time.perf_counter() - t0) * 1e3)
        kern.append(ctx.last_timing()[0])
    idx = rng.choice(n, size=2000, replace=False)
    t0 = time.perf_counter()
    for i in idx:
        x = lens[off[i]:off[i + 1]]
        w = [np.percentile(x, p) for p in pctl]
        assert out[i].tobytes() == np.array(w).tobytes()
    host_ms = (time.perf_counter() - t0) * 1e3 * n / len(idx)
    return dict(reads=n, lengths=int(off[-1]), kernel_ms=float(np.median(kern)),
                end_to_end_ms=float(np.median(e2e)), host_numpy_ms_est=host_ms)


def coverage(ctx, n, reps):
    rng = np.random.RandomState(2)
    G = 5000000
    strand = rng.randint(0, 2, size=n)
    order = np.argsort(strand, kind='stable')
    start = rng.randint(0, G - 20000, size=n)[order].astype(np.int64)
    end = (start + rng.randint(300, 20000, size=n)).astype(np.int64)
    n_minus = int((strand == 0).sum())
    grp_off = np.array([0, n_minus, n], dtype=np.int64)
    ctx.read_mid_coverage(np.array([0, 10]), start[:10], end[:10])     # warm-up
    kern, e2e = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = ctx.read_mid_coverage(grp_off, start, end)
        e2e.append((time.perf_counter() - t0) * 1e3)
        kern.append(ctx.last_timing()[0])
    t0 = time.perf_counter()                       # the reference's loop (_filter_reads.py:113-126)
    want = np.empty(n, dtype=np.int64)
    for a, b in zip(grp_off[:-1], grp_off[1:]):
        cov = np.zeros(int(end[a:b].max()), dtype=np.int64)
        for i in range(a, b):
            cov[start[i]:end[i]] += 1
        for i in range(a, b):
            want[i] = cov[start[i] + (end[i] - start[i]) // 2]
    host_ms = (time.perf_counter() - t0) * 1e3
    assert np.array_equal(out, want)
    return dict(reads=n, genome=G, strands=2, kernel_ms=float(np.median(kern)),
                end_to_end_ms=float(np.median(e2e)), host_reference_ms=host_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reads', type=int, default=100000)
    ap.add_argument('--pctl-reads', type=int, default=1000000)
    ap.add_argument('--cov-reads', type=int, default=1000000)
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    ctx = _lib.Context(0)
    out = dict(bench='read_filters', gpu=gpu_info(),
               resident=resident(ctx, a.reads, a.reps),
               stuck=stuck(ctx, a.pctl_reads, a.reps),
               coverage=coverage(ctx, a.cov_reads, a.reps))
    ctx.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
