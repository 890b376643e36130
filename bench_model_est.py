#!/usr/bin/env python
"""Per-k-mer Gaussian kernel densities on the device (tb2_kernel_densities, the cost of
`tombo build_model estimate_alt_reference`): seeded level sets at the reference's default
shape, bandwidth 0.05 (--kernel-density-bandwidth) and 500 points over (-5, 5).

Prints one JSON line, per workload (a) 4 096 sets x 10 000 levels, (b) 1 024 sets x
1 000 levels and (c) one set of 10^6 levels, after a warm-up call:
  kernel_ms   device time of the two kernels (tb2_last_timing), terms_per_s from it
              (terms = levels x grid points, the reference's per-term work);
  setup_ms    the part of kernel_ms spent in the per-set setup kernel (std, factor, c);
  call_ms     host clock around the whole call, upload of the levels and download included.
Also the GPU's name and power limit (queried in the same run), parity against scipy's
gaussian_kde on a seeded sample of sets (within the bound of tests/kde_cases.py), and
scipy's ns per term measured on the host in the same run, with the reference's time per
sample extrapolated from it (not run: labelled as such)."""
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

from tombo_b200 import _lib  # noqa: E402

BW = 0.05
GRID = np.linspace(-5, 5, 500)


def make_sets(rs, n_sets, n_levels):
    centres = rs.normal(0, 1, n_sets)
    levels = (rs.normal(0, 0.25, (n_sets, n_levels)) + centres[:, None]).ravel()
    return levels, np.arange(n_sets + 1, dtype=np.int64) * n_levels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--parity-sets', type=int, default=8)
    args = ap.parse_args()
    import kde_cases as kc
    out = {'workload': 'bandwidth %g, %d grid points' % (BW, GRID.shape[0]), 'results': [],
           'parity_checked': 0, 'parity_mismatches': 0}
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    out['gpu'] = q[0] if q else 'unknown'
    ctx = _lib.Context(0)
    rs = np.random.RandomState(1914)
    for n_sets, n_levels in ((4096, 10000), (1024, 1000), (1, 10 ** 6)):
        levels, off = make_sets(rs, n_sets, n_levels)
        ctx.kernel_densities(levels, off, GRID, BW)                 # warm-up
        kern, setup, call = [], [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            dens, cho, factor = ctx.kernel_densities(levels, off, GRID, BW)
            call.append((time.perf_counter() - t0) * 1e3)
            kern.append(ctx.last_timing()[0])
            setup.append(ctx.last_timing()[1])
        terms = float(levels.shape[0]) * GRID.shape[0]
        out['results'].append(dict(
            sets=n_sets, levels_per_set=n_levels, kernel_ms=float(np.median(kern)),
            setup_ms=float(np.median(setup)), call_ms=float(np.median(call)), terms_per_s=terms / (np.median(kern) * 1e-3),
            call_terms_per_s=terms / (np.median(call) * 1e-3)))
        for i in rs.choice(n_sets, min(n_sets, args.parity_sets), replace=False):
            x = levels[off[i]:off[i + 1]]
            want, c_ref = kc.scipy_kde(x, GRID, BW)
            bound = (kc.density_bound(x, GRID, cho[i], want) +
                     kc.c_widening(x, GRID, cho[i], c_ref))
            ok = (np.abs(dens[i] - want) <= bound).all() and abs(cho[i] - c_ref) <= kc.c_bound(x.shape[0]) * c_ref
            out['parity_checked'] += 1
            out['parity_mismatches'] += int(not ok)
    ctx.close()
    # scipy on the host, one thread's worth: n = 3 000 levels, 500 points
    x = rs.normal(0, 0.25, 3000)
    t0 = time.perf_counter()
    reps = 3
    for _ in range(reps):
        kc.scipy_kde(x, GRID, BW)
    ns = (time.perf_counter() - t0) / reps / (x.shape[0] * GRID.shape[0]) * 1e9
    out['scipy_ns_per_term'] = ns
    out['reference_min_per_sample_extrapolated'] = {
        '4096 k-mers x 1000 levels': 4096 * 1000 * 500 * ns * 1e-9 / 60,
        '4096 k-mers x 10000 levels': 4096 * 10000 * 500 * ns * 1e-9 / 60}
    out['parity_against'] = 'scipy.stats.gaussian_kde within the bound of tests/kde_cases.py'
    print(json.dumps(out))


if __name__ == '__main__':
    main()
