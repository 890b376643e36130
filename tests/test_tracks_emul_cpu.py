"""The genome browser tracks' device source (csrc/browser_tracks.cuh with the coverage scan of
read_filter.cuh and radix_sort.cuh) run on the host through tests/emul: coverage runs against
the np.diff encoding, slot means bit for bit against the reference's slice-add loop, and every
golden case of `tombo text_output browser_files` through text_output."""
import os
import sys

import numpy as np
import pytest

import tracks_cases as tc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emul'))
import emul_tracks as et     # noqa: E402

GOLD = tc.load_golden()


def _reads(rng, sizes, max_reads, max_span):
    grp_off, start, end = [0], [], []
    for s in sizes:
        k = rng.randint(1, max_reads + 1) if s else 0
        for _ in range(k):
            a = rng.randint(0, s)
            start.append(a)
            end.append(a + rng.randint(1, min(max_span, s - a) + 1))
        grp_off.append(grp_off[-1] + k)
    return np.array(grp_off), np.array(start, np.int64), np.array(end, np.int64)


def test_coverage_runs_match_numpy():
    # groups across several 4096-entry scan tiles, empty groups, one-read groups
    rng = np.random.RandomState(11)
    grp_off, start, end = _reads(rng, [0, 1, 300, 5000, 9000, 0, 17000, 2], 60, 3000)
    one = np.array([0, 1, 1, 2])
    for args in [(grp_off, start, end), (one, np.array([5, 0]), np.array([9, 4100]))]:
        got = et.EmulContext().coverage_runs(*args)
        want = tc.HostContext().coverage_runs(*args)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)


def _batches(rng, n_reads, chrm_len, split):
    start = rng.randint(0, chrm_len - 200, size=n_reads)
    nv = rng.randint(0, 200, size=n_reads)
    rev = rng.rand(n_reads) < 0.5
    vals = rng.choice([-1, 1], size=nv.sum()) * 10.0 ** rng.uniform(-10, 6, size=nv.sum())
    vals[rng.rand(vals.shape[0]) < 0.001] = np.nan
    vals[rng.rand(vals.shape[0]) < 0.01] = -0.0
    off = np.concatenate([[0], np.cumsum(nv)])
    cuts = [0] + sorted(rng.choice(np.arange(1, n_reads), size=split - 1, replace=False)) + [n_reads]
    return [(start[a:b], off[a:b + 1] - off[a], vals[off[a]:off[b]], rev[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]


@pytest.mark.parametrize('split', [1, 3, 8])
def test_slot_means_bit_exact(split):
    rng = np.random.RandomState(split)
    batches = _batches(rng, 900, 6000, split)
    got = et.EmulContext().slot_means(6000, batches)
    want = tc.HostContext().slot_means(6000, batches)
    assert got.tobytes() == want.tobytes()


def test_slot_means_deep_position():
    # 3000 values on one position, then split over two calls: the running sum continues
    rng = np.random.RandomState(5)
    vals = rng.choice([-1, 1], size=3000) * 10.0 ** rng.uniform(-12, 6, size=3000)
    b = [(np.full(1500, 7), np.arange(1501), vals[:1500], np.zeros(1500, bool)),
         (np.full(1500, 7), np.arange(1501), vals[1500:], np.ones(1500, bool))]
    got = et.EmulContext().slot_means(10, b)
    want = tc.HostContext().slot_means(10, b)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize('case', GOLD['cases'], ids=lambda c: c['name'])
def test_browser_files_match_reference(case, tmp_path):
    tc.same_files(tc.run_case(case, str(tmp_path), et.EmulContext()), case['files'])
