"""The read filters' device source (csrc/read_filter.cuh) run on the host through tests/emul:
percentiles bit for bit against np.percentile, coverage against numpy, and every filter
command and the index batch against the unmodified reference's goldens."""
import os
import sys

import numpy as np
import pytest

import filters_cases as fc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emul'))
import emul_read_filter as erf     # noqa: E402

GOLD = fc.load_golden()
PCTL_SETS = [[0, 100], [50], [33, 67, 25, 75], [12.5, 99.9, 0.1, 37.0], [90, 10]]


def _ragged(rng, n, sizes, hi=40):
    lens = [rng.randint(1, hi, size=int(rng.choice(sizes))) for _ in range(n)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lens])]).astype(np.int64)
    return lens, off


@pytest.mark.parametrize('pctl', PCTL_SETS)
def test_percentiles_bit_exact(pctl):
    rng = np.random.RandomState(len(pctl))
    lens, off = _ragged(rng, 60, [1, 2, 3, 4, 5, 64, 257, 3000])
    got = erf.EmulContext().dwell_percentiles(np.concatenate(lens), off, pctl)
    want = np.array([[np.percentile(x, p) for p in pctl] for x in lens])
    assert got.tobytes() == want.tobytes()


def test_mid_coverage_matches_numpy():
    rng = np.random.RandomState(3)
    sizes = [0, 1, 300, 5000, 9000]
    grp_off = np.concatenate([[0], np.cumsum([rng.randint(0, 40) if s else 0 for s in sizes])])
    start, end = [], []
    for g, s in enumerate(sizes):
        for _ in range(grp_off[g + 1] - grp_off[g]):
            a = rng.randint(0, max(s - 1, 1))
            start.append(a)
            end.append(a + rng.randint(1, max(2, min(3000, s - a + 1))))
    start, end = np.array(start), np.array(end)
    got = erf.EmulContext().read_mid_coverage(grp_off, start, end)
    assert np.array_equal(got, fc.HostContext().read_mid_coverage(grp_off, start, end))


@pytest.mark.parametrize('case', [c for c in GOLD['filters'] if c['cmd'] in ('stuck', 'coverage')],
                         ids=lambda c: c['name'])
def test_filter_commands_match_reference(case, tmp_path):
    kind, got = fc.run_filter_case(case, erf.EmulContext(), str(tmp_path))
    if 'error' in case:
        assert kind == 'error'
    else:
        assert got == case['output']


@pytest.mark.parametrize('case', GOLD['io'], ids=lambda c: c['name'])
def test_index_batch_matches_io_and_map_read(case):
    r = case['reads']
    segs = [x['segs'] for x in r]
    ok = [not x['failed'] for x in r]
    codes, pv = erf.EmulContext().batch_read_filters_on(
        segs, [x['score'] for x in r], ok, case['sig_match_thresh'], case['obs_filter'])
    assert list(codes) == fc.host_codes(segs, [x['score'] for x in r], ok,
                                         case['sig_match_thresh'], case['obs_filter'])
    for i, s in enumerate(segs):
        want = [np.percentile(np.diff(s), p) for p, _ in (case['obs_filter'] or [])]
        assert pv[i].tobytes() == (np.array(want) if ok[i] else np.full(len(want), np.nan)).tobytes()
    index, failed = fc.run_io_case(case, codes)
    assert index.records() == fc.golden_io_index(case).records()
    assert [list(f) for f in failed] == case['failed']
