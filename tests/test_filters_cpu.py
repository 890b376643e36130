"""`tombo filter` and the resquiggle-time index filters, host logic, against the unmodified
reference (tests/golden/filters.npz, tests/golden/make_filters_golden.py).  The device calls
are stood in for by a numpy restatement here; tests/test_filters_emul_cpu.py and
tests/test_filters_gpu.py run the device source."""
import os

import numpy as np
import pytest

import filters_cases as fc
from tombo_b200 import formats, tombo_helper as th

GOLD = fc.load_golden()


def test_parse_obs_filter():
    assert th.parse_obs_filter([]) is None
    assert th.parse_obs_filter(['90:10', '50:4']) == [[90, 10], [50, 4]]
    assert th.parse_obs_filter(['0:1', '100:3']) == [[0, 1], [100, 3]]
    with pytest.raises(th.TomboError, match='Invalid format for observation filter'):
        th.parse_obs_filter(['90-10'])
    with pytest.raises(th.TomboError, match='Invalid percentile value.'):
        th.parse_obs_filter(['101:10'])
    with pytest.raises(th.TomboError, match='Invalid percentile value.'):
        th.parse_obs_filter(['-1:10'])


def test_mean_q_score():
    q = '!+5?I'
    assert th.get_mean_q_score(q) == np.mean([ord(c) - 33 for c in q])


@pytest.mark.parametrize('case', GOLD['filters'], ids=lambda c: c['name'])
def test_filter_commands_match_reference(case, tmp_path):
    kind, got = fc.run_filter_case(case, fc.HostContext(), str(tmp_path))
    if 'error' in case:
        assert kind == 'error' and got == 'No unfiltered reads present in current Tombo index.'
    else:
        assert kind == 'output'
        assert got == case['output']


@pytest.mark.parametrize('case', GOLD['io'], ids=lambda c: c['name'])
def test_index_batch_matches_io_and_map_read(case):
    r = case['reads']
    codes = fc.host_codes([x['segs'] for x in r], [x['score'] for x in r],
                          [not x['failed'] for x in r], case['sig_match_thresh'], case['obs_filter'])
    index, failed = fc.run_io_case(case, codes)
    assert index.records() == fc.golden_io_index(case).records()
    assert [list(f) for f in failed] == case['failed']


def test_obs_message_queued_for_every_tested_read():
    """the reference queues the observation-filter message for each read that passes the
    signal matching test, filtered or not"""
    case = [c for c in GOLD['io'] if c['obs_filter'] is not None][0]
    kept = [rd for _, _, rd in case['index'] if not rd[2]]
    assert kept
    obs = [f for f in case['failed'] if f[0].startswith('Read filtered by observation')]
    tested = [rd for _, _, rd in case['index'] if not (rd[8] > case['sig_match_thresh'])]
    assert len(obs) == len(tested) > len([rd for rd in tested if rd[2]])


def test_load_index_remove_filtered(tmp_path):
    case = [c for c in GOLD['filters'] if c['name'] == 'stuck'][0]
    d = str(tmp_path / 'f5') + '/'
    os.makedirs(d)
    fn = fc.write_index(d, case['output'])
    full = formats.load_index(fn, d, fc.CORR_GRP)
    kept = formats.load_index(fn, d, fc.CORR_GRP, remove_filtered=True)
    assert sum(map(len, full.values())) == sum(len(r) for _, r in case['output'])
    for (k, recs) in case['output']:
        want = [r for r in recs if not r[6]]
        if want:
            assert [rd.fn for rd in kept[tuple(k)]] == [os.path.join(d, r[0]) for r in want]
        else:
            assert tuple(k) not in kept
    assert not any(rd.filtered for rds in kept.values() for rd in rds)
