"""The numpy / scipy restatement of the de novo and sample-compare per-read tests
(reg_stats_cases) against the unmodified reference's results in tests/golden/reg_stats.npz:
positions and error messages exact, p-values within rtol 1e-7.  No GPU needed."""
import os

import numpy as np
import pytest

import reg_stats_cases as rc
from tombo_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'reg_stats.npz')


@pytest.fixture(scope='module')
def g():
    return dict(np.load(GOLDEN))


def kmer_tables():
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    m, s = syn.kmer_table(kmer_ref)
    return m, s, len(kmer_ref[0][0]), cpos


def test_golden_covers_the_cases(g):
    seen = set()
    for k in range(int(g['n_calls'])):
        st, reg, fm = rc.golden_settings(g, k)[:3]
        seen.add((st, fm))
        if st != 'model_compare':
            seen |= set(('msg', m) for m, _, _ in rc.golden_results(g, k))
    for fm in (0, 1, 2, 10):
        assert ('de_novo', fm) in seen
    assert ('msg', rc.NO_INFO) in seen and ('msg', rc.FISHER_SHORT) in seen
    assert ('msg', rc.NO_VALID_Z) in seen
    assert set(g['reads_strand']) == {0, 1}


def test_restatement_matches_reference(g):
    kmeans, ksds, K, cpos = kmer_tables()
    assert int(g['cpos']) == cpos
    checked = 0
    for k in range(int(g['n_calls'])):
        st, reg, fm = rc.golden_settings(g, k)[:3]
        if st == 'model_compare':
            continue
        start, end = [int(x) for x in g['g%d_region' % reg]]
        for ri, (want_msg, want_pv, want_pos) in zip(g['q%d_reads' % k], rc.golden_results(g, k)):
            r = rc.golden_read(g, int(ri))
            try:
                if st == 'de_novo':
                    pv, pos = rc.de_novo(r['means'], r['bases'], r['start'], r['end'], r['strand'],
                                         kmeans, ksds, K, cpos, fm, start, end)
                else:
                    pv, pos = rc.sample_compare(r['means'], r['start'], r['end'], r['strand'],
                                                g['q%d_ctrl_means' % k], g['q%d_ctrl_sds' % k],
                                                fm, start, end)
                msg = ''
            except rc.CaseError as e:
                msg = str(e)
            assert msg == want_msg, (k, ri, msg, want_msg)
            if msg:
                continue
            np.testing.assert_array_equal(pos, want_pos)
            np.testing.assert_allclose(pv, want_pv, rtol=1e-7, atol=0)
            checked += 1
    assert checked > 300
