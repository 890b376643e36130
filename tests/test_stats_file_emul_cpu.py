"""The statistics-file kernels' device source on the host (tests/emul): aggregation with
shared-memory and chunked global counters, the row packing, the radix sort's digit skipping
and the table's sort cadence, through aggregate_per_read_stats and the writers, against the
reference's files and the numpy restatement."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(HERE, 'emul')]
import emul_stats_file as ef  # noqa: E402
import stats_file_cases as sc  # noqa: E402
from tombo_b200 import formats, tombo_helper as th, tombo_stats as ts  # noqa: E402

G = np.load(os.path.join(HERE, 'golden', 'stats_file.npz'))


def same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize('q,smem,batch', [('q3', True, 1 << 24), ('q7', False, 1 << 24)])
def test_model_golden_emulated(q, smem, batch):
    """one block per call or all at once, shared or global counters (3 blocks a launch)"""
    prs, thresh, lower, damp, n_keep, mtr = sc.golden_model_input(G, q)
    root = sc.FakeGroup()
    ts.aggregate_per_read_stats(prs, thresh, lower, root, damp, mtr, n_keep, batch_entries=batch,
                                ctx=ef.EmulContext(smem=smem, per=3))
    assert sc.file_layout(root) == json.loads(str(G[q + '_layout']))
    off = G[q + '_tab_off']
    for b, t in enumerate(sc.file_tables(root)):
        assert same(t, G[q + '_tab'][off[b]:off[b + 1]]), b
    assert same(root['Most_Significant_Stats']['Most_Significant_Stats'], G[q + '_ms'])


@pytest.mark.parametrize('n_keep,seed', [(7, 0), (60, 1)])
def test_random_cadences_emulated(n_keep, seed):
    """host rows one block at a time: with N small the table sorts every few blocks"""
    rng = np.random.default_rng(seed)
    blocks = sc.random_blocks(rng, 8, 48, 1.5, quantum=0.25, nan_frac=0.1)
    ctx = ef.EmulContext()
    ctx.most_signif_begin(False, n_keep)
    rows = []
    for b, (chrm, strand, start, t) in enumerate(blocks):
        tab = sc.restate_block(t['pos'], t['stat'], 0.5, None, False, 1, 1)
        r = sc.with_chrm_strand(tab, b % 3, strand)
        rows.append(r)
        ctx.most_signif_add_rows(r['damp_frac'], r['pos'], r['cov'], r['control_cov'], b % 3, strand.encode(),
                                 frac=r['frac'], valid_cov=r['valid_cov'])
    c = ctx.most_signif_get()
    ref = sc.restate_most_signif(np.concatenate(rows), n_keep)
    assert same(c['key'], ref['damp_frac'])
    for name in ('frac', 'pos', 'cov', 'valid_cov', 'chrm', 'strand'):
        assert np.array_equal(c[name], ref[name]), name
