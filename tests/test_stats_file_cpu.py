"""Statistics files without a device: the numpy restatements of aggregate_per_read_stats'
block tables and of the most-significant table against the reference's files
(tests/golden/stats_file.npz), and the writers' file layout over an in-memory h5py-like file
with the restatements standing in for the device table."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]
import stats_file_cases as sc  # noqa: E402
from tombo_b200 import formats, tombo_helper as th, tombo_stats as ts  # noqa: E402

G = np.load(os.path.join(HERE, 'golden', 'stats_file.npz'))
MODEL = sc.golden_cases(G, 'q')
LEVEL = sc.golden_cases(G, 'l')


def same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def restated_model(q):
    prs, thresh, lower, damp, n_keep, _ = sc.golden_model_input(G, q)
    ids, tabs, rows = {}, [], []
    for chrm, strand, start, _, t in prs:
        cid = ids.setdefault(chrm, len(ids))
        tab = sc.restate_block(t['pos'], t['stat'], thresh, lower, prs.stat_type == 'model_compare', *damp)
        tabs.append(tab)
        rows.append(sc.with_chrm_strand(tab, cid, strand))
    return tabs, sc.restate_most_signif(np.concatenate(rows), n_keep), ids


@pytest.mark.parametrize('q', MODEL)
def test_model_restatement_matches_reference(q):
    tabs, ms, ids = restated_model(q)
    off = G[q + '_tab_off']
    assert len(tabs) == off.shape[0] - 1
    for b, t in enumerate(tabs):
        assert same(t, G[q + '_tab'][off[b]:off[b + 1]]), b
    assert same(ms, G[q + '_ms'])
    assert sorted(ids.items()) == sorted(tuple(x) for x in json.loads(str(G[q + '_ids'])))


@pytest.mark.parametrize('q', LEVEL)
def test_level_restatement_matches_reference(q):
    blocks, n_keep = sc.golden_level_input(G, q)
    ids, rows = {}, []
    for chrm, strand, start, stat, poss, cov, ctrl in blocks:
        keep = ~np.isnan(stat)
        t = np.zeros(int(keep.sum()), formats.LEVEL_STATS_DTYPE)
        t['stat'], t['pos'], t['cov'], t['control_cov'] = stat[keep], poss[keep], cov[keep], ctrl[keep]
        rows.append(sc.with_chrm_strand(t, ids.setdefault(chrm, len(ids)), strand, level=True))
    assert same(sc.restate_most_signif(np.concatenate(rows), n_keep), G[q + '_ms'])


def test_table_does_not_depend_on_cadence():
    """the reference at most_signif_num_batches 1, 10 and 1000 writes one table; the
    cases are tie-heavy (quantised statistics), so the tie rule decides much of it"""
    qs = [q for q in MODEL if str(G[q + '_tag']).startswith('quant_b')]
    assert len(qs) == 3
    ms = G[qs[0] + '_ms']
    assert np.unique(ms['damp_frac']).shape[0] < ms.shape[0] // 4
    for q in qs[1:]:
        assert same(G[q + '_ms'], ms)


def test_ties_break_on_the_other_fields():
    """numpy's sort(order=key) orders equal keys by the remaining fields, not by arrival"""
    rows = np.zeros(3, sc.MODEL_MS_DTYPE)
    rows['damp_frac'] = 0.5
    rows['pos'] = [9, 3, 5]
    ref = rows.copy()
    ref.sort(kind='mergesort', order='damp_frac')
    assert list(ref['pos']) == [3, 5, 9]
    assert same(sc.restate_most_signif(rows, 3), ref)


@pytest.mark.parametrize('q', MODEL)
def test_aggregate_writer_layout(q):
    prs, thresh, lower, damp, n_keep, mtr = sc.golden_model_input(G, q)
    root = sc.FakeGroup()
    ts.aggregate_per_read_stats(prs, thresh, lower, root, damp, mtr, n_keep,
                                batch_entries=500, ctx=sc.RestatedContext())
    assert sc.file_layout(root) == json.loads(str(G[q + '_layout']))
    off = G[q + '_tab_off']
    for b, t in enumerate(sc.file_tables(root)):
        assert same(t, G[q + '_tab'][off[b]:off[b + 1]])
    ms = root['Most_Significant_Stats']
    assert same(ms['Most_Significant_Stats'], G[q + '_ms'])
    assert [list(x) for x in ms['chrm_ids'].attrs.items()] == json.loads(str(G[q + '_ids']))


@pytest.mark.parametrize('q', LEVEL)
def test_level_writer_layout(q):
    blocks, n_keep = sc.golden_level_input(G, q)
    root = sc.FakeGroup()
    w = formats.LevelStatsWriter(root, 'ks_test', 200, 1, n_keep, ctx=sc.RestatedContext())
    for chrm, strand, start, stat, poss, cov, ctrl in blocks:
        w._write_stat_block(th.groupStats(stat, poss, chrm, strand, start, cov, ctrl))
    w.close()
    assert sc.file_layout(root) == json.loads(str(G[q + '_layout']))
    assert same(root['Most_Significant_Stats']['Most_Significant_Stats'], G[q + '_ms'])


def test_empty_input_raises():
    prs = sc.PerReadBlocks('de_novo', 200, [])
    with pytest.raises(th.TomboError, match='No genomic positions contain --minimum-test-reads.'):
        ts.aggregate_per_read_stats(prs, 0.1, None, sc.FakeGroup(), (2, 0), 1, 10,
                                    ctx=sc.RestatedContext())
