"""Statistics files on the device: every golden case bit-identical (block tables, the
most-significant table's columns and row order, chromosome ids and the file layout), and
genome-scale tie-heavy random cases against the numpy restatement whatever the add cadence
or path (resident aggregate, host rows)."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]
import stats_file_cases as sc  # noqa: E402
from tombo_b200 import _lib, formats, tombo_helper as th, tombo_stats as ts  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(HERE, 'golden', 'stats_file.npz'))


def same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.fixture(scope='module')
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize('q', sc.golden_cases(G, 'q'))
@pytest.mark.parametrize('batch', [1, 1 << 24])
def test_model_golden(ctx, q, batch):
    prs, thresh, lower, damp, n_keep, mtr = sc.golden_model_input(G, q)
    root = sc.FakeGroup()
    ts.aggregate_per_read_stats(prs, thresh, lower, root, damp, mtr, n_keep, batch_entries=batch, ctx=ctx)
    assert sc.file_layout(root) == json.loads(str(G[q + '_layout']))
    off = G[q + '_tab_off']
    for b, t in enumerate(sc.file_tables(root)):
        assert same(t, G[q + '_tab'][off[b]:off[b + 1]]), b
    ms = root['Most_Significant_Stats']
    assert same(ms['Most_Significant_Stats'], G[q + '_ms'])
    assert [list(x) for x in ms['chrm_ids'].attrs.items()] == json.loads(str(G[q + '_ids']))


@pytest.mark.parametrize('q', sc.golden_cases(G, 'l'))
def test_level_golden(ctx, q):
    blocks, n_keep = sc.golden_level_input(G, q)
    root = sc.FakeGroup()
    w = formats.LevelStatsWriter(root, 'ks_test', 200, 1, n_keep, ctx=ctx)
    for chrm, strand, start, stat, poss, cov, ctrl in blocks:
        w._write_stat_block(th.groupStats(stat, poss, chrm, strand, start, cov, ctrl))
    w.close()
    assert sc.file_layout(root) == json.loads(str(G[q + '_layout']))
    assert same(root['Most_Significant_Stats']['Most_Significant_Stats'], G[q + '_ms'])


def restated(blocks, thresh, lower, llr, damp, n_keep):
    ids, tabs, rows = {}, [], []
    for chrm, strand, start, t in blocks:
        tab = sc.restate_block(t['pos'], t['stat'], thresh, lower, llr, *damp)
        tabs.append(tab)
        rows.append(sc.with_chrm_strand(tab, ids.setdefault(chrm, len(ids)), strand))
    return tabs, sc.restate_most_signif(np.concatenate(rows), n_keep)


def test_genome_scale_cadences(ctx):
    """2 000 blocks x 10 kb of quantised p-values at N = 100 000: one block per call, all
    blocks in one call and host rows one block at a time give the restatement's table"""
    rng = np.random.default_rng(11)
    blocks = sc.random_blocks(rng, 2000, 10000, 0.5, chrms=('c1', 'c2', 'c3'), quantum=0.125)
    args = (0.25, None, False, (1, 1), 100000)
    tabs, ms = restated(blocks, *args)
    assert np.unique(ms['damp_frac']).shape[0] < 100
    prs = sc.PerReadBlocks('de_novo', 10000, blocks)
    for batch in (1, 1 << 30):
        root = sc.FakeGroup()
        ts.aggregate_per_read_stats(prs, 0.25, None, root, (1, 1), 1, 100000, batch_entries=batch, ctx=ctx)
        assert same(root['Most_Significant_Stats']['Most_Significant_Stats'], ms), batch
        for b in (0, 777, 1999):
            assert same(sc.file_tables(root)[b], tabs[b])
    root = sc.FakeGroup()
    w = formats.ModelStatsWriter(root, 'de_novo', 10000, (1, 1), 1, 100000, ctx=ctx)
    for (chrm, strand, start, _), t in zip(blocks, tabs):
        w._write_stat_block(th.regionStats(t['frac'], t['pos'], chrm, strand, start, t['cov'],
                                           [0] * t.shape[0], t['valid_cov']))
    w.close()
    assert same(root['Most_Significant_Stats']['Most_Significant_Stats'], ms)


def test_region_past_shared_memory(ctx):
    """40 kb blocks: 480 KB of counters per block run from global memory"""
    rng = np.random.default_rng(12)
    blocks = sc.random_blocks(rng, 6, 40000, 1.0, llr=True, quantum=0.5, nan_frac=0.05)
    tabs, ms = restated(blocks, 1.0, -0.5, True, (2, 0), 5000)
    root = sc.FakeGroup()
    ts.aggregate_per_read_stats(sc.PerReadBlocks('model_compare', 40000, blocks), 1.0, -0.5, root, (2, 0), 1,
                                5000, ctx=ctx)
    for t, r in zip(sc.file_tables(root), tabs):
        assert same(t, r)
    assert same(root['Most_Significant_Stats']['Most_Significant_Stats'], ms)


def test_position_outside_block(ctx):
    t = sc.per_read_table(np.array([5, 250]), np.array([0.1, 0.2]))
    prs = sc.PerReadBlocks('de_novo', 200, [('c', '+', 0, t)])
    with pytest.raises(_lib.TomboB200Error, match='outside its block'):
        ts.aggregate_per_read_stats(prs, 0.1, None, sc.FakeGroup(), (2, 0), 1, 10, ctx=ctx)


def test_empty_input(ctx):
    with pytest.raises(th.TomboError, match='No genomic positions contain --minimum-test-reads.'):
        ts.aggregate_per_read_stats(sc.PerReadBlocks('de_novo', 200, []), 0.1, None, sc.FakeGroup(),
                                    (2, 0), 1, 10, ctx=ctx)


def test_reset_and_reuse(ctx):
    rng = np.random.default_rng(13)
    rows = [sc.with_chrm_strand(sc.restate_block(t['pos'], t['stat'], 0.5, None, False, 1, 1), i % 2, s)
            for i, (_, s, _, t) in enumerate(sc.random_blocks(rng, 8, 300, 1.0, quantum=0.25))]

    def add(rs):
        for r in rs:
            ctx.most_signif_add_rows(r['damp_frac'], r['pos'], r['cov'], r['control_cov'], r['chrm'][0],
                                     r['strand'][0], frac=r['frac'], valid_cov=r['valid_cov'])

    def table():
        c = ctx.most_signif_get()
        out = np.zeros(c['key'].shape[0], sc.MODEL_MS_DTYPE)
        out['damp_frac'] = c['key']
        for name in sc.MODEL_MS_DTYPE[1:]:
            out[name[0]] = c[name[0]]
        return out
    ctx.most_signif_begin(False, 50)
    add(rows[:4])
    assert same(table(), sc.restate_most_signif(np.concatenate(rows[:4]), 50))
    ctx.most_signif_reset()
    add(rows[4:])
    assert same(table(), sc.restate_most_signif(np.concatenate(rows[4:]), 50))
    with pytest.raises(_lib.TomboB200Error, match='table is open'):
        ctx.most_signif_begin(False, 10 ** 6)
    ctx.most_signif_end()
    ctx.most_signif_begin(False, 10 ** 6)
    assert ctx.most_signif_count() == 0
    add(rows)
    assert same(table(), sc.restate_most_signif(np.concatenate(rows), 10 ** 6))
    ctx.most_signif_end()


def test_interleaved_writers():
    """two writers open at once (test_significance with two alternative models) keep their
    own tables and chromosome ids"""
    rng = np.random.default_rng(14)
    cases = []
    for k in range(2):
        blocks = sc.random_blocks(rng, 10, 500, 1.0, chrms=('x%d' % k, 'y'), quantum=0.25)
        tabs = [sc.restate_block(t['pos'], t['stat'], 0.5, None, False, 2, 0) for _, _, _, t in blocks]
        cases.append((blocks, tabs))
    roots = [sc.FakeGroup(), sc.FakeGroup()]
    ws = [formats.ModelStatsWriter(r, 'de_novo', 500, (2, 0), 1, 200) for r in roots]
    for b in range(10):
        for w, (blocks, tabs) in zip(ws, cases):
            chrm, strand, start, _ = blocks[b]
            t = tabs[b]
            w._write_stat_block(th.regionStats(t['frac'], t['pos'], chrm, strand, start, t['cov'],
                                               [0] * t.shape[0], t['valid_cov']))
    for w in ws:
        w.close()
    for root, (blocks, tabs) in zip(roots, cases):
        ids, rows = {}, []
        for (chrm, strand, _, _), t in zip(blocks, tabs):
            rows.append(sc.with_chrm_strand(t, ids.setdefault(chrm, len(ids)), strand))
        ms = root['Most_Significant_Stats']
        assert same(ms['Most_Significant_Stats'], sc.restate_most_signif(np.concatenate(rows), 200))
        assert dict(ms['chrm_ids'].attrs) == ids


def test_global_counters_over_several_launches(ctx):
    """4 Mb blocks: 48 MB of counters each, five blocks a launch, so 12 blocks take three"""
    rng = np.random.default_rng(15)
    R = 1 << 22
    blocks = []
    for b in range(12):
        pos = rng.integers(0, R, 3000) + (b // 2) * R
        stat = np.round(rng.uniform(0, 1, 3000) * 8) / 8
        blocks.append(('c', '+-'[b % 2], (b // 2) * R, sc.per_read_table(pos, stat)))
    tabs, ms = restated(blocks, 0.5, None, False, (2, 0), 1000)
    root = sc.FakeGroup()
    ts.aggregate_per_read_stats(sc.PerReadBlocks('de_novo', R, blocks), 0.5, None, root, (2, 0), 1, 1000,
                                ctx=ctx)
    for t, r in zip(sc.file_tables(root), tabs):
        assert same(t, r)
    assert same(root['Most_Significant_Stats']['Most_Significant_Stats'], ms)
