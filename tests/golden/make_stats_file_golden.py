#!/usr/bin/env python
"""Writes tests/golden/stats_file.npz: statistics files written by the UNMODIFIED reference
(oracle/_ref) in-process.

Model cases run _agg_stats_worker then _write_stats (ModelStats) exactly as
aggregate_per_read_stats wires them, with queue.Queue for the multiprocessing queues and one
aggregation process (with more, the arrival order depends on process scheduling).  Level
cases write groupStats blocks through LevelStats._write_stat_block and close().  The writers
pre-fill the running table with ``[:] = np.NAN``, which numpy 2 refuses for the integer
fields; while they run, np.NAN is a tuple of NaN floats and zero integers, which fills the
fields as numpy 1 did (those rows sort last and are trimmed).  h5py.File is
replaced by the in-memory FakeGroup of tests/stats_file_cases.py (ts.h5py.File = ...), and
ModelStats / LevelStats get the case's most_signif_num_batches.

Key scheme, case q<k> (model) or l<k> (level):
  _par     thresh, lower (NaN: None), llr (0/1), unmod, mod, num_most_signif, region_size,
           most_signif_num_batches, min_test_reads
  _chrms   chromosome names; _blk (chrm index, strand 0 '+' / 1 '-', start) per block in
           arrival order; _off block offsets into the inputs
  model inputs: _pos, _stat (per-read entries);  level inputs: _lstat, _lpos, _lcov, _lctrl
  _tab, _tab_off  every Block_<n>/block_stats, concatenated
  _ms      Most_Significant_Stats/Most_Significant_Stats
  _ids     chrm_ids attributes as (name, id) in stored order, JSON
  _layout  group paths, their attributes and dataset paths in creation order, JSON

    python oracle/build_ref.py && python tests/golden/make_stats_file_golden.py
"""
import contextlib
import json
import os
import queue
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
for p in (REPO, os.path.join(REPO, 'oracle'), os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)
import ref_harness as rh                      # noqa: E402
import stats_file_cases as sc                 # noqa: E402

REGION = 200


def model_cases():
    """(tag, stat_type, thresh, lower, damp counts, N, batches, blocks kwargs, seed)"""
    return [
        ('llr', 'model_compare', 1.5, None, (2, 0), 40, 10, dict(llr=True, quantum=0.5), 1),
        ('llr_lower', 'model_compare', 1.0, -1.0, (2, 0), 500, 10, dict(llr=True, quantum=0.25), 2),
        ('denovo', 'de_novo', 0.05, None, (2, 0), 100000, 10, dict(), 3),
        ('quant_b1', 'de_novo', 0.25, None, (1, 1), 120, 1, dict(quantum=0.25), 4),
        ('quant_b10', 'de_novo', 0.25, None, (1, 1), 120, 10, dict(quantum=0.25), 4),
        ('quant_b1000', 'de_novo', 0.25, None, (1, 1), 120, 1000, dict(quantum=0.25), 4),
        ('nan_pval', 'de_novo', 0.3, None, (2, 0), 300, 10, dict(quantum=0.1, nan_frac=0.2), 5),
        ('nan_llr', 'model_compare', 1.0, None, (0, 0), 300, 10, dict(llr=True, nan_frac=0.2), 6),
        ('nan_lower', 'sample_compare', 0.3, 0.1, (2, 1), 300, 3, dict(nan_frac=0.2, quantum=0.1), 7),
        ('n1', 'de_novo', 0.25, None, (2, 0), 1, 10, dict(quantum=0.25), 8),
    ]


def model_blocks(seed, kw):
    """two chromosomes x both strands; the first (chrm, strand) out of start order, the rest
    sorted, as PerReadStats.__iter__ yields them"""
    rng = np.random.default_rng(seed)
    blocks = sc.random_blocks(rng, 16, REGION, 2.0, **kw)
    groups = {}
    for b in blocks:
        groups.setdefault((b[0], b[1]), []).append(b)
    order = list(groups)
    rng.shuffle(order)
    out = []
    for g, key in enumerate(order):
        bl = sorted(groups[key], key=lambda b: b[2])
        if g == 0:
            bl = [bl[i] for i in rng.permutation(len(bl))]
        out.extend(bl)
    return out


def level_blocks(seed):
    """groupStats blocks: quantised negative and positive stats with -0.0 and NaN"""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(12):
        chrm, strand = (('chrA', '+'), ('chrB', '-'), ('chrA', '-'))[b % 3]
        start = (b // 3) * REGION
        n = int(rng.integers(20, REGION))
        poss = np.sort(rng.choice(REGION, n, replace=False)) + start
        stat = np.round(rng.normal(0, 1, n) * 2) / 4
        stat[rng.random(n) < 0.2] = -0.0
        stat[rng.random(n) < 0.1] = np.nan
        cov = rng.integers(1, 4, n)
        ctrl = rng.integers(0, 3, n)
        out.append((chrm, strand, start, stat, poss, cov, ctrl))
    return out


@contextlib.contextmanager
def nan_fill(row):
    old = np.NAN
    np.NAN = row
    try:
        yield
    finally:
        np.NAN = old


def jsonable(v):
    if isinstance(v, bytes):
        return v.decode()
    if isinstance(v, np.generic):
        return v.item()
    return v


def dump_layout(root):
    out = []
    for path, kind, val in sc.layout(root):
        if kind == 'group':
            out.append([path, kind, [[k, jsonable(a)] for k, a in val.items()]])
        else:
            out.append([path, kind, str(val.dtype)])
    return json.dumps(out)


def store_file(store, tag, root):
    blocks = root['Statistic_Blocks']
    tabs = [blocks['Block_%d' % i]['block_stats'] for i in range(len(blocks.children))]
    store[tag + '_tab'] = np.concatenate(tabs) if tabs else np.zeros(0)
    store[tag + '_tab_off'] = np.concatenate([[0], np.cumsum([t.shape[0] for t in tabs])]).astype(np.int64)
    ms = root['Most_Significant_Stats']
    store[tag + '_ms'] = ms['Most_Significant_Stats']
    store[tag + '_ids'] = np.array(json.dumps([[k, jsonable(v)] for k, v in ms['chrm_ids'].attrs.items()]))
    store[tag + '_layout'] = np.array(dump_layout(root))


def main():
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    files = {}

    def h5_file(fn, mode='r'):
        files[fn] = sc.FakeGroup()
        return files[fn]
    ts.h5py.File = h5_file
    orig_model, orig_level = ts.ModelStats, ts.LevelStats
    store = {}
    for k, (tag, stype, thresh, lower, damp, N, nb, kw, seed) in enumerate(model_cases()):
        blocks = model_blocks(seed, kw)
        chrms = sorted(set(b[0] for b in blocks))

        class MS(orig_model):
            def __init__(self, *a, **kw):
                kw['most_signif_num_batches'] = nb
                orig_model.__init__(self, *a, **kw)
        ts.ModelStats = MS
        pr_q, stats_q = queue.Queue(), queue.Queue()
        for chrm, strand, start, table in blocks:
            pr_q.put((chrm, strand, start, start + REGION, table.copy()))
        pr_q.put(None)
        fn = 'q%d.tombo.stats' % k
        with rh.ref_errstate(), np.errstate(invalid='ignore', divide='ignore'):
            ts._agg_stats_worker(pr_q, stats_q, stype, thresh, lower)
            with nan_fill((np.nan, np.nan, 0, 0, 0, 0, 0, b'')):
                ts._write_stats(stats_q, fn, stype, REGION, damp, 1, N, len(blocks), 1)
        ts.ModelStats = orig_model
        q = 'q%d' % k
        store[q + '_tag'] = np.array(tag)
        store[q + '_stype'] = np.array(stype)
        store[q + '_par'] = np.array([thresh, np.nan if lower is None else lower, stype == 'model_compare',
                                      damp[0], damp[1], N, REGION, nb, 1], dtype=np.float64)
        store[q + '_chrms'] = np.array(chrms)
        store[q + '_blk'] = np.array([(chrms.index(c), s == '-', st) for c, s, st, _ in blocks], dtype=np.int64)
        store[q + '_off'] = np.concatenate([[0], np.cumsum([b[3].shape[0] for b in blocks])]).astype(np.int64)
        store[q + '_pos'] = np.concatenate([b[3]['pos'] for b in blocks])
        store[q + '_stat'] = np.concatenate([b[3]['stat'] for b in blocks])
        store_file(store, q, files[fn])
    for k, (N, nb) in enumerate([(30, 10), (1, 1), (1000, 1000), (30, 1)]):
        blocks = level_blocks(100 + (k % 2))
        chrms = sorted(set(b[0] for b in blocks))
        fn = 'l%d.tombo.stats' % k
        with rh.ref_errstate(), np.errstate(invalid='ignore'), nan_fill((np.nan, 0, 0, 0, 0, b'')):
            ls = orig_level(fn, stat_type='ks_test', region_size=REGION, cov_thresh=1, num_most_signif=N,
                            most_signif_num_batches=nb)
            for chrm, strand, start, stat, poss, cov, ctrl in blocks:
                ls._write_stat_block(th.groupStats(stat, poss, chrm, strand, start, cov, ctrl))
            ls.close()
        q = 'l%d' % k
        store[q + '_par'] = np.array([np.nan, np.nan, 0, np.nan, np.nan, N, REGION, nb, 1])
        store[q + '_chrms'] = np.array(chrms)
        store[q + '_blk'] = np.array([(chrms.index(b[0]), b[1] == '-', b[2]) for b in blocks], dtype=np.int64)
        store[q + '_off'] = np.concatenate([[0], np.cumsum([b[3].shape[0] for b in blocks])]).astype(np.int64)
        for j, name in ((3, '_lstat'), (4, '_lpos'), (5, '_lcov'), (6, '_lctrl')):
            store[q + name] = np.concatenate([b[j] for b in blocks])
        store_file(store, q, files[fn])
    np.savez_compressed(os.path.join(HERE, 'stats_file.npz'), **store)
    print('stats_file.npz:', len(store), 'arrays')


if __name__ == '__main__':
    main()
