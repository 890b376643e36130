#!/usr/bin/env python
"""Writes tests/golden/filters.npz: `tombo filter` commands and the resquiggle-time index
filters run by the UNMODIFIED reference in-process.

* Each filter_reads_for_* / clear_filters of tombo/_filter_reads.py runs on a synthetic index
  written to a temporary directory (tests/filters_cases.py).  h5py.File is the in-memory
  FakeFile there, serving Events lengths, Fastq strings and signal_match_score attributes.
  _filter_reads.py:138 uses np.float, which numpy 2 removed: np.float = float while the
  reference runs.  np.random.seed(case seed) precedes level_coverage.  The reference orders
  (chromosome, strand) groups as a set of the loaded keys; each input index is written in
  that order, so the file order is the order the reference iterates.
* resquiggle._io_and_map_read runs with map_read, map_conn and write_new_fast5_group stubbed;
  the index queue and the failed-reads queue are recorded for chosen segs, scores,
  thresholds and obs_filter.

_filter_reads is imported from the reference checkout (TOMBO_REFERENCE_ROOT) into the
package oracle/_ref provides.  One JSON document under key 'json':
  filters: [{name, cmd, args, seed, input, store, output | error}]
  io: [{name, sig_match_thresh, obs_filter, reads: [{segs, score, failed}], index, failed}]

    python oracle/build_ref.py && python tests/golden/make_filters_golden.py
"""
import importlib.util
import json
import os
import queue
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
for p in (REPO, os.path.join(REPO, 'oracle'), os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)
import ref_harness as rh                      # noqa: E402
import filters_cases as fc                    # noqa: E402

REF_ROOT = os.environ.get('TOMBO_REFERENCE_ROOT', '/root/reference')


def load_filter_module():
    m = rh.load_reference()
    spec = importlib.util.spec_from_file_location(
        'tombo._filter_reads', os.path.join(REF_ROOT, 'tombo', '_filter_reads.py'))
    fr = importlib.util.module_from_spec(spec)
    sys.modules['tombo._filter_reads'] = fr
    spec.loader.exec_module(fr)
    return m, fr


def set_order(groups):
    """the group order a TomboReads built from these keys iterates in"""
    for _ in range(10):
        keys = [tuple(k) for k, _ in groups]
        order = list(set(keys))
        if order == keys:
            return groups
        by = dict((tuple(k), r) for k, r in groups)
        groups = [[list(k), by[k]] for k in order]
    raise RuntimeError('no stable group order')


FILTER_CASES = [
    # name, cmd, args, case seed, groups, reads per group, kwargs of make_case
    ('clear', 'clear', [], 1, [('chr1', '+', 2000), ('chr1', '-', 2000)], 30, {}),
    ('stuck', 'stuck', [[[50, 4], [90, 9]]], 2, [('chr1', '+', 3000), ('chr2', '-', 1500), ('chr2', '+', 900)], 60, dict(long_reads=True)),
    ('stuck_ends', 'stuck', [[[0, 2], [100, 25]]], 3, [('chr1', '+', 3000)], 80, {}),
    ('stuck_gamma', 'stuck', [[[33, 3], [67, 5], [25, 2], [75, 6]]], 4, [('c', '+', 3000), ('c', '-', 3000)], 60, {}),
    ('coverage', 'coverage', [0.3], 5, [('chr1', '+', 2500), ('chr1', '-', 2500), ('chr3', '+', 700)], 80, {}),
    ('coverage_one', 'coverage', [0.5], 6, [('chr1', '+', 600)], 40, dict(filt_frac=0.5)),
    ('qscore', 'qscore', [10.0], 7, [('chr1', '+', 2000), ('chr2', '+', 2000)], 60, {}),
    ('sigmatch', 'sigmatch', [1.2], 8, [('chr1', '+', 2000), ('chr2', '-', 2000)], 60, {}),
    ('genome', 'genome', [{'chr1': [[100, 900], [1200, 1900]], 'chr2': None}, False], 9,
     [('chr1', '+', 2000), ('chr2', '-', 2000), ('chr3', '+', 2000)], 50, {}),
    ('genome_partial', 'genome', [{'chr1': [[100, 900], [1200, 1900]]}, True], 10,
     [('chr1', '+', 2000), ('chr1', '-', 2000)], 50, {}),
    ('none_unfiltered', 'stuck', [[[50, 4]]], 11, [('chr1', '+', 2000)], 20, dict(filt_frac=1.0)),
    ('none_unfiltered_cov', 'coverage', [0.2], 12, [('chr1', '+', 2000)], 20, dict(filt_frac=1.0)),
]


def run_filter(fr, cmd, d, args, seed):
    if cmd == 'clear':
        fr.clear_filters(d, fc.CORR_GRP)
    elif cmd == 'stuck':
        fr.filter_reads_for_stuck(d, fc.CORR_GRP, args[0])
    elif cmd == 'coverage':
        np.random.seed(seed)
        fr.filter_reads_for_coverage(d, fc.CORR_GRP, args[0])
    elif cmd == 'qscore':
        fr.filter_reads_for_qscore(d, fc.BC_GRP, fc.CORR_GRP, args[0])
    elif cmd == 'sigmatch':
        fr.filter_reads_for_signal_matching(d, fc.CORR_GRP, args[0])
    elif cmd == 'genome':
        regs = dict((c, None if r is None else [tuple(x) for x in r]) for c, r in args[0].items())
        fr.filter_reads_for_genome_pos(d, fc.CORR_GRP, regs, args[1])


def filter_goldens(m, fr):
    out = []
    np.float = float
    for name, cmd, args, seed, groups, n, kw in FILTER_CASES:
        groups_in, store = fc.make_case(seed, groups, n, **kw)
        groups_in = set_order(groups_in)
        with tempfile.TemporaryDirectory() as tmp:
            d = os.path.join(tmp, 'fast5s') + '/'
            os.makedirs(d)
            index_fn = fc.write_index(d, groups_in)
            rec = dict(name=name, cmd=cmd, args=args, seed=seed, input=groups_in, store=store)
            with fc.fake_h5py(fc.full_store(store, d)) as mod:
                fr.h5py = mod
                m['th'].h5py = mod
                try:
                    with rh.ref_errstate():
                        run_filter(fr, cmd, d, args, seed)
                    rec['output'] = fc.read_index(index_fn)
                except SystemExit:
                    rec['error'] = 'exit'
        out.append(rec)
    del np.float
    return out


IO_CASES = [
    ('sig_only', 1.1, None, 21),
    ('obs', 1.1, [[50, 4], [90, 9]], 22),
    ('obs_loose_sig', 1.6, [[0, 2], [100, 12], [37, 4]], 23),
]


def io_reads(seed):
    rng = np.random.RandomState(seed)
    reads = []
    for i in range(40):
        nb = int(rng.choice([1, 2, 5, 30, 300]))
        segs = np.concatenate([[0], np.cumsum(rng.choice([1, 2, 3, 4, 8, 15], size=nb))]).astype(np.int64)
        reads.append(dict(segs=[int(v) for v in segs], score=float(np.round(rng.uniform(0.4, 2.0), 3)),
                          failed=bool(rng.rand() < 0.1), start=int(rng.randint(0, 10000)),
                          chrm='chr%d' % rng.randint(1, 3), strand='+-'[rng.randint(2)],
                          q=float(np.round(rng.uniform(5, 15), 3)), rsrtr=int(rng.randint(0, 500))))
    return reads


def io_goldens(m):
    th, rsq = m['th'], m['rsq']
    out = []
    for name, thresh, obs, seed in IO_CASES:
        reads = io_reads(seed)
        index_q, failed_q = queue.Queue(), queue.Queue()
        saved = (rsq.map_read, th.get_channel_info, th.get_raw_read_slot, th.write_new_fast5_group)
        for i, r in enumerate(reads):
            fn = '/data/r%03d.fast5' % i

            class Conn(object):
                def send(self, msg):
                    pass

                def recv(self, r=r, fn=fn):
                    if r['failed']:
                        return True, ['Alignment not produced', fn, True]
                    return False, th.resquiggleResults(
                        align_info=th.alignInfo('rid%d' % i, 'BaseCalled_template', 0, 0, 0, 0, 0, 0),
                        genome_loc=th.genomeLocation(r['start'], r['strand'], r['chrm']),
                        genome_seq='ACGT', mean_q_score=r['q'], raw_signal=None,
                        read_start_rel_to_raw=r['rsrtr'], segs=np.array(r['segs'], dtype=np.int64),
                        sig_match_score=r['score'])
            rsq.map_read = lambda *a, **k: th.resquiggleResults(
                align_info=None, genome_loc=None, genome_seq='ACGT', mean_q_score=None)
            th.get_channel_info = lambda f: None
            th.get_raw_read_slot = lambda f: {'Signal': np.zeros(10, dtype=np.int16)}
            th.write_new_fast5_group = lambda *a, **k: None
            try:
                with rh.ref_errstate():
                    rsq._io_and_map_read(
                        None, failed_q, ['BaseCalled_template'], fc.BC_GRP, fc.CORR_GRP, None,
                        th.seqSampleType('DNA', False), None, fn, None, Conn(), None, False, obs,
                        index_q, 0, thresh, None, None, None)
            finally:
                rsq.map_read, th.get_channel_info, th.get_raw_read_slot, th.write_new_fast5_group = saved
        index = []
        while not index_q.empty():
            chrm, strand, rd = index_q.get()
            index.append([chrm, strand, [v.item() if hasattr(v, 'item') else v for v in rd]])
        failed = []
        while not failed_q.empty():
            failed.append(list(failed_q.get()))
        out.append(dict(name=name, sig_match_thresh=thresh, obs_filter=obs, reads=reads,
                        index=index, failed=failed))
    return out


def main():
    m, fr = load_filter_module()
    doc = dict(filters=filter_goldens(m, fr), io=io_goldens(m))
    np.savez_compressed(fc.GOLDEN, json=np.array(json.dumps(doc)))
    print('wrote', fc.GOLDEN, len(doc['filters']), 'filter cases', len(doc['io']), 'io cases')


if __name__ == '__main__':
    main()
