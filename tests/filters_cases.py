"""Shared by tests/golden/make_filters_golden.py and the read-filter tests: synthetic resquiggle
indexes, an in-memory stand-in for h5py.File that serves each read's Events lengths, Fastq
string and signal_match_score attribute, and the host restatement of the resquiggle-time
filter codes."""
import contextlib
import io
import json
import os
import pickle
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'filters.npz')
CORR_GRP = 'RawGenomeCorrected_000'
BC_GRP = 'Basecall_1D_000'
SUBGRP = 'BaseCalled_template'


class _Dset(object):
    def __init__(self, value):
        self.value = value

    def __getitem__(self, k):
        return self.value


class _Grp(object):
    def __init__(self, attrs):
        self.attrs = attrs


class FakeFile(object):
    """h5py.File(fn, 'r') over STORE[fn] = dict(lengths, fastq, score); a missing entry raises
    KeyError as a missing HDF5 path does"""
    STORE = {}

    def __init__(self, fn, mode='r'):
        self.d = self.STORE[fn]

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def close(self):
        pass

    def __getitem__(self, path):
        parts = path.strip('/').split('/')
        if parts[-1] == 'Events':
            if self.d.get('lengths') is None:
                raise KeyError(path)
            ev = np.zeros(len(self.d['lengths']), dtype=[('norm_mean', 'f8'), ('length', 'u4')])
            ev['length'] = self.d['lengths']
            return ev
        if parts[-1] == 'Fastq':
            if self.d.get('fastq') is None:
                raise KeyError(path)
            return _Dset(self.d['fastq'].encode())
        if self.d.get('score') is None:
            return _Grp({})
        return _Grp({'signal_match_score': self.d['score']})


@contextlib.contextmanager
def fake_h5py(store):
    """serve ``store`` to every ``import h5py`` (and to modules holding h5py already)"""
    FakeFile.STORE = store
    mod = types.ModuleType('h5py')
    mod.File = FakeFile
    old = sys.modules.get('h5py')
    sys.modules['h5py'] = mod
    try:
        yield mod
    finally:
        if old is None:
            sys.modules.pop('h5py', None)
        else:
            sys.modules['h5py'] = old


def write_index(fast5s_dir, groups):
    """groups: [[[chrm, strand], [11-field records]]] in order -> the index file's path"""
    base = fast5s_dir.rstrip('/')
    head, tail = os.path.split(base)
    fn = os.path.join(head, '.' + tail + '.' + CORR_GRP + '.tombo.index')
    data = dict((tuple(k), [tuple(r) for r in recs]) for k, recs in groups)
    with io.open(fn, 'wb') as fp:
        pickle.dump(data, fp, protocol=2)
    return fn


def read_index(index_fn):
    """the index file as [[[chrm, strand], [records as lists]]] in stored order"""
    with io.open(index_fn, 'rb') as fp:
        data = pickle.load(fp)
    return [[list(k), [list(r) for r in recs]] for k, recs in data.items()]


def make_case(seed, groups, n_reads, filt_frac=0.2, long_reads=False, missing=0.05):
    """synthetic index groups and FAST5 store: reads with ragged dwell lengths (ties, n = 1
    and 2 included), mean q-scores (some None, read from the Fastq instead), signal matching
    scores (some None, read from the attribute)"""
    rng = np.random.RandomState(seed)
    out, store = [], {}
    k = 0
    for chrm, strand, glen in groups:
        recs = []
        for _ in range(n_reads):
            fn = 'reads/r%05d.fast5' % k
            k += 1
            start = int(rng.randint(0, glen - 50))
            end = int(start + rng.randint(1, min(400, glen - start)))
            nb = int(rng.choice([1, 2, 3, 7, 50, 400] + ([5000] if long_reads else [])))
            lens = rng.choice([1, 2, 3, 4, 6, 10, 30], size=nb,
                              p=[.1, .2, .25, .2, .15, .07, .03]).astype(np.int64)
            q = None if rng.rand() < 0.3 else float(np.round(rng.uniform(5, 15), 2))
            sc = None if rng.rand() < 0.3 else float(np.round(rng.uniform(0.5, 2.0), 3))
            fq = ''.join(chr(33 + int(v)) for v in rng.randint(2, 20, size=20))
            store[fn] = dict(
                lengths=None if rng.rand() < missing else [int(v) for v in lens],
                fastq=None if rng.rand() < missing else '@r\nACGT\n+\n' + fq,
                score=None if rng.rand() < missing else float(np.round(rng.uniform(0.5, 2.0), 3)))
            recs.append([fn, start, end, 0, CORR_GRP, SUBGRP, bool(rng.rand() < filt_frac), False,
                         sc, q, 'id%d' % k])
        out.append([[chrm, strand], recs])
    return out, store


def full_store(store, fast5s_dir):
    return dict((os.path.join(fast5s_dir, fn), v) for fn, v in store.items())


def host_codes(segs_list, scores, ok, sig_thresh, obs_filter):
    """_io_and_map_read's filter decision per read: -1 failed, 1, 2 or 0"""
    codes = []
    for segs, sc, good in zip(segs_list, scores, ok):
        if not good:
            codes.append(-1)
        elif sc > sig_thresh:
            codes.append(1)
        elif obs_filter is not None and any(
                np.percentile(np.diff(segs), p) > t for p, t in obs_filter):
            codes.append(2)
        else:
            codes.append(0)
    return codes


def load_golden():
    z = np.load(GOLDEN)
    return json.loads(str(z['json']))


class HostContext(object):
    """numpy restatement of the read-filter calls (np.percentile; coverage by slice adds)"""

    def dwell_percentiles(self, lens, len_off, pctl):
        return np.array([[np.percentile(lens[a:b], p) for p in pctl]
                         for a, b in zip(len_off[:-1], len_off[1:])]).reshape(-1, len(pctl))

    def read_mid_coverage(self, grp_off, start, end):
        out = np.zeros(len(start), dtype=np.int64)
        for a, b in zip(grp_off[:-1], grp_off[1:]):
            if b == a:
                continue
            cov = np.zeros(int(np.max(end[a:b])), dtype=np.int64)
            for i in range(a, b):
                cov[start[i]:end[i]] += 1
            for i in range(a, b):
                out[i] = cov[start[i] + (end[i] - start[i]) // 2]
        return out


def run_filter_case(case, ctx, tmp):
    """one golden filter case through tombo_b200.filters: the written index, or 'error' with
    the TomboError message"""
    from tombo_b200 import filters, tombo_helper as th
    d = os.path.join(tmp, case['name']) + '/'
    os.makedirs(d)
    index_fn = write_index(d, case['input'])
    cmd, args = case['cmd'], case['args']
    with fake_h5py(full_store(case['store'], d)):
        try:
            if cmd == 'clear':
                filters.clear_filters(d, CORR_GRP)
            elif cmd == 'stuck':
                filters.filter_reads_for_stuck(d, CORR_GRP, args[0], ctx=ctx)
            elif cmd == 'coverage':
                np.random.seed(case['seed'])
                filters.filter_reads_for_coverage(d, CORR_GRP, args[0], ctx=ctx)
            elif cmd == 'qscore':
                filters.filter_reads_for_qscore(d, BC_GRP, CORR_GRP, args[0])
            elif cmd == 'sigmatch':
                filters.filter_reads_for_signal_matching(d, CORR_GRP, args[0])
            elif cmd == 'genome':
                regs = dict((c, None if r is None else [tuple(x) for x in r])
                            for c, r in args[0].items())
                filters.filter_reads_for_genome_pos(d, CORR_GRP, regs, args[1])
        except th.TomboError as e:
            return 'error', str(e)
    return 'output', read_index(index_fn)


def run_io_case(case, codes):
    """the golden _io_and_map_read reads through worker.ReadBatcher with the index opt-in,
    ``codes`` standing in for the device's filter codes: (index records, failed messages)"""
    from tombo_b200 import formats, worker, tombo_helper as th
    reads = case['reads']
    results = []
    for i, r in enumerate(reads):
        if r['failed']:
            results.append(th.TomboError('Alignment not produced'))
        else:
            results.append(th.resquiggleResults(
                align_info=th.alignInfo('rid%d' % i, SUBGRP, 0, 0, 0, 0, 0, 0),
                genome_loc=th.genomeLocation(r['start'], r['strand'], r['chrm']),
                genome_seq='ACGT', mean_q_score=r['q'], raw_signal=np.zeros(10, np.int16),
                read_start_rel_to_raw=r['rsrtr'], segs=np.array(r['segs'], dtype=np.int64),
                sig_match_score=r['score']))

    def fn(map_results, *a, **k):
        return [(results[m.read_start_rel_to_raw], int(codes[m.read_start_rel_to_raw]))
                for m in map_results]
    index = formats.ReadsIndex('/data', CORR_GRP)
    b = worker.ReadBatcher(None, None, max_reads=7, resquiggle_fn=fn, index=index,
                           corr_grp=CORR_GRP, bc_subgrp=SUBGRP, obs_filter=case['obs_filter'])
    for i in range(len(reads)):
        # read_start_rel_to_raw carries the read's position to the stand-in resquiggle
        b.add(th.resquiggleResults(None, None, 'ACGT', None, np.zeros(10, np.int16),
                                   read_start_rel_to_raw=i), '/data/r%03d.fast5' % i)
    b.flush()
    return index, b.failed_reads


def golden_io_index(case):
    """the golden index queue as a formats.ReadsIndex"""
    from tombo_b200 import formats, tombo_helper as th
    index = formats.ReadsIndex('/data', CORR_GRP)
    for chrm, strand, rd in case['index']:
        index.add_read_data(chrm, strand, th.readData(*rd))
    return index
