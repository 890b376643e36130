"""Shared by tests/golden/make_tracks_golden.py and the browser-track tests: synthetic
resquiggle indexes whose reads carry Events tables (norm_mean, norm_stdev, length), served by
the FakeFile stand-in of filters_cases, the golden cases of `tombo text_output browser_files`,
and a numpy restatement of the device calls (the reference's slice-add loop)."""
import contextlib
import hashlib
import json
import os

import numpy as np

import filters_cases as fc

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'tracks.npz')
CORR_GRP = fc.CORR_GRP
SUBGRP = fc.SUBGRP
SUBGRP2 = 'BaseCalled_complement'
WIG_BASE = 'tracks'                  # relative: the track headers carry it


class EventsFile(fc.FakeFile):
    """FakeFile whose STORE entries may hold a whole Events table: dict(events=dict(norm_mean,
    norm_stdev, length) or None); None (or a missing entry) raises KeyError as a missing HDF5
    path does"""

    def __getitem__(self, path):
        if path.strip('/').split('/')[-1] != 'Events' or 'events' not in self.d:
            return fc.FakeFile.__getitem__(self, path)
        e = self.d['events']
        if e is None:
            raise KeyError(path)
        ev = np.zeros(len(e['length']), dtype=[('norm_mean', 'f8'), ('norm_stdev', 'f8'), ('length', 'u4')])
        for k in ('norm_mean', 'norm_stdev', 'length'):
            ev[k] = e[k]
        return ev


@contextlib.contextmanager
def events_h5py(store):
    with fc.fake_h5py(store) as mod:
        mod.File = EventsFile
        yield mod


def _read_events(rng, n, kind):
    if kind == 'zeros':
        mean = rng.choice([0.0, -0.0, 1e-5, -1e-5, 2.5], size=n)
    elif kind == 'deep':
        mean = rng.choice([-1, 1], size=n) * 10.0 ** rng.uniform(-12, 6, size=n)
    else:
        mean = rng.normal(0, 1.3, size=n)
    sd = np.full(n, np.nan) if kind == 'sd_nan' else rng.gamma(2.0, 0.15, size=n)
    length = rng.choice([1, 2, 3, 4, 5, 8, 13, 40], size=n)
    return dict(norm_mean=[float(x) for x in mean], norm_stdev=[float(x) for x in sd],
                length=[int(x) for x in length])


def make_dir(rng, groups, prefix, kind='normal', filt_frac=0.1, missing=0.05, short_frac=0.2,
             subgrps=(SUBGRP,)):
    """index groups [[chrm, strand], 11-field records] and the FAST5 store of one directory;
    groups: (chrm, strand, genome length, reads); a read's Events may be shorter than its span"""
    out, store = [], {}
    k = 0
    for chrm, strand, glen, n_reads in groups:
        recs = []
        for _ in range(n_reads):
            fn = '%s/r%05d.fast5' % (prefix, k)
            k += 1
            start = int(rng.randint(0, glen - 5))
            end = int(start + rng.randint(1, min(120, glen - start) + 1))
            n = end - start
            if rng.rand() < short_frac:
                n = int(rng.randint(0, n + 1))
            store[fn] = dict(events=None if rng.rand() < missing else _read_events(rng, n, kind))
            recs.append([fn, start, end, 0, CORR_GRP, str(rng.choice(list(subgrps))),
                         bool(rng.rand() < filt_frac), False, None, None, 'id%s%d' % (prefix, k)])
        out.append([[chrm, strand], recs])
    return out, store


def make_deep_dir(rng, n_reads=2400, pos=57):
    """every read covers position ``pos`` (values across 18 decades, both signs)"""
    recs, store = [], {}
    for k in range(n_reads):
        fn = 'deep/r%05d.fast5' % k
        start = int(rng.randint(max(0, pos - 6), pos + 1))
        end = int(max(pos + 1, start + rng.randint(1, 9)))
        strand = '+'
        store[fn] = dict(events=_read_events(rng, end - start, 'deep'))
        recs.append([fn, start, end, 0, CORR_GRP, SUBGRP, False, False, None, None, 'idd%d' % k])
    return [[['chrD', strand], recs]], store


def index_dirs(tmp, dirs):
    """write each directory's index under ``tmp``: ([dir paths], FakeFile store by full path)"""
    paths, store = [], {}
    for name, groups, dstore in dirs:
        d = os.path.join(tmp, name) + '/'
        os.makedirs(d, exist_ok=True)
        fc.write_index(d, groups)
        paths.append(d)
        store.update(fc.full_store(dstore, d))
    return paths, store


def output_files(tmp):
    """{file name: text} of every browser file written in ``tmp``"""
    out = {}
    for fn in sorted(os.listdir(tmp)):
        if fn.startswith(WIG_BASE + '.'):
            with open(os.path.join(tmp, fn), 'rb') as fp:
                out[fn] = fp.read().decode()
    return out


def bedgraph_groups(text):
    """(header, {chrm: lines}) of one bedgraph: the reference writes its groups in set order"""
    lines = text.split('\n')
    groups = {}
    for ln in lines[1:]:
        if ln:
            groups.setdefault(ln.split('\t')[0], []).append(ln)
    return lines[0], groups


def same_files(got, want):
    """wiggles byte for byte, bedgraphs group by group"""
    assert sorted(got) == sorted(want)
    for fn in want:
        if fn.endswith('.bedgraph'):
            assert bedgraph_groups(got[fn]) == bedgraph_groups(want[fn]), fn
        else:
            assert got[fn] == want[fn], fn


def case_inputs():
    """the golden cases' inputs as JSON-ready dicts: name, sample / control ([dir, groups,
    store] each), bc_subgrps, wig_types"""
    return [dict(name=name, sample=[list(d) for d in sample],
                 control=[list(d) for d in control] if control else None,
                 bc_subgrps=bc_subgrps, wig_types=wig_types)
            for name, sample, control, bc_subgrps, wig_types in golden_cases()]


def inputs_digest(case):
    """sha256 of one case's inputs, so a golden is only compared with the inputs it was made from"""
    doc = [case['sample'], case['control'], case['bc_subgrps'], case['wig_types']]
    return hashlib.sha256(json.dumps(doc, sort_keys=True).encode()).hexdigest()


def load_golden():
    """{'cases': [inputs + files]}: the golden holds the reference's files and a digest of each
    case's inputs; the inputs themselves are regenerated from their fixed seeds"""
    z = np.load(GOLDEN)
    gold = dict((c['name'], c) for c in json.loads(str(z['json']))['cases'])
    cases = case_inputs()
    assert sorted(gold) == sorted(c['name'] for c in cases)
    for c in cases:
        g = gold[c['name']]
        assert inputs_digest(c) == g['digest'], 'inputs of %s differ from the golden\'s' % c['name']
        c['files'] = g['files']
    return dict(cases=cases)


def run_case(case, tmp, ctx):
    """one golden case through tombo_b200.text_output: {file name: text}"""
    from tombo_b200 import text_output
    sample, s_store = index_dirs(tmp, case['sample'])
    ctrl, c_store = index_dirs(tmp, case['control']) if case['control'] else (None, {})
    s_store.update(c_store)
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        with events_h5py(s_store):
            text_output.write_all_browser_files(sample, ctrl, CORR_GRP, case['bc_subgrps'], None, WIG_BASE,
                                                case['wig_types'], ctx=ctx)
    finally:
        os.chdir(cwd)
    return output_files(tmp)


class HostContext(object):
    """numpy restatement of tb2_coverage_runs and tb2_slot_sums_*: the reference's coverage
    loop and np.diff encoding, and its slice-add loop (base_sums[s:s + n] += values)"""

    def coverage_runs(self, grp_off, start, end):
        run_off, rs, rc = [0], [], []
        for a, b in zip(grp_off[:-1], grp_off[1:]):
            if b > a:
                cov = np.zeros(int(np.max(end[a:b])), dtype=np.int64)
                for i in range(a, b):
                    cov[start[i]:end[i]] += 1
                starts = np.concatenate([[0], np.where(np.diff(cov))[0] + 1])
                rs.append(starts)
                rc.append(cov[starts])
                run_off.append(run_off[-1] + starts.shape[0])
            else:
                run_off.append(run_off[-1])
        cat = (lambda x: np.concatenate(x).astype(np.int64) if x else np.zeros(0, np.int64))
        return np.array(run_off, dtype=np.int64), cat(rs), cat(rc)

    def slot_means(self, chrm_len, batches):
        base_sums = np.zeros(chrm_len)
        base_cov = np.zeros(chrm_len, dtype=np.int64)
        for start, val_off, vals, reverse in batches:
            for r in range(len(start)):
                v = np.asarray(vals[val_off[r]:val_off[r + 1]], dtype=np.float64)
                if reverse[r]:
                    v = v[::-1]
                s = int(start[r])
                if s < 0 or s + v.shape[0] > chrm_len:
                    raise ValueError('read values past the chromosome end')
                base_sums[s:s + v.shape[0]] += v
                base_cov[s:s + v.shape[0]] += 1
        with np.errstate(invalid='ignore', divide='ignore'):
            return base_sums / base_cov


def golden_cases():
    """(name, sample dirs, control dirs or None, bc_subgrps, wig_types) with seeds fixed"""
    all_types = ['coverage', 'signal', 'signal_sd', 'dwell']
    rng = np.random.RandomState(101)
    cases = []
    g3 = [('chr1', '+', 1500, 30), ('chr1', '-', 1500, 25), ('chr2', '+', 450, 15)]
    s, st = make_dir(rng, g3, 'a')
    cases.append(('single_all', [('s1', s, st)], None, None, all_types))
    # sample + control: (chr2, -) only in the sample, (chr3, +) only in the control, chr4 one strand
    s, st = make_dir(rng, [('chr1', '+', 1000, 20), ('chr1', '-', 1000, 20), ('chr2', '-', 400, 10),
                           ('chr4', '+', 600, 12)], 'b')
    c, ct = make_dir(rng, [('chr1', '+', 1150, 20), ('chr1', '-', 750, 15), ('chr3', '+', 350, 10),
                           ('chr4', '+', 500, 7)], 'c')
    cases.append(('sample_control', [('s1', s, st)], [('c1', c, ct)], None,
                  ['coverage', 'signal', 'difference', 'signal_sd', 'dwell']))
    s, st = make_dir(rng, [('chr1', '+', 750, 20), ('chr2', '-', 750, 20)], 'd')
    c, ct = make_dir(rng, [('chr1', '+', 750, 20), ('chr2', '-', 750, 20)], 'e')
    cases.append(('difference_only', [('s1', s, st)], [('c1', c, ct)], None, ['difference']))
    s, st = make_dir(rng, [('chr1', '+', 750, 20), ('chr1', '-', 750, 20)], 'f', kind='sd_nan')
    cases.append(('sd_all_nan', [('s1', s, st)], None, None, ['signal', 'signal_sd']))
    s, st = make_dir(rng, [('chr1', '+', 300, 15)], 'g', filt_frac=0.0, missing=0.0, short_frac=0.0)
    nan_read = st[s[0][1][3][0]]['events']
    nan_read['norm_mean'][len(nan_read['norm_mean']) // 2] = float('nan')
    cases.append(('nan_mean', [('s1', s, st)], None, None, ['signal', 'dwell']))
    s, st = make_dir(rng, [('chr1', '+', 200, 20), ('chr1', '-', 200, 20)], 'h', kind='zeros')
    c, ct = make_dir(rng, [('chr1', '+', 200, 20), ('chr1', '-', 200, 20)], 'i', kind='zeros')
    cases.append(('signed_zeros', [('s1', s, st)], [('c1', c, ct)], None, ['signal', 'difference']))
    s, st = make_dir(rng, [('chr1', '-', 1250, 40), ('chr2', '-', 500, 15)], 'j')
    cases.append(('minus_strand', [('s1', s, st)], None, None, all_types))
    s, st = make_dir(rng, [('chr1', '+', 750, 25), ('chr2', '+', 400, 10)], 'k', missing=0.3)
    cases.append(('unreadable_events', [('s1', s, st)], None, None, all_types))
    s, st = make_dir(rng, [('chr1', '+', 750, 25), ('chr1', '-', 450, 3)], 'l', filt_frac=0.5)
    for rec in s[1][1]:
        rec[6] = True                # (chr1, -) left without unfiltered reads
    cases.append(('filtered_reads', [('s1', s, st)], None, None, all_types))
    s1, st1 = make_dir(rng, [('chr1', '+', 750, 15), ('chr2', '-', 450, 10)], 'm')
    s2, st2 = make_dir(rng, [('chr1', '+', 850, 15), ('chr3', '+', 300, 10)], 'n')
    cases.append(('two_dirs', [('s1', s1, st1), ('s2', s2, st2)], None, None, all_types))
    s, st = make_dir(rng, [('chr1', '+', 750, 30), ('chr1', '-', 750, 30)], 'o', subgrps=(SUBGRP, SUBGRP2))
    cases.append(('bc_subgrps', [('s1', s, st)], None, [SUBGRP], all_types))
    s, st = make_deep_dir(rng)
    cases.append(('deep_order', [('s1', s, st)], None, None, ['coverage', 'signal']))
    return cases
