#!/usr/bin/env python
"""Generate tests/golden/rsqgl_inputs.npz from the UNMODIFIED reference (oracle/_ref):
resquiggle with caller-supplied map_res.scale_values and map_res.stall_ints.

    python oracle/build_ref.py && python tests/golden/make_inputs_golden.py

Sections:
  * nm_*  normalize_raw_signal(raw, outlier_thresh=t, scale_values=sv) on seeded signals:
          odd / even n, continuous / integer-valued, finite / None limits, t = 5, 0.5, None.
  * c_* / o_*  resquiggle cases.  c_call 0: one resquiggle_read call on the data as given
          (DNA sample type); c_call 1: the worker policy (iterate, rescue, RNA flip and
          stall detection), run as batches grouped by c_group in c_read_index order.
Every input is stored (scale values, stall lists) or regenerated from its seed with
tombo_b200.synthetic; a checksum of each raw signal detects generator drift.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'oracle'))
sys.path.insert(0, os.path.dirname(HERE))

import ref_harness as rh  # noqa: E402
from read_inputs_cases import (NORM_THRESHOLDS, norm_scale_values, norm_signal,  # noqa: E402
                               stall_lists)
from tombo_b200 import synthetic as syn  # noqa: E402

ALN_ADAPT = (4.2, 4.2, 200, 1500, 20.0, 40, 300, 2500, 100)
ALN_NARROW = (4.2, 4.2, 100, 1500, 20.0, 40, 300, 2500, 100)
RNA_ALN = (6, 4, 500, 1500, 20.0, 50, 1000, 3000, 250)
NAN5 = (np.nan,) * 5


def _nan(v):
    return np.nan if v is None else float(v)


def _none(v):
    return None if np.isnan(v) else float(v)


def norm_cases():
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    rows = []
    for n, seed in ((601, 31), (600, 32)):
        for integer in (0, 1):
            raw = norm_signal(n, seed, integer)
            for name, sv in norm_scale_values(raw):
                for t in NORM_THRESHOLDS + (None,):
                    if t is None and name != 'shifted_none':
                        continue
                    with rh.ref_errstate():
                        norm, out = ts.normalize_raw_signal(raw, outlier_thresh=t,
                                                            scale_values=th.scaleValues(*sv))
                    rows.append((n, seed, integer, sv, t, norm, tuple(out)))
    return dict(
        nm_n=np.array([r[0] for r in rows], dtype=np.int64),
        nm_seed=np.array([r[1] for r in rows], dtype=np.int64),
        nm_int=np.array([r[2] for r in rows], dtype=np.int64),
        nm_sv=np.array([[_nan(v) for v in r[3]] for r in rows]),
        nm_t=np.array([_nan(r[4]) for r in rows]),
        nm_norm=np.concatenate([r[5] for r in rows]),
        nm_off=np.concatenate([[0], np.cumsum([r[0] for r in rows])]).astype(np.int64),
        nm_out=np.array([[_nan(v) for v in r[6]] for r in rows]),
        nm_out_none=np.array([[v is None for v in r[6]] for r in rows]))


class Cases(object):
    def __init__(self):
        self.c, self.o = [], []

    def add(self, call, kind, rna_params, aln, nbases, seed, plant=(-1, -1), skip=False,
            const_scale=None, sv=None, stalls=None, group=-1, read_index=0):
        self.c.append(dict(call=call, kind=kind, rna_params=rna_params, aln=aln, nbases=nbases,
                           seed=seed, plant=plant, skip=skip, const_scale=const_scale, sv=sv,
                           stalls=stalls, group=group, read_index=read_index))


def read_of(c):
    kmer_ref, cpos = syn.make_kmer_ref(c['kind'], 0)
    plant = c.get('plant', (-1, -1))
    kw = {} if plant[0] < 0 else dict(stall=tuple(plant))
    return syn.make_read(kmer_ref, cpos, c['nbases'], c['seed'], kind=c['kind'], **kw)


def run_case(c):
    m = rh.load_reference()
    th, ts, rsq = m['th'], m['ts'], m['rsq']
    kmer_ref, cpos = syn.make_kmer_ref(c['kind'], 0)
    std_ref, _ = rh.make_models(kmer_ref, cpos)
    sst, p, sp = rh.make_params('RNA' if c['rna_params'] else 'DNA', c['aln'])
    r = read_of(c)
    sv = None if c['sv'] is None else th.scaleValues(*c['sv'])
    if c['call'] == 1:
        wsst = th.seqSampleType(c['kind'], c['kind'] == 'RNA')
        res, err, info = rh.run_read(r.raw, r.genome_seq, std_ref, wsst, p, sp,
                                     read_index=c['read_index'], scale_values=sv,
                                     stall_ints=c['stalls'])
    else:
        from tombo_b200.synthetic import subsample_key
        mr = rh.make_map_res(r.raw, r.genome_seq)._replace(scale_values=sv,
                                                          stall_ints=c['stalls'])
        info = dict(calls=1, rescued=False, n_iters=1)
        res = err = None
        with rh.ref_errstate(), rh.keyed_choice(subsample_key(0, 0, 0)):
            try:
                res = rsq.resquiggle_read(
                    mr, std_ref, p, 5.0, const_scale=c['const_scale'],
                    skip_seq_scaling=c['skip'], seq_samp_type=th.seqSampleType('DNA', False))
            except th.TomboError as e:
                err = str(e)
            except Exception as e:   # noqa
                err = 'UNEXPECTED: ' + repr(e)
    return r, res, err, info


def ref_cpts(c, raw):
    """the sorted changepoints of the first call without inputs (for the lists whose
    endpoints sit on changepoints)"""
    m = rh.load_reference()
    ts, ch = m['ts'], m['ch']
    sst, p, sp = rh.make_params('RNA' if c['rna_params'] else 'DNA', c['aln'])
    k = 6 if c['kind'] == 'DNA' else 5
    num_events = ts.compute_num_events(raw.shape[0], c['nbases'] - k + 1, p.mean_obs_per_event,
                                       1.1)
    with rh.ref_errstate():
        if p.use_t_test_seg:
            cp = ch.c_valid_cpts_w_cap_t_test(raw, p.min_obs_per_base, p.running_stat_width,
                                              num_events)
        else:
            norm, _ = ts.normalize_raw_signal(raw, outlier_thresh=5.0)
            cp = ch.c_valid_cpts_w_cap(norm, p.min_obs_per_base, p.running_stat_width,
                                       num_events)
    return np.sort(cp)


def build_cases():
    m = rh.load_reference()
    ts = m['ts']
    cs = Cases()
    # single DNA calls with supplied scale values
    base = dict(kind='DNA', rna_params=False, aln=ALN_ADAPT, nbases=500, seed=25000)
    raw = np.asarray(read_of(base).raw, dtype=np.float64)
    with rh.ref_errstate():
        _, own = ts.normalize_raw_signal(raw, outlier_thresh=5.0)
    svs = [tuple(own),
           (own.shift + 3.7, own.scale * 1.13, own.lower_lim, own.upper_lim, 5.0),
           (own.shift, own.scale, None, None, None)]
    for sv in svs:
        for skip in (False, True):
            for const_scale in (None, 61.5):
                cs.add(0, sv=sv, skip=skip, const_scale=const_scale, **base)
    # single DNA calls with stall lists
    base = dict(kind='DNA', rna_params=False, aln=ALN_ADAPT, nbases=500, seed=25100,
                plant=(120, 1500))
    raw = np.asarray(read_of(base).raw, dtype=np.float64)
    lists = stall_lists(raw.shape[0], ref_cpts(base, raw))
    with rh.ref_errstate():
        lists['planted'] = [tuple(int(v) for v in iv) for iv in ts.identify_stalls(raw, m['rsq'].DEFAULT_STALL_PARAMS)]
    assert len(lists['planted']) >= 1
    lists['most_of_read'] = [(5, raw.shape[0] - 5)]
    for name, si in lists.items():
        cs.add(0, stalls=si, **base)
    # single calls with RNA parameters (t-test segmentation, no flip)
    base = dict(kind='RNA', rna_params=True, aln=RNA_ALN, nbases=270, seed=25200)
    raw = np.asarray(read_of(base).raw, dtype=np.float64)
    lists = stall_lists(raw.shape[0], ref_cpts(base, raw))
    for name in ('sorted', 'unsorted', 'overlapping', 'endpoints'):
        cs.add(0, stalls=lists[name], **base)
    for name, sv in norm_scale_values(raw):
        for skip in (False, True):
            cs.add(0, sv=sv, skip=skip, **base)
    # worker policy: DNA with scale values on a narrow band (some reads are rescued)
    rs = np.random.RandomState(253)
    for i in range(24):
        c = dict(kind='DNA', rna_params=False, aln=ALN_NARROW, nbases=int(rs.randint(300, 900)),
                 seed=25300 + i)
        raw = np.asarray(read_of(c).raw, dtype=np.float64)
        sv = norm_scale_values(raw)[i % 2][1]
        cs.add(1, sv=sv, group=0, read_index=i, **c)
    # worker policy: DNA with stall lists
    for i in range(12):
        c = dict(kind='DNA', rna_params=False, aln=ALN_NARROW, nbases=int(rs.randint(300, 900)),
                 seed=25400 + i)
        n = read_of(c).raw.shape[0]
        si = [[(int(n * .3), int(n * .35)), (int(n * .6), int(n * .62))],
              [(int(n * .6), int(n * .62)), (int(n * .1), int(n * .35))], []][i % 3]
        cs.add(1, stalls=si, group=1, read_index=i, **c)
    # worker policy: RNA with caller stalls (replaced by the worker's own) and scale values
    for i in range(6):
        c = dict(kind='RNA', rna_params=True, aln=None, nbases=270, seed=25500 + i)
        raw = np.asarray(read_of(c).raw, dtype=np.float64)
        n = raw.shape[0]
        sv = norm_scale_values(raw)[0][1] if i % 2 else None
        cs.add(1, stalls=[(int(n * .1), int(n * .2))], sv=sv, group=2, read_index=i, **c)
    return cs


def pack(cs):
    c = cs.c
    flat, off = [], [0]
    segs, seg_off, scal, none, msgs, chk = [], [0], [], [], [], []
    for case in c:
        si = case['stalls'] or []
        flat.extend([(int(a), int(b)) for a, b in si])
        off.append(len(flat))
        r, res, err, info = run_case(case)
        chk.append(float(np.sum(np.asarray(r.raw, dtype=np.float64))))
        if res is None:
            msgs.append(err)
            scal.append([np.nan] * 8 + [info['calls'], int(info['rescued']), -1])
            none.append([False] * 5)
            seg_off.append(seg_off[-1])
            continue
        msgs.append('')
        segs.append(res.segs.astype(np.int64))
        seg_off.append(seg_off[-1] + res.segs.shape[0])
        sv = tuple(res.scale_values)
        scal.append([_nan(v) for v in sv] + [res.sig_match_score, res.read_start_rel_to_raw,
                                             int(res.norm_params_changed), info['calls'],
                                             int(info['rescued']), info['n_iters']])
        none.append([v is None for v in sv])
    aln = [x['aln'] if x['aln'] is not None else (np.nan,) * 9 for x in c]
    return dict(
        c_call=np.array([x['call'] for x in c], dtype=np.int64),
        c_kind=np.array([x['kind'] for x in c]),
        c_rna_params=np.array([x['rna_params'] for x in c], dtype=np.int64),
        c_aln=np.array(aln, dtype=np.float64),
        c_nbases=np.array([x['nbases'] for x in c], dtype=np.int64),
        c_seed=np.array([x['seed'] for x in c], dtype=np.int64),
        c_plant=np.array([x['plant'] for x in c], dtype=np.int64),
        c_skip=np.array([x['skip'] for x in c], dtype=np.int64),
        c_const_scale=np.array([_nan(x['const_scale']) for x in c]),
        c_has_sv=np.array([x['sv'] is not None for x in c]),
        c_sv=np.array([[_nan(v) for v in (x['sv'] or NAN5)] for x in c]),
        c_has_stalls=np.array([x['stalls'] is not None for x in c]),
        c_stalls=np.array(flat, dtype=np.int64).reshape(-1, 2),
        c_stall_off=np.array(off, dtype=np.int64),
        c_group=np.array([x['group'] for x in c], dtype=np.int64),
        c_read_index=np.array([x['read_index'] for x in c], dtype=np.int64),
        raw_checksum=np.array(chk),
        o_segs=np.concatenate(segs) if segs else np.zeros(0, np.int64),
        o_seg_off=np.array(seg_off, dtype=np.int64),
        o_scalars=np.array(scal, dtype=np.float64),
        o_none=np.array(none, dtype=bool),
        o_messages=np.array(msgs))


if __name__ == '__main__':
    out = norm_cases()
    out.update(pack(build_cases()))
    np.savez_compressed(os.path.join(HERE, 'rsqgl_inputs.npz'), **out)
    msgs = out['o_messages']
    print('rsqgl_inputs: %d normalisation cases, %d resquiggle cases, %d failures, %d rescued'
          % (len(out['nm_n']), len(msgs), int((msgs != '').sum()),
             int(np.nansum(out['o_scalars'][:, 9]))))
    for i, mm in enumerate(msgs):
        if mm:
            print('  case %d: %s' % (i, mm))
