#!/usr/bin/env python
"""Generate tests/golden/rsqgl_params.npz from the UNMODIFIED reference (oracle/_ref): the
worker policy of resquiggle at the parameter points of tests/params_cases.py (alignment and
segmentation parameters, outlier threshold, scaling iterations, sequence rescaling, fixed
scale, max_raw_cpts, min_event_to_seq_ratio, per-k-mer model sds, int16 raw).

    python oracle/build_ref.py && python tests/golden/make_params_golden.py

Per read it records what make_golden.py records: segs, read_start_rel_to_raw, the scale
values, score, call count, rescued flag, or the error message.  Reads are regenerated from
the stored seeds with tombo_b200.synthetic; a checksum of each raw signal detects drift.
The lp_* arrays hold load_resquiggle_parameters of float CLI-style tuples, field by field.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'oracle'))
sys.path.insert(0, os.path.dirname(HERE))

import params_cases as pc  # noqa: E402
import ref_harness as rh  # noqa: E402
from tombo_b200 import synthetic as syn  # noqa: E402

SEED0 = 30000


def _nan(v):
    return np.nan if v is None else float(v)


def run_point(pt, seed0):
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    kmer_ref, cpos = syn.make_kmer_ref(pt['kind'], 0, sd_range=pt['sd_range'])
    std_ref, _ = rh.make_models(kmer_ref, cpos)
    sst = th.seqSampleType(pt['kind'], pt['kind'] == 'RNA')
    p = ts.load_resquiggle_parameters(sst, pt['aln'], pt['seg'])
    sp = ts.load_resquiggle_parameters(sst, pt['aln'], pt['seg'], use_save_bandwidth=True)
    pol = pt['pol']
    rows = []
    for i, nb in enumerate(pt['nbases']):
        kw = dict(kind=pt['kind'], int16=pt['int16'])
        stall = pt['stall'].get(i)
        if stall is not None:
            kw['stall'] = stall
        r = syn.make_read(kmer_ref, cpos, nb, seed0 + i, **kw)
        res, err, info = rh.run_read(
            r.raw, r.genome_seq, std_ref, sst, p, sp, outlier_thresh=pol['outlier_thresh'],
            max_scaling_iters=pol['max_scaling_iters'], read_index=i, stable_ties=pt['stable'],
            const_scale=pol['const_scale'], skip_seq_scaling=pol['skip_seq_scaling'],
            max_raw_cpts=pol['max_raw_cpts'],
            min_event_to_seq_ratio=pol['min_event_to_seq_ratio'])
        rows.append((nb, seed0 + i, stall or (-1, -1),
                     float(np.sum(np.asarray(r.raw, dtype=np.float64))), res, err, info))
    return rows


def load_param_cases():
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    vals, is_int, is_none = [], [], []
    for kind, aln, seg in pc.LOAD_PARAM_CASES:
        for save in (False, True):
            sst = th.seqSampleType(kind, kind == 'RNA')
            p = ts.load_resquiggle_parameters(sst, aln, seg, use_save_bandwidth=save)
            vals.append([_nan(v) for v in p])
            is_int.append([isinstance(v, (int, np.integer)) and not isinstance(v, bool)
                           for v in p])
            is_none.append([v is None for v in p])
    aln = [(np.nan,) * 9 if a is None else tuple(_nan(v) for v in a)
           for _, a, _ in pc.LOAD_PARAM_CASES]
    seg = [(-1,) * 4 if s is None else s for _, _, s in pc.LOAD_PARAM_CASES]
    return dict(lp_kind=np.array([k for k, _, _ in pc.LOAD_PARAM_CASES]),
                lp_aln=np.array(aln, dtype=np.float64), lp_seg=np.array(seg, dtype=np.int64),
                lp_fields=np.array(m['th'].resquiggleParams._fields),
                lp_values=np.array(vals, dtype=np.float64), lp_is_int=np.array(is_int),
                lp_is_none=np.array(is_none))


def build():
    P = pc.points()
    read_off, nbs, seeds, stalls, chk, scal, msgs, segs, seg_off = [0], [], [], [], [], [], [], [], [0]
    for j, pt in enumerate(P):
        for nb, seed, stall, c, res, err, info in run_point(pt, SEED0 + 100 * j):
            nbs.append(nb); seeds.append(seed); stalls.append(stall); chk.append(c)
            if res is None:
                msgs.append(err)
                scal.append([np.nan] * 6 + [info['calls'], int(info['rescued']), -1, 0])
                seg_off.append(seg_off[-1])
                continue
            msgs.append('')
            segs.append(res.segs.astype(np.int64))
            seg_off.append(seg_off[-1] + res.segs.shape[0])
            sv = res.scale_values
            scal.append([sv.shift, sv.scale, sv.lower_lim, sv.upper_lim, res.sig_match_score,
                         res.read_start_rel_to_raw, info['calls'], int(info['rescued']),
                         info['n_iters'], int(res.norm_params_changed)])
        read_off.append(len(nbs))
    out = dict(
        p_name=np.array([pt['name'] for pt in P]), p_kind=np.array([pt['kind'] for pt in P]),
        p_aln=np.array([[_nan(v) for v in pt['aln']] for pt in P]),
        p_seg=np.array([pt['seg'] for pt in P], dtype=np.int64),
        p_outlier=np.array([_nan(pt['pol']['outlier_thresh']) for pt in P]),
        p_iters=np.array([pt['pol']['max_scaling_iters'] for pt in P], dtype=np.int64),
        p_skip=np.array([pt['pol']['skip_seq_scaling'] for pt in P], dtype=np.int64),
        p_const_scale=np.array([_nan(pt['pol']['const_scale']) for pt in P]),
        p_max_raw_cpts=np.array([pt['pol']['max_raw_cpts'] for pt in P], dtype=np.int64),
        p_ev_ratio=np.array([pt['pol']['min_event_to_seq_ratio'] for pt in P]),
        p_sd_range=np.array([pt['sd_range'] or (np.nan, np.nan) for pt in P], dtype=np.float64),
        p_int16=np.array([pt['int16'] for pt in P], dtype=np.int64),
        p_stable=np.array([pt['stable'] for pt in P], dtype=np.int64),
        p_read_off=np.array(read_off, dtype=np.int64),
        r_nbases=np.array(nbs, dtype=np.int64), r_seed=np.array(seeds, dtype=np.int64),
        r_stall=np.array(stalls, dtype=np.int64), raw_checksum=np.array(chk),
        # int32 keeps the file small; every boundary fits (reads are < 2^31 samples)
        segs=(np.concatenate(segs) if segs else np.zeros(0)).astype(np.int32),
        seg_off=np.array(seg_off, dtype=np.int64), scalars=np.array(scal, dtype=np.float64),
        messages=np.array(msgs))
    out.update(load_param_cases())
    return out


if __name__ == '__main__':
    o = build()
    path = os.path.join(HERE, 'rsqgl_params.npz')
    np.savez_compressed(path, **o)
    print('rsqgl_params: %d points, %d reads, %d bytes' % (len(o['p_name']), len(o['r_seed']),
                                                           os.path.getsize(path)))
    for j, name in enumerate(o['p_name']):
        a, b = o['p_read_off'][j], o['p_read_off'][j + 1]
        m = o['messages'][a:b]
        print('  %-28s reads %d ok %d rescued %d %s' % (
            name, b - a, int((m == '').sum()), int(np.nansum(o['scalars'][a:b, 7])),
            sorted(set(x for x in m if x))))
