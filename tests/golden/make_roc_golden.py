#!/usr/bin/env python
"""Writes tests/golden/roc.npz: the labelled statistics and the accuracy curves of the
UNMODIFIED reference (oracle/_ref) for the cases of tests/roc_cases.py.

Each case is rebuilt from its recorded seeds (roc_cases.build_case) and run through the
reference's _compute_motif_stats, _compute_ground_truth_stats or _compute_ctrl_motif_stats
(motif descriptions through its parse_motif_descs).  Then every non-empty modification name
goes through prep_accuracy_rates' steps (_plot_commands.py:60-82): sorted() of the tuples,
compute_accuracy_rates, compute_auc and compute_mean_avg_precison.  The reference runs under
numpy's default error state, so 0 / 0 gives NaN with a warning, as it does for a user.

Keys: <case>__names (mod names in dict order), <case>__error (exception type or ''),
<case>__pulled (blocks taken from the iterator), <case>__get_seq (chrm index, start, end of
each get_seq call), <case>__get_reg (the same for get_reg_stats), and per name j
<case>__<j>__stat / __label (the tuple list), __tp / __fp / __prec, __auc_ap.

    python oracle/build_ref.py && python tests/golden/make_roc_golden.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
for p in (REPO, os.path.join(REPO, 'oracle'), os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)
import ref_harness as rh                      # noqa: E402
import roc_cases as rc                        # noqa: E402

CHRM_IDX = {c: i for i, (c, _) in enumerate(rc.CHRMS)}


def calls_array(calls, width):
    """(chrm, start, end) or (chrm, strand, start, end) calls -> int64 rows, strand 0 '+'"""
    rows = [[CHRM_IDX[c[0]]] + [(0 if x == '+' else 1) if isinstance(x, str) else int(x)
                                for x in c[1:]] for c in calls]
    return np.array(rows, dtype=np.int64).reshape(len(calls), width)


def run(c, th, ts):
    stats, genome, extra = rc.build_case(c)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        try:
            if c['path'] == 'truth':
                res = ts._compute_ground_truth_stats(stats, extra)
            else:
                descs = th.parse_motif_descs(c['descs'])
                if c['path'] == 'ctrl':
                    res = ts._compute_ctrl_motif_stats(
                        stats, extra, descs, genome, None, c.get('total_stats_limit'))
                else:
                    if c.get('rng_seed') is not None:
                        np.random.seed(c['rng_seed'])
                    res = ts._compute_motif_stats(
                        stats, descs, genome, c.get('stats_per_block'), c.get('total_stats_limit'))
            err = ''
        except Exception as e:                # noqa: the exception type is the record
            res, err = None, type(e).__name__
    out = {'__error': np.array(err), '__pulled': np.array(stats.pulled),
           '__get_seq': calls_array(genome.calls, 3),
           '__get_reg': calls_array(extra.calls if c['path'] == 'ctrl' else [], 4)}
    names = list(res) if res is not None else []
    out['__names'] = np.array(names, dtype='U16')
    for j, name in enumerate(names):
        tuples = res[name]
        out['__%d__stat' % j] = np.array([t[0] for t in tuples], dtype=np.float64)
        out['__%d__label' % j] = np.array([bool(t[1]) for t in tuples], dtype=bool)
        if tuples:
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                ordered = list(zip(*sorted(tuples)))[1]
                tp, fp, prec = ts.compute_accuracy_rates(ordered)
                out['__%d__tp' % j], out['__%d__fp' % j], out['__%d__prec' % j] = tp, fp, prec
                out['__%d__auc_ap' % j] = np.array([ts.compute_auc(tp, fp),
                                                    ts.compute_mean_avg_precison(tp, prec)])
    return out


def main():
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    arrays = {}
    for c in rc.CASES:
        for k, v in run(c, th, ts).items():
            arrays[c['name'] + k] = v
        print(c['name'], str(arrays[c['name'] + '__error']) or 'ok',
              [(str(n), arrays['%s__%d__stat' % (c['name'], j)].shape[0])
               for j, n in enumerate(arrays[c['name'] + '__names'])])
    np.savez_compressed(os.path.join(HERE, 'roc.npz'), **arrays)


if __name__ == '__main__':
    main()
