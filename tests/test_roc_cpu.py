"""CPU checks of the accuracy restatement (tests/roc_cases.py) against the reference's
labelled statistics and curves (tests/golden/roc.npz), of the golden's coverage, of the tie
rule, and of parse_motif_descs."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import roc_cases as rc  # noqa: E402
from golden_util import load  # noqa: E402


@pytest.fixture(scope='module')
def g():
    return load('roc')


def golden_case(g, name):
    names = [str(n) for n in g[name + '__names']]
    out = {}
    for j, n in enumerate(names):
        out[n] = dict(stat=g['%s__%d__stat' % (name, j)], label=g['%s__%d__label' % (name, j)])
        if ('%s__%d__tp' % (name, j)) in g.files:
            for k in ('tp', 'fp', 'prec', 'auc_ap'):
                out[n][k] = g['%s__%d__%s' % (name, j, k)]
    return out, str(g[name + '__error'])


@pytest.mark.parametrize('case', rc.CASES, ids=[c['name'] for c in rc.CASES])
def test_restatement_matches_reference(g, case):
    from tombo_b200 import tombo_helper as th
    want, err = golden_case(g, case['name'])
    got, got_err = rc.run_case(case, th)
    assert (got_err or '') == err
    if err:
        return
    assert list(got) == list(want)
    for name, (st, lab) in got.items():
        w = want[name]
        assert np.array_equal(st, w['stat'], equal_nan=True)
        assert np.array_equal(np.signbit(st), np.signbit(w['stat']))
        assert np.array_equal(lab, w['label'])
        if st.shape[0]:
            tp, fp, prec, auc, ap = rc.curve(st, lab)
            assert np.array_equal(tp, w['tp'], equal_nan=True)
            assert np.array_equal(fp, w['fp'], equal_nan=True)
            assert np.array_equal(prec, w['prec'], equal_nan=True)
            assert np.array_equal([auc, ap], w['auc_ap'], equal_nan=True)


def test_golden_covers_the_cases(g):
    """both paths' limits, subsampling, both dtypes, n below and above the plot points, an
    all-True and an all-False name, the shifted '-' window and both IndexError cases"""
    seen = {c['name']: golden_case(g, c['name']) for c in rc.CASES}
    assert seen['motif_err_start'][1] == 'IndexError' and seen['motif_err_end'][1] == 'IndexError'
    sizes = [v['stat'].shape[0] for res, _ in seen.values() for v in res.values()]
    assert min(sizes) < rc.ROC_PLOT_POINTS < max(sizes)
    labels = [v['label'] for res, _ in seen.values() for v in res.values() if v['label'].shape[0]]
    assert any(l.all() for l in labels) and any(not l.any() for l in labels)
    stats = np.concatenate([v['stat'] for res, _ in seen.values() for v in res.values()])
    assert np.isinf(stats).any() and (stats == 0).any()
    assert np.signbit(stats[stats == 0]).any() and (~np.signbit(stats[stats == 0])).any()
    # the limits stop both paths mid-run: fewer blocks pulled than exist
    for name in ('motif_limit', 'ctrl_limit'):
        c = [x for x in rc.CASES if x['name'] == name][0]
        n_blocks = len(rc.build_case(c)[0].blocks)
        assert 0 < int(g[name + '__pulled']) < n_blocks
    # the '-' chromosome-end window is labelled by the base upstream of pos
    c = [x for x in rc.CASES if x['name'] == 'motif_minus_end'][0]
    stats_obj, genome, _ = rc.build_case(c)
    n = dict(rc.CHRMS)['chr2']
    seq = genome.seqs['chr2']
    first = seen['motif_minus_end'][0]['g3']['stat'][:4]
    b = stats_obj.blocks[0][4]
    # window[bb] of pos n - 2 is the complement of base n - 3: appended iff that base is T
    want = [s for p, s in zip(b['pos'], b['stat'])
            if seq[(n - 3) if p == n - 2 else p] == 'T']
    assert np.array_equal(first[:len(want)], want)
    # the ground truth has a missing (chrm, strand), a position in both sets, and locations
    # outside every block
    mod, unmod, _ = rc.build_case([x for x in rc.CASES if x['name'] == 'truth_read'][0])[2]
    assert ('chr1', '-') not in mod and ('chr1', '-') in unmod
    assert any(np.intersect1d(mod[k], unmod[k]).size for k in mod)
    assert any(np.max(v) >= dict(rc.CHRMS)[k[0]] for k, v in mod.items())
    # get_seq / get_reg_stats calls recorded for every path that makes them
    assert g['ctrl_read__get_reg'].shape[0] == g['ctrl_read__get_seq'].shape[0] > 0


def test_tie_rule_is_python_tuple_sort():
    rs = np.random.RandomState(5)
    for _ in range(50):
        n = rs.randint(1, 300)
        st = rs.choice([-np.inf, -1.0, -0.25, -0.0, 0.0, 0.25, 1.0, np.inf], n)
        lab = rs.rand(n) < 0.5
        want = [t[1] for t in sorted(zip(st.tolist(), lab.tolist()))]
        assert rc.ordered_labels(st, lab).tolist() == want


def test_parse_motif_descs():
    from tombo_b200 import tombo_helper as th
    d = th.parse_motif_descs('CG:1:cpg::GATC:2:dam')
    assert [(m.raw_motif, m.mod_pos, m.mod_base, n) for m, n in d] == [
        ('CG', 1, 'C', 'cpg'), ('GATC', 2, 'A', 'dam')]
    assert th.parse_motif_descs('CCWGG:2:dcm')[0][0].motif_pat.pattern == 'CC[AT]GG'
    for bad in ('CG:1', 'CG:x:cpg', 'CG:3:cpg', 'CZ:1:z', 'CG:1:cpg::'):
        with pytest.raises(th.TomboError):
            th.parse_motif_descs(bad)
