"""GPU tests of the accuracy of modified-base calls (csrc/accuracy.cu): the drop-ins against
the reference's golden (tests/golden/roc.npz), the fused accuracy_curves against the drop-ins
and the numpy restatement at 10^7 statistics, the radix sort against np.lexsort on
adversarial keys, errors, and the other modules' device results."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import roc_cases as rc  # noqa: E402
from golden_util import load  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def g():
    return load('roc')


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _run_dropin(c):
    from tombo_b200 import tombo_helper as th, tombo_stats as ts
    stats, genome, extra = rc.build_case(c)
    if c['path'] == 'truth':
        res = ts._compute_ground_truth_stats(stats, extra)
    else:
        descs = th.parse_motif_descs(c['descs'])
        if c['path'] == 'ctrl':
            res = ts._compute_ctrl_motif_stats(stats, extra, descs, genome, None,
                                               c.get('total_stats_limit'))
        else:
            if c.get('rng_seed') is not None:
                np.random.seed(c['rng_seed'])
            res = ts._compute_motif_stats(stats, descs, genome, c.get('stats_per_block'),
                                          c.get('total_stats_limit'))
    return res, stats, genome, extra


@pytest.mark.parametrize('case', rc.CASES, ids=[c['name'] for c in rc.CASES])
def test_dropins_match_reference(g, case):
    from tombo_b200 import tombo_stats as ts
    name = case['name']
    err = str(g[name + '__error'])
    if err:
        with pytest.raises(IndexError):
            _run_dropin(case)
        return
    res, stats, genome, extra = _run_dropin(case)
    # the same get_seq / get_reg_stats calls and blocks pulled as the reference
    assert stats.pulled == int(g[name + '__pulled'])
    assert [(rc.CHRMS[r[0]][0], r[1], r[2]) for r in g[name + '__get_seq'].tolist()] == genome.calls
    if case['path'] == 'ctrl':
        assert [(rc.CHRMS[r[0]][0], '+-'[r[1]], r[2], r[3])
                for r in g[name + '__get_reg'].tolist()] == extra.calls
    names = [str(n) for n in g[name + '__names']]
    assert list(res) == names
    for j, n in enumerate(names):
        st = np.array([t[0] for t in res[n]], dtype=np.float64)
        lab = [t[1] for t in res[n]]
        assert all(isinstance(x, (bool, np.bool_)) for x in lab)
        assert _same(st, g['%s__%d__stat' % (name, j)])
        assert np.array_equal(np.signbit(st), np.signbit(g['%s__%d__stat' % (name, j)]))
        assert np.array_equal(np.array(lab, dtype=bool), g['%s__%d__label' % (name, j)])
    nonempty = {n: res[n] for n in names if res[n]}
    tp, fp, prec, mods = ts.prep_accuracy_rates(nonempty)
    k = 0
    for j, n in enumerate(names):
        if not res[n]:
            continue
        sl = slice(k * rc.ROC_PLOT_POINTS, (k + 1) * rc.ROC_PLOT_POINTS)
        k += 1
        for got, key in ((tp, 'tp'), (fp, 'fp'), (prec, 'prec')):
            assert _same(got[sl], g['%s__%d__%s' % (name, j, key)]), (n, key)
        assert mods[sl] == [n] * rc.ROC_PLOT_POINTS
        t, f, p = (g['%s__%d__%s' % (name, j, key)] for key in ('tp', 'fp', 'prec'))
        assert _same([ts.compute_auc(t, f), ts.compute_mean_avg_precison(t, p)],
                     g['%s__%d__auc_ap' % (name, j)])
        # compute_accuracy_rates on the ordered labels
        ordered = [x[1] for x in sorted(res[n])]
        for got, want in zip(ts.compute_accuracy_rates(ordered), (t, f, p)):
            assert _same(got, want)
    # the fused path: the same curves, None for a name without statistics
    stats, genome, extra = rc.build_case(case)
    kw = {}
    if case['path'] == 'truth':
        kw['ground_truth_locs'] = extra
    else:
        from tombo_b200 import tombo_helper as th
        kw.update(motif_descs=th.parse_motif_descs(case['descs']), genome_index=genome)
        if case['path'] == 'ctrl':
            kw['ctrl_stats'] = extra
    if case.get('rng_seed') is not None:
        np.random.seed(case['rng_seed'])
    fused = ts.accuracy_curves(stats, stats_per_block=case.get('stats_per_block'),
                               total_stats_limit=case.get('total_stats_limit'), **kw)
    assert list(fused) == names
    for j, n in enumerate(names):
        if not res[n]:
            assert fused[n] is None
            continue
        for got, key in zip(fused[n][:3], ('tp', 'fp', 'prec')):
            assert _same(got, g['%s__%d__%s' % (name, j, key)])
        assert _same(fused[n][3:], g['%s__%d__auc_ap' % (name, j)])


# ---- fused path at scale ----------------------------------------------------------------
def _big(seed, chrm_len=400000, cov=6.5, block=10000):
    """two chromosomes, both strands, 10 kb blocks, ~10^7 per-read statistics"""
    rs = np.random.RandomState(seed)
    seqs = [(c, ''.join(rs.choice(list('ACGT'), chrm_len))) for c in ('chrA', 'chrB')]
    genome = rc.Genome(seqs)
    blocks = []
    for chrm, _ in seqs:
        for strand in ('+', '-'):
            for start in range(0, chrm_len, block):
                end = min(chrm_len, start + block)
                poss = np.arange(max(start, 8), min(end, chrm_len - 8))
                pos = np.repeat(poss, rs.poisson(cov, poss.shape[0]))
                b = np.zeros(pos.shape[0], dtype=rc.PER_READ_DT)
                b['pos'] = pos
                b['stat'] = np.round(rs.normal(0, 2, pos.shape[0]) * 8) / 8
                blocks.append((chrm, strand, start, end, b))
    return genome, blocks


def _restated_curves(res):
    return {n: (rc.curve(st, lab) if st.shape[0] else None) for n, (st, lab) in res.items()}


def _assert_curves(got, want):
    assert list(got) == list(want)
    for n in want:
        if want[n] is None:
            assert got[n] is None
            continue
        for a, b in zip(got[n], want[n]):
            assert _same(a, b), n


@pytest.mark.parametrize('path', ['motif', 'truth', 'ctrl'])
def test_fused_equals_restatement_and_dropins_at_scale(path):
    from tombo_b200 import tombo_helper as th, tombo_stats as ts
    genome, blocks = _big(71 + len(path))
    n_stats = sum(b[4].shape[0] for b in blocks)
    assert n_stats >= 10 ** 7 and len(blocks) >= 100
    descs = th.parse_motif_descs('CG:1:cpg::GATC:2:dam::CCWGG:2:dcm')
    if path == 'motif':
        fused = ts.accuracy_curves(rc.Stats(blocks, 'stat'), descs, genome)
        want, err = rc.motif_stats(rc.Stats(blocks, 'stat'), descs, genome)
        assert err is None
    elif path == 'truth':
        rs = np.random.RandomState(3)
        locs = {(c, s): np.sort(rs.choice(400000, 60000, replace=False))
                for c in ('chrA', 'chrB') for s in '+-'}
        gt = ({k: v[:20000] for k, v in locs.items()}, {k: v[15000:] for k, v in locs.items()}, 'gt')
        fused = ts.accuracy_curves(rc.Stats(blocks, 'stat'), ground_truth_locs=gt)
        want = rc.truth_stats(rc.Stats(blocks, 'stat'), gt)
    else:
        ctrl_genome, ctrl_blocks = _big(99)
        ctrl = rc.CtrlStats(ctrl_blocks)
        fused = ts.accuracy_curves(rc.Stats(blocks, 'stat'), descs, genome, ctrl_stats=ctrl)
        want = rc.ctrl_stats_of(rc.Stats(blocks, 'stat'), rc.CtrlStats(ctrl_blocks), descs, genome)
    assert sum(v[0].shape[0] for v in want.values()) > 10 ** 6
    _assert_curves(fused, _restated_curves(want))
    # the drop-ins' composition on a part of the blocks (tuples are the slow return type)
    part = blocks[:40]
    if path == 'motif':
        tuples = ts._compute_motif_stats(rc.Stats(part, 'stat'), descs, genome)
        fused = ts.accuracy_curves(rc.Stats(part, 'stat'), descs, genome)
    elif path == 'truth':
        tuples = ts._compute_ground_truth_stats(rc.Stats(part, 'stat'), gt)
        fused = ts.accuracy_curves(rc.Stats(part, 'stat'), ground_truth_locs=gt)
    else:
        tuples = ts._compute_ctrl_motif_stats(rc.Stats(part, 'stat'), rc.CtrlStats(ctrl_blocks),
                                              descs, genome)
        fused = ts.accuracy_curves(rc.Stats(part, 'stat'), descs, genome,
                                   ctrl_stats=rc.CtrlStats(ctrl_blocks))
    for n, tl in tuples.items():
        if not tl:
            assert fused[n] is None
            continue
        tp, fp, prec, _ = ts.prep_accuracy_rates({n: tl})
        assert _same(tp, fused[n][0]) and _same(fp, fused[n][1]) and _same(prec, fused[n][2])


# ---- the sort ---------------------------------------------------------------------------
def _adversarial(rs):
    one = np.nextafter(1.0, 2.0) - 1.0
    yield 'all_equal', np.full(5000, 0.25)
    yield 'one_ulp', 1.0 + one * rs.randint(0, 4, 9000)
    yield 'denormal_inf_zero', rs.choice([5e-324, -5e-324, 1e-310, -1e-310, 0.0, -0.0, np.inf,
                                          -np.inf, 2.2250738585072014e-308], 7000)
    yield 'shared_top_bytes', 1000.0 + one * 1024 * rs.randint(0, 1 << 20, 50000)
    yield 'n1', np.array([0.5])
    yield 'tile_plus', rs.normal(0, 1, 3 * 4096 + 17)
    yield 'wide', rs.standard_cauchy(200000) * np.exp(rs.normal(0, 30, 200000))


def test_sort_matches_lexsort_on_adversarial_keys(ctx):
    rs = np.random.RandomState(8)
    for name, st in _adversarial(rs):
        n = st.shape[0]
        for lab in (rs.rand(n) < 0.3, np.ones(n, dtype=bool), np.zeros(n, dtype=bool)):
            ctx.accuracy_load(3, st, lab)
            # every index sampled: the rates fix the whole label order
            idx = np.arange(n, dtype=np.int64)
            tp, fp, prec = ctx.accuracy_curve(3, idx, idx)
            want = rc.accuracy_rates(rc.ordered_labels(st, lab), n)
            ordered = rc.ordered_labels(st, lab)
            assert _same(prec, np.cumsum(ordered) / np.arange(1, n + 1, dtype=float)), name
            for a, b in zip((tp, fp), want[:2]):
                assert _same(a, b), name


# ---- errors -------------------------------------------------------------------------------
def test_errors(ctx):
    from tombo_b200 import _lib, tombo_helper as th, tombo_stats as ts
    with pytest.raises(th.TomboError):
        ts.prep_accuracy_rates({'m': [(0.5, True), (float('nan'), False)]})
    with pytest.raises(IndexError):
        ts.prep_accuracy_rates({'m': []})
    with pytest.raises(IndexError):
        ts.compute_accuracy_rates([])
    lib, h = ctx.lib, ctx.handle
    ctx.accuracy_reset()
    idx = np.zeros(4, dtype=np.int64)
    with pytest.raises(_lib.TomboB200Error):
        ctx.accuracy_curve(0, idx, idx)                 # empty slot
    with pytest.raises(_lib.TomboB200Error):
        ctx.accuracy_curve(16, idx, idx)                # no such slot
    ctx.accuracy_load(0, [1.0, 2.0], [True, False])
    with pytest.raises(_lib.TomboB200Error):
        ctx.accuracy_curve(0, idx + 2, idx)             # index past the end
    m = th.TomboMotif('CG', 1)
    motifs = [_lib.motif_struct(m)]
    blocks = np.zeros(1, dtype=_lib.ACC_BLOCK_DTYPE)
    blocks['seq_len'], blocks['n_stat'] = 10, 1
    seq, pos, st = np.zeros(10, np.uint8), np.array([5], np.uint32), np.array([0.1])
    ctx.accuracy_label_motif(blocks, seq, pos, st, motifs, [0], 0, 1)
    bad = blocks.copy()
    bad['strand'] = 2
    for args in ((bad, seq, pos, st, motifs, [0], 0, 1),       # strand
                 (blocks, seq, pos, st, motifs, [16], 0, 1),   # slot
                 (blocks, seq, pos, st, motifs, [0], 1, 1),    # bb not max(mod_pos) - 1
                 (blocks, seq[:5], pos, st, motifs, [0], 0, 1)):   # block past the sequence
        with pytest.raises(_lib.TomboB200Error) as e:
            ctx.accuracy_label_motif(*args)
        assert '(201)' in str(e.value)
    unsorted = np.array([5, 3], dtype=np.int64)
    tb = np.zeros(1, dtype=_lib.ACC_BLOCK_DTYPE)
    tb['n_stat'], tb['n_mod'] = 1, 2
    with pytest.raises(_lib.TomboB200Error) as e:
        ctx.accuracy_label_truth(tb, pos, st, unsorted, np.zeros(0, np.int64))
    assert '(201)' in str(e.value)
    with pytest.raises(_lib.TomboB200Error):
        ctx.accuracy_rates_ordered(np.zeros(0, bool), idx, idx)


# ---- workspace isolation ---------------------------------------------------------------
def test_other_device_results_survive(ctx, RPcls):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    kmeans, ksds = syn.kmer_table(kmer_ref)
    K = len(kmer_ref[0][0])
    ctx.set_model(kmeans, ksds, K, cpos)
    ctx.set_alt_model(np.full((4 ** K, K), 1.0), K)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 64, 200, 99)
    aln = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    pol = _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    before = {k: v.copy() for k, v in ctx.batch_download().items() if isinstance(v, np.ndarray)}
    start = np.arange(64, dtype=np.int64) * 11
    ctx.batch_alt_llr(start, 1)
    llr_before = [a.copy() for a in ctx.batch_llr_download()]
    ctx.region_stats_begin(0, 2000)
    ctx.region_stats_add(np.array([0.5, 0.01]), np.array([3, 4]), 0.05, None, 1)
    cnt_before = ctx.region_counts_get()
    lv = np.random.RandomState(1).normal(0, 1, 300)
    med_before = ctx.kmer_medians(8, np.arange(300) % 8, lv, np.abs(lv))
    # the accuracy calls
    rs = np.random.RandomState(2)
    st = np.round(rs.normal(0, 1, 300000) * 4) / 4
    ctx.accuracy_load(0, st, rs.rand(st.shape[0]) < 0.4)
    idx = np.linspace(0, st.shape[0] - 1, 1000).astype(np.int64)
    ctx.accuracy_curve(0, idx, idx)
    ctx.accuracy_rates_ordered(rs.rand(5000) < 0.5, idx % 5000, idx % 5000)
    after = ctx.batch_download()
    for k, v in before.items():
        assert np.array_equal(after[k], v, equal_nan=True), k
    for a, b in zip(ctx.batch_llr_download(), llr_before):
        assert np.array_equal(a, b, equal_nan=True)
    assert np.array_equal(ctx.region_counts_get(), cnt_before)
    for a, b in zip(ctx.kmer_medians(8, np.arange(300) % 8, lv, np.abs(lv)), med_before):
        assert np.array_equal(a, b, equal_nan=True)
