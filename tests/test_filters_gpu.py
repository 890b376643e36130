"""Read filters on the device (csrc/read_filter.cu): percentiles bit for bit against
np.percentile, the resquiggle-time filter codes on a real resident batch, mid-read coverage,
every `tombo filter` command against the unmodified reference's goldens, and the error paths."""
import numpy as np
import pytest

import filters_cases as fc

pytestmark = pytest.mark.gpu

GOLD = fc.load_golden()
ALN_DNA = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
ALN_RNA = (6, 4, 500, 1500, 20.0, 50, 1000, 3000, 250)
SEG_RNA = (12, 6, 2, 15)
OBS = [[50, 4], [90, 9], [0, 1], [100, 40], [33, 6]]


@pytest.fixture
def ctx():
    from tombo_b200 import _lib
    c = _lib.Context(0)
    yield c
    c.close()


def _last_error(c):
    return c.lib.tb2_last_error(c.handle).decode()


@pytest.mark.parametrize('pctl', [[0, 100], [50, 90], [33, 67, 25, 75, 12.5, 99.9], [37.5, 0.1]])
def test_dwell_percentiles_bit_exact(ctx, pctl):
    rng = np.random.RandomState(int(sum(pctl)))
    n = 12000
    sizes = rng.choice([1, 2, 3, 5, 17, 256, 257, 600, 9000], size=n,
                       p=[.1, .1, .1, .2, .2, .1, .1, .09, .01])
    lens = rng.randint(1, 60, size=int(sizes.sum())).astype(np.int64)
    lens[rng.rand(lens.shape[0]) < 0.3] = 3              # many ties
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    got = ctx.dwell_percentiles(lens, off, pctl)
    want = np.empty_like(got)
    for r in range(n):
        x = lens[off[r]:off[r + 1]]
        for j, p in enumerate(pctl):
            want[r, j] = np.percentile(x, p)
    assert got.tobytes() == want.tobytes()


def test_dwell_percentiles_long_reads(ctx):
    """reads far longer than a block's shared memory"""
    rng = np.random.RandomState(5)
    sizes = np.array([1 << 20, 300001, 1, 2])
    lens = rng.randint(1, 1 << 30, size=int(sizes.sum())).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    pctl = [0, 13.7, 50, 99.99, 100]
    got = ctx.dwell_percentiles(lens, off, pctl)
    want = np.array([[np.percentile(lens[a:b], p) for p in pctl] for a, b in zip(off[:-1], off[1:])])
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize('kind', ['DNA', 'RNA'])
def test_batch_read_filters_match_host(ctx, RPcls, kind):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, len(kmer_ref[0][0]), cpos)
    if kind == 'DNA':
        rp, sp = RPcls(ALN_DNA), RPcls(ALN_DNA, save=True)
        raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 3000, 444, 77)
    else:
        rp, sp = RPcls(ALN_RNA, SEG_RNA, rna=True), RPcls(ALN_RNA, SEG_RNA, rna=True, save=True)
        raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 1000, 270, 78, kind='RNA')
    pol = _lib.make_policy(kind)
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    res = ctx.batch_download()
    ok = res['status'] == 0
    assert ok.mean() > 0.8
    segs = [res['segs'][a:b] for a, b in zip(res['seg_off'][:-1], res['seg_off'][1:])]
    score = res['sig_match_score']
    thr = float(np.median(score[ok]))                 # about half the reads above it
    p90 = [np.percentile(np.diff(s), 90) for s, g in zip(segs, ok) if g]
    split = [[90, int(np.median(p90))]]               # about half the tested reads stuck
    for obs in (None, OBS, split):
        code, pv = ctx.batch_read_filters(thr, obs, want_percentiles=True)
        assert list(code) == fc.host_codes(segs, score, ok, thr, obs)
        assert (code[~ok] == -1).all()
        if obs:
            want = np.array([[np.percentile(np.diff(s), p) for p, _ in obs] if g else [np.nan] * len(obs)
                             for s, g in zip(segs, ok)])
            assert pv.tobytes() == want.tobytes()
        if obs is split:
            assert (code == 2).any() and (code == 1).any() and (code == 0).any()
        assert np.array_equal(ctx.batch_read_filters(thr, obs), code)


def test_mid_coverage_matches_numpy(ctx):
    rng = np.random.RandomState(9)
    sizes = [5000, 1, 700000, 0, 300]
    counts = [400, 1, 20000, 0, 50]
    grp_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    start, end = [], []
    for s, n in zip(sizes, counts):
        a = rng.randint(0, max(s - 1, 1), size=n)
        start.append(a)
        end.append(a + rng.randint(1, 20000, size=n))
    start, end = np.concatenate(start), np.concatenate(end)
    got = ctx.read_mid_coverage(grp_off, start, end)
    assert np.array_equal(got, fc.HostContext().read_mid_coverage(grp_off, start, end))


@pytest.mark.parametrize('case', GOLD['filters'], ids=lambda c: c['name'])
def test_filter_commands_match_reference(ctx, case, tmp_path):
    kind, got = fc.run_filter_case(case, ctx, str(tmp_path))
    if 'error' in case:
        assert kind == 'error' and got == 'No unfiltered reads present in current Tombo index.'
    else:
        assert got == case['output']


def test_error_paths(ctx, RPcls):
    from tombo_b200 import _lib, synthetic as syn
    E = _lib.TomboB200Error
    lens, off = np.arange(1, 7, dtype=np.int64), np.array([0, 2, 6], dtype=np.int64)
    for pctl in ([-1.0], [100.5], [np.nan], []):
        with pytest.raises(E, match=r'\(201\)'):
            ctx.dwell_percentiles(lens, off, pctl)
    for bad in (np.array([0, 2, 2]), np.array([0, 4, 2]), np.array([-1, 2, 6])):
        with pytest.raises(E, match=r'\(201\)'):
            ctx.dwell_percentiles(lens, bad, [50])
    with pytest.raises(E, match=r'\(201\)'):
        ctx.read_mid_coverage([0, 2], [5, 3], [5, 9])          # end <= start
    with pytest.raises(E, match=r'\(201\)'):
        ctx.read_mid_coverage([0, 2, 1], [0, 3], [5, 9])       # decreasing groups
    # before any compute
    with pytest.raises(E, match='tb2_batch_compute has not been called'):
        ctx.batch_read_filters(1.1, [[50, 4]])
    # a good batch, then a failed compute: no stale codes
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, len(kmer_ref[0][0]), cpos)
    rp, sp, pol = RPcls(ALN_DNA), RPcls(ALN_DNA, save=True), _lib.make_policy('DNA')
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 16, 200, 4242)
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    assert ctx.batch_read_filters(1.1, [[50, 4]]).shape == (16,)
    with pytest.raises(E, match=r'\(201\)'):
        ctx.batch_read_filters(1.1, [[150, 4]])
    assert _last_error(ctx) == ''
    with pytest.raises(E, match=r'\(201\)'):
        ctx.batch_compute(rp, None, pol)                      # rescue without save parameters
    with pytest.raises(E, match='tb2_batch_compute has not been called'):
        ctx.batch_read_filters(1.1, [[50, 4]])
    # a clean call after the failures carries no message
    ctx.read_mid_coverage([0, 1], [0], [3])
    assert _last_error(ctx) == ''


def test_resquiggle_reads_for_index(RPcls):
    """the batched resquiggle call with filter codes: same results as resquiggle_reads"""
    from tombo_b200 import resquiggle as rsq, synthetic as syn, tombo_helper as th, tombo_stats as ts
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    reads = syn.make_reads(kmer_ref, cpos, 40, 444, seed0=99)
    maps = [th.resquiggleResults(align_info=th.alignInfo('r%d' % i, 'BaseCalled_template', 0, 0, 0, 0, 0, 0),
                                 genome_loc=th.genomeLocation(100 * i, '+', 'chr1'),
                                 genome_seq=r.genome_seq, mean_q_score=10.0, raw_signal=r.raw)
            for i, r in enumerate(reads)]
    rp, sp = RPcls(ALN_DNA), RPcls(ALN_DNA, save=True)
    plain = rsq.resquiggle_reads(maps, std_ref, rp, sp)
    both = rsq.resquiggle_reads_for_index(maps, std_ref, rp, sp, index_sig_match_thresh=0.9,
                                          obs_filter=[[90, 6]])
    assert len(both) == len(plain)
    segs, score, ok = [], [], []
    for a, (b, code) in zip(plain, both):
        good = not isinstance(a, Exception)
        ok.append(good)
        segs.append(a.segs if good else None)
        score.append(a.sig_match_score if good else 0.0)
        if good:
            assert np.array_equal(a.segs, b.segs) and a.sig_match_score == b.sig_match_score
    assert [c for _, c in both] == fc.host_codes(segs, score, ok, 0.9, [[90, 6]])
