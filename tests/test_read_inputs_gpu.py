"""GPU: caller-supplied per-read inputs of resquiggle_read -- map_res.scale_values and
map_res.stall_ints (resquiggle.py:1079-1118) -- through the Python mirrors and through
tb2_batch_set_read_inputs at batch scale, bit for bit against the C oracle
(orc_resquiggle_read / orc_run_read_inputs) and against the reference's own outputs
(tests/golden/rsqgl_inputs.npz); the state those inputs leave between calls; and the checks
on them."""
import ctypes as C
from multiprocessing.pool import ThreadPool

import numpy as np
import pytest

import golden_util as gu
from read_inputs_cases import norm_scale_values, stall_lists

pytestmark = pytest.mark.gpu

ALN_C1 = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
ALN_NARROW = (4.2, 4.2, 100, 1500, 20.0, 40, 300, 2500, 100)
INVALID_ARG = 201
CAPACITY = 202


def _same(a, b):
    """equal doubles, None on one side <-> NaN on the other"""
    a = [np.nan if v is None else float(v) for v in a]
    b = [np.nan if v is None else float(v) for v in b]
    return all(x == y or (np.isnan(x) and np.isnan(y)) for x, y in zip(a, b))


def _setup(kind, aln):
    from tombo_b200 import tombo_helper as th, tombo_stats as ts, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
    sst = th.seqSampleType(kind, kind == 'RNA')
    p = ts.load_resquiggle_parameters(sst, aln)
    sp = ts.load_resquiggle_parameters(sst, aln, use_save_bandwidth=True)
    return th, syn, kmer_ref, cpos, std_ref, sst, p, sp


def _map_res(th, raw, seq, **kw):
    return th.resquiggleResults(
        align_info=th.alignInfo('r', 'BaseCalled_template', 0, 0, 0, 0, len(seq), 0),
        genome_loc=th.genomeLocation(0, '+', 'chr'), genome_seq=seq, mean_q_score=10.0,
        raw_signal=raw, **kw)


def _check_single(res, o):
    """a resquiggleResults (or TomboError) against orc_resquiggle_read / orc_run_read output"""
    from tombo_b200 import _lib, tombo_helper as th
    if o['status'] != 0:
        assert isinstance(res, Exception), o['status']
        assert str(res) == _lib.status_message(o['status']), (res, o['status'])
        return
    assert not isinstance(res, Exception), (res, o['status'])
    assert np.array_equal(res.segs, o['segs'])
    assert res.read_start_rel_to_raw == o['read_start_rel_to_raw']
    sv = o['scale_values'] if 'scale_values' in o else (
        o['shift'], o['scale'], o['lower_lim'], o['upper_lim'], o['outlier_thresh'])
    assert _same(res.scale_values, sv), (res.scale_values, sv)
    # the outlier_threshold attribute write_new_fast5_group writes (tombo_helper.py:2407-2409)
    assert (res.scale_values.outlier_thresh is None) == bool(np.isnan(sv[4]))
    assert res.sig_match_score == o['sig_match_score']
    assert res.norm_params_changed == o['norm_params_changed']
    if 'norm_signal' in o:
        assert np.array_equal(res.raw_signal, o['norm_signal'])
    assert isinstance(res, th.resquiggleResults)


def _run_single(mr, std_ref, p, sst, kw):
    from tombo_b200 import resquiggle, tombo_helper as th
    try:
        return resquiggle.resquiggle_read(mr, std_ref, p, seq_samp_type=sst, **kw)
    except (th.TomboError, resquiggle.LibraryError) as e:
        return e


def test_normalize_raw_signal_mirror_with_scale_values_and_threshold(orc):
    """tombo_stats.normalize_raw_signal(raw, outlier_thresh=t, scale_values=sv): odd and even n,
    continuous and integer-valued raw, finite and None limits, t = 5 and 0.5, and None limits
    without a threshold -- signal and all five scale values equal the oracle's"""
    from tombo_b200 import tombo_helper as th, tombo_stats as ts
    rs = np.random.RandomState(31)
    for n in (4001, 4000, 257, 20012):
        for integer in (False, True):
            raw = 480 + 60 * rs.standard_t(5, n)
            if integer:
                raw = np.round(raw)
            for name, sv in norm_scale_values(raw):
                for t in (5.0, 0.5, None):
                    if t is None and name != 'shifted_none':
                        continue
                    s0, n0, sv0 = orc.normalize_raw_signal(raw, outlier_thresh=t, scale_values=sv)
                    norm, sv1 = ts.normalize_raw_signal(raw, outlier_thresh=t,
                                                        scale_values=th.scaleValues(*sv))
                    assert s0 == 0
                    assert np.array_equal(norm, n0), (n, integer, name, t)
                    assert _same(sv1, sv0), (n, integer, name, t, sv1, sv0)


@pytest.mark.parametrize('kind', ['DNA', 'RNA_params'])
def test_resquiggle_read_supplied_scale_values(orc, kind):
    """single resquiggle_read calls with map_res.scale_values: the read's own values, a
    shifted and scaled copy, None limits; skip_seq_scaling on and off; with const_scale the
    supplied values win.  RNA parameters (t-test segmentation, no flip) skip event scaling"""
    rna = kind != 'DNA'
    aln = gu.RNA_ALN if rna else (4.2, 4.2, 200, 1500, 20.0, 40, 300, 2500, 100)
    th, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup('RNA' if rna else 'DNA', aln)
    sst_dna = th.seqSampleType('DNA', False)      # one call on the data as given
    for seed in (23000, 23001):
        r = syn.make_read(kmer_ref, cpos, 270 if rna else 500, seed, kind='RNA' if rna else 'DNA')
        rm, rsd = gu.levels(r.genome_seq, kmer_ref)
        raw = np.asarray(r.raw, dtype=np.float64)
        for name, sv in norm_scale_values(raw):
            for skip in (False, True):
                for cs in (None, 61.5):
                    mr = _map_res(th, r.raw, r.genome_seq, scale_values=th.scaleValues(*sv))
                    res = _run_single(mr, std_ref, p, sst_dna,
                                      dict(outlier_thresh=5.0, skip_seq_scaling=skip, const_scale=cs))
                    pol = orc.policy('DNA', skip_seq_scaling=skip, const_scale=cs)
                    o = orc.resquiggle_read(raw, rm, rsd, p, pol, scale_values=sv)
                    _check_single(res, o)


@pytest.mark.parametrize('kind', ['DNA', 'RNA_params'])
def test_resquiggle_read_stall_lists(orc, kind):
    """single calls with map_res.stall_ints: identify_stalls of a planted stall, sorted,
    unsorted, overlapping and nested lists, endpoints on changepoints, an empty list, +-2^40,
    and one interval over most of the read (the call fails with the oracle's message)"""
    rna = kind != 'DNA'
    aln = gu.RNA_ALN if rna else (4.2, 4.2, 200, 1500, 20.0, 40, 300, 2500, 100)
    th, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup('RNA' if rna else 'DNA', aln)
    sst_dna = th.seqSampleType('DNA', False)
    pol = orc.policy('DNA')
    nbases = 270 if rna else 500
    r = syn.make_read(kmer_ref, cpos, nbases, 23100, kind='RNA' if rna else 'DNA', stall=(120, 1500))
    rm, rsd = gu.levels(r.genome_seq, kmer_ref)
    raw = np.asarray(r.raw, dtype=np.float64)
    n = raw.shape[0]
    n_ev = max(n // p.mean_obs_per_event, int((len(r.genome_seq) - len(kmer_ref[0][0]) + 1) * 1.1))
    if rna:
        st, cp = orc.valid_cpts_w_cap(raw, p.min_obs_per_base, p.running_stat_width, n_ev, t_test=True)
    else:
        st, n0, _ = orc.normalize_raw_signal(raw, 5.0)
        st, cp = orc.valid_cpts_w_cap(n0, p.min_obs_per_base, p.running_stat_width, n_ev)
    assert st == 0
    lists = stall_lists(n, np.sort(cp))
    lists['planted'] = [tuple(int(v) for v in iv) for iv in orc.identify_stalls(raw)]
    lists['most_of_read'] = [(5, n - 5)]
    assert len(lists['planted']) >= 1
    for name, si in lists.items():
        mr = _map_res(th, r.raw, r.genome_seq, stall_ints=si)
        res = _run_single(mr, std_ref, p, sst_dna, dict(outlier_thresh=5.0))
        o = orc.resquiggle_read(raw, rm, rsd, p, pol, stall_ints=si)
        if name == 'most_of_read':
            assert o['status'] != 0
        _check_single(res, o)


def test_resquiggle_reads_worker_policy_with_inputs(orc):
    """resquiggle_reads (worker policy): DNA with supplied scale values on a narrow band, so
    that rescued reads start again from the caller's values; DNA with stalls; RNA with caller
    stalls, which the worker replaces with its own (adjust_map_res)"""
    from tombo_b200 import resquiggle
    for kind, aln in (('DNA', ALN_NARROW), ('RNA', gu.RNA_ALN)):
        th, syn, kmer_ref, cpos, std_ref, sst, p, sp = _setup(kind, aln)
        pol = orc.policy(kind)
        nbs = np.random.RandomState(5).randint(300, 700, 48) if kind == 'DNA' else [270] * 24
        mrs, args = [], []
        for i, nb in enumerate(nbs):
            r = syn.make_read(kmer_ref, cpos, int(nb), 24000 + i, kind=kind)
            raw = np.asarray(r.raw, dtype=np.float64)
            n = raw.shape[0]
            sv = si = None
            if i % 3 == 0:
                sv = norm_scale_values(raw)[i % 2][1] if kind == 'DNA' else norm_scale_values(raw[::-1])[0][1]
            if i % 3 == 1 or kind == 'RNA':
                si = [(int(n * .4), int(n * .45)), (int(n * .1), int(n * .15))]
            mrs.append(_map_res(th, r.raw, r.genome_seq,
                                scale_values=None if sv is None else th.scaleValues(*sv), stall_ints=si))
            args.append((raw, gu.levels(r.genome_seq, kmer_ref), sv, si))
        out = resquiggle.resquiggle_reads(mrs, std_ref, p, sp, outlier_thresh=5.0, seq_samp_type=sst)
        rescued_sv = 0
        for i, (raw, (rm, rsd), sv, si) in enumerate(args):
            o = orc.run_read(raw, rm, rsd, p, sp, pol, read_index=i, scale_values=sv, stall_ints=si)
            rescued_sv += o['rescued'] and sv is not None
            _check_single(out[i], o)
        if kind == 'DNA':
            assert rescued_sv > 0, 'no read with supplied scale values went through the rescue'


# ---------------------------------------------------------------- staged C API, batch scale
def _stall_arrays(lists):
    off = np.zeros(len(lists) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in lists])
    flat = np.zeros(max(1, int(off[-1])) * 2, dtype=np.int64)
    k = 0
    for s in lists:
        for a, b in s:
            flat[2 * k], flat[2 * k + 1] = a, b
            k += 1
    return flat, off


def _set_inputs(ctx, sv, stall_flat, stall_off):
    from tombo_b200 import _lib
    return ctx.lib.tb2_batch_set_read_inputs(
        ctx.handle, _lib.ptr(sv, _lib.ScaleValues) if sv is not None else None,
        _lib.ptr(stall_flat, C.c_int64) if stall_flat is not None else None,
        _lib.ptr(stall_off, C.c_int64) if stall_off is not None else None)


def _batch_inputs(raw_off, seed, with_sv=True, with_stalls=True):
    """a third of the reads carry scale values (the rest NaN shift), a third stall lists:
    sorted, unsorted, empty, +-2^40 in turn"""
    n = raw_off.shape[0] - 1
    rs = np.random.RandomState(seed)
    sv = np.full((n, 5), np.nan)
    lists = [[] for _ in range(n)]
    for i in range(n):
        ln = int(raw_off[i + 1] - raw_off[i])
        if with_sv and i % 3 == 0:
            sv[i] = (480.0 + rs.normal(0, 4), 60.0 * (1 + rs.normal(0, .05)),
                     -5.0 if i % 2 else np.nan, 5.0 if i % 2 else np.nan, np.nan)
        if with_stalls and i % 3 == 1:
            a = lambda f: int(ln * f)   # noqa: E731
            lists[i] = [[(a(.3), a(.35)), (a(.6), a(.62))], [(a(.6), a(.62)), (a(.3), a(.35))], [],
                        [(-2 ** 40, a(.02)), (a(.97), 2 ** 40)]][(i // 3) % 4]
    return (sv if with_sv else None), (lists if with_stalls else None)


def _oracle_batch(orc, raw, raw_off, seq, seq_off, means, sds, k, p, sp, pol, sv, lists):
    def one(i):
        rm, rs = orc.levels_from_codes(seq[seq_off[i]:seq_off[i + 1]], means, sds, k)
        r = np.asarray(raw[raw_off[i]:raw_off[i + 1]], dtype=np.float64)
        svi = None if sv is None or np.isnan(sv[i][0]) else tuple(sv[i])
        si = None if lists is None else lists[i]
        return i, orc.run_read(r, rm, rs, p, sp, pol, read_index=i, scale_values=svi, stall_ints=si)
    with ThreadPool(32) as tp:
        return dict(tp.imap_unordered(one, range(raw_off.shape[0] - 1), chunksize=16))


def _compare(res, out):
    import oracle as orc
    bad = orc.compare_batch(res, out)
    for i, o in out.items():
        if o['status'] == 0 and int(res['status'][i]) == 0:
            t = res['scale_values'][i][4]
            if not (t == o['outlier_thresh'] or (np.isnan(t) and np.isnan(o['outlier_thresh']))):
                bad.append((i, 'outlier_thresh'))
    return bad


def _staged(ctx, raw, raw_off, seq, seq_off, p, sp, pol, sv=None, lists=None, withdraw=False):
    ctx.batch_upload(raw, raw_off, seq, seq_off, p, pol)
    if sv is not None or lists is not None:
        flat, off = _stall_arrays(lists) if lists is not None else (None, None)
        assert _set_inputs(ctx, sv, flat, off) == 0
    if withdraw:
        assert _set_inputs(ctx, None, None, None) == 0
    ctx.batch_compute(p, sp, pol)
    return ctx.batch_download()


@pytest.mark.parametrize('aln', [ALN_C1, ALN_NARROW], ids=['default_band', 'narrow_band'])
def test_batch_inputs_config1_2048_reads(ctx, orc, RPcls, aln):
    """2048 configs[1]-shaped DNA reads, a third with scale values and a third with stall lists,
    worker policy with rescue: every read bit for bit against orc_run_read_inputs"""
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    k = len(kmer_ref[0][0])
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, k, cpos)
    rp, sp = RPcls(aln, (5, 3, 1, 5)), RPcls(aln, (5, 3, 1, 5), save=True)
    nb = 444 if aln is ALN_C1 else np.random.RandomState(7).randint(300, 900, 2048)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 2048, nb, 301)
    sv, lists = _batch_inputs(raw_off, 302)
    pol = _lib.make_policy('DNA', subsample_seed=301)
    res = _staged(ctx, raw, raw_off, seq, seq_off, rp, sp, pol, sv, lists)
    out = _oracle_batch(orc, raw, raw_off, seq, seq_off, means, sds, k, rp, sp,
                        orc.policy('DNA', subsample_seed=301), sv, lists)
    bad = _compare(res, out)
    assert not bad, bad[:10]
    assert (res['status'] == 0).mean() > (0.8 if aln is ALN_C1 else 0.2)
    if aln is ALN_NARROW:
        with_sv = ~np.isnan(sv[:, 0])
        assert ((res['flags'] & 2 != 0) & with_sv).any(), 'no read with scale values was rescued'
        has_st = np.array([len(s) > 0 for s in lists])
        assert ((res['flags'] & 2 != 0) & has_st).any(), 'no read with stalls was rescued'


def test_batch_inputs_rna_params_dna_policy_512_reads(ctx, orc, RPcls):
    """512 RNA-parameter reads (t-test segmentation) under a DNA policy, single call, with
    scale values and stall lists"""
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('RNA', 0)
    k = len(kmer_ref[0][0])
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, k, cpos)
    rp, sp = RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True), RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True, save=True)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 512, 270, 303, kind='RNA')
    sv, lists = _batch_inputs(raw_off, 304)
    pol = _lib.make_policy('DNA', max_scaling_iters=1, rescue=False, subsample_seed=303)
    res = _staged(ctx, raw, raw_off, seq, seq_off, rp, sp, pol, sv, lists)
    out = _oracle_batch(orc, raw, raw_off, seq, seq_off, means, sds, k, rp, sp,
                        orc.policy('DNA', max_scaling_iters=1, subsample_seed=303), sv, lists)
    bad = _compare(res, out)
    assert not bad, bad[:10]
    assert (res['status'] == 0).mean() > 0.5


def test_batch_inputs_rna_policy_scale_values(ctx, orc, RPcls):
    """an RNA-policy batch (flip, own stalls, iterations, rescue) with supplied scale values"""
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('RNA', 0)
    k = len(kmer_ref[0][0])
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, k, cpos)
    rp, sp = RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True), RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True, save=True)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, 256, 270, 305, kind='RNA')
    sv, _ = _batch_inputs(raw_off, 306, with_stalls=False)
    pol = _lib.make_policy('RNA', subsample_seed=305)
    res = _staged(ctx, raw, raw_off, seq, seq_off, rp, sp, pol, sv, None)
    out = _oracle_batch(orc, raw, raw_off, seq, seq_off, means, sds, k, rp, sp,
                        orc.policy('RNA', subsample_seed=305), sv, None)
    bad = _compare(res, out)
    assert not bad, bad[:10]
    assert (res['status'] == 0).mean() > 0.5


# ---------------------------------------------------------------- state between calls, bad input
def _small_batch(RPcls, seed, n=64):
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    means, sds = syn.kmer_table(kmer_ref)
    batch = syn.make_read_batch(kmer_ref, n, 444, seed)
    model = (means, sds, len(kmer_ref[0][0]), cpos)
    return batch, model, RPcls(ALN_C1), RPcls(ALN_C1, save=True), _lib.make_policy('DNA')


def _same_result(a, b):
    for key in ('segs', 'read_start_rel_to_raw', 'sig_match_score', 'status', 'n_iters', 'flags'):
        if not np.array_equal(a[key], b[key], equal_nan=key == 'sig_match_score'):
            return False
    return np.array_equal(a['scale_values'], b['scale_values'], equal_nan=True)


def test_inputs_do_not_outlive_their_upload(RPcls):
    """set_read_inputs before any upload fails; inputs of one upload do not reach the next
    upload's reads (equal to a fresh context's result); withdrawing them with a second call
    passing NULL gives the no-input result"""
    from tombo_b200 import _lib
    (raw, raw_off, seq, seq_off), model, rp, sp, pol = _small_batch(RPcls, 401)
    (raw2, raw_off2, seq2, seq_off2), _, _, _, _ = _small_batch(RPcls, 402)
    sv, lists = _batch_inputs(raw_off, 403)
    flat, off = _stall_arrays(lists)
    a = _lib.Context(0)
    b = _lib.Context(0)
    try:
        assert _set_inputs(a, sv, flat, off) == INVALID_ARG
        for c in (a, b):
            c.set_model(*model)
        with_inputs = _staged(a, raw, raw_off, seq, seq_off, rp, sp, pol, sv, lists)
        plain = _staged(b, raw, raw_off, seq, seq_off, rp, sp, pol)
        assert not _same_result(with_inputs, plain), 'the inputs changed nothing'
        second = _staged(a, raw2, raw_off2, seq2, seq_off2, rp, sp, pol)
        fresh = _staged(b, raw2, raw_off2, seq2, seq_off2, rp, sp, pol)
        assert _same_result(second, fresh)
        withdrawn = _staged(a, raw, raw_off, seq, seq_off, rp, sp, pol, sv, lists, withdraw=True)
        assert _same_result(withdrawn, plain)
    finally:
        a.close()
        b.close()


def test_set_read_inputs_rejects_bad_stall_input(ctx, orc, RPcls):
    """stall_off not starting at 0 or decreasing, and stall inputs on an RNA-policy upload:
    TB2_ERR_INVALID_ARG.  +-2^40 stall values give the oracle's result on the int64 values"""
    from tombo_b200 import _lib, synthetic as syn
    (raw, raw_off, seq, seq_off), model, rp, sp, pol = _small_batch(RPcls, 404, n=32)
    ctx.set_model(*model)
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    n = raw_off.shape[0] - 1
    flat = np.zeros(8, dtype=np.int64)
    off = np.zeros(n + 1, dtype=np.int64)
    off[0] = 1
    off[1:] = 1
    assert _set_inputs(ctx, None, flat, off) == INVALID_ARG
    off = np.zeros(n + 1, dtype=np.int64)
    off[1], off[2:] = 2, 1
    assert _set_inputs(ctx, None, flat, off) == INVALID_ARG
    # a pair count far beyond the batch's signal: refused before stall_ints is read
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = 1 << 29
    assert _set_inputs(ctx, None, flat, off) == CAPACITY
    # +-2^40 against the oracle on the int64 values
    lists = [[(-2 ** 40, 2 ** 40)] if i % 4 == 0 else
             [(-2 ** 41, int(raw_off[i + 1] - raw_off[i]) // 3), (2 ** 40, 2 ** 40 + 5)] if i % 4 == 1 else
             [(int(raw_off[i + 1] - raw_off[i]) // 2, 2 ** 40)] if i % 4 == 2 else []
             for i in range(n)]
    res = _staged(ctx, raw, raw_off, seq, seq_off, rp, sp, pol, None, lists)
    means, sds, k, cpos = model
    out = _oracle_batch(orc, raw, raw_off, seq, seq_off, means, sds, k, rp, sp, orc.policy('DNA'),
                        None, lists)
    bad = _compare(res, out)
    assert not bad, bad[:10]
    assert (res['status'][::4] != 0).all()          # one interval over the whole read
    # RNA-policy upload: the worker detects stalls itself
    kmer_ref, cpos = syn.make_kmer_ref('RNA', 0)
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, len(kmer_ref[0][0]), cpos)
    rraw, rraw_off, rseq, rseq_off = syn.make_read_batch(kmer_ref, 8, 270, 405, kind='RNA')
    rrp = RPcls(gu.RNA_ALN, gu.RNA_SEG, rna=True)
    ctx.batch_upload(rraw, rraw_off, rseq, rseq_off, rrp, _lib.make_policy('RNA'))
    flat, off = _stall_arrays([[(10, 20)]] * 8)
    assert _set_inputs(ctx, None, flat, off) == INVALID_ARG
    sv = np.full((8, 5), np.nan)
    assert _set_inputs(ctx, sv, None, None) == 0


# ---------------------------------------------------------------- the reference's own outputs
def _check_golden(res, e, i):
    """a resquiggleResults / exception of the Python mirrors against the reference's output
    recorded in tests/golden/rsqgl_inputs.npz"""
    from tombo_b200 import _lib, resquiggle, tombo_helper as th
    if e['message']:
        if e['message'].startswith('UNEXPECTED'):
            assert isinstance(res, resquiggle.LibraryError), (i, res)
            assert str(res) == _lib.status_message(100), (i, res)
        else:
            assert isinstance(res, th.TomboError) and str(res) == e['message'], (i, res)
        return
    assert not isinstance(res, Exception), (i, res)
    assert np.array_equal(res.segs, e['segs']), i
    assert res.read_start_rel_to_raw == e['read_start_rel_to_raw'], i
    # all five values, None where the reference has None (the outlier_threshold attribute)
    assert tuple(res.scale_values) == e['scale_values'], (i, tuple(res.scale_values), e['scale_values'])
    assert res.sig_match_score == e['sig_match_score'], i
    assert res.norm_params_changed == e['norm_params_changed'], i


def test_normalize_raw_signal_matches_reference_golden():
    """tombo_stats.normalize_raw_signal with scale values and a threshold, against the
    reference: signal and all five values, None included"""
    import read_inputs_cases as ric
    from tombo_b200 import tombo_helper as th, tombo_stats as ts
    for raw, t, sv, want_norm, want in ric.golden_norm_cases(ric.golden()):
        norm, out = ts.normalize_raw_signal(raw, outlier_thresh=t, scale_values=th.scaleValues(*sv))
        assert np.array_equal(norm, want_norm), (len(raw), t, sv)
        assert tuple(out) == want, (tuple(out), want)


def test_resquiggle_read_and_reads_match_reference_golden(RPcls):
    """resquiggle_read (single calls: supplied scale values with skip_seq_scaling and
    const_scale, every stall-list shape, RNA parameters) and resquiggle_reads (worker policy:
    DNA scale values with rescues, DNA stalls, RNA with caller stalls) against the reference"""
    import read_inputs_cases as ric
    from tombo_b200 import resquiggle, tombo_helper as th, tombo_stats as ts
    cases = ric.golden_cases(ric.golden(), RPcls)
    models = {}

    def model(c):
        if c['kind'] not in models:
            models[c['kind']] = ts.TomboModel(kmer_ref=c['kmer_ref'], central_pos=c['cpos'])
        return models[c['kind']]

    def map_res(c):
        sv = None if c['scale_values'] is None else th.scaleValues(*c['scale_values'])
        return _map_res(th, c['read'].raw, c['read'].genome_seq, scale_values=sv,
                        stall_ints=c['stall_ints'])
    dna = th.seqSampleType('DNA', False)
    for i, c in enumerate(cases):
        if c['call'] != 0:
            continue
        res = _run_single(map_res(c), model(c), c['rp'], dna,
                          dict(outlier_thresh=5.0, skip_seq_scaling=c['skip'],
                               const_scale=c['const_scale']))
        _check_golden(res, c['expected'], i)
    for grp in sorted(set(c['group'] for c in cases if c['call'] == 1)):
        idx = sorted((c['read_index'], i) for i, c in enumerate(cases)
                     if c['call'] == 1 and c['group'] == grp)
        cs = [cases[i] for _, i in idx]
        assert [c['read_index'] for c in cs] == list(range(len(cs)))
        kind = cs[0]['kind']
        out = resquiggle.resquiggle_reads([map_res(c) for c in cs], model(cs[0]), cs[0]['rp'],
                                          cs[0]['sp'], outlier_thresh=5.0,
                                          seq_samp_type=th.seqSampleType(kind, kind == 'RNA'))
        for (_, i), c, res in zip(idx, cs, out):
            _check_golden(res, c['expected'], i)
