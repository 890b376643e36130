"""tb2_resquiggle_batch above 6 U reads (U = SMs x 32): the pipelined branch cuts the batch
into chunks of 2 U, 4 U and then 6 U reads and runs them alternately on two lane contexts.

Every chunk, lane and context is held to the staged single-upload path bit for bit and to
the C oracle under the read's global index.  Chunk boundaries come from the device's SM
count and tb2_pipeline_chunks, so the file means the same thing on any SM count.  Batches are
short filler reads with planted reads at chosen indices: the first and last read of every
chunk, reads of more than 1000 bases (keyed Theil-Sen sub-sampling) in every chunk, reads that
fail, and stall reads that are rescued at the save bandwidth."""
import threading
from types import SimpleNamespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DNA_ALN = (4.2, 4.2, 120, 1500, 20.0, 40, 300, 2500, 100)   # planted stalls need the rescue
DNA_ALN_BW400 = (4.2, 4.2, 400, 1500, 20.0, 40, 750, 2500, 250)
DNA_SEG = (5, 3, 1, 5)
RNA_ALN = (6, 4, 500, 1500, 20.0, 50, 1000, 3000, 250)
RNA_SEG = (12, 6, 2, 15)
TB2_ERR_INVALID_ARG = 201
NOT_COMPUTED = 'tb2_batch_compute has not been called'
SUBSAMPLE_BASES = 1000          # Theil-Sen sub-samples reads with more bases than this
ORACLE_SAMPLE = 512


# ---------------------------------------------------------------------------- fixtures
@pytest.fixture(scope='module')
def sm_count():
    """SMs of device 0, read at run time (cudaDevAttrMultiProcessorCount through torch)"""
    import torch
    return int(torch.cuda.get_device_properties(0).multi_processor_count)


@pytest.fixture(scope='module')
def models():
    from tombo_b200 import synthetic as syn
    out = {}
    for name, kind, seed, sd_range in (('dna', 'DNA', 0, None), ('dna_b', 'DNA', 3, (0.15, 0.3)),
                                       ('rna', 'RNA', 0, None)):
        kmer_ref, cpos = syn.make_kmer_ref(kind, seed, sd_range=sd_range)
        means, sds = syn.kmer_table(kmer_ref)
        out[name] = dict(kind=kind, kmer_ref=kmer_ref, cpos=cpos, means=means, sds=sds,
                         k=len(kmer_ref[0][0]))
    return out


def _params(RPcls, kind, aln=None):
    if kind == 'RNA':
        return RPcls(RNA_ALN, RNA_SEG, rna=True), RPcls(RNA_ALN, RNA_SEG, rna=True, save=True)
    aln = DNA_ALN if aln is None else aln
    return RPcls(aln, DNA_SEG), RPcls(aln, DNA_SEG, save=True)


def chunk_starts(sm, n):
    from tombo_b200 import _lib
    out = np.zeros(64, dtype=np.int64)
    k = _lib.load().tb2_pipeline_chunks(int(sm), int(n), _lib.ptr(out, _lib.i64), 64)
    assert k > 0, k
    return out[:k + 1]


def n_reads_for(sm, chunks):
    """the smallest batch plus half a U that runs `chunks` (3: > 6 U, 4: > 12 U) chunks"""
    u = sm * 32
    return {3: 6 * u, 4: 12 * u}[chunks] + u // 2


# ---------------------------------------------------------------------------- batches
def _one(m, nb, seed, int16=False, **kw):
    from tombo_b200 import synthetic as syn
    r = syn.make_read(m['kmer_ref'], m['cpos'], nb, seed, kind=m['kind'], int16=int16, **kw)
    return r.raw, syn.seq_to_codes(r.genome_seq)


def planted_reads(m, cs, seed, int16=False):
    """{index: (raw, codes, what)} for chunks [cs[k], cs[k+1]): the chunk's first read is a
    long read (a stall read in chunk 0), the second a stall read, the middle one a long read,
    four failing reads follow it and the chunk's last read fails too"""
    K = m['k']

    def failing(j, s):
        if j == 0:                                   # constant signal: MAD scale of zero
            raw, codes = _one(m, 100, s, int16)
            return np.full_like(raw, 480), codes, 'fail'
        if j == 1:                                   # too much signal for one base
            raw, codes = _one(m, 1000, s, int16)
            return raw, codes[:K], 'fail'
        if j == 2:                                   # sequence unrelated to the signal
            return _one(m, 120, s, int16)[0], _one(m, 120, s + 1, int16)[1], 'unrelated'
        raw, codes = _one(m, 100, s, int16)          # sequence shorter than the k-mer
        return raw, codes[:K - 1], 'fail'

    def stall(s):
        if m['kind'] == 'RNA':
            return _one(m, 300, s, int16, stall=(150, 3000)) + ('stall',)
        return _one(m, 600, s, int16, stall=(300, 1500)) + ('stall',)

    def long(k, s):
        return _one(m, 1100 + 97 * k, s, int16) + ('long',)

    out = {}
    for k in range(len(cs) - 1):
        a, b = int(cs[k]), int(cs[k + 1])
        mid = (a + b) // 2
        s = seed + 100 * k
        out[a] = long(k, s) if k else stall(s)
        out[a + 1] = stall(s + 1)
        out[mid] = long(k, s + 2)
        for j in range(4):
            out[mid + 1 + j] = failing(j, s + 10 + 2 * j)
        out[b - 1] = failing(k % 4, s + 20)
    return out


def build_batch(m, n, filler_nb, seed, planted, int16=False):
    """n short filler reads (make_read_batch) with the planted reads in place"""
    from tombo_b200 import synthetic as syn
    raw, ro, sq, so = syn.make_read_batch(m['kmer_ref'], n, filler_nb, seed, kind=m['kind'],
                                          int16=int16)
    if not planted:
        return raw, ro, sq, so
    idx = np.array(sorted(planted), dtype=np.int64)
    rl, sl = np.diff(ro), np.diff(so)
    keep = np.ones(n, dtype=bool)
    keep[idx] = False
    nrl, nsl = rl.copy(), sl.copy()
    nrl[idx] = [planted[i][0].shape[0] for i in idx]
    nsl[idx] = [planted[i][1].shape[0] for i in idx]
    nro = np.concatenate([[0], np.cumsum(nrl)]).astype(np.int64)
    nso = np.concatenate([[0], np.cumsum(nsl)]).astype(np.int64)
    nraw = np.empty(int(nro[-1]), dtype=raw.dtype)
    nsq = np.empty(int(nso[-1]), dtype=np.uint8)
    nraw[np.repeat(keep, nrl)] = raw[np.repeat(keep, rl)]
    nsq[np.repeat(keep, nsl)] = sq[np.repeat(keep, sl)]
    for i in idx:
        nraw[nro[i]:nro[i + 1]] = planted[i][0]
        nsq[nso[i]:nso[i + 1]] = planted[i][1]
    return nraw, nro, nsq, nso


def filler_lengths(n, seed, lo=60, hi=150, mixed=False):
    rs = np.random.RandomState(seed)
    nb = rs.randint(lo, hi + 1, n)
    if mixed:
        # a few reads several times longer: the longest-first launch order of every chunk
        # then moves reads far from their place in the batch
        sel = rs.rand(n) < 0.02
        nb[sel] = rs.randint(300, 900, int(sel.sum()))
    return nb


# ---------------------------------------------------------------------------- checks
def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8)


def _ranges(off, lengths, sel):
    """sample indices of [off[i], off[i] + lengths[i]) for the reads sel, in that order"""
    st, ln = off[sel], lengths[sel]
    return np.repeat(st - (np.cumsum(ln) - ln), ln) + np.arange(int(ln.sum()))


def read_fields(res, raw_off, order=None, want_norm=False):
    """per-read results of reads `order` (all by default), concatenated in that order; the
    per-base means and the normalised signal only of reads that succeeded (nothing defines
    them for failed reads)"""
    n = res['status'].shape[0]
    order = np.arange(n) if order is None else np.asarray(order)
    so, bo = res['seg_off'], res['base_off']
    ok = order[res['status'][order] == 0]
    out = {k: res[k][order] for k in ('status', 'n_iters', 'flags', 'read_start_rel_to_raw',
                                      'sig_match_score', 'scale_values')}
    out['segs'] = res['segs'][_ranges(so, np.diff(so), order)]
    out['norm_mean'] = res['norm_mean'][_ranges(bo, np.diff(bo), ok)]
    if want_norm:
        out['norm_signal'] = res['norm_signal'][_ranges(raw_off, res['segs'][so[1:] - 1], ok)]
    return out


def assert_same_bits(a, b, what):
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].shape == b[k].shape, (what, k)
        if not np.array_equal(_bits(a[k]), _bits(b[k])):
            bad = np.flatnonzero(np.any((_bits(a[k]) != _bits(b[k])).reshape(a[k].shape[0], -1),
                                        axis=1))
            raise AssertionError('%s: %s differs at %d entries, first %s'
                                 % (what, k, bad.shape[0], bad[:8].tolist()))


def staged(ctx, batch, rp, sp, pol, want_norm):
    raw, ro, sq, so = batch
    ctx.batch_upload(raw, ro, sq, so, rp, pol)
    ctx.batch_compute(rp, sp, pol, want_norm_signal=want_norm)
    return {k: v.copy() for k, v in ctx.batch_download(want_norm_signal=want_norm).items()}


def oracle_indices(cs, planted, n, seed, sample=ORACLE_SAMPLE):
    edges = {int(x) for a in cs[:-1] for x in (a, a + 1)} | {int(b) - 1 for b in cs[1:]}
    fixed = sorted(set(planted) | edges)
    rest = np.setdiff1d(np.arange(n), fixed)
    pick = np.random.RandomState(seed).choice(rest, min(sample, rest.shape[0]), replace=False)
    return sorted(fixed + [int(i) for i in pick])


def check_oracle(orc, res, batch, m, rp, sp, opol, indices):
    """every field _compare in test_pipeline_gpu.py checks, with the read's global index"""
    raw, ro, sq, so = batch
    out = orc.run_batch(raw, ro, sq, so, m['means'], m['sds'], m['k'], rp, sp, opol,
                        indices=indices, want_norm=True)
    bad = orc.compare_batch(res, out)
    assert not bad, bad[:10]
    for i, o in out.items():
        if o['status'] != 0:
            continue
        ns = o['norm_signal']
        if 'norm_signal' in res:
            assert np.array_equal(res['norm_signal'][ro[i]:ro[i] + ns.shape[0]], ns), i
        bo = res['base_off'][i]
        nm = orc.new_means(ns, o['segs'])
        assert np.array_equal(res['norm_mean'][bo:bo + nm.shape[0]], nm), i
    return out


def run_case(ctx, orc, m, batch, cs, planted, rp, sp, seed, want_norm, int16=False):
    """chunked call vs the staged path (every read) and the oracle (planted reads, chunk
    edges and a sample); returns the chunked result and the oracle's"""
    from tombo_b200 import _lib
    raw, ro, sq, so = batch
    ctx.set_model(m['means'], m['sds'], m['k'], m['cpos'])
    pol = _lib.make_policy(m['kind'], subsample_seed=seed)
    got = ctx.resquiggle_batch(raw, ro, sq, so, rp, sp, pol, want_norm_signal=want_norm)
    got = {k: v.copy() for k, v in got.items()}
    ref = staged(ctx, batch, rp, sp, pol, want_norm)
    assert_same_bits(read_fields(got, ro, want_norm=want_norm),
                     read_fields(ref, ro, want_norm=want_norm), 'chunked vs staged')
    idx = oracle_indices(cs, planted, ro.shape[0] - 1, seed)
    out = check_oracle(orc, got, batch, m, rp, sp, orc.policy(m['kind'], subsample_seed=seed),
                       idx)
    return got, out, pol


# ---------------------------------------------------------------------------- chunk cases
CASES = {
    # name: model, chunks, int16, want_norm_signal, filler lengths
    'dna_f64_norm_signal': ('dna', 4, False, True, dict()),
    'dna_int16': ('dna', 3, True, False, dict()),
    'dna_mixed_lengths': ('dna', 3, False, False, dict(mixed=True)),
    'rna': ('rna', 3, False, True, dict(lo=40, hi=70)),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_chunked_batch_matches_staged_and_oracle(ctx, orc, models, RPcls, sm_count, case):
    name, chunks, int16, want_norm, fk = CASES[case]
    m = models[name]
    seed = 900 + sorted(CASES).index(case)
    n = n_reads_for(sm_count, chunks)
    cs = chunk_starts(sm_count, n)
    assert len(cs) - 1 >= chunks >= 3, cs
    planted = planted_reads(m, cs, 10000 * seed, int16)
    batch = build_batch(m, n, filler_lengths(n, seed, **fk), seed, planted, int16)
    rp, sp = _params(RPcls, m['kind'])
    got, out, _ = run_case(ctx, orc, m, batch, cs, planted, rp, sp, seed, want_norm, int16)

    chunk_of = lambda i: int(np.searchsorted(cs, i, side='right')) - 1
    what = {i: p[2] for i, p in planted.items()}
    long_ok = [i for i, w in what.items() if w == 'long' and out[i]['status'] == 0]
    assert {chunk_of(i) for i in long_ok} >= set(range(1, len(cs) - 1)), long_ok
    assert all(out[i]['status'] != 0 for i, w in what.items() if w == 'fail')
    if m['kind'] == 'DNA':
        assert any(out[i]['rescued'] and out[i]['status'] == 0
                   for i, w in what.items() if w == 'stall')
    # the sub-sampling key really is the global index: under a chunk-local index the oracle
    # gives a long read of chunk >= 1 other scale values
    raw, ro, sq, so = batch
    i = max(long_ok)
    rm, rs = orc.levels_from_codes(sq[so[i]:so[i + 1]], m['means'], m['sds'], m['k'])
    local = orc.run_read(np.asarray(raw[ro[i]:ro[i + 1]], dtype=np.float64), rm, rs, rp, sp,
                         orc.policy(m['kind'], subsample_seed=seed),
                         read_index=i - int(cs[chunk_of(i)]))
    assert (local.get('shift'), local.get('scale')) != (out[i]['shift'], out[i]['scale'])


def test_placement_of_short_reads_does_not_matter(ctx, models, RPcls, sm_count):
    """reads of <= 1000 bases are not sub-sampled, so moving them across chunk boundaries
    (and so onto the other lane and into another longest-first order) changes nothing"""
    from tombo_b200 import _lib
    m = models['dna']
    n = n_reads_for(sm_count, 3)
    cs = chunk_starts(sm_count, n)
    assert len(cs) - 1 >= 3
    planted = planted_reads(m, cs, 4242)
    raw, ro, sq, so = build_batch(m, n, filler_lengths(n, 77), 77, planted)
    nb = np.diff(so) - (m['k'] - 1)
    short = np.flatnonzero(nb <= SUBSAMPLE_BASES)
    perm = np.arange(n)
    perm[short] = np.random.RandomState(5).permutation(short)   # long reads keep their index
    moved = short[perm[short] != short]
    chunk_of = np.searchsorted(cs, np.arange(n), side='right') - 1
    assert (chunk_of[moved] != chunk_of[perm[moved]]).sum() > n // 4
    praw = np.concatenate([raw[ro[i]:ro[i + 1]] for i in perm])
    psq = np.concatenate([sq[so[i]:so[i + 1]] for i in perm])
    pro = np.concatenate([[0], np.cumsum(np.diff(ro)[perm])]).astype(np.int64)
    pso = np.concatenate([[0], np.cumsum(np.diff(so)[perm])]).astype(np.int64)
    rp, sp = _params(RPcls, 'DNA')
    pol = _lib.make_policy('DNA', subsample_seed=11)
    ctx.set_model(m['means'], m['sds'], m['k'], m['cpos'])
    a = {k: v.copy() for k, v in
         ctx.resquiggle_batch(raw, ro, sq, so, rp, sp, pol, want_norm_signal=True).items()}
    b = ctx.resquiggle_batch(praw, pro, psq, pso, rp, sp, pol, want_norm_signal=True)
    # read perm[j] of the original batch is read j of the permuted one
    assert_same_bits(read_fields(a, ro, perm, want_norm=True),
                     read_fields(b, pro, want_norm=True), 'permuted batch')
    assert (a['status'] == 0).mean() > 0.9


def test_lanes_across_calls_with_other_models_and_sizes(orc, models, RPcls, sm_count):
    """one Context: chunked DNA, then set_model RNA and a chunked RNA call, then DNA with
    another model and a smaller chunked batch (lane buffers reused at a smaller size), then
    a single-chunk call; each against an oracle sample"""
    from tombo_b200 import _lib
    u = sm_count * 32
    steps = [('dna', 7 * u, 3), ('rna', 6 * u + u // 3, 3), ('dna_b', 6 * u + u // 5, 3),
             ('dna', 1000, 1)]
    c = _lib.Context(0)
    try:
        for j, (name, n, chunks) in enumerate(steps):
            m = models[name]
            cs = chunk_starts(sm_count, n)
            assert len(cs) - 1 == chunks if chunks == 1 else len(cs) - 1 >= chunks, cs
            planted = planted_reads(m, cs, 3000 + 100 * j) if chunks > 1 else {}
            lo, hi = (40, 70) if m['kind'] == 'RNA' else (60, 150)
            batch = build_batch(m, n, filler_lengths(n, 30 + j, lo, hi), 30 + j, planted)
            rp, sp = _params(RPcls, m['kind'])
            c.set_model(m['means'], m['sds'], m['k'], m['cpos'])
            pol = _lib.make_policy(m['kind'], subsample_seed=50 + j)
            res = c.resquiggle_batch(*batch, rp, sp, pol, want_norm_signal=True)
            idx = oracle_indices(cs, planted, n, 60 + j, sample=256)
            check_oracle(orc, res, batch, m, rp, sp, orc.policy(m['kind'], subsample_seed=50 + j),
                         idx)
            assert (res['status'] == 0).mean() > 0.9, (name, n)
    finally:
        c.close()


# ---------------------------------------------------------------------------- defects
def _last_error(c):
    return c.lib.tb2_last_error(c.handle).decode()


def _expect_invalid(c, fn, *args, **kw):
    from tombo_b200 import _lib
    with pytest.raises(_lib.TomboB200Error) as e:
        fn(*args, **kw)
    assert '(%d)' % TB2_ERR_INVALID_ARG in str(e.value), str(e.value)
    return _last_error(c)


def test_resquiggle_batch_leaves_no_resident_batch(models, RPcls, sm_count):
    """batch A staged and computed, then tb2_resquiggle_batch on batch B (one chunk, then
    >= 3 chunks): no resident call may act on A afterwards, nor on B"""
    from tombo_b200 import _lib, synthetic as syn
    m = models['dna']
    K = m['k']
    rp, sp = _params(RPcls, 'DNA')
    pol = _lib.make_policy('DNA')
    # B has as many reads as A and fewer bases, so that a call which (wrongly) acts on B
    # after it stays inside the arrays sized for A
    n_a = 500
    batch_a = syn.make_read_batch(m['kmer_ref'], n_a, 200, 321)
    start = np.arange(n_a, dtype=np.int64) * 1000
    strand = np.zeros(n_a, dtype=np.int8)
    cg = _lib.motif_struct(SimpleNamespace(raw_motif='CG', mod_pos=1))
    c = _lib.Context(0)
    try:
        c.set_model(m['means'], m['sds'], K, m['cpos'])
        c.set_alt_model(np.repeat(m['means'][:, None], K, axis=1) + 0.5, K)

        def resident_calls():
            yield 'download', lambda: c.batch_download()
            yield 'alt_llr', lambda: c.batch_alt_llr(start, 1)
            yield 'alt_llr_motif', lambda: c.batch_alt_llr_motif(start, strand, cg, 1, 1, 0,
                                                                 10 ** 6)
            yield 'de_novo_region', lambda: c.batch_de_novo_region(start, strand, 1, 0, 10 ** 6)

        for n_b in (n_a, n_reads_for(sm_count, 3)):
            chunks = len(chunk_starts(sm_count, n_b)) - 1
            assert chunks == 1 if n_b == n_a else chunks >= 3
            c.batch_upload(*batch_a, rp, pol)
            c.batch_compute(rp, sp, pol)
            for name, call in resident_calls():     # A is resident: every call works
                call()
            batch_b = syn.make_read_batch(m['kmer_ref'], n_b, 80, 654 + n_b)
            res = c.resquiggle_batch(*batch_b, rp, sp, pol)
            assert (res['status'] == 0).mean() > 0.9
            for name, call in resident_calls():
                err = _expect_invalid(c, call)
                assert err == NOT_COMPUTED, (n_b, chunks, name, err)
    finally:
        c.close()


def test_bad_offsets_same_error_in_both_branches(models, RPcls, sm_count):
    """raw_off[0] != 0, seq_off[0] != 0 and decreasing offsets: the same status and error
    text whether the batch goes as one chunk or is pipelined"""
    from tombo_b200 import _lib, synthetic as syn
    m = models['dna']
    rp, sp = _params(RPcls, 'DNA')
    pol = _lib.make_policy('DNA')
    c = _lib.Context(0)
    try:
        c.set_model(m['means'], m['sds'], m['k'], m['cpos'])
        errors = {}
        for n in (500, n_reads_for(sm_count, 3)):
            cs = chunk_starts(sm_count, n)
            raw, ro, sq, so = syn.make_read_batch(m['kmer_ref'], n, 60, 99)
            j = int(cs[1]) + 7 if len(cs) > 2 else n // 2       # inside chunk 1
            bad = {
                # the inputs are padded in front, so a call that accepts them stays in bounds
                'raw_off0': (np.concatenate([np.full(5, 480.0), raw]), ro + 5, sq, so),
                'seq_off0': (raw, ro, np.concatenate([np.zeros(3, np.uint8), sq]), so + 3),
            }
            ro_dec = ro.copy()
            ro_dec[j] = ro[j + 1] + 10
            bad['raw_off_decreasing'] = (raw, ro_dec, sq, so)
            so_dec = so.copy()
            so_dec[j] = so[j + 1] + 4
            bad['seq_off_decreasing'] = (raw, ro, sq, so_dec)
            for what, b in bad.items():
                err = _expect_invalid(c, c.resquiggle_batch, *b, rp, sp, pol,
                                      want_norm_signal=True)
                errors.setdefault(what, []).append(err)
            # a valid call on the same context still works afterwards
            res = c.resquiggle_batch(raw, ro, sq, so, rp, sp, pol)
            assert (res['status'] == 0).mean() > 0.9
        for what, (one, piped) in errors.items():
            assert one == piped and one, (what, one, piped)
            assert 'off' in one, (what, one)
    finally:
        c.close()


# ---------------------------------------------------------------------------- concurrency
def _context_plan(models, RPcls, sm_count, t):
    """thread t's model, parameters, policy and inputs: DNA at bandwidth 200 / 400, RNA, and
    int16 DNA"""
    from tombo_b200 import synthetic as syn
    u = sm_count * 32
    name, aln, int16 = [('dna', DNA_ALN_BW400[:2] + (200,) + DNA_ALN_BW400[3:], False),
                        ('dna_b', DNA_ALN_BW400, False), ('rna', None, False),
                        ('dna', DNA_ALN, True)][t]
    m = models[name]
    rp, sp = _params(RPcls, m['kind'], aln)
    lo, hi = (40, 70) if m['kind'] == 'RNA' else (60, 150)
    n_big = 6 * u + u // 4
    cs = chunk_starts(sm_count, n_big)
    planted = {i: p for i, p in planted_reads(m, cs, 7000 + 100 * t, int16).items()
               if p[2] == 'long'}
    big = build_batch(m, n_big, filler_lengths(n_big, 40 + t, lo, hi), 40 + t, planted, int16)
    small = build_batch(m, 700, filler_lengths(700, 50 + t, lo, hi), 50 + t, {}, int16)
    staged_b = syn.make_read_batch(m['kmer_ref'], 300, 200 if m['kind'] == 'DNA' else 60,
                                   60 + t, kind=m['kind'], int16=int16)
    K = m['k']
    alt = np.repeat(m['means'][:, None], K, axis=1) + np.linspace(-0.6, 0.6, K)[None, :]
    return dict(m=m, rp=rp, sp=sp, seed=70 + t, big=big, big_cs=cs, planted=planted,
                small=small, staged=staged_b, alt=alt)


def _run_plan(c, p, fail_midway=False):
    """the thread's calls in order: chunked, single-chunk, staged + LLR + region counters"""
    from tombo_b200 import _lib
    m = p['m']
    c.set_model(m['means'], m['sds'], m['k'], m['cpos'])
    c.set_alt_model(p['alt'], m['k'])
    pol = _lib.make_policy(m['kind'], subsample_seed=p['seed'])
    out = {}
    out['big'] = {k: v.copy() for k, v in
                  c.resquiggle_batch(*p['big'], p['rp'], p['sp'], pol).items()}
    if fail_midway:
        raw, ro, sq, so = p['small']
        out['error'] = _expect_invalid(c, c.resquiggle_batch, raw, ro + 1, sq, so, p['rp'],
                                       p['sp'], pol)
    out['small'] = {k: v.copy() for k, v in
                    c.resquiggle_batch(*p['small'], p['rp'], p['sp'], pol).items()}
    n = p['staged'][1].shape[0] - 1
    c.batch_upload(*p['staged'], p['rp'], pol)
    c.batch_compute(p['rp'], p['sp'], pol)
    out['staged'] = {k: v.copy() for k, v in c.batch_download().items()}
    start = np.arange(n, dtype=np.int64) * 37
    c.batch_alt_llr(start, 1)
    out['llr'] = [a.copy() for a in c.batch_llr_download()]
    c.region_stats_begin(0, 37 * n + 400)
    c.region_stats_add_batch_llr(2.5, -1.5, 0)
    out['counts'] = c.region_counts_get().copy()
    return out


def _same_run(a, b, what):
    for k in ('big', 'small', 'staged'):
        assert sorted(a[k]) == sorted(b[k])
        for f in a[k]:
            assert np.array_equal(_bits(a[k][f]), _bits(b[k][f])), (what, k, f)
    for x, y in zip(a['llr'], b['llr']):
        assert np.array_equal(_bits(x), _bits(y)), (what, 'llr')
    assert np.array_equal(a['counts'], b['counts']), (what, 'counts')


def test_concurrent_contexts_match_serial_runs_and_oracle(orc, models, RPcls, sm_count):
    """four threads, one Context each (ctypes releases the GIL, so the calls overlap); one
    thread also makes an invalid call while the others run"""
    from tombo_b200 import _lib
    plans = [_context_plan(models, RPcls, sm_count, t) for t in range(4)]
    ctxs = []
    threads = []
    try:
        ctxs = [_lib.Context(0) for _ in plans]
        serial = [_run_plan(c, p) for c, p in zip(ctxs, plans)]
        got, errs = [None] * 4, [None] * 4
        go = threading.Barrier(4)

        def work(t):
            try:
                go.wait()
                got[t] = _run_plan(ctxs[t], plans[t], fail_midway=(t == 3))
            except BaseException as e:           # reported by the main thread
                errs[t] = e
        threads = [threading.Thread(target=work, args=(t,)) for t in range(4)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        threads = []
        for t in range(4):
            if errs[t] is not None:
                raise errs[t]
        for t in range(4):
            _same_run(got[t], serial[t], 'context %d concurrent vs serial' % t)
        assert 'raw_off' in got[3]['error']
        for t in range(3):
            assert _last_error(ctxs[t]) != got[3]['error'], t
        for t, p in enumerate(plans):
            m = p['m']
            opol = orc.policy(m['kind'], subsample_seed=p['seed'])
            idx = oracle_indices(p['big_cs'], p['planted'], p['big'][1].shape[0] - 1, t,
                                 sample=128)
            check_oracle(orc, got[t]['big'], p['big'], m, p['rp'], p['sp'], opol, idx)
            check_oracle(orc, got[t]['small'], p['small'], m, p['rp'], p['sp'], opol,
                         range(0, 700, 11))
            assert (got[t]['big']['status'] == 0).mean() > 0.9, t
    finally:
        for th in threads:
            th.join()
        for c in ctxs:
            c.close()


def test_queue_buckets_match_serial_and_oracle(orc, models, RPcls, sm_count, tmp_path):
    """the bench's --queue pattern: length buckets (one above 6 U reads) pulled by 3 threads,
    one Context each, from a WorkQueue; the sub-sampling key is the index in the bucket"""
    from tombo_b200 import _lib, multi_gpu as mg
    m = models['dna']
    u = sm_count * 32
    n_short, n_mid = 7 * u, 1000
    nb = np.concatenate([filler_lengths(n_short, 81), np.random.RandomState(82).randint(
        300, 900, n_mid), [1100, 1250, 1400]])
    raw, ro, sq, so = build_batch(m, nb.shape[0], nb, 83, {})
    lens = np.diff(ro)
    nbases = np.diff(so) - (m['k'] - 1)
    order = np.lexsort((nbases, lens))[::-1]
    first = int(6 * u + u // 2)
    target = int(lens[order[:first]].sum())
    buckets = mg.length_buckets(lens, nbases, target_samples=target, tail_fraction=0.1,
                                tail_divisor=32)
    assert len(buckets) >= 3 and max(len(b) for b in buckets) > 6 * u, [len(b) for b in buckets]
    packed = []
    for b in buckets:
        bro = np.concatenate([[0], np.cumsum(lens[b])]).astype(np.int64)
        bso = np.concatenate([[0], np.cumsum(so[b + 1] - so[b])]).astype(np.int64)
        braw = np.concatenate([raw[ro[i]:ro[i + 1]] for i in b])
        bsq = np.concatenate([sq[so[i]:so[i + 1]] for i in b])
        packed.append((braw, bro, bsq, bso))
    rp, sp = _params(RPcls, 'DNA', DNA_ALN_BW400)
    pol = _lib.make_policy('DNA', subsample_seed=0)
    ctxs, threads = [], []
    q = mg.WorkQueue('tb2_test_queue', len(buckets), create=True, directory=str(tmp_path))
    try:
        ctxs = [_lib.Context(0) for _ in range(4)]
        for c in ctxs:
            c.set_model(m['means'], m['sds'], m['k'], m['cpos'])
        serial = [{k: v.copy() for k, v in ctxs[3].resquiggle_batch(*pb, rp, sp, pol).items()}
                  for pb in packed]
        results, errs = {}, []

        def worker(c):
            try:
                while True:
                    i = q.next()
                    if i is None:
                        break
                    r = c.resquiggle_batch(*packed[i], rp, sp, pol)
                    results[i] = {k: v.copy() for k, v in r.items()}
            except BaseException as e:
                errs.append(e)
        threads = [threading.Thread(target=worker, args=(c,)) for c in ctxs[:3]]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        threads = []
        if errs:
            raise errs[0]
        assert sorted(results) == list(range(len(buckets)))
        opol = orc.policy('DNA', subsample_seed=0)
        for i, pb in enumerate(packed):
            for k in serial[i]:
                assert np.array_equal(_bits(results[i][k]), _bits(serial[i][k])), (i, k)
            n = pb[1].shape[0] - 1
            long_ = np.flatnonzero(np.diff(pb[3]) - (m['k'] - 1) > SUBSAMPLE_BASES)
            idx = sorted(set(long_.tolist()) | {0, n - 1} |
                         set(np.random.RandomState(i).choice(n, min(n, 96), replace=False).tolist()))
            check_oracle(orc, results[i], pb, m, rp, sp, opol, idx)
    finally:
        for th in threads:
            th.join()
        for c in ctxs:
            c.close()
        q.close(unlink=True)
