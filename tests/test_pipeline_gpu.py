"""GPU parity of the batched hot path (tb2_resquiggle_batch) against the C oracle:
bit-exact segs / read_start_rel_to_raw / scale values / score, per-read status."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALN = {
    'static4k': (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250),
    'adapt4k': (4.2, 4.2, 200, 1500, 20.0, 40, 300, 2500, 100),
    'adapt_bw400': (4.2, 4.2, 400, 1500, 20.0, 40, 750, 2500, 250),
}


def _flatten(reads):
    from tombo_b200 import synthetic as syn
    raw = np.concatenate([r.raw for r in reads])
    raw_off = np.concatenate([[0], np.cumsum([r.raw.shape[0] for r in reads])]).astype(np.int64)
    codes = [syn.seq_to_codes(r.genome_seq) for r in reads]
    seq = np.concatenate(codes)
    seq_off = np.concatenate([[0], np.cumsum([c.shape[0] for c in codes])]).astype(np.int64)
    return raw, raw_off, seq, seq_off


def _levels(genome_seq, means, sds, k):
    from tombo_b200 import synthetic as syn
    codes = syn.seq_to_codes(genome_seq).astype(np.int64)
    nb = codes.shape[0] - k + 1
    kidx = np.zeros(nb, dtype=np.int64)
    for j in range(k):
        kidx = kidx * 4 + codes[j:j + nb]
    return means[kidx], sds[kidx]


def _compare(ctx, orc, reads, means, sds, k, cpos, rp, sp, kind='DNA', want_norm=True,
             seed=0):
    from tombo_b200 import _lib
    ctx.set_model(means, sds, k, cpos)
    raw, raw_off, seq, seq_off = _flatten(reads)
    pol = _lib.make_policy(kind, subsample_seed=seed)
    res = ctx.resquiggle_batch(raw, raw_off, seq, seq_off, rp, sp, pol,
                               want_norm_signal=want_norm)
    opol = orc.policy(kind, subsample_seed=seed)
    n_fail = 0
    for i, r in enumerate(reads):
        rm, rsd = _levels(r.genome_seq, means, sds, k)
        o = orc.run_read(np.asarray(r.raw, dtype=np.float64), rm, rsd, rp, sp, opol,
                         read_index=i, want_norm=True)
        assert res['status'][i] == o['status'], (i, res['status'][i], o['status'], o['message'])
        if o['status'] != 0:
            n_fail += 1
            continue
        a, b = res['seg_off'][i], res['seg_off'][i + 1]
        assert np.array_equal(res['segs'][a:b], o['segs']), i
        assert res['read_start_rel_to_raw'][i] == o['read_start_rel_to_raw']
        assert res['scale_values'][i, 0] == o['shift']
        assert res['scale_values'][i, 1] == o['scale']
        assert res['scale_values'][i, 2] == o['lower_lim']
        assert res['scale_values'][i, 3] == o['upper_lim']
        assert res['sig_match_score'][i] == o['sig_match_score']
        assert res['n_iters'][i] == o['n_iters']
        assert bool(res['flags'][i] & 2) == o['rescued']
        assert bool(res['flags'][i] & 1) == o['norm_params_changed']
        ns = o['norm_signal']
        ro = raw_off[i]
        assert np.array_equal(res['norm_signal'][ro:ro + ns.shape[0]], ns)
        # norm_mean == per-base means of the final signal
        bo = res['base_off'][i]
        nm = orc.new_means(ns, o['segs'])
        assert np.array_equal(res['norm_mean'][bo:bo + nm.shape[0]], nm)
    return res, n_fail


@pytest.mark.parametrize('name,nbases,nreads', [('static4k', 444, 24), ('adapt4k', 444, 24),
                                                ('adapt_bw400', 2222, 4)])
def test_batch_matches_oracle(ctx, orc, dna_model, RPcls, name, nbases, nreads):
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    rp, sp = RPcls(ALN[name]), RPcls(ALN[name], save=True)
    reads = syn.make_reads(kmer_ref, cpos, nreads, nbases, seed0=5000)
    _compare(ctx, orc, reads, means, sds, 6, cpos, rp, sp)


def test_batch_mixed_lengths_and_int16(ctx, orc, dna_model, RPcls):
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    rp, sp = RPcls(ALN['adapt_bw400']), RPcls(ALN['adapt_bw400'], save=True)
    rs = np.random.RandomState(5)
    nbs = rs.randint(222, 2222, 10)
    reads = syn.make_reads(kmer_ref, cpos, 10, nbs, seed0=6000, int16=True)
    _compare(ctx, orc, reads, means, sds, 6, cpos, rp, sp)


def test_batch_rescue_and_failures(ctx, orc, dna_model, RPcls):
    """reads with a planted stall leave the narrow adaptive band and are rescued
    with the save bandwidth; hopeless reads fail with the reference's message."""
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    aln = (4.2, 4.2, 120, 1500, 20.0, 40, 300, 2500, 100)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    reads = []
    for i in range(6):
        reads.append(syn.make_read(kmer_ref, cpos, 600, 7000 + i, stall=(300 + i, 1500)))
    reads.append(syn.make_read(kmer_ref, cpos, 600, 7100))
    # sequence unrelated to the signal
    r = syn.make_read(kmer_ref, cpos, 600, 7200)
    r2 = syn.make_read(kmer_ref, cpos, 600, 7201)
    reads.append(r._replace(genome_seq=r2.genome_seq))
    # far too much signal for the sequence
    r3 = syn.make_read(kmer_ref, cpos, 2000, 7300)
    reads.append(r3._replace(genome_seq=r3.genome_seq[:12]))
    # constant signal: MAD scale of zero (FloatingPointError in the reference)
    r4 = syn.make_read(kmer_ref, cpos, 300, 7400)
    reads.append(r4._replace(raw=np.full(r4.raw.shape[0], 480.0)))
    res, n_fail = _compare(ctx, orc, reads, means, sds, 6, cpos, rp, sp)
    assert (res['flags'] & 2).any(), 'no read exercised the rescue path'
    assert n_fail >= 1


def test_batch_long_reads_subsample(ctx, orc, dna_model, RPcls):
    """> 1000 bases: keyed Theil-Sen sub-sampling identical on both sides"""
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    aln = (4.2, 4.2, 400, 1500, 20.0, 40, 750, 2500, 250)
    rp, sp = RPcls(aln), RPcls(aln, save=True)
    reads = syn.make_reads(kmer_ref, cpos, 3, 1400, seed0=8000)
    _compare(ctx, orc, reads, means, sds, 6, cpos, rp, sp, seed=99)


def test_large_batch_pipelined_chunks_match_single_chunk(ctx, dna_model, RPcls):
    """tb2_resquiggle_batch splits big batches into chunks over two lanes (H2D of the
    next chunk overlaps compute); results must equal the unchunked staged path"""
    from tombo_b200 import _lib, synthetic as syn
    import bench
    import torch
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    ctx.set_model(means, sds, 6, cpos)
    u = torch.cuda.get_device_properties(0).multi_processor_count * 32
    n = 8 * u + 1234                      # > 6 U reads (U = SMs x 32): chunks of 2 U, 4 U, rest
    nb = np.full(n, 60)
    # a few long reads (> 1000 bases) in every chunk after the first, so that the keyed
    # Theil-Sen sub-sampling is exercised with a chunk's non-zero global read index
    long_at = [2 * u, 2 * u + 5, 4 * u, 6 * u, 6 * u + 777, n - 1]
    nb[long_at] = [1100, 1400, 1250, 1333, 1200, 1150]
    raw, raw_off, codes, seq_off = syn.make_read_batch(kmer_ref, n, nb, 77)
    rp, sp = RPcls(bench.ALN_DNA), RPcls(bench.ALN_DNA, save=True)
    pol = _lib.make_policy('DNA', subsample_seed=5)
    a = ctx.resquiggle_batch(raw, raw_off, codes, seq_off, rp, sp, pol)
    a = {k: v.copy() for k, v in a.items()}
    ctx.batch_upload(raw, raw_off, codes, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    b = ctx.batch_download()
    for k in ('segs', 'read_start_rel_to_raw', 'status', 'n_iters', 'flags'):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a['scale_values'][:, :4], b['scale_values'][:, :4], equal_nan=True)
    assert np.array_equal(a['sig_match_score'], b['sig_match_score'], equal_nan=True)
    assert np.array_equal(a['norm_mean'], b['norm_mean'], equal_nan=True)
    assert (a['status'] == 0).mean() > 0.9
    assert (a['status'][long_at] == 0).all()
