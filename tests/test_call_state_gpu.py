"""What a call leaves on its context: the error text is the last call's own, and a producer of
resident results that fails leaves none for the calls that consume them (DESIGN.md, section 3)."""
from types import SimpleNamespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALN = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
N_READS = 16
NOT_UPLOADED = 'tb2_batch_upload has not been called'
NOT_COMPUTED = 'tb2_batch_compute has not been called'


@pytest.fixture
def fresh():
    from tombo_b200 import _lib
    c = _lib.Context(0)
    yield c
    c.close()


def _last_error(c):
    return c.lib.tb2_last_error(c.handle).decode()


def _set_models(c):
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    kmeans, ksds = syn.kmer_table(kmer_ref)
    K = len(kmer_ref[0][0])
    c.set_model(kmeans, ksds, K, cpos)
    c.set_alt_model(np.repeat(kmeans[:, None], K, axis=1) + 0.5, K)
    return kmer_ref


def _resident_batch(c, RPcls):
    """N_READS DNA reads resquiggled and resident on c -> (seq, seq_off, read starts, the
    batch's download)"""
    from tombo_b200 import _lib, synthetic as syn
    kmer_ref = _set_models(c)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, N_READS, 200, 4242)
    rp, sp = RPcls(ALN), RPcls(ALN, save=True)
    pol = _lib.make_policy('DNA')
    c.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    c.batch_compute(rp, sp, pol)
    res = c.batch_download()
    assert (res['status'] == 0).mean() > 0.9
    return seq, seq_off, np.arange(N_READS, dtype=np.int64) * 1000, res


def test_error_text_belongs_to_the_last_call(fresh, RPcls):
    """a message is reported with the call that set it, and never with a later one"""
    from tombo_b200 import _lib
    _set_models(fresh)
    pol = _lib.make_policy('DNA')
    with pytest.raises(_lib.TomboB200Error) as compute_error:
        fresh.batch_compute(RPcls(ALN), RPcls(ALN, save=True), pol)
    assert _last_error(fresh) == NOT_UPLOADED
    fresh.new_means(np.arange(10.0), np.array([0, 4, 10]))
    assert _last_error(fresh) == ''
    with pytest.raises(_lib.TomboB200Error) as e:
        fresh.most_signif_begin(True, 0)           # refused without a message of its own
    assert '(201)' in str(e.value)
    assert NOT_UPLOADED not in str(e.value), str(e.value)
    # the exception carries the message of the call that set it, whatever the status
    assert NOT_UPLOADED in str(compute_error.value), str(compute_error.value)


def test_failed_batch_call_leaves_no_batch(fresh, RPcls):
    """a rejected tb2_batch_compute or tb2_batch_upload leaves no resident batch for the calls
    after it"""
    from tombo_b200 import _lib
    rp, sp, pol = RPcls(ALN), RPcls(ALN, save=True), _lib.make_policy('DNA')
    _resident_batch(fresh, RPcls)
    with pytest.raises(_lib.TomboB200Error, match=r'\(201\)'):
        fresh.batch_compute(rp, None, pol)            # rescue without save parameters
    with pytest.raises(_lib.TomboB200Error, match=NOT_COMPUTED):
        fresh.batch_download()
    _resident_batch(fresh, RPcls)
    empty = np.zeros(1, np.int64)
    with pytest.raises(_lib.TomboB200Error, match=r'\(201\)'):
        fresh.batch_upload(np.zeros(0), empty, np.zeros(0, np.uint8), empty, rp, pol)   # no reads
    with pytest.raises(_lib.TomboB200Error, match=NOT_COMPUTED):
        fresh.batch_download()
    with pytest.raises(_lib.TomboB200Error, match=NOT_UPLOADED):
        fresh.batch_compute(rp, sp, pol)


def test_failed_llr_call_leaves_no_llrs(fresh, RPcls):
    """after a rejected tb2_batch_alt_llr_motif, neither the download nor the region counters
    see the LLRs of the successful call before it"""
    from tombo_b200 import _lib
    _, _, start, _ = _resident_batch(fresh, RPcls)
    assert fresh.batch_alt_llr(start, 1) > 0
    cg = _lib.motif_struct(SimpleNamespace(raw_motif='CG', mod_pos=1))
    with pytest.raises(_lib.TomboB200Error, match=r'\(201\)'):
        fresh.batch_alt_llr_motif(start, np.full(N_READS, 2, np.int8), cg, 1, 1, 0, 10 ** 6)
    with pytest.raises(_lib.TomboB200Error, match='no successful tb2_batch_alt_llr'):
        fresh.batch_llr_download()
    fresh.region_stats_begin(0, 1000 * N_READS + 1000)
    with pytest.raises(_lib.TomboB200Error, match='no successful tb2_batch_alt_llr'):
        fresh.region_stats_add_batch_llr(2.5, -1.5, 0)
    assert not fresh.region_counts_get().any()


@pytest.mark.parametrize('producer', ['de_novo', 'batch_de_novo', 'sample_compare'])
def test_failed_region_call_leaves_no_tests(fresh, RPcls, producer):
    """after a region test rejected for its strands, tb2_region_stats_add_tests refuses
    instead of adding the statistics of the successful call before it"""
    from tombo_b200 import _lib
    seq, seq_off, start, res = _resident_batch(fresh, RPcls)
    fm, reg = 2, (0, 1000 * N_READS + 1000)
    ctrl = np.zeros(reg[1] - reg[0] + 2 * fm), np.ones(reg[1] - reg[0] + 2 * fm)

    def call(strand):
        if producer == 'de_novo':
            return fresh.de_novo_region_stats(res['norm_mean'], res['base_off'], seq, seq_off,
                                              start, strand, fm, *reg)
        if producer == 'batch_de_novo':
            return fresh.batch_de_novo_region(start, strand, fm, *reg)
        return fresh.sample_compare_region_stats(res['norm_mean'], res['base_off'], start,
                                                 strand, *ctrl, fm, *reg)
    strand = np.zeros(N_READS, np.int8)
    assert call(strand)[2][-1] > 0
    strand[3] = 2
    with pytest.raises(_lib.TomboB200Error, match=r'\(201\)'):
        call(strand)
    assert _last_error(fresh) == 'strand outside {-1, 0, 1}'
    fresh.region_stats_begin(*reg)
    with pytest.raises(_lib.TomboB200Error, match='no de novo or sample-compare region call'):
        fresh.region_stats_add_tests(0.05)
    assert not fresh.region_counts_get().any()
