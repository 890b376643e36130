"""CPU: the banded-DP device source (tombo_b200/csrc/dp_*.cuh, the files nvcc compiles for
sm_90a) executed on the host emulation of tests/emul and compared bit for bit with the
oracle's find_adaptive_base_assignment -- static band, start search, masked start,
adaptive rows, traceback.  An algorithm check of the kernel source; the GPU parity tests
remain the proof for the compiled kernel."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emul'))


def _events(orc, read, means, sds, rp, k=6):
    """first-call inputs of the assignment: changepoints + event means (oracle stages)"""
    from tombo_b200 import synthetic as syn
    codes = syn.seq_to_codes(read.genome_seq).astype(np.int64)
    nb = codes.shape[0] - k + 1
    kidx = np.zeros(nb, dtype=np.int64)
    for j in range(k):
        kidx = kidx * 4 + codes[j:j + nb]
    rm, rs = means[kidx], sds[kidx]
    st, norm, sv = orc.normalize_raw_signal(np.asarray(read.raw, dtype=np.float64), 5.0)
    assert st == 0
    n_ev = max(norm.shape[0] // rp.mean_obs_per_event, int(nb * 1.1))
    st, cp = orc.valid_cpts_w_cap(norm, rp.min_obs_per_base, rp.running_stat_width, n_ev)
    assert st == 0
    cp = np.sort(cp)
    em = orc.new_means(norm, cp)
    return cp.astype(np.int32), em, rm, rs


CASES = [
    # name, aln params, n_bases list, klass
    ('static4k', (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250), [444, 444, 300, 61], 1),
    ('adapt4k', (4.2, 4.2, 200, 1500, 20.0, 40, 300, 2500, 100), [444, 444, 380], 2),
    ('adapt_bw400', (4.2, 4.2, 400, 1500, 20.0, 40, 750, 2500, 250), [900, 700], 2),
    ('adapt_bw120_narrow', (4.2, 4.2, 120, 1500, 20.0, 40, 300, 2500, 100), [500, 444], 0),
    # the register engine's chunk widths 7 / 10 / 13 / 17 at their widest bands, the
    # DNA / RNA default bandwidths, and a band too wide for it (lane-chunk engine)
    ('abs_ch7_w218', (4.2, 4.2, 218, 1500, 20.0, 40, 300, 2500, 100), [500, 700], 2),
    ('abs_ch10_w300', (4.2, 4.2, 300, 1500, 20.0, 40, 750, 2500, 250), [1300, 900], 2),
    ('abs_ch10_w311', (4.2, 4.2, 311, 1500, 20.0, 40, 750, 2500, 250), [1100], 2),
    ('abs_ch13_w404', (4.2, 4.2, 404, 1500, 20.0, 40, 750, 2500, 250), [1200], 2),
    ('abs_ch17_w500', (4.2, 4.2, 500, 1500, 20.0, 40, 750, 2500, 250), [1300], 2),
    ('abs_ch17_w528', (4.2, 4.2, 528, 1500, 20.0, 40, 750, 2500, 250), [1300], 2),
    # wide bands: three chunks per lane (bandwidth 1200 of BASELINE configs[4], the save
    # bandwidth 1500, the widest bands of both chunk widths), and the lane-chunk engine beyond
    ('abs_ms13_w600', (4.2, 4.2, 600, 1500, 20.0, 40, 750, 2500, 250), [1300], 2),
    ('abs_ms13_w1200', (4.2, 4.2, 1200, 1500, 20.0, 40, 750, 2500, 250), [1500], 2),
    ('abs_ms13_w1236', (4.2, 4.2, 1236, 1500, 20.0, 40, 750, 2500, 250), [1600], 2),
    ('abs_ms17_w1500', (4.2, 4.2, 1500, 1500, 20.0, 40, 750, 2500, 250), [2000], 2),
    ('abs_ms17_w1616', (4.2, 4.2, 1616, 1500, 20.0, 40, 750, 2500, 250), [2200], 2),
    ('chunk_engine_w1700', (4.2, 4.2, 1700, 1500, 20.0, 40, 750, 2500, 250), [2200], 2),
    # a start window (150 events) narrower than the start bases (250): the start score's scratch
    # no longer fits the row buffer and moves to the (free) move scratch
    ('start_window_lt_start_bases', (4.2, 4.2, 200, 1500, 20.0, 40, 150, 2500, 250), [700, 300], 2),
]


def test_band_edge_failures_match_oracle(orc, dna_model, RPcls):
    """reads with a planted stall leave a 60-cell adaptive band: the traceback reports
    'extends beyond bandwidth' (status 2) exactly where the oracle does"""
    import emul
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    rp = RPcls((4.2, 4.2, 60, 1500, 20.0, 40, 200, 2500, 80))
    reads = [syn.make_read(kmer_ref, cpos, nb, 500 + i, stall=(250 + i, 200 + 150 * i))
             for i, nb in enumerate([600, 600, 600, 600, 500, 700])]
    ins = [_events(orc, r, means, sds, rp) for r in reads]
    res = emul.align_batch(ins, rp, klass=2)
    sts = []
    for (cp, em, rm, rs), o in zip(ins, res):
        st, segs, rsrtr, dbg, epb = orc.find_adaptive_base_assignment(cp, em, rp, rm, rs)
        assert o['status'] == st
        if st == 0:
            assert np.array_equal(o['segs'], segs) and o['rsrtr'] == rsrtr
        sts.append(st)
    assert 2 in sts and 0 in sts


@pytest.mark.parametrize('name,aln,nbs,klass', CASES)
def test_device_source_matches_oracle(orc, dna_model, RPcls, name, aln, nbs, klass):
    import emul
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    rp = RPcls(aln)
    reads = syn.make_reads(kmer_ref, cpos, len(nbs), nbs, seed0=4100)
    ins = [_events(orc, r, means, sds, rp) for r in reads]
    res = emul.align_batch(ins, rp, klass=klass)
    for (cp, em, rm, rs), o in zip(ins, res):
        st, segs, rsrtr, dbg, epb = orc.find_adaptive_base_assignment(cp, em, rp, rm, rs)
        assert o['status'] == st
        if st == 0:
            assert np.array_equal(o['segs'], segs)
            assert o['rsrtr'] == rsrtr
            assert o['dbg'][0] == dbg[0]


def test_randomized_parameters_match_oracle(orc, dna_model, RPcls):
    """a seeded sweep over odd parameter combinations (band widths at and around the chunk-width
    limits, start windows narrower than the start bases, tiny reads): statuses and assignments
    equal the oracle's.  The sweep this is cut from found the start-score scratch limit."""
    import emul
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    means, sds = syn.kmer_table(kmer_ref)
    rs = np.random.RandomState(77)
    n_ok = n_fail = 0
    for it in range(14):
        bw = int(rs.choice([33, 64, 97, 128, 218, 219, 312, 404, 405, 529, 700]))
        sbw = int(rs.choice([64, 150, 300, 750, 1000]))
        snb = int(rs.choice([33, 64, 100, 250]))
        aln = (float(rs.choice([4.2, 3.0])), float(rs.choice([4.2, 2.0, 6.0])), bw, 1500,
               float(rs.choice([20.0, 5.0])), int(rs.choice([5, 40])), sbw, int(rs.choice([1500, 2500])), snb)
        rp = RPcls(aln)
        nbs = [int(x) for x in rs.randint(20, 1100, size=2)]
        reads = syn.make_reads(kmer_ref, cpos, len(nbs), nbs, seed0=9000 + it * 10)
        try:
            ins = [_events(orc, r, means, sds, rp) for r in reads]
        except AssertionError:          # the oracle's own stages reject the read (too short)
            continue
        res = emul.align_batch(ins, rp, klass=0)
        for (cp, em, rm, rs_), o in zip(ins, res):
            st, segs, rsrtr, dbg, epb = orc.find_adaptive_base_assignment(cp, em, rp, rm, rs_)
            assert o['status'] == st, (it, aln, len(rm), o['status'], st)
            if st == 0:
                assert np.array_equal(o['segs'], segs) and o['rsrtr'] == rsrtr, (it, aln, len(rm))
                n_ok += 1
            else:
                n_fail += 1
    assert n_ok >= 15
