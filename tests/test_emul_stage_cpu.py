"""CPU: stage kernels' device source (tombo_b200/csrc/stage_kernels.cuh) on the host emulation
of tests/emul, bit-compared with the oracle: skipped-base raw DP (32-row wavefront for DNA,
serial recurrence for RNA, overflow arena) and Theil-Sen.  An algorithm check of the kernel
source; the GPU parity tests remain the proof for the compiled kernels."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emul'))
from test_emul_dp_cpu import _events  # noqa: E402

ALN = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)


def _dp_segs(orc, kmer_ref, cpos, rp, nb, seed, stall=None, kind='DNA'):
    from tombo_b200 import synthetic as syn
    means, sds = syn.kmer_table(kmer_ref)
    r = syn.make_read(kmer_ref, cpos, nb, seed, stall=stall, kind=kind)
    cp, em, rm, rs = _events(orc, r, means, sds, rp, k=len(kmer_ref[0][0]))
    st, norm, sv = orc.normalize_raw_signal(np.asarray(r.raw, dtype=np.float64), 5.0)
    st, segs, rsrtr, dbg, epb = orc.find_adaptive_base_assignment(cp, em, rp, rm, rs)
    assert st == 0
    return segs, rm, rs, norm[rsrtr:rsrtr + segs[-1]], sv


@pytest.mark.parametrize('nb,seed,stall,raw_min_obs,cap', [
    (444, 9000, None, 1, 1 << 15), (300, 9001, None, 1, 1 << 15),
    (600, 9002, (300, 1500), 1, 1 << 15),          # a stall: 78 skipped bases, big windows
    (800, 9004, (400, 3000), 1, 4096),             # windows beyond the slab: overflow arena
    (444, 9005, None, 2, 1 << 15),                 # raw_min_obs_per_base 2: serial recurrence
    (600, 9006, (300, 1500), 2, 1 << 15),
])
def test_resolve_skipped_bases_matches_oracle(orc, dna_model, RPcls, nb, seed, stall, raw_min_obs, cap):
    import emul
    kmer_ref, cpos = dna_model
    rp = RPcls(ALN, (5, 3, raw_min_obs, 5))
    segs, rm, rs, nsig, sv = _dp_segs(orc, kmer_ref, cpos, rp, nb, seed, stall)
    so, oseg = orc.resolve_skipped_bases_with_raw(segs, rm, rs, nsig, rp)
    se, eseg = emul.resolve(segs, rm, rs, nsig, rp, cap_doubles=cap)
    assert se == so
    if so == 0:
        assert np.array_equal(eseg, oseg)


def test_resolve_failure_statuses_and_capacity(orc, dna_model, RPcls):
    import emul
    kmer_ref, cpos = dna_model
    rp = RPcls(ALN)
    segs, rm, rs, nsig, sv = _dp_segs(orc, kmer_ref, cpos, rp, 800, 9004, (400, 3000))
    # too many deletions in one window (max_raw_cpts): the reference's message, same status
    so, _ = orc.resolve_skipped_bases_with_raw(segs, rm, rs, nsig, rp, max_raw_cpts=20)
    se, _ = emul.resolve(segs, rm, rs, nsig, rp, max_raw_cpts=20)
    assert so == se == 5
    # slab and arena both too small: a loud capacity failure, never a different answer
    se, _ = emul.resolve(segs, rm, rs, nsig, rp, cap_doubles=1024, big_cap_doubles=1024)
    assert se == 202


@pytest.mark.parametrize('nb,seed', [(444, 9100), (61, 9101), (999, 9102), (1400, 9103)])
def test_theil_sen_matches_oracle(orc, dna_model, RPcls, nb, seed):
    """> 1000 bases: keyed sub-sampling, identical on both sides"""
    import emul
    kmer_ref, cpos = dna_model
    rp = RPcls((4.2, 4.2, 400, 1500, 20.0, 40, 750, 2500, 250))
    segs, rm, rs, nsig, sv = _dp_segs(orc, kmer_ref, cpos, rp, nb, seed)
    st, seg2 = orc.resolve_skipped_bases_with_raw(segs, rm, rs, nsig, rp)
    assert st == 0
    bm = orc.new_means(nsig, seg2)
    s1, o1 = orc.theil_sen(sv[0], sv[1], bm, rm, key=77)
    s2, o2 = emul.theil_sen(sv[0], sv[1], bm, rm, key=77)
    assert s1 == s2 and o1 == o2


def test_theil_sen_adversarial_inputs_match_oracle(orc):
    """quantised values (ties, collinear triples), clipped plateaus (equal ev), heavy tails,
    nearly collinear points: whichever path the kernel takes, the doubles are the oracle's"""
    import emul
    rs = np.random.RandomState(1)
    for it in range(36):
        n = int(rs.choice([128, 129, 200, 257, 444, 511, 512, 513, 700, 1000]))
        kind = it % 6
        ev = rs.normal(0, 1.5, n)
        if kind == 0:
            md = ev * 1.03 + 0.05 + rs.normal(0, 0.1, n)
        elif kind == 1:
            md = ev * 0.9 + rs.standard_cauchy(n) * 0.05
        elif kind == 2:
            ev = np.round(ev * 64) / 64
            md = np.round((ev * 1.1 + rs.normal(0, 0.2, n)) * 64) / 64
        elif kind == 3:
            md = rs.normal(0, 1, n)
        elif kind == 4:
            ev = np.clip(ev, -2.0, 2.0)
            md = ev + rs.normal(0, 0.05, n)
        else:
            md = ev * 1.0 + rs.normal(0, 1e-9, n)
        s1, o1 = orc.theil_sen(0.3, 1.7, ev, md, key=9)
        s2, o2 = emul.theil_sen(0.3, 1.7, ev, md, key=9)
        assert s1 == s2, (it, n, kind)
        if s1 == 0:
            assert o1 == o2, (it, n, kind)


def test_block_select_on_integer_and_tied_values():
    """the radix select skips every byte in which no two keys differ: integer-valued signal (the
    int16 DAC dtype: five constant trailing bytes), heavy ties, negative values, all-equal input"""
    import emul
    rng = np.random.RandomState(11)
    cases = [rng.randint(300, 700, size=4150).astype(np.float64),          # DAC-like
             rng.randint(-5, 6, size=777).astype(np.float64),              # sign changes, many ties
             np.full(500, 412.0),                                          # all equal
             np.concatenate([np.full(300, 7.0), rng.randn(5)]),            # one dominant value
             rng.randn(1000),                                              # generic doubles
             (rng.randint(0, 8192, size=2000) * 0.25)]                     # few fractional bits
    for v in cases:
        sv = np.sort(v)
        for k in (0, len(v) // 2 - 1, len(v) // 2, len(v) - 2):
            a, b = emul.select2(v, k)
            assert a == sv[k] and b == sv[k + 1], (len(v), k, a, b, sv[k], sv[k + 1])


def test_theil_sen_equal_levels_stay_on_the_sort_and_sweep_path(orc):
    """integer-valued signal (the int16 DAC dtype) makes base means ratios of small integers:
    equal ev values are the rule, not the exception.  Such pairs have the reference slope 1000.0;
    the sort-and-sweep path must handle them (same doubles as the oracle) instead of abandoning
    to the exhaustive path"""
    import ctypes as C
    import emul
    L = emul.stage_lib()
    rs = np.random.RandomState(5)
    out = (C.c_ulonglong * 8)()
    L.emul_ts_counters(out, 1)
    n_cases = 0
    for it in range(12):
        n = int(rs.choice([200, 444, 445, 700]))
        rm = rs.normal(0, 1.0, n)
        if it % 3 == 0:       # means of 5-12 integer samples, then an affine map: many exact ties
            cnt = rs.randint(5, 13, size=n)
            tot = np.round((rm * 80 + 400) * cnt + rs.normal(0, 12, n) * np.sqrt(cnt))
            bm = ((tot / cnt) - 400.0) / 80.0
            bm[rs.randint(0, n, size=n // 10)] = bm[rs.randint(0, n, size=n // 10)]   # forced ties
        elif it % 3 == 1:     # a 1/16 grid on both axes: ties and identical points
            bm = np.round((rm * 1.05 + rs.normal(0, 0.15, n)) * 16) / 16
            rm = np.round(rm * 16) / 16
        else:                 # a few large tie groups
            bm = rm * 0.97 + rs.normal(0, 0.1, n)
            bm[: n // 4] = np.round(bm[: n // 4] * 4) / 4
        assert len(np.unique(bm)) < n
        s1, o1 = orc.theil_sen(0.1, 1.2, bm, rm, key=3)
        s2, o2 = emul.theil_sen(0.1, 1.2, bm, rm, key=3)
        assert s1 == s2, (it, n)
        if s1 == 0:
            assert o1 == o2, (it, n, o1, o2)
            n_cases += 1
    L.emul_ts_counters(out, 0)
    c = list(out)
    # [5] reads finished by sort-and-sweep, [6] reads that abandoned it
    assert c[5] >= n_cases - 1 and c[6] <= 1, c


def _oracle_segment(orc, raw, rp, n_ev, thresh=5.0, const_scale=None):
    st, norm, sv = orc.normalize_raw_signal(raw, thresh, const_scale=const_scale)
    if st != 0:
        return st, None, None, None, None
    st, cp = orc.valid_cpts_w_cap(norm, rp.min_obs_per_base, rp.running_stat_width, n_ev,
                                  t_test=rp.use_t_test_seg)
    if st != 0:
        return st, norm, sv, None, None
    cp = np.sort(cp)
    return 0, norm, sv, cp, orc.new_means(norm, cp)


@pytest.mark.parametrize('case', ['dna', 'dna_even_n', 'dna_integer_signal', 'dna_few_levels',
                                  'rna_t_test', 'const_scale', 'too_many_events', 'flat_signal'])
def test_segmentation_kernels_match_oracle(orc, dna_model, RPcls, case):
    """k_normalize (radix-select medians, closed-form clipping medians), k_cumsum, k_cpts (greedy
    exclusion as a bit-parallel fixed point, ties, N-best cut) and k_event_means on the host
    emulation: normalised signal, scale values, changepoints and event means equal the oracle's
    normalize_raw_signal / c_valid_cpts_w_cap(_t_test) / c_new_means bit for bit"""
    import emul
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    rna = case == 'rna_t_test'
    rp = RPcls(seg=(12, 6, 2, 15) if rna else (5, 3, 1, 5), rna=rna)
    r = syn.make_read(kmer_ref, cpos, 300, 4242)
    raw = np.asarray(r.raw, dtype=np.float64)
    const_scale = None
    if case == 'dna_even_n':
        raw = raw[:len(raw) - (len(raw) & 1)]
    elif case == 'dna' and not (len(raw) & 1):
        raw = raw[:-1]
    elif case == 'dna_integer_signal':
        raw = np.round(raw)                       # the int16 DAC dtype: ties everywhere
    elif case == 'dna_few_levels':
        raw = np.round(raw / 25.0) * 25.0         # plateaus of equal candidate scores
    elif case == 'const_scale':
        const_scale = 61.5
    elif case == 'flat_signal':
        raw = np.full(1200, 417.0)                # MAD 0: FloatingPointError in the reference
    n_ev = max(raw.shape[0] // rp.mean_obs_per_event, 330)
    if case == 'too_many_events':
        n_ev = raw.shape[0] // 2                  # more events than the exclusion zones allow
    so, onorm, osv, ocp, oem = _oracle_segment(orc, raw, rp, n_ev, const_scale=const_scale)
    se, norm, sv, cp, em = emul.segment(raw, rp, n_ev, const_scale=const_scale)
    assert (se == 0) == (so == 0), (case, se, so)
    if so != 0:
        assert se == so, (case, se, so)
        return
    assert np.array_equal(norm, onorm)
    assert sv[:2] == tuple(osv[:2]) and sv[2:4] == tuple(osv[2:4]), (sv, osv)
    assert np.array_equal(cp, ocp), (len(cp), len(ocp))
    assert np.array_equal(em, oem)


def test_segmentation_kernels_randomized(orc, dna_model, RPcls):
    import emul
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = dna_model
    rs = np.random.RandomState(8)
    n_ok = 0
    for it in range(16):
        rna = it % 4 == 3
        rp = RPcls(seg=(int(rs.choice([8, 12])), int(rs.choice([4, 6])), 2, 15) if rna
                   else (int(rs.choice([3, 5, 7])), int(rs.choice([2, 3, 4])), 1, int(rs.choice([4, 5, 8]))), rna=rna)
        nb = int(rs.choice([40, 100, 270, 444]))
        raw = np.asarray(syn.make_read(kmer_ref, cpos, nb, 5000 + it).raw, dtype=np.float64)
        if it % 3 == 1:
            raw = np.round(raw)
        n_ev = max(raw.shape[0] // rp.mean_obs_per_event, int(nb * 1.1))
        so, onorm, osv, ocp, oem = _oracle_segment(orc, raw, rp, n_ev)
        se, norm, sv, cp, em = emul.segment(raw, rp, n_ev)
        assert (se == 0) == (so == 0), (it, se, so)
        if so == 0:
            assert np.array_equal(norm, onorm) and np.array_equal(cp, ocp) and np.array_equal(em, oem), it
            assert sv[:4] == tuple(osv[:4])
            n_ok += 1
    assert n_ok >= 12


def test_stall_detection_kernel_matches_oracle(orc):
    """k_stalls (mean-window stall detection of direct-RNA reads) on the host emulation:
    the intervals of identify_stalls, none / one / several stalls, merged neighbours, a read
    shorter than one window, and an interval buffer that is too small (loud capacity status)"""
    import emul
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('RNA', 0)
    rs = np.random.RandomState(4)
    seen = set()
    for seed, stall in [(1, None), (2, (100, 1500)), (3, (50, 700)), (4, (200, 3000)), (5, (20, 260))]:
        raw = np.asarray(syn.make_read(kmer_ref, cpos, 270, seed, stall=stall, kind='RNA').raw,
                         dtype=np.float64)
        if seed == 4:          # a second and a third flat stretch, two of them close together
            raw = np.concatenate([raw[:1500], np.full(600, raw[1500]) + rs.normal(0, 2, 600),
                                  raw[1500:1700], np.full(500, raw[1700]) + rs.normal(0, 2, 500), raw[1700:]])
        o = orc.identify_stalls(raw)
        st, e, k = emul.stalls(raw)
        assert st == 0 and k == len(o) and np.array_equal(o, e), (seed, o.tolist(), e.tolist())
        seen.add(len(o))
    assert 0 in seen and max(seen) >= 2
    st, e, k = emul.stalls(np.full(100, 400.0))          # shorter than the 350-sample window
    assert st == 0 and k == 0
    # capacity: more intervals than the buffer holds is a loud failure, never a truncation
    many = np.concatenate([np.asarray(syn.make_read(kmer_ref, cpos, 150, 30 + q, stall=(60, 900), kind='RNA').raw,
                                      dtype=np.float64) for q in range(4)])
    o = orc.identify_stalls(many)
    st, e, k = emul.stalls(many, stall_cap=2)
    assert len(o) > 2 and st == 202
    st, e, k = emul.stalls(many, stall_cap=64)
    assert st == 0 and np.array_equal(o, e)


def test_finalize_kernel_matches_oracle(orc, dna_model, RPcls):
    """k_finalize: (norm - shift_corr) / scale_corr, per-base means in c_new_means' order and the
    numpy pairwise-sum mean of |mean - level| / sd"""
    import emul
    kmer_ref, cpos = dna_model
    rp = RPcls(ALN)
    for nb, seed in [(444, 9100), (129, 9101), (1000, 9102)]:
        segs, rm, rs, nsig, sv = _dp_segs(orc, kmer_ref, cpos, rp, nb, seed)
        so, segs = orc.resolve_skipped_bases_with_raw(segs, rm, rs, nsig, rp)    # no empty bases
        assert so == 0
        shc, scc = 0.0123, 1.0456
        for rescale in (True, False):
            want_sig = (nsig - shc) / scc if rescale else nsig
            want_bm = orc.new_means(want_sig, segs)
            want_score = orc.get_read_seg_score(want_bm, rm, rs)
            bm, sig, score = emul.finalize(nsig, segs, rm, rs, shc, scc, rescale)
            assert np.array_equal(bm, want_bm) and np.array_equal(sig[:segs[-1]], want_sig[:segs[-1]])
            assert score == want_score
