"""CPU: resquiggle at caller-chosen parameters.  The C restatement (oracle/oracle.c) against
the reference's own outputs at every parameter point of tests/golden/rsqgl_params.npz, bit
for bit; the Python mirror of load_resquiggle_parameters against the reference's; and the
banded-DP device source (host emulation, tests/emul) against the oracle on both sides of every
register-engine and three-chunk boundary of the adaptive band."""
import os
import sys

import numpy as np
import pytest

import golden_util as gu
import params_cases as pc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emul'))

POINTS = [p['name'] for p in pc.points()]


@pytest.fixture(scope='module')
def golden():
    g = pc.golden()
    assert list(g['p_name']) == POINTS, 'tests/params_cases.py and rsqgl_params.npz disagree'
    return g


@pytest.mark.parametrize('name', POINTS)
def test_oracle_reproduces_reference_at_parameter_point(orc, RPcls, golden, name):
    g = golden
    j = POINTS.index(name)
    pt = pc.point_of(g, j, RPcls)
    kmer_ref, cpos, reads = pc.reads_of_point(g, j)
    pol = orc.policy(pt['kind'], **pt['pol'])
    for k, r in enumerate(reads):
        i = int(g['p_read_off'][j]) + k
        rm, rsd = gu.levels(r.genome_seq, kmer_ref)
        o = orc.run_read(np.asarray(r.raw, dtype=np.float64), rm, rsd, pt['rp'], pt['sp'], pol,
                         read_index=k)
        e = pc.expected(g, i)
        assert o['message'] == e['message'], (k, o['message'], e['message'])
        assert o['calls'] == e['calls'] and o['rescued'] == e['rescued'], k
        if e['message']:
            continue
        assert np.array_equal(o['segs'], e['segs']), k
        assert o['read_start_rel_to_raw'] == e['read_start_rel_to_raw'], k
        for key in ('shift', 'scale', 'lower_lim', 'upper_lim', 'sig_match_score'):
            # None limits (no outlier threshold) are NaN on both sides
            assert o[key] == e[key] or (np.isnan(o[key]) and np.isnan(e[key])), (k, key)
        assert o['n_iters'] == e['n_iters'], k
        assert o['norm_params_changed'] == e['norm_params_changed'], k


def test_parameter_points_reach_their_paths(golden):
    """the facts that make the points meaningful, as the reference recorded them"""
    g = golden
    msgs, sc = g['messages'], g['scalars']

    def rows(name):
        j = POINTS.index(name)
        return slice(int(g['p_read_off'][j]), int(g['p_read_off'][j + 1]))
    # wide bands: every read long enough for the band succeeds
    for W in pc.BOUNDARY_BWS:
        assert (msgs[rows('bw_%d' % W)] == '').all(), W
    assert sc[rows('save_bw_2100'), 7].sum() >= 2, 'no rescue at save bandwidth 2100'
    assert sc[rows('bbt_half_bw_m1'), 7].sum() >= 1
    for name in ('min_obs_6', 'min_obs_10', 'mean_obs_1', 'mean_obs_3'):
        assert (msgs[rows(name)] != '').any(), name
    assert (sc[rows('iters_1'), 8] == 1).all()
    assert (msgs[rows('rna_min_obs_10')] == '').all()


def test_load_resquiggle_parameters_matches_reference(golden):
    """tombo_stats.load_resquiggle_parameters on float tuples as Tombo's CLI parses them
    (bandwidth 333.7 and friends), default tables and segmentation tuples: every field of the
    reference's resquiggleParams, its value and whether it is an int or None"""
    from tombo_b200 import tombo_helper as th, tombo_stats as ts
    g = golden
    assert tuple(g['lp_fields']) == th.resquiggleParams._fields
    row = 0
    for kind, aln, seg in pc.LOAD_PARAM_CASES:
        for save in (False, True):
            p = ts.load_resquiggle_parameters(th.seqSampleType(kind, kind == 'RNA'), aln, seg,
                                              use_save_bandwidth=save)
            for f, v in enumerate(p):
                if g['lp_is_none'][row][f]:
                    assert v is None, (kind, aln, save, p._fields[f])
                    continue
                assert v == g['lp_values'][row][f], (kind, aln, save, p._fields[f], v)
                is_int = isinstance(v, (int, np.integer)) and not isinstance(v, bool)
                assert is_int == bool(g['lp_is_int'][row][f]), (kind, aln, save, p._fields[f])
            row += 1


def _events(orc, read, rm, rs, rp):
    """first-call inputs of the assignment: changepoints and event means (oracle stages)"""
    st, norm, _ = orc.normalize_raw_signal(np.asarray(read.raw, dtype=np.float64), 5.0)
    assert st == 0
    n_ev = max(norm.shape[0] // rp.mean_obs_per_event, int(rm.shape[0] * 1.1))
    st, cp = orc.valid_cpts_w_cap(norm, rp.min_obs_per_base, rp.running_stat_width, n_ev)
    assert st == 0
    cp = np.sort(cp)
    return cp.astype(np.int32), orc.new_means(norm, cp), rm, rs


EMUL_BWS = [W for W in pc.BOUNDARY_BWS if pc.engine_of(W)[0] in ('reg', 'ms')] + [1617]


@pytest.mark.parametrize('W', EMUL_BWS)
def test_emulated_adaptive_band_at_engine_boundary(orc, RPcls, golden, W):
    """the golden reads of point bw_W (events from the oracle's stages) through the host
    emulation of k_align's long-read kernel: status, segs, read start and path equal the
    oracle's, and the reads take the adaptive band the boundary is about"""
    import emul
    g = golden
    j = POINTS.index('bw_%d' % W)
    pt = pc.point_of(g, j, RPcls)
    kmer_ref, cpos, reads = pc.reads_of_point(g, j)
    reads = reads[:2]
    ins = []
    for r in reads:
        rm, rsd = gu.levels(r.genome_seq, kmer_ref)
        ins.append(_events(orc, r, rm, rsd, pt['rp']))
    res = emul.align_batch(ins, pt['rp'], klass=2)
    for k, ((cp, em, rm, rs), o) in enumerate(zip(ins, res)):
        st, segs, rsrtr, dbg, epb = orc.find_adaptive_base_assignment(cp, em, pt['rp'], rm, rs)
        assert dbg[0] == 1, (W, k, 'read takes the static band')
        assert o['status'] == st == 0, (W, k, o['status'], st)
        assert np.array_equal(o['segs'], segs), (W, k)
        assert o['rsrtr'] == rsrtr and o['dbg'][0] == dbg[0], (W, k)


def _device_engine(L, W):
    """the engine the device source picks for an adaptive band of W cells (dp_align.cuh
    tb2_assign_adaptive: register engine, three chunks per lane, lane-chunk engine with
    tb2_wpl_of words, capacity beyond TB2_MAX_WPL), as compiled into the emulation"""
    ch = L.emul_abs_chunk(W)
    if ch:
        return 'reg', ch
    ch = L.emul_abs_ms_chunk(W)
    if ch:
        return 'ms', ch
    wpl = L.emul_wpl_of((W + 31) // 32)
    return ('lane', wpl) if wpl <= 16 else ('capacity', None)


def test_engine_of_matches_the_device_source():
    """engine_of (which places the bandwidth points) equals the choice compiled from
    kernels.h / dp_align.cuh at W - 1, W and W + 1 of every boundary point, and every boundary
    point is the last or first bandwidth of an engine.  A boundary moved in the device source
    fails here even where the moved engine still computes the same alignment."""
    import emul
    L = emul.lib()
    for W in pc.BOUNDARY_BWS + (333, 2100, 2560, 2561, 8193):
        for w in (W - 1, W, W + 1):
            assert pc.engine_of(w) == _device_engine(L, w), (w, pc.engine_of(w), _device_engine(L, w))
    for W in pc.BOUNDARY_BWS:
        assert pc.engine_of(W - 1) != pc.engine_of(W) or pc.engine_of(W + 1) != pc.engine_of(W), W
    sides = [pc.engine_of(W) for W in pc.BOUNDARY_BWS]
    assert sides[:8] == [('reg', 7), ('reg', 10), ('reg', 10), ('reg', 13), ('reg', 13),
                         ('reg', 17), ('reg', 17), ('ms', 13)]
    assert sides[8:12] == [('ms', 13), ('ms', 17), ('ms', 17), ('lane', 4)]
    assert sides[12:] == [('lane', 4), ('lane', 5), ('lane', 8), ('lane', 16), ('lane', 16)]
    assert pc.engine_of(8193) == ('capacity', None)
