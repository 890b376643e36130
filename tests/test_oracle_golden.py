"""CPU: pin the C restatement (oracle/oracle.c) against the golden vectors produced
by the unmodified reference (tests/golden/make_golden.py)."""
import numpy as np
import pytest

import golden_util as gu


@pytest.mark.parametrize('name', gu.READ_CONFIGS)
def test_oracle_reproduces_reference_reads(orc, RPcls, name):
    g = gu.load(name)
    kind, kmer_ref, cpos, reads = gu.reads_of(g)
    rp, sp = gu.params_of(g, RPcls)
    pol = orc.policy(kind, const_scale=gu.const_scale_of(g))
    for i, r in enumerate(reads):
        rm, rsd = gu.levels(r.genome_seq, kmer_ref)
        o = orc.run_read(np.asarray(r.raw, dtype=np.float64), rm, rsd, rp, sp, pol, read_index=i)
        e = gu.expected(g, i)
        assert o['message'] == e['message']
        if e['message']:
            continue
        assert np.array_equal(o['segs'], e['segs'])
        assert o['read_start_rel_to_raw'] == e['read_start_rel_to_raw']
        for k in ('shift', 'scale', 'lower_lim', 'upper_lim', 'sig_match_score'):
            assert o[k] == e[k], k
        assert o['calls'] == e['calls'] and o['rescued'] == e['rescued']
        assert o['n_iters'] == e['n_iters']
        assert o['norm_params_changed'] == e['norm_params_changed']


def test_oracle_kernel_known_answers(orc):
    k = gu.load('kernel_kats')
    fwd, tb = orc.banded_forward_pass(k['bfp_z'], k['bfp_es'], 4.2, 4.2)
    assert np.array_equal(fwd, k['bfp_fwd'])
    assert np.array_equal(tb[1:], k['bfp_tb'])
    st, tbk = orc.banded_traceback(tb, k['bfp_es'], int(np.argmax(fwd[-1])), -1)
    assert st == 0 and np.array_equal(tbk, k['bfp_traceback'])
    f, t, e = k['ad_seed_fwd'].copy(), k['ad_seed_tb'].copy(), k['ad_seed_es'].copy()
    st, _ = orc.adaptive_banded_forward_pass(f, t, e, k['ad_em'], k['ad_rm'], k['ad_rs'], 5.0,
                                             4.2, 4.2, int(k['ad_ssp']), -15.0, True, 20.0)
    assert (st == 0) == bool(k['ad_ok'])
    if st == 0:
        ssp = int(k['ad_ssp'])
        assert np.array_equal(e, k['ad_es'])
        assert np.array_equal(f[ssp + 1:], k['ad_fwd'][ssp + 1:])
        assert np.array_equal(t[ssp + 1:], k['ad_tb'][ssp + 1:])
    assert np.array_equal(orc.new_means(k['h_sig'], k['h_segs']), k['h_means'])
    m, s = orc.new_mean_stds(k['h_sig'], k['h_segs'])
    assert np.array_equal(m, k['h_mean_stds_m']) and np.array_equal(s, k['h_mean_stds_s'])
    st, cp = orc.valid_cpts_w_cap(k['h_sig'], 3, 5, 500)
    assert st == 0 and np.array_equal(cp, k['h_cpts'])
    st, cp = orc.valid_cpts_w_cap(k['h_sig'], 6, 12, 150, t_test=True)
    assert st == 0 and np.array_equal(cp, k['h_cpts_t'])
    assert np.array_equal(orc.compute_slopes(k['h_ev'], k['h_md']), k['h_slopes'])
    assert orc.calc_scaled_llh_ratio_const_var(k['l_m'], k['l_r'], k['l_a'], 0.04, 4.0, 1.0,
                                               0.2) == float(k['l_scaled'])
    assert orc.calc_llh_ratio_const_var(k['l_m'], k['l_r'], k['l_a'], 0.04) == float(k['l_const'])
    assert orc.calc_llh_ratio(k['l_m'], k['l_r'], k['l_a'], np.full(6, 0.04),
                              np.full(6, 0.05)) == float(k['l_full'])


def test_numpy_restatements(orc):
    rs = np.random.RandomState(1)
    for n in [1, 2, 5, 7, 8, 9, 15, 16, 17, 100, 127, 128, 129, 130, 200, 255, 256, 257, 443, 444,
              1000, 1001, 5000]:
        a = rs.normal(0, 1, n) * rs.uniform(0.1, 100)
        assert np.mean(a) == orc.np_mean(a)
        assert np.median(a) == orc.median(a)
    for (a, b, n) in [(0, 111, 222), (-90, -90 + 151 * 2.3, 151), (101, 1173, 50), (0, 37, 8),
                      (0, 5, 1), (0, 5, 2)]:
        assert np.array_equal(np.linspace(a, b, n), orc.linspace(a, b, n))


def test_subsampler_matches_python_definition(orc):
    import ctypes as C
    from tombo_b200 import synthetic as syn
    lib = orc.lib()
    for n, key in [(1001, 5), (1300, 77), (4000, 123456), (65537, 9)]:
        idx = syn.theil_sen_subsample(n, 1000, key)
        assert len(set(idx.tolist())) == 1000 and idx.min() >= 0 and idx.max() < n
        for i in (0, 1, 500, 999):
            assert lib.orc_perm_index(C.c_int64(i), C.c_int64(n), C.c_uint32(key)) == idx[i]
    assert lib.orc_subsample_key(C.c_uint32(3), C.c_uint32(7), C.c_uint32(2)) == \
        syn.subsample_key(3, 7, 2)


def test_oracle_normalize_with_scale_values_matches_reference():
    """normalize_raw_signal(raw, outlier_thresh, scale_values) as the reference returned it
    (tests/golden/rsqgl_inputs.npz): signal and all five values, None <-> NaN"""
    import oracle as orc
    import read_inputs_cases as ric
    for raw, t, sv, want_norm, want in ric.golden_norm_cases(ric.golden()):
        st, norm, out = orc.normalize_raw_signal(raw, outlier_thresh=t, scale_values=sv)
        assert st == 0
        assert np.array_equal(norm, want_norm), (len(raw), t, sv)
        assert all((w is None and np.isnan(o)) or o == w for o, w in zip(out, want)), (out, want)


def test_oracle_read_inputs_match_reference(orc, RPcls):
    """resquiggle_read with caller scale values / stall lists (single calls, orc_resquiggle_read)
    and the worker policy from such a map_res (orc_run_read_inputs) against the reference"""
    import read_inputs_cases as ric
    cases = ric.golden_cases(ric.golden(), RPcls)
    for i, c in enumerate(cases):
        rm, rsd = gu.levels(c['read'].genome_seq, c['kmer_ref'])
        raw = np.asarray(c['read'].raw, dtype=np.float64)
        e = c['expected']
        if c['call'] == 0:
            pol = orc.policy('DNA', skip_seq_scaling=c['skip'], const_scale=c['const_scale'])
            o = orc.resquiggle_read(raw, rm, rsd, c['rp'], pol, scale_values=c['scale_values'],
                                    stall_ints=c['stall_ints'])
            sv = o.get('scale_values')
        else:
            o = orc.run_read(raw, rm, rsd, c['rp'], c['sp'], orc.policy(c['kind']),
                             read_index=c['read_index'], scale_values=c['scale_values'],
                             stall_ints=c['stall_ints'])
            assert (o['calls'], o['rescued']) == (e['calls'], e['rescued']), i
            sv = None if o['status'] else tuple(o[k] for k in ('shift', 'scale', 'lower_lim',
                                                               'upper_lim', 'outlier_thresh'))
        if e['message']:
            assert ric.same_message(o['status'], o['message'], e['message']), (i, o['message'])
            continue
        assert o['status'] == 0, (i, o['message'])
        assert np.array_equal(o['segs'], e['segs']), i
        assert o['read_start_rel_to_raw'] == e['read_start_rel_to_raw'], i
        assert all((w is None and np.isnan(v)) or v == w for v, w in zip(sv, e['scale_values'])), \
            (i, sv, e['scale_values'])
        assert o['sig_match_score'] == e['sig_match_score'], i
        assert o['norm_params_changed'] == e['norm_params_changed'], i
        if c['call'] == 1:
            assert o['n_iters'] == e['n_iters'], i
    # what the cases are there for
    worker_sv = [c for c in cases if c['call'] == 1 and c['scale_values'] is not None and c['kind'] == 'DNA']
    assert any(c['expected']['rescued'] for c in worker_sv), 'no read with scale values rescued'
    assert any(c['expected']['message'] for c in cases), 'no failing case'
