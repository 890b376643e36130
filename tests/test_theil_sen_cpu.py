"""CPU: Theil-Sen rescaling against an exact numpy restatement of the reference
(tests/theil_sen_cases.py).  The restatement, the C oracle and k_theil_sen's device source on
the host emulation (tests/emul) must give the same status and the same four doubles, bit for
bit, on every case family; the emulation must take the selection path each case declares.
The GPU counterpart is test_theil_sen_gpu.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import theil_sen_cases as tc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emul'))

CASES = tc.all_cases()
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES), 'case names must be unique'


def _bits(out):
    return np.array(out, dtype=np.float64).view(np.int64)


def assert_same(got, want, what):
    """status and all four outputs bit for bit; no outputs to compare on a failed read"""
    (s0, o0), (s1, o1) = want, got
    assert s1 == s0, (what, s0, s1)
    if s0 == tc.OK:
        assert np.array_equal(_bits(o1), _bits(o0)), (what, o0, o1)


def _emul_run(case):
    """the emulated kernel's result and the set of path slots [1]-[6] its call moved"""
    import emul
    L = emul.stage_lib()
    before, after = (C.c_ulonglong * 8)(), (C.c_ulonglong * 8)()
    L.emul_ts_counters(before, 0)
    res = emul.theil_sen(case.prev_shift, case.prev_scale, case.ev, case.md, key=case.key)
    L.emul_ts_counters(after, 0)
    delta = [after[i] - before[i] for i in range(8)]
    return res, delta


@pytest.mark.parametrize('name', sorted(BY_NAME))
def test_restatement_matches_oracle(orc, name):
    c = BY_NAME[name]
    want = tc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)
    got = orc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, key=c.key)
    assert_same(got, want, name)


@pytest.mark.parametrize('name', sorted(BY_NAME))
def test_emulated_kernel_matches_restatement_and_takes_declared_path(name):
    c = BY_NAME[name]
    want = tc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)
    got, delta = _emul_run(c)
    assert_same(got, want, name)
    assert delta[tc.READS] == 1, delta
    if c.expected_path is not None:
        moved = {s for s in tc.PATH_SLOTS if delta[s]}
        assert moved == set(c.expected_path), (name, sorted(moved), c.expected_path, delta)
        assert all(delta[s] == 1 for s in moved), delta


def test_every_path_is_some_cases_declared_path():
    declared = set()
    for c in CASES:
        declared.update(c.expected_path or ())
    assert declared >= set(tc.PATH_SLOTS), sorted(declared)
    # and, apart from the fp32 paths, on the device as well
    on_device = set()
    for c in CASES:
        if not c.emul_only:
            on_device.update(c.expected_path or ())
    assert on_device >= {tc.HISTOGRAM, tc.GENERIC, tc.SWEEP, tc.SWEEP_ABANDONED}, sorted(on_device)


def test_size_cases_cover_both_parities_and_both_kinds_of_even_median():
    """np.median averages the two middle slopes of an even count: those two are unequal for
    smooth data and tie inside the outlier mixture's block of exactly equal slopes"""
    seen = set()
    for c in tc.size_cases():
        a, b = tc.middle_slopes(c.ev, c.md, c.key)
        n = c.ev.shape[0]
        kind = 'odd' if b is None else 'even_equal' if a == b else 'even_unequal'
        seen.add((n, kind))
    kinds = {k for _, k in seen}
    assert kinds == {'odd', 'even_equal', 'even_unequal'}, seen
    for n in tc.SIZES:
        if (n * (n - 1) // 2) % 2 == 0 and n >= 17:
            assert (n, 'even_unequal') in seen and (n, 'even_equal') in seen, (n, seen)


def test_power_of_two_rescalings_are_exact():
    """ev * 2^k, md * 2^k: the same slopes, the intercept times 2^k -- on the restatement,
    the oracle and the emulated kernel, whichever path the kernel takes"""
    import emul
    import oracle
    cases = {c.name: c for c in tc.rescaled_cases()}
    base = cases.pop('rescaled_base')
    s, base_out = tc.theil_sen(base.prev_shift, base.prev_scale, base.ev, base.md)
    assert s == tc.OK and base.prev_shift == 0.0 and base.prev_scale == 1.0
    for k in tc.RESCALE_EXPONENTS:
        c = cases['rescaled_2^%d' % k]
        want = (tc.OK, tc.rescale_expectation(base_out, k))
        for fn in (tc.theil_sen, oracle.theil_sen, emul.theil_sen):
            assert_same(fn(c.prev_shift, c.prev_scale, c.ev, c.md, c.key), want, (k, fn.__module__))


def test_zero_slope_fails_with_the_reference_status_and_message(orc):
    from tombo_b200 import _lib
    import emul
    n_zero = 0
    for c in CASES:
        if not c.name.startswith('family_constant_md'):
            continue
        assert tc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)[0] == tc.ERR_THEIL_SEN_ZERO
        assert orc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)[0] == tc.ERR_THEIL_SEN_ZERO
        assert emul.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)[0] == tc.ERR_THEIL_SEN_ZERO
        n_zero += 1
    assert n_zero >= 3
    assert orc.status_message(tc.ERR_THEIL_SEN_ZERO) == tc.ZERO_SLOPE_MESSAGE
    assert _lib.status_message(tc.ERR_THEIL_SEN_ZERO) == tc.ZERO_SLOPE_MESSAGE


def test_emulated_kernel_random_sweep():
    """seeded cases over every family, size class and a share of 2^k rescalings"""
    rs = np.random.RandomState(2024)
    moved = np.zeros(8, dtype=np.int64)
    for it in range(150):
        c = tc.random_case(rs)
        want = tc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)
        got, delta = _emul_run(c)
        assert_same(got, want, (it, c.name, c.key))
        moved += np.array(delta, dtype=np.int64)
    assert moved[tc.READS] == 150
    assert all(moved[s] > 0 for s in (tc.HISTOGRAM, tc.GENERIC, tc.SWEEP, tc.SWEEP_ABANDONED)), moved
