"""GPU: k_theil_sen through tb2_theil_sen against the exact numpy restatement of the reference
(tests/theil_sen_cases.py): status and all four doubles bit for bit on every case family, the
selection path each case's construction fixes, and a seeded sweep that must reach every path
on the device."""
import ctypes as C
import time

import numpy as np
import pytest

import theil_sen_cases as tc

pytestmark = pytest.mark.gpu

CASES = tc.all_cases()
BY_NAME = {c.name: c for c in CASES}


def debug_counters(ctx):
    """g_tb2_counters (include/tombo_b200.h); device-global, so callers compare deltas"""
    out = (C.c_ulonglong * 8)()
    ctx.check(ctx.lib.tb2_debug_counters(ctx.handle, out, 0))
    return np.array(list(out), dtype=np.int64)


def _run(ctx, c):
    before = debug_counters(ctx)
    res = ctx.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)
    return res, debug_counters(ctx) - before


def assert_same(got, want, what):
    (s0, o0), (s1, o1) = want, got
    assert s1 == s0, (what, s0, s1)
    if s0 == tc.OK:
        assert np.array_equal(np.array(o1, np.float64).view(np.int64),
                              np.array(o0, np.float64).view(np.int64)), (what, o0, o1)


@pytest.mark.parametrize('name', sorted(BY_NAME))
def test_theil_sen_matches_restatement(ctx, name):
    c = BY_NAME[name]
    want = tc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)
    got = ctx.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)
    assert_same(got, want, name)


@pytest.mark.parametrize('name', sorted(c.name for c in CASES
                                        if c.expected_path is not None and not c.emul_only))
def test_theil_sen_takes_declared_path(ctx, name):
    """exactly the declared slots move, each once; slot [0] counts the call"""
    c = BY_NAME[name]
    _, delta = _run(ctx, c)
    assert delta[tc.READS] == 1, delta
    moved = {s for s in tc.PATH_SLOTS if delta[s]}
    assert moved == set(c.expected_path), (name, sorted(moved), c.expected_path, delta)
    assert all(delta[s] == 1 for s in moved), delta


# Minimum count of each path slot over the sweep below.  Measured on one H100 (80 GB) with
# the kernel of this commit, 3000 reads: [1] 98, [2] 599, [3] 714, [4] 20, [5] 1569, [6] 693.
# The inputs are seeded and the path decisions depend on counts, not on the order of atomic
# updates, so the counts repeat; the
# minimums sit at about half of them, so a kernel that stops reaching a path fails here
# instead of passing with that path unexercised.
SWEEP_CASES = 3000
SWEEP_MIN = {tc.FP32_ALL: 49, tc.HISTOGRAM: 300, tc.GENERIC: 357, tc.FP32_SAMPLED: 10,
             tc.SWEEP: 785, tc.SWEEP_ABANDONED: 346}


def test_theil_sen_random_sweep(ctx):
    rs = np.random.RandomState(20261015)
    moved = np.zeros(8, dtype=np.int64)
    t0 = time.time()
    for it in range(SWEEP_CASES):
        c = tc.random_case(rs)
        want = tc.theil_sen(c.prev_shift, c.prev_scale, c.ev, c.md, c.key)
        got, delta = _run(ctx, c)
        assert_same(got, want, (it, c.name, c.key))
        assert delta[tc.READS] == 1
        moved += delta
    print('theil-sen sweep: %d reads in %.1f s, path counts %s' % (
        SWEEP_CASES, time.time() - t0, {s: int(moved[s]) for s in tc.PATH_SLOTS}))
    for s, lo in SWEEP_MIN.items():
        assert moved[s] >= lo, (s, moved.tolist())
