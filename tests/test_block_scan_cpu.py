"""CPU check of the block-wide scan (tb2_block_excl_scan, csrc/common.cuh) in its 1024-thread,
64-bit, looped use: the offsets kernel k_scan_offsets run on the host emulation against
np.cumsum, across chunk edges, for int and unsigned long long counts, separate and in place."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.join(HERE, 'emul') not in sys.path:
    sys.path.insert(0, os.path.join(HERE, 'emul'))
import emul_motif as em     # noqa: E402

SIZES = [0, 1, 1023, 1024, 1025, 4999]


def expected(cnt):
    off = np.zeros(cnt.shape[0] + 1, dtype=np.uint64)
    np.cumsum(cnt.astype(np.uint64), out=off[1:])
    return off.view(np.int64)


@pytest.mark.parametrize('n', SIZES)
def test_int_counts(n):
    rng = np.random.default_rng(n)
    cnt = rng.integers(0, 1 << 21, n).astype(np.int32)
    if n:
        cnt[n // 2] = (1 << 31) - 1
    off = em.scan_offsets(cnt)
    assert np.array_equal(off, expected(cnt))
    if n > 4096:
        assert off[-1] > 1 << 32             # a 64-bit total of 32-bit counts


@pytest.mark.parametrize('in_place', [False, True])
@pytest.mark.parametrize('n', SIZES)
def test_u64_counts_past_2_32(n, in_place):
    rng = np.random.default_rng(1000 + n)
    cnt = rng.integers(0, 1 << 24, n).astype(np.uint64)
    if n:
        cnt[n // 2] = (1 << 33) + 5          # totals past 2^32 from the middle on
    off = em.scan_offsets(cnt, in_place=in_place)
    assert np.array_equal(off, expected(cnt))
    if n > 1:
        assert off[-1] > 1 << 32
