"""GPU: the reciprocal-based division used in the DP rows is bit-identical to IEEE
division (the reference divides; SURVEY.md section 7)."""
import ctypes as C

import pytest

pytestmark = pytest.mark.gpu


def test_div_by_reciprocal_is_correctly_rounded(ctx):
    fn = ctx.lib.tb2_debug_div_check
    total = 0
    for seed in (1, 2, 3, 4):
        mism = C.c_uint64(0)
        ex = (C.c_double * 4)()
        blocks, per_thread = 2048, 1024          # 2^29 pairs per seed
        ctx.check(fn(ctx.handle, C.c_uint64(seed), C.c_int(blocks), C.c_int(per_thread),
                     C.byref(mism), ex))
        assert mism.value == 0, (mism.value, list(ex))
        total += blocks * 256 * per_thread
    assert total == 2 ** 31
