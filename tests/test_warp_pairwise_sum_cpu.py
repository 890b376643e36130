"""CPU: warp_pairwise_sum (tombo_b200/csrc/common.cuh), the one-lane-per-subtree form of numpy's
pairwise sum that k_finalize and k_kde_setup use, against np.sum bit for bit on the host
emulation of tests/emul."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emul')
PD = C.POINTER(C.c_double)


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp('emul') / 'libemul_pairwise.so')
    subprocess.check_call(['g++', '-O1', '-g', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared',
                           '-o', so, os.path.join(EMUL, 'emul_pairwise.cpp'),
                           os.path.join(EMUL, 'cuda_emul.cpp')])
    return C.CDLL(so)


def test_warp_pairwise_sum_is_np_sum(lib):
    """every n from 1 to 2000: n < 8, the 8-accumulator leaf (n <= 128), and splits of numpy's
    tree that are not multiples of 8"""
    rng = np.random.default_rng(4242)
    # magnitudes over many binades make every change of summation order visible
    base = rng.normal(0.0, 1.0, 2000) * np.exp2(rng.integers(-30, 30, 2000))
    out = np.zeros(1)
    for n in range(1, 2001):
        v = np.ascontiguousarray(base[:n])
        lib.emul_warp_pairwise_sum(v.ctypes.data_as(PD), C.c_int(n), out.ctypes.data_as(PD))
        assert out.view(np.uint64)[0] == np.sum(v).view(np.uint64), n
