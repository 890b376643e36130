import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, 'oracle')):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (H100)')


@pytest.fixture(scope='session')
def orc():
    """The C restatement of the reference (oracle/oracle.c) -- the checker."""
    import oracle
    oracle.lib()
    return oracle


@pytest.fixture(scope='session')
def ctx():
    """A tombo_b200 CUDA context (GPU tests only)."""
    from tombo_b200 import _lib
    c = _lib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope='session')
def dna_model():
    from tombo_b200 import synthetic as syn
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    return kmer_ref, cpos


class RP(object):
    """Minimal stand-in for resquiggleParams (attribute access only)."""

    def __init__(self, aln=(4.2, 4.2, 300, 1500, 20.0, 40, 750, 2500, 250),
                 seg=(5, 3, 1, 5), rna=False, save=False):
        (self.match_evalue, self.skip_pen, bw, sbw, self.max_half_z_score,
         self.band_bound_thresh, self.start_bw, self.start_save_bw,
         self.start_n_bases) = aln
        self.bandwidth = sbw if save else bw
        (self.running_stat_width, self.min_obs_per_base,
         self.raw_min_obs_per_base, self.mean_obs_per_event) = seg
        self.z_shift = float(np.sqrt(2.0 / np.pi)) + self.match_evalue
        self.stay_pen = self.match_evalue
        self.use_t_test_seg = rna


@pytest.fixture(scope='session')
def RPcls():
    return RP
