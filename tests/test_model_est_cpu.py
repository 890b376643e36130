"""Alternative-model estimation without a GPU: the kernel-density restatement against scipy,
and parse_base_levels / isolate_alt_density / the density files against the unmodified
reference's goldens (tests/golden/model_est.npz, make_model_est_golden.py)."""
import hashlib
import os
import sys
from collections import namedtuple

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import kde_cases as kc  # noqa: E402
from tombo_b200 import synthetic as syn, tombo_helper as th, tombo_stats as ts  # noqa: E402
from tombo_b200 import _default_parameters as dp  # noqa: E402

GOLD = os.path.join(HERE, 'golden', 'model_est.npz')
Read = namedtuple('Read', ('fn', 'corr_group'))


class Index(object):
    def __init__(self, reads):
        self.reads = reads

    def iter_reads(self):
        return list(self.reads)


def golden():
    return np.load(GOLD)


def cfg_of(g, key):
    return g[key].item()


def serve(monkeypatch, g, tag, n_reads=None):
    """regenerate one sample's reads from the golden's seeds and serve them at the Events
    seam; returns its reads index"""
    alt = tag == 'alt'
    kmer_ref = syn.make_event_model(cfg_of(g, 'kmer_width'), cfg_of(g, 'model_seed'))
    seed0 = cfg_of(g, 'alt_seed0' if alt else 'ctrl_seed0')
    n = cfg_of(g, 'n_reads') if n_reads is None else n_reads
    served = {}
    for i in range(n):
        served['%s%d' % (tag, i)] = syn.make_event_read(
            kmer_ref, cfg_of(g, 'central_pos'), cfg_of(g, 'n_bases'), seed0 + i,
            alt_base='C' if alt else None, alt_frac=cfg_of(g, 'alt_frac'),
            alt_shift=cfg_of(g, 'alt_shift'), shift=cfg_of(g, 'alt_level_shift') if alt else 0.0)
    monkeypatch.setattr(th, 'get_multiple_slots_read_centric',
                        lambda r, slots, corr=None: list(served[r.fn]))
    return Index([Read('%s%d' % (tag, i), 'RawGenomeCorrected_000') for i in range(n)]), kmer_ref


def digests(levels):
    return np.stack([np.frombuffer(hashlib.sha256(np.asarray(v, np.float64).tobytes()).digest(),
                                   dtype=np.uint8) for v in levels.values()])


def shuffled(index, seed):
    np.random.seed(seed)
    reads = list(index.iter_reads())
    np.random.shuffle(reads)
    return reads


def message(stderr):
    """the message inside the reference's '*** ERROR ***' / '*** WARNING ***' block"""
    return str(stderr).split('\n\t', 1)[1].rstrip('\n')


# ---------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------
def test_restatement_is_scipy_bit_for_bit():
    for x, grid, bw in kc.seeded_sets():
        want, c = kc.scipy_kde(x, grid, bw)
        got = kc.restate_kde(x, grid, c)
        assert np.array_equal(got, want), (x.shape[0], bw)
        assert np.array_equal(kc.scipy_kde_at(x, grid, c), want)
    # the far tails underflow to exactly 0 in some of them
    x, grid, bw = kc.seeded_sets()[6]
    assert (kc.scipy_kde(x, grid, bw)[0] == 0).sum() > 50


def test_pairwise_cho_cov_within_bound_of_scipy():
    rs = np.random.RandomState(2071)
    worst = 0.0
    for i in range(300):
        n = int(rs.randint(2, 5000))
        x = rs.normal(rs.uniform(-3, 3), rs.uniform(0.01, 2), n)
        bw = rs.uniform(0.01, 0.5)
        _, c_ref = kc.scipy_kde(x, np.zeros(1), bw)
        c = kc.cho_cov_pairwise(x, kc.factor_of(x, bw))
        rel = abs(c - c_ref) / c_ref
        assert rel <= kc.c_bound(n), (i, n, rel)
        worst = max(worst, rel / kc.U)
    assert worst < 16          # measured: a few u


# ---------------------------------------------------------------------------
# parse_base_levels against the reference
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('tag', ['alt', 'ctrl'])
def test_parse_base_levels_matches_reference(monkeypatch, tag):
    g = golden()
    index, kmer_ref = serve(monkeypatch, g, tag)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cfg_of(g, 'central_pos'))
    levels = ts.parse_base_levels(
        shuffled(index, cfg_of(g, 'shuffle_' + tag)), std_ref, cfg_of(g, 'batch'),
        cfg_of(g, 'kmer_obs_thresh'), cfg_of(g, 'max_kmer_obs'), cfg_of(g, 'min_kmer_obs_to_est'), 1)
    assert list(levels) == syn.all_kmers(cfg_of(g, 'kmer_width'))
    counts = np.array([v.shape[0] for v in levels.values()])
    np.testing.assert_array_equal(counts, g[tag + '_counts'])
    # k-mers completed mid-run and the stop rule fired before the reads ran out
    assert counts.max() > cfg_of(g, 'max_kmer_obs') and counts.min() > cfg_of(g, 'kmer_obs_thresh')
    assert counts.sum() < cfg_of(g, 'n_reads') * (cfg_of(g, 'n_bases') - 3)
    np.testing.assert_array_equal(digests(levels), g[tag + '_sha'])


def test_parse_base_levels_warning_and_failure_messages(monkeypatch, capsys):
    g = golden()
    index, kmer_ref = serve(monkeypatch, g, 'ctrl', cfg_of(g, 'out_reads'))
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cfg_of(g, 'central_pos'))
    args = (std_ref, cfg_of(g, 'batch'), cfg_of(g, 'out_thresh'), cfg_of(g, 'max_kmer_obs'))
    levels = ts.parse_base_levels(shuffled(index, cfg_of(g, 'shuffle_out')), *args,
                                  cfg_of(g, 'out_min'), 1)
    assert capsys.readouterr().err == str(g['out_stderr'])
    np.testing.assert_array_equal([v.shape[0] for v in levels.values()], g['out_counts'])
    np.testing.assert_array_equal(digests(levels), g['out_sha'])
    with pytest.raises(th.TomboError) as e:
        ts.parse_base_levels(shuffled(index, cfg_of(g, 'shuffle_fail')), *args,
                             cfg_of(g, 'fail_min'), 1)
    assert str(e.value) == message(g['fail_stderr'])


def test_no_downstream_bases_gives_no_levels(monkeypatch):
    g = golden()
    index, kmer_ref = serve(monkeypatch, g, 'ctrl', cfg_of(g, 'dn0_reads'))
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cfg_of(g, 'dn0_central_pos'))
    np.random.seed(cfg_of(g, 'shuffle_dn0'))
    with pytest.raises(th.TomboError) as e:
        ts.est_kernel_density(index, std_ref, cfg_of(g, 'dn0_thresh'), None, np.linspace(-5, 5, 10),
                              cfg_of(g, 'bw'), 1, 'alt', cfg_of(g, 'batch'), cfg_of(g, 'max_kmer_obs'),
                              cfg_of(g, 'dn0_min'))
    assert str(e.value) == message(g['dn0_stderr'])
    assert 'has 0 total observations' in str(e.value)


def test_non_acgt_kmers_are_skipped(monkeypatch):
    kmer_ref = syn.make_event_model(3, 1)
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=1)
    lv = np.arange(8, dtype=np.float64)
    base = np.frombuffer(b'ACGNTACG', dtype='S1')
    monkeypatch.setattr(th, 'get_multiple_slots_read_centric', lambda r, s, c=None: [lv, base])
    levels = ts.parse_base_levels([Read('r', 'g')], std_ref, 10, 0, 100, 0, 1)
    got = dict((k, list(v)) for k, v in levels.items() if v.shape[0])
    # ACG -> level 1, TAC -> 5, ACG -> 6; k-mers with the N are dropped
    assert got == {'ACG': [1.0, 6.0], 'TAC': [5.0]}


# ---------------------------------------------------------------------------
# isolate_alt_density and the density files against the reference
# ---------------------------------------------------------------------------
def golden_densities(g):
    kmers = syn.all_kmers(cfg_of(g, 'kmer_width'))
    return (dict(zip(kmers, g['alt_dens'])), dict(zip(kmers, g['ctrl_dens'])),
            np.linspace(-5, 5, cfg_of(g, 'n_points')))


def test_isolate_alt_density_matches_reference():
    g = golden()
    alt, ctrl, save_x = golden_densities(g)
    kmer_ref = syn.make_event_model(cfg_of(g, 'kmer_width'), cfg_of(g, 'model_seed'))
    std_ref = ts.TomboModel(kmer_ref=kmer_ref, central_pos=cfg_of(g, 'central_pos'))
    alt_ref, dec = ts._isolate_alt_density(alt, ctrl, 'C', cfg_of(g, 'alt_pctl'), std_ref, save_x)
    assert isinstance(alt_ref, ts.AltModel)
    assert [k for k, _ in alt_ref.means] == list(g['alt_kmers'])
    assert [p for _, p in alt_ref.means] == list(g['alt_pos'])
    assert np.array_equal(np.array(list(alt_ref.means.values())), g['alt_means'])
    assert np.array_equal(np.array(list(alt_ref.sds.values())), g['alt_sds'])
    np.testing.assert_array_equal(list(dec['offsets'].values()), g['dec_offsets'])
    np.testing.assert_array_equal(list(dec['peaks'].values()), g['dec_peaks'])
    # every decision is far from flipping under the device's density error (< 1e-11)
    for k in ('mask', 'offset', 'ctrl_peak', 'alt_peaks'):
        assert float(g['dec_margin_' + k]) > 1e-7, k
    assert int(g['dec_peak_distance_gap']) >= 1     # no tie for the nearest alternative peak
    assert min(dec['offsets'].values()) != 0       # the alternative densities were moved


def test_density_file_round_trip(tmp_path):
    g = golden()
    alt, _, save_x = golden_densities(g)
    fn = str(tmp_path / 'x.alt_density.txt')
    first = dict(list(alt.items())[:3])
    ts.write_kmer_densities_file(fn, first, save_x)
    with open(fn) as fp:
        assert fp.read() == str(g['density_file'])
    back = ts.parse_kmer_densities_file(fn)
    assert list(back) == list(first)
    for k in first:
        assert np.array_equal(back[k], first[k])
    with open(fn, 'a') as fp:
        fp.write('AAAA\t0.1\t0.5\n')
    with pytest.raises(th.TomboError):
        ts.parse_kmer_densities_file(fn)


def test_defaults_and_exports():
    assert (dp.ALT_EST_BATCH, dp.MAX_KMER_OBS, dp.MIN_KMER_OBS_TO_EST, dp.KERNEL_DENSITY_RANGE,
            dp.ALT_EST_PCTL, dp.NUM_DENS_POINTS) == (1000, 10000, 50, (-5, 5), 5, 500)
    for name in ('parse_base_levels', 'est_kernel_density', 'write_kmer_densities_file',
                 'parse_kmer_densities_file', 'isolate_alt_density'):
        assert name in ts.__all__
