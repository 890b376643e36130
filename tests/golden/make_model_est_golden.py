#!/usr/bin/env python
"""Goldens for alternative-model estimation from the UNMODIFIED reference (oracle/_ref):
est_kernel_density (parse_base_levels + gaussian_kde per k-mer), isolate_alt_density and
write_kmer_densities_file on a 4-mer synthetic model, a C-spiked sample and a control.

Reads are served at the Events seam: the reference's worker opens each read with
``h5py.File`` (a mock under the harness) and reads it with
``tombo_helper.get_multiple_slots_read_centric``; both are patched to serve in-memory
columns.  The worker runs in a forked process (num_processes=1), so the patches reach it.
Reads are regenerated from the seeds stored here (tombo_b200.synthetic.make_event_read).

Stored: per-k-mer level counts and SHA-256 of the level bytes (order-sensitive), scipy's
cho_cov, the densities, the alternative model, the decisions of isolate_alt_density with
their margins, the text of one density file, and the messages of the warning, failure and
dnstrm_bases == 0 cases.

    python oracle/build_ref.py && python tests/golden/make_model_est_golden.py
"""
import contextlib
import hashlib
import io
import os
import sys
import tempfile
from collections import namedtuple

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'oracle'))

import ref_harness as rh  # noqa: E402
from tombo_b200 import synthetic as syn  # noqa: E402

Read = namedtuple('Read', ('fn', 'corr_group'))
# densities below this are left out of the neighbour margins: the device bound's absolute
# term (< 1e-300 here) dominates there
PEAK_FLOOR = 1e-290

# recorded inputs (tests regenerate the reads from these)
CFG = dict(kmer_width=4, central_pos=1, model_seed=7, n_bases=300, alt_frac=0.6,
           alt_shift=0.7, alt_level_shift=0.3, alt_seed0=5000, ctrl_seed0=9000, n_reads=400, n_points=120,
           bw=0.1, batch=40, max_kmer_obs=150, kmer_obs_thresh=120, min_kmer_obs_to_est=50,
           alt_pctl=5, shuffle_alt=11, shuffle_ctrl=12,
           # reads run out: warning
           out_reads=50, out_thresh=1000, out_min=10, shuffle_out=13,
           # too few observations: error
           fail_min=100, shuffle_fail=14,
           # dnstrm_bases == 0: no read contributes
           dn0_central_pos=3, dn0_reads=30, dn0_thresh=10, dn0_min=5, shuffle_dn0=15)


def sample_reads(kmer_ref, cfg, seed0, n, alt):
    return [syn.make_event_read(kmer_ref, cfg['central_pos'], cfg['n_bases'], seed0 + i,
                                alt_base='C' if alt else None, alt_frac=cfg['alt_frac'],
                                alt_shift=cfg['alt_shift'],
                                shift=cfg['alt_level_shift'] if alt else 0.0)
            for i in range(n)]


class Index(object):
    def __init__(self, reads):
        self.reads = reads

    def iter_reads(self):
        return list(self.reads)


def level_digest(levels):
    return np.frombuffer(hashlib.sha256(np.asarray(levels, dtype=np.float64).tobytes()).digest(),
                         dtype=np.uint8)


def decisions(alt_dens, std_dens, save_x, alt_base='C'):
    """isolate_alt_density's discrete steps on the reference's densities, with margins"""
    def dens_mean(d):
        return np.average(save_x[d > 1e-10], weights=d[d > 1e-10])
    xs, ys = [], []
    for k in std_dens:
        if alt_base not in k:
            xs.append(dens_mean(std_dens[k]))
            ys.append(dens_mean(alt_dens[k]) - xs[-1])
    fit = np.poly1d(np.polyfit(xs, ys, 2))
    step = save_x[1] - save_x[0]
    kmers = list(alt_dens)
    v = np.array([fit(dens_mean(std_dens[k])) / step for k in kmers])
    offsets = np.array([int(t) for t in v], dtype=np.int64)
    all_d = np.concatenate([np.concatenate(list(alt_dens.values())),
                            np.concatenate(list(std_dens.values()))])
    peaks, m_ctrl, m_alt, m_dist = [], np.inf, np.inf, np.inf
    for k, off in zip(kmers, offsets):
        if k.count(alt_base) != 1:
            continue
        d = alt_dens[k]
        alt = (np.concatenate([np.zeros(-off), d[:off]]) if off < 0 else
               np.concatenate([d[off:], np.zeros(off)]))
        ctrl = std_dens[k]
        cp = int(np.argmax(ctrl))
        srt = np.sort(ctrl)
        m_ctrl = min(m_ctrl, (srt[-1] - srt[-2]) / srt[-1])
        inner = alt[1:-1]
        pk = np.nonzero((inner > alt[:-2]) & (inner > alt[2:]))[0] + 1
        dist = np.abs(pk - cp)
        ap = int(pk[np.argmin(dist)])
        # every local-peak candidate: each comparison of neighbours decides one, so the
        # smallest relative gap between neighbours (above the subnormal floor of the bound)
        hi = np.maximum(alt[1:], alt[:-1])
        live = hi > PEAK_FLOOR
        m_alt = min(m_alt, np.min(np.abs(alt[1:] - alt[:-1])[live] / hi[live]))
        # the matched peak: the nearest candidate, by a whole number of grid points
        srt_d = np.sort(dist)
        if srt_d.shape[0] > 1:
            m_dist = min(m_dist, int(srt_d[1] - srt_d[0]))
        peaks.append((cp, ap))
    return dict(offsets=offsets, peaks=np.array(peaks, dtype=np.int64),
                margin_mask=np.min(np.abs(all_d / 1e-10 - 1.0)),
                margin_offset=np.min(np.abs(v - np.round(v))),
                margin_ctrl_peak=m_ctrl, margin_alt_peaks=m_alt, peak_distance_gap=m_dist)


def main():
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    ts.VERBOSE = False
    cfg = CFG
    kmer_ref = syn.make_event_model(cfg['kmer_width'], cfg['model_seed'])
    std_ref, _ = rh.make_models(kmer_ref, cfg['central_pos'])
    alt_reads = sample_reads(kmer_ref, cfg, cfg['alt_seed0'], cfg['n_reads'], True)
    ctrl_reads = sample_reads(kmer_ref, cfg, cfg['ctrl_seed0'], cfg['n_reads'], False)
    served = {}

    class Served(object):
        def __init__(self, fn, mode='r'):
            self.fn = fn

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False
    ts.h5py.File = Served
    th.get_multiple_slots_read_centric = lambda f5, slots, corr_grp=None: list(served[f5.fn])

    def index(tag, reads):
        rd = []
        for i, (lv, base) in enumerate(reads):
            served['%s%d' % (tag, i)] = (lv, base)
            rd.append(Read('%s%d' % (tag, i), 'RawGenomeCorrected_000'))
        return Index(rd)

    captured = {}
    orig_parse, orig_kde = ts.parse_base_levels, ts.stats.gaussian_kde

    def parse(*a, **k):
        captured['levels'] = orig_parse(*a, **k)
        return captured['levels']

    def kde(*a, **k):
        est = orig_kde(*a, **k)
        captured['cho'].append(float(est.cho_cov[0, 0]))
        return est
    ts.parse_base_levels = parse
    out = dict((k, np.array(v)) for k, v in cfg.items())
    save_x = np.linspace(-5, 5, cfg['n_points'])
    dens = {}
    try:
        ts.stats.gaussian_kde = kde
        with rh.ref_errstate():
            for tag, reads, seed in (('alt', alt_reads, cfg['shuffle_alt']),
                                     ('ctrl', ctrl_reads, cfg['shuffle_ctrl'])):
                captured['cho'] = []
                np.random.seed(seed)
                d = ts.est_kernel_density(
                    index(tag, reads), std_ref, cfg['kmer_obs_thresh'], None, save_x, cfg['bw'], 1,
                    tag, cfg['batch'], cfg['max_kmer_obs'], cfg['min_kmer_obs_to_est'])
                lv = captured['levels']
                out[tag + '_counts'] = np.array([len(lv[k]) for k in lv], dtype=np.int64)
                out[tag + '_sha'] = np.stack([level_digest(lv[k]) for k in lv])
                out[tag + '_cho_cov'] = np.array(captured['cho'])
                out[tag + '_dens'] = np.stack([d[k] for k in d])
                dens[tag] = d
            alt_ref = ts.isolate_alt_density(dens['alt'], dens['ctrl'], 'C', cfg['alt_pctl'],
                                             std_ref, save_x)
            out['alt_kmers'] = np.array([k for k, _ in alt_ref.means])
            out['alt_pos'] = np.array([p for _, p in alt_ref.means], dtype=np.int64)
            out['alt_means'] = np.array(list(alt_ref.means.values()))
            out['alt_sds'] = np.array(list(alt_ref.sds.values()))
            with np.errstate(under='ignore'):
                for k, v in decisions(dens['alt'], dens['ctrl'], save_x).items():
                    out['dec_' + k] = np.asarray(v)
            with tempfile.TemporaryDirectory() as tmp:
                fn = os.path.join(tmp, 'dens.txt')
                ts.write_kmer_densities_file(fn, dict(list(dens['alt'].items())[:3]), save_x)
                with open(fn) as fp:
                    out['density_file'] = np.array(fp.read())

            # reads run out (warning), too few observations (error), dnstrm_bases == 0
            short = index('out', ctrl_reads[:cfg['out_reads']])
            for tag, mn in (('out', cfg['out_min']), ('fail', cfg['fail_min'])):
                err = io.StringIO()
                np.random.seed(cfg['shuffle_' + tag])
                all_reads = list(short.iter_reads())
                np.random.shuffle(all_reads)
                try:
                    with contextlib.redirect_stderr(err):
                        lv = orig_parse(all_reads, std_ref, cfg['batch'], cfg['out_thresh'],
                                        cfg['max_kmer_obs'], mn, 1)
                    out[tag + '_counts'] = np.array([len(lv[k]) for k in lv], dtype=np.int64)
                    out[tag + '_sha'] = np.stack([level_digest(lv[k]) for k in lv])
                except SystemExit:
                    pass
                out[tag + '_stderr'] = np.array(err.getvalue())
            dn0_ref, _ = rh.make_models(kmer_ref, cfg['dn0_central_pos'])
            dn0 = index('dn0', ctrl_reads[:cfg['dn0_reads']])
            err = io.StringIO()
            np.random.seed(cfg['shuffle_dn0'])
            try:
                with contextlib.redirect_stderr(err):
                    ts.est_kernel_density(dn0, dn0_ref, cfg['dn0_thresh'], None, save_x, cfg['bw'], 1,
                                          'alt', cfg['batch'], cfg['max_kmer_obs'], cfg['dn0_min'])
            except SystemExit:
                pass
            out['dn0_stderr'] = np.array(err.getvalue())
    finally:
        ts.parse_base_levels, ts.stats.gaussian_kde = orig_parse, orig_kde
    assert 'ERROR' in str(out['fail_stderr']) and 'WARNING' in str(out['out_stderr'])
    assert 'ERROR' in str(out['dn0_stderr'])
    np.savez_compressed(os.path.join(HERE, 'model_est.npz'), **out)
    print('model_est.npz:', len(out), 'arrays;', dict(
        (k, float(out[k])) for k in out if k.startswith('dec_margin')),
        'counts alt', out['alt_counts'].min(), out['alt_counts'].max(),
        'ctrl', out['ctrl_counts'].min(), out['ctrl_counts'].max())


if __name__ == '__main__':
    main()
