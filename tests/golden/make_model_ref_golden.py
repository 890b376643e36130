#!/usr/bin/env python
"""Goldens for standard and motif model estimation from the UNMODIFIED reference
(oracle/_ref): extract_kmer_levels (get_region_kmer_levels in its one-worker order),
tabulate_kmer_levels, tabulate_mod_kmer_levels, center_model_to_median_norm and
TomboModel._make_constant_sd on
tests/model_ref_cases.py's reads, in median and mean mode, with subsampling, a region
smaller than a read, CG:1 and CCWGG:2 motifs and valid_poss.

The reference's TomboReads is built with ``object.__new__`` around the in-memory reads, so
its own iter_cov_regs runs; the regions go through the reference's get_region_kmer_levels
in this process, in the one-worker order.  Reads are served at the Events seam
(``tombo_helper.get_single_slot_read_centric`` patched).

Stored per case: the row count of every (region, key) and all rows in order; per row whether
the reference summarised the position's levels in read order, their count and mean |level|;
the tabulated medians and tabulate's messages, also with one key emptied ("not covered").

Centering (center_model_to_median_norm, then _make_constant_sd) on the median-mode model,
after the extraction's shuffles, with DNA reads, all DNA reads (warning), RNA reads (event
scaling, stall removal) and unreadable reads (error): the per-read correction factors in
fit order, the model before and after, the messages and the RNG state after the call.  The
reference's calc_kmer_fitted_shift_scale, h5py.File, get_raw_read_slot and
get_multiple_slots_read_centric are patched to record the factors and serve the reads.

    python oracle/build_ref.py && python tests/golden/make_model_ref_golden.py
"""
import contextlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'oracle'))
sys.path.insert(0, os.path.dirname(HERE))

import ref_harness as rh  # noqa: E402
import model_ref_cases as mc  # noqa: E402


def object_index(th, reads):
    index = object.__new__(th.TomboReads)
    index.reads_index = mc.Index(reads).reads_index
    index.coverage = None
    return index


def worker_regions(th, ts, index, region_size, cov_thresh, upstrm_bases, dnstrm_bases,
                   cs_cov_thresh, est_mean, motif=None, valid_poss=None):
    """extract_kmer_levels :1398-1452 as its one worker runs it (:1361-1388), in this
    process: the worker's draws come from a copy of the RNG state, so the state is restored
    afterwards as the fork leaves the parent's untouched.  A region whose
    get_region_kmer_levels raises ends the worker, as it does in the reference."""
    state = np.random.get_state()
    out = []
    try:
        for chrm, strand, reg_start in index.iter_cov_regs(cov_thresh, region_size):
            reg_data = th.intervalData(chrm=chrm, start=reg_start, end=reg_start + region_size,
                                       strand=strand).add_reads(index)
            if len(reg_data.reads) == 0:
                continue
            try:
                r = ts.get_region_kmer_levels(reg_data, cov_thresh, upstrm_bases, dnstrm_bases,
                                              cs_cov_thresh, est_mean, region_size, motif, valid_poss)
            except TypeError:
                break
            if r is not None:
                out.append(r)
    finally:
        np.random.set_state(state)
    return out


class LevelOrder(object):
    """records, for every row get_region_kmer_levels appends, whether the reference summarised
    that position's levels in read order (the device's order), their count and mean |level|"""

    def __init__(self, th, ts, served):
        self.th, self.ts, self.served = th, ts, served
        self.rows = {}
        self.orig = th.get_reads_events, ts.calc_med_sd, ts.c_mean_std

    def __enter__(self):
        th, ts = self.th, self.ts
        orig_events, orig_med, orig_mean = self.orig
        cur = {}

        def events(cs_reads):
            be = orig_events(cs_reads)
            cur.clear()
            if be is None:
                return be
            per = {}
            for r in cs_reads:
                m = self.served[r.fn]['norm_mean']
                if m is None or m.shape[0] != r.end - r.start:
                    continue
                m = m[::-1] if r.strand == '-' else m
                for j, v in enumerate(m):
                    per.setdefault(r.start + j, []).append(v)
            for pos, v in be.items():
                cur[id(v)] = np.array(per[pos])
            return be

        def wrap(fn):
            def rec(vals):
                res = fn(vals)
                self.rows[id(res)] = (np.array_equal(vals, cur[id(vals)]), vals.shape[0],
                                      np.mean(np.abs(vals)), res)
                return res
            return rec
        th.get_reads_events = events
        ts.calc_med_sd, ts.c_mean_std = wrap(orig_med), wrap(orig_mean)
        return self

    def __exit__(self, *a):
        self.th.get_reads_events, self.ts.calc_med_sd, self.ts.c_mean_std = self.orig
        return False

    def flags(self, regs):
        """(same order, n, mean |level|) per row, in mc.flatten's order"""
        got = [self.rows[id(row)][:3] for reg in regs for v in reg.values() for row in v]
        return np.array(got, dtype=np.float64).reshape(-1, 3)


def stderr_of(fn, *args):
    """(result or None, stderr text) of a reference call that may exit"""
    err = io.StringIO()
    res = None
    try:
        with contextlib.redirect_stderr(err):
            res = fn(*args)
    except SystemExit:
        pass
    # status lines carry the time of day; the messages that matter are the warnings and errors
    return res, '\n'.join(l for l in err.getvalue().splitlines() if not l.startswith('['))


def model_arrays(ref, kmers):
    return (np.array([ref.means[k] for k in kmers], dtype=np.float64),
            np.array([ref.sds[k] for k in kmers], dtype=np.float64))


def centering(th, ts, out, tag, index, init_tab, up, kmers, max_reads):
    """center_model_to_median_norm (and _make_constant_sd) of the unmodified reference on
    ``index``, starting from the model ``init_tab``: per-read factors in the order they were
    fitted, the model before and after, the RNG state after the call and the messages"""
    factors = []
    orig_fit = ts.calc_kmer_fitted_shift_scale

    def fit(*a, **k):
        res = orig_fit(*a, **k)
        factors.append(res[2:4])
        return res
    ts.calc_kmer_fitted_shift_scale = fit
    try:
        init_ref = ts.TomboModel(kmer_ref=init_tab, central_pos=up)
        out[tag + '_before'] = np.stack(model_arrays(init_ref, kmers))
        ref, err = stderr_of(ts.center_model_to_median_norm, index, init_ref, max_reads)
    finally:
        ts.calc_kmer_fitted_shift_scale = orig_fit
    out[tag + '_stderr'] = np.array(err)
    out[tag + '_rng_after'] = np.array(np.random.get_state()[1])
    out[tag + '_rng_pos'] = np.array(np.random.get_state()[2])
    if ref is None:
        return
    out[tag + '_factors'] = np.array(factors, dtype=np.float64).reshape(-1, 2)
    out[tag + '_after'] = np.stack(model_arrays(ref, kmers))
    ref._make_constant_sd()
    out[tag + '_after_const_sd'] = np.stack(model_arrays(ref, kmers))


def main():
    m = rh.load_reference()
    th, ts = m['th'], m['ts']
    ts.VERBOSE = False
    th.VERBOSE = False
    cfg = mc.CFG
    kmer_ref, genome, reads, served = mc.make_inputs()

    th.get_single_slot_read_centric = lambda r, slot, corr_grp=None: served[r.fn].get(slot)

    class Served(object):
        def __init__(self, fn, mode='r'):
            self.fn = fn

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False
    ts.h5py.File = Served
    th.get_raw_read_slot = lambda f5: dict(Signal=served[f5.fn]['Signal'])
    th.get_multiple_slots_read_centric = (
        lambda f5, slots, corr_grp=None: [served[f5.fn][n] for n in slots])
    index = object_index(th, reads)
    out = dict((k, np.array(v)) for k, v in cfg.items())
    for name, kw in mc.extraction_cases():
        kw = dict(kw)
        motif = kw.pop('motif', None)
        if motif is not None:
            raw, pos = motif.split(':')
            motif = th.TomboMotif(raw, int(pos))
        if kw.pop('valid_poss', None):
            kw['valid_poss'] = mc.valid_poss_of(genome)
        np.random.seed(cfg['shuffle_seed'])
        with LevelOrder(th, ts, served) as lo:
            regs = worker_regions(th, ts, index, motif=motif, **kw)
        counts, rows = mc.flatten(regs)
        out[name + '_counts'], out[name + '_rows'] = counts, rows
        out[name + '_order'] = lo.flags(regs)
        tabulate = ((lambda r: ts.tabulate_kmer_levels(r, cfg['min_kmer_obs'])) if motif is None else
                    (lambda r: ts.tabulate_mod_kmer_levels(r, cfg['min_kmer_obs'], motif)))
        try:
            tab, err = stderr_of(tabulate, regs)
        except NameError as e:
            # tabulate_kmer_levels' "fewer observations" path names an undefined motif
            tab, err = None, 'NameError: %s' % e
        out[name + '_tab_stderr'] = np.array(err)
        out[name + '_tab'] = (np.zeros((0, 2)) if tab is None else
                              np.array([t[-2:] for t in tab], dtype=np.float64))
        # "not covered": the first key loses every row
        first = next(iter(regs[0]))
        gap = [dict((k, [] if k == first else v) for k, v in reg.items()) for reg in regs]
        out[name + '_gap_stderr'] = np.array(stderr_of(tabulate, gap)[1])
        if name == 'median':
            median_tab = tab

    # centering on the median-mode model: DNA reads, then RNA reads (event scaling with
    # stall removal); the region shuffles before it leave the RNG as the fork leaves it
    up = cfg['central_pos']
    kmers = [t[0] for t in median_tab]
    np.random.seed(cfg['shuffle_seed'])
    worker_regions(th, ts, index, **dict(mc.extraction_cases()[0][1]))
    centering(th, ts, out, 'center_dna', index, median_tab, up, kmers, cfg['center_reads'])
    np.random.seed(cfg['shuffle_seed'])
    centering(th, ts, out, 'center_dna_all', index, median_tab, up, kmers, 5000)
    _, _, rna_reads, rna_served = mc.make_inputs(rna=True)
    served.update(rna_served)
    np.random.seed(cfg['shuffle_seed'])
    centering(th, ts, out, 'center_rna', object_index(th, rna_reads), median_tab, up, kmers,
              cfg['center_reads'])
    np.random.seed(cfg['shuffle_seed'])
    centering(th, ts, out, 'center_none', object_index(th, mc.unreadable(reads)), median_tab, up,
              kmers, cfg['center_reads'])
    np.savez_compressed(os.path.join(HERE, 'model_ref.npz'), **out)
    print('model_ref.npz:', sorted((k, out[k].shape) for k in out if k.endswith('_counts')))


if __name__ == '__main__':
    main()
