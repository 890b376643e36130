"""Shared inputs of the standard / motif model estimation tests (golden: make_model_ref_golden.py).

* ``Index``: a reads index with TomboReads' coverage and region iteration
  (tombo_helper.py:1394-1404, 1430-1485), ``get_cs_reads`` and ``iter_reads``.
* ``serve``: patches the Events / raw-signal seam to serve in-memory reads.
* ``RestatedContext``: tb2_kmer_level_summaries / tb2_kmer_medians restated in numpy, in
  read order -- what the device must reproduce bit for bit.
"""
import contextlib

import numpy as np

from tombo_b200 import synthetic as syn
from tombo_b200 import tombo_helper as th
from tombo_b200 import tombo_stats as ts

CFG = dict(kmer_width=3, central_pos=1, model_seed=3, genome_len=1200, n_reads=60, read_len=300,
           read_seed=21, region_size=200, cov_thresh=3, min_kmer_obs=2, cs_cov_thresh=12,
           small_region=100, shuffle_seed=5, motifs=('CG:1', 'CCWGG:2'), center_reads=25)


def make_inputs(cfg=CFG, rna=False):
    """(kmer_ref, genome, reads, served): reads on both strands; read 0 has a norm_mean one
    base short (mismatched length), one read has no bases (sequence gap source), and reads
    are absent from [900, 1000) of the '+' strand (a region below the threshold).  With
    ``rna`` the reads are RNA (raw signal reversed) on chromosome 'rna'."""
    chrm = 'rna' if rna else 'chr'
    kmer_ref = syn.make_event_model(cfg['kmer_width'], cfg['model_seed'])
    genome, reads, served = syn.make_mapped_reads(
        kmer_ref, cfg['central_pos'], cfg['genome_len'], cfg['n_reads'], cfg['read_len'],
        cfg['read_seed'], chrm=chrm, rna=rna, obs_per_base=12 if rna else 6)
    served[reads[0].fn]['norm_mean'] = served[reads[0].fn]['norm_mean'][:-1]
    gap = chrm + '_gap_read'
    reads = [r for r in reads if not (r.strand == '+' and r.start < 1000 and r.end > 900)] + [
        syn.MappedRead(50, 150, '+', gap, 'RawGenomeCorrected_000', rna, 0, chrm)]
    served[gap] = dict(norm_mean=np.zeros(100), base=None, start=None, Signal=None)
    return kmer_ref, genome, reads, served


def unreadable(reads):
    """the same reads under file names nothing serves: every read fails to open"""
    return [r._replace(fn='missing_' + r.fn) for r in reads]


class Index(object):
    """reads index stand-in: TomboReads' coverage and iter_cov_regs over in-memory reads"""

    def __init__(self, reads):
        self.reads_index = {}
        for r in reads:
            self.reads_index.setdefault((r.chrm, r.strand), []).append(r)

    def get_cs_reads(self, chrm, strand, invalid_return=[]):
        return self.reads_index.get((chrm, strand), invalid_return)

    def iter_reads(self):
        for cs_reads in self.reads_index.values():
            for r in cs_reads:
                yield r

    def iter_cov_regs(self, cov_thresh, region_size=None):
        for (chrm, strand), cs_reads in self.reads_index.items():
            if len(cs_reads) == 0:
                continue
            cov = np.zeros(max(r.end for r in cs_reads), dtype=np.int64)
            for r in cs_reads:
                cov[r.start:r.end] += 1
            starts = np.concatenate([[0], np.where(np.diff(cov))[0] + 1, [cov.shape[0]]])
            cov = cov[starts[:-1]]
            curr_reg_start = -1
            valid = np.where(np.diff(np.concatenate([[False], np.greater_equal(cov, cov_thresh), [False]])))[0]
            for a, b in zip(valid[:-1], valid[1:]):
                cov_start, cov_end = starts[a], starts[b]
                for reg_start in range(int(region_size * np.floor(cov_start / float(region_size))),
                                       int(region_size * np.ceil(cov_end / float(region_size))), region_size):
                    if reg_start != curr_reg_start:
                        yield chrm, strand, reg_start
                        curr_reg_start = reg_start


class _Fast5(object):
    def __init__(self, cols):
        self.cols = cols

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@contextlib.contextmanager
def serve(served):
    """serve reads' Events columns and raw signal from ``served`` through the mirrors' seam"""
    orig = th.get_multiple_slots_read_centric, th.get_raw_read_slot, ts._open_read

    def slots(r_data, slot_names, corr_grp=None):
        cols = r_data.cols if isinstance(r_data, _Fast5) else served.get(r_data.fn, {})
        return [cols.get(n) for n in slot_names]
    th.get_multiple_slots_read_centric = slots
    th.get_raw_read_slot = lambda f5: dict(Signal=f5.cols['Signal'])
    ts._open_read = lambda r_data: _Fast5(served[r_data.fn])
    try:
        yield
    finally:
        th.get_multiple_slots_read_centric, th.get_raw_read_slot, ts._open_read = orig


def summaries(n_pos, reads, cov_thresh, est_mean=False):
    """tb2_kmer_level_summaries restated: per position, the levels in read order; calc_med_sd
    or c_mean_std where coverage > cov_thresh"""
    lv, off, st = reads
    per = [[] for _ in range(n_pos)]
    for r in range(len(off) - 1):
        for j, v in enumerate(lv[off[r]:off[r + 1]]):
            p = st[r] + j
            if 0 <= p < n_pos and not np.isnan(v):
                per[p].append(v)
    cov = np.array([len(v) for v in per], dtype=np.int64)
    out_lv, out_sd = np.full(n_pos, np.nan), np.full(n_pos, np.nan)
    for p in np.nonzero(cov > cov_thresh)[0]:
        v = np.array(per[p])
        if est_mean:
            m = 0.0
            for x in v:
                m += x
            m /= v.shape[0]
            var = 0.0
            for x in v:
                var += (x - m) * (x - m)
            out_lv[p], out_sd[p] = m, np.sqrt(var / v.shape[0])
        else:
            out_lv[p], out_sd[p] = np.median(v), np.std(v)
    return out_lv, out_sd, cov


def medians(n_keys, keys, levels, sds):
    """tb2_kmer_medians restated"""
    keys = np.asarray(keys, dtype=np.int64)
    cnt = np.bincount(keys, minlength=n_keys).astype(np.int64)
    ml, ms = np.full(n_keys, np.nan), np.full(n_keys, np.nan)
    for k in np.nonzero(cnt)[0]:
        ml[k], ms[k] = np.median(levels[keys == k]), np.median(sds[keys == k])
    return cnt, ml, ms


class RestatedContext(object):
    def kmer_level_summaries(self, n_pos, reads, cov_thresh, est_mean=False):
        return summaries(n_pos, reads, cov_thresh, est_mean)

    def kmer_medians(self, n_keys, keys, levels, sds):
        return medians(n_keys, keys, levels, sds)


def extraction_cases(cfg=CFG):
    """(name, extract_kmer_levels keyword arguments beyond the reads index) of the goldens"""
    base = dict(region_size=cfg['region_size'], cov_thresh=cfg['cov_thresh'],
                upstrm_bases=cfg['central_pos'], dnstrm_bases=cfg['kmer_width'] - cfg['central_pos'] - 1)
    out = [('median', dict(base, cs_cov_thresh=None, est_mean=False)),
           ('mean', dict(base, cs_cov_thresh=None, est_mean=True)),
           ('subsample', dict(base, cs_cov_thresh=cfg['cs_cov_thresh'], est_mean=False)),
           ('small_region', dict(base, region_size=cfg['small_region'], cs_cov_thresh=None,
                                 est_mean=False))]
    for i, desc in enumerate(cfg['motifs']):
        out.append(('motif%d' % i, dict(base, cs_cov_thresh=None, est_mean=False, motif=desc)))
    out.append(('valid_poss', dict(base, cs_cov_thresh=None, est_mean=False, motif='CG:1',
                                   valid_poss=True)))
    return out


def valid_poss_of(genome):
    """every C of a CpG on '+', and the G on '-', as parse_locs_file returns them"""
    cg = np.array([i for i in range(len(genome) - 1) if genome[i:i + 2] == 'CG'])
    return {('chr', '+'): cg, ('chr', '-'): cg + 1}


def flatten(all_reg_kmer_levels):
    """per region and key (in dict order): counts, and the rows concatenated"""
    counts = np.array([[len(v) for v in reg.values()] for reg in all_reg_kmer_levels], dtype=np.int64)
    rows = [np.asarray(v, dtype=np.float64).reshape(-1, 2) for reg in all_reg_kmer_levels for v in reg.values()]
    return counts, (np.concatenate(rows) if rows else np.zeros((0, 2)))


U = 2.0 ** -53


def gamma(n):
    return n * U / (1 - n * U)


def order_tol(order, sd):
    """per-row bound between a summary in read order and the reference's in its own order:
    0 where the reference used read order; else 2 gamma_{n+2} (sum|x| / n + sd) -- the mean's
    summation error is gamma_n sum|x| / n in either order, and the sd's is that plus
    (gamma_{n+1} / 2 + 2u) sd (DESIGN.md §2)"""
    same, n, absmean = order[:, 0], order[:, 1], order[:, 2]
    return np.where(same > 0, 0.0, 2 * gamma(n + 2) * (absmean + np.abs(sd)))


def message(stderr):
    """the message of a reference error / warning banner"""
    return str(stderr).split('********************\n\t', 1)[1]
