"""``tombo filter``: rewrite the filtered flags of a resquiggle index (_filter_reads.py).

Every command loads the index next to ``fast5s_dir`` with the filtered reads kept, rewrites
the flags, and writes the index back, with the reads in the order the reference writes them.
Two commands have work for the device:

* ``filter_reads_for_stuck`` takes every read's dwell percentiles from
  ``tb2_dwell_percentiles``, in batches across the index;
* ``filter_reads_for_coverage`` takes every read's mid-read coverage from
  ``tb2_read_mid_coverage``.  The draw itself (``np.random.choice`` on the global RNG) stays
  on the host, so a seeded run filters the reads the reference filters.

The others are host logic.  Per-read FAST5 values are read through ``_open_fast5`` (and, for
the Events lengths, ``tombo_helper.get_multiple_slots_read_centric``); a read whose value
cannot be read counts as filtered, as in the reference.  ``ctx`` is any object with the
Context methods used here (default: the device's shared context)."""
from __future__ import division

import numpy as np

from . import _lib
from . import formats
from . import tombo_helper as th

NO_UNFILT_MESSAGE = 'No unfiltered reads present in current Tombo index.'
STUCK_BATCH_READS = 1 << 16          # reads per tb2_dwell_percentiles call


def _open_fast5(fn):
    import h5py
    return h5py.File(fn, 'r')


def _context(ctx, device):
    return ctx if ctx is not None else _lib.get_context(device)


def _load(fast5s_dir, corr_grp):
    index_fn = formats.index_filename(fast5s_dir, corr_grp)
    return formats.load_index(index_fn, fast5s_dir, corr_grp, remove_filtered=False)


def _write(fast5s_dir, corr_grp, reads_index):
    """replace_index + write_index_file (tombo_helper.py:1137-1187)"""
    if sum(len(x) for x in reads_index.values()) == 0:
        raise th.TomboError('Cannot replace with an empty index.')
    th.status_message('Saving Tombo reads index to file.')
    out = formats.ReadsIndex(fast5s_dir, corr_grp)
    for (chrm, strand), cs_reads in reads_index.items():
        for rd in cs_reads:
            out.add_read_data(chrm, strand, rd)
    return out.write_index_file()


def _filter_mess(num_filt_reads, prev_unfilt_reads, total_reads, fast5s_dir, filter_text):
    """print_filter_mess (_filter_reads.py:44-56)"""
    if prev_unfilt_reads == 0:
        raise th.TomboError(NO_UNFILT_MESSAGE)
    th.status_message(
        'Filtered {:d} reads ({:.1%} of previously filtered and '.format(
            num_filt_reads, float(num_filt_reads) / prev_unfilt_reads) +
        '{:.1%} of all valid reads)'.format(float(num_filt_reads) / total_reads) +
        ' reads due to ' + filter_text + ' filter from ' + fast5s_dir + '.')


def _filter_each(fast5s_dir, corr_grp, reads_index, is_filtered, filter_text):
    """the loop shared by the q-score, signal-matching and genome-location filters: filtered
    reads are kept as they are, every other read is tested, order unchanged"""
    filt = dict((cs, []) for cs in reads_index)
    num_filt, prev_unfilt, total = 0, 0, 0
    for cs, cs_reads in reads_index.items():
        for rd in cs_reads:
            total += 1
            if rd.filtered:
                filt[cs].append(rd)
                continue
            prev_unfilt += 1
            if is_filtered(cs, rd):
                num_filt += 1
                rd = rd._replace(filtered=True)
            filt[cs].append(rd)
    _filter_mess(num_filt, prev_unfilt, total, fast5s_dir, filter_text)
    return _write(fast5s_dir, corr_grp, filt)


def clear_filters(fast5s_dir, corr_grp):
    """_filter_reads.py:29-42"""
    reads_index = _load(fast5s_dir, corr_grp)
    th.status_message('Clearing all filters.')
    fn = _write(fast5s_dir, corr_grp, dict(
        (cs, [rd._replace(filtered=False) for rd in cs_reads])
        for cs, cs_reads in reads_index.items()))
    th.status_message('All filters successfully cleared!')
    return fn


def _read_lengths(rd):
    """the Events `length` column of one read, or None when it cannot be read"""
    try:
        lens = th.get_multiple_slots_read_centric(rd, ['length'])[0]
        if lens is None:
            return None
        lens = np.asarray(lens).astype(np.int64)
        return lens if lens.shape[0] > 0 else None   # np.percentile of nothing raises
    except Exception:
        return None


def filter_reads_for_stuck(fast5s_dir, corr_grp, obs_filter, ctx=None, device=0):
    """_filter_reads.py:58-96: a read is filtered when any np.percentile(lengths, pctl) >
    thresh of ``obs_filter`` ([[pctl, thresh]], see tombo_helper.parse_obs_filter)"""
    reads_index = _load(fast5s_dir, corr_grp)
    th.status_message('Filtering stuck reads.')
    pctl = [float(p) for p, _ in obs_filter]
    thresh = np.array([t for _, t in obs_filter], dtype=np.float64)
    todo = [(cs, i) for cs, cs_reads in reads_index.items()
            for i, rd in enumerate(cs_reads) if not rd.filtered]
    stuck = set()
    if todo and len(pctl):
        c = _context(ctx, device)
        for b0 in range(0, len(todo), STUCK_BATCH_READS):
            batch = todo[b0:b0 + STUCK_BATCH_READS]
            lens = [_read_lengths(reads_index[cs][i]) for cs, i in batch]
            ok = [k for k, l in enumerate(lens) if l is not None]
            stuck.update(batch[k] for k, l in enumerate(lens) if l is None)
            if not ok:
                continue
            off = np.zeros(len(ok) + 1, dtype=np.int64)
            off[1:] = np.cumsum([lens[k].shape[0] for k in ok])
            pv = c.dwell_percentiles(np.concatenate([lens[k] for k in ok]), off, pctl)
            hit = (pv > thresh[None, :]).any(axis=1)
            stuck.update(batch[k] for k, h in zip(ok, hit) if h)
    elif todo:
        stuck.update(b for b in todo if _read_lengths(reads_index[b[0]][b[1]]) is None)
    filt = {}
    num_filt, prev_unfilt, total = 0, 0, 0
    for cs, cs_reads in reads_index.items():
        out = []
        for i, rd in enumerate(cs_reads):
            total += 1
            if not rd.filtered:
                prev_unfilt += 1
                if (cs, i) in stuck:
                    num_filt += 1
                    rd = rd._replace(filtered=True)
            out.append(rd)
        filt[cs] = out
    _filter_mess(num_filt, prev_unfilt, total, fast5s_dir, 'observations per base')
    return _write(fast5s_dir, corr_grp, filt)


def filter_reads_for_coverage(fast5s_dir, corr_grp, frac_to_filter, ctx=None, device=0):
    """_filter_reads.py:98-151: per (chrm, strand), reads already filtered go first; the rest
    follow, filtered at random with probability proportional to the coverage at their middle"""
    reads_index = _load(fast5s_dir, corr_grp)
    th.status_message('Filtering reads to obtain more uniform coverage.')
    filt = dict((cs, []) for cs in reads_index)
    groups = list(reads_index.items())
    total_reads = sum(len(r) for _, r in groups)
    unfilt_reads = []
    for cs, cs_reads in groups:
        filt[cs].extend(rd for rd in cs_reads if rd.filtered)
    for cs, cs_reads in groups:
        unfilt_reads.extend((cs, rd) for rd in cs_reads if not rd.filtered)
    prev_unfilt_reads = len(unfilt_reads)
    if prev_unfilt_reads == 0:
        raise th.TomboError(NO_UNFILT_MESSAGE)
    # coverage counts every read of the group, filtered ones included
    grp_off = np.zeros(len(groups) + 1, dtype=np.int64)
    grp_off[1:] = np.cumsum([len(r) for _, r in groups])
    start = np.array([rd.start for _, r in groups for rd in r], dtype=np.int64)
    end = np.array([rd.end for _, r in groups for rd in r], dtype=np.int64)
    mid = _context(ctx, device).read_mid_coverage(grp_off, start, end)
    unfilt_mask = np.array([not rd.filtered for _, r in groups for rd in r], dtype=bool)
    num_filt_reads = int(frac_to_filter * prev_unfilt_reads)
    _filter_mess(num_filt_reads, prev_unfilt_reads, total_reads, fast5s_dir, 'even coverage')
    unfilt_reads_cov = mid[unfilt_mask].astype(np.float64)
    unfilt_reads_p = unfilt_reads_cov / unfilt_reads_cov.sum()
    filt_indices = set(np.random.choice(
        prev_unfilt_reads, size=num_filt_reads, replace=False, p=unfilt_reads_p))
    for i, (cs, rd) in enumerate(unfilt_reads):
        if i in filt_indices:
            rd = rd._replace(filtered=True)
        filt[cs].append(rd)
    return _write(fast5s_dir, corr_grp, filt)


def filter_reads_for_qscore(fast5s_dir, bc_grp, corr_grp, q_score_thresh, ctx=None, device=0):
    """_filter_reads.py:153-194 (host only; ctx and device are accepted for a uniform call)"""
    def fails(rd):
        if rd.mean_q_score is not None:
            return rd.mean_q_score < q_score_thresh
        try:
            with _open_fast5(rd.fn) as fast5_data:
                r_q_scores = fast5_data['/Analyses/' + bc_grp + '/' + rd.corr_group.split('/')[-1] +
                                        '/Fastq'][:].decode().split('\n')[3]
                return th.get_mean_q_score(r_q_scores) < q_score_thresh
        except Exception:
            return True
    reads_index = _load(fast5s_dir, corr_grp)
    th.status_message('Filtering reads below a mean q-score cutoff.')
    return _filter_each(fast5s_dir, corr_grp, reads_index, lambda cs, rd: fails(rd), 'q-score')


def filter_reads_for_signal_matching(fast5s_dir, corr_grp, sig_match_thresh, ctx=None, device=0):
    """_filter_reads.py:196-235 (host only)"""
    def fails(rd):
        if rd.sig_match_score is not None:
            return rd.sig_match_score > sig_match_thresh
        try:
            with _open_fast5(rd.fn) as fast5_data:
                return fast5_data['/Analyses/' + rd.corr_group].attrs.get(
                    'signal_match_score') > sig_match_thresh
        except Exception:
            return True
    reads_index = _load(fast5s_dir, corr_grp)
    th.status_message('Filtering reads above a signal matching score threshold.')
    return _filter_each(fast5s_dir, corr_grp, reads_index, lambda cs, rd: fails(rd),
                        'signal matching')


def filter_reads_for_genome_pos(fast5s_dir, corr_grp, include_regs, include_partial=False,
                                ctx=None, device=0):
    """_filter_reads.py:237-280: ``include_regs`` {chrm: [(start, end)] or None}"""
    def included(start, end, regs):
        if regs is None:
            return True
        if include_partial:
            return any(not (start > i_end or end < i_start) for i_start, i_end in regs)
        return any(start >= i_start and end <= i_end for i_start, i_end in regs)

    def fails(cs, rd):
        chrm = cs[0]
        return chrm not in include_regs or not included(rd.start, rd.end, include_regs[chrm])
    reads_index = _load(fast5s_dir, corr_grp)
    th.status_message('Filtering reads outside of the specified genomic location.')
    return _filter_each(fast5s_dir, corr_grp, reads_index, fails, 'genomic position')
