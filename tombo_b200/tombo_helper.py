"""Data model and thin native wrappers of the resquiggle hot path -- the part of
``tombo.tombo_helper`` the path needs (tombo_helper.py:67-337, 526-563), with the
Cython wrappers (:76-102) re-bound to the CUDA library through the C ABI.

FAST5 / index / HDF5 machinery of the reference module is out of scope (SURVEY.md
section 2, row 8)."""
import re
from collections import namedtuple

import os
import sys

import numpy as np

from . import _lib
from ._default_parameters import DNA_SAMP_TYPE, RNA_SAMP_TYPE  # noqa: F401

__all__ = [
    'TomboError', 'readData', 'TomboMotif', 'resquiggleParams', 'startClipParams',
    'stallParams', 'resquiggleResults', 'alignInfo', 'genomeLocation', 'sequenceData',
    'channelInfo', 'dpResults', 'scaleValues', 'seqSampleType', 'regionStats', 'groupStats',
    'get_seq_kmers', 'rev_comp', 'warning_message',
    'valid_cpts_w_cap', 'valid_cpts_w_cap_t_test', 'banded_traceback',
    'adaptive_banded_forward_pass', 'get_raw_read_slot', 'get_multiple_slots_read_centric']

SINGLE_LETTER_CODE = {
    'A': 'A', 'C': 'C', 'G': 'G', 'T': 'T', 'B': '[CGT]', 'D': '[AGT]', 'H': '[ACT]',
    'K': '[GT]', 'M': '[AC]', 'N': '[ACGT]', 'R': '[AG]', 'S': '[CG]', 'V': '[ACG]',
    'W': '[AT]', 'Y': '[CT]'}
INVALID_BASES = re.compile('[^ACGT]')
INVALID_BASE_RUNS = re.compile('[^ACGT]+')


class TomboError(Exception):
    """tombo_helper.py:67"""
    pass


def warning_message(message):
    """tombo_helper.py:350-355"""
    sys.stderr.write('*' * 20 + ' WARNING ' + '*' * 20 + '\n\t' + message + '\n')
    sys.stderr.flush()


def _raise_status(st):
    if st != 0:
        raise TomboError(_lib.status_message(st))


# ---- namedtuples (field lists identical to tombo_helper.py:109-337) ----------
class alignInfo(namedtuple('alignInfo', (
        'ID', 'Subgroup', 'ClipStart', 'ClipEnd', 'Insertions', 'Deletions', 'Matches',
        'Mismatches'))):
    """Information from genomic read alignment (tombo_helper.py:109)"""


class readData(namedtuple('readData', (
        'start', 'end', 'filtered', 'read_start_rel_to_raw', 'strand', 'fn', 'corr_group',
        'rna', 'sig_match_score', 'mean_q_score', 'read_id'))):
    """Nanopore read meta-data (tombo_helper.py:126)"""


readData.__new__.__defaults__ = (None, None, None)


class scaleValues(namedtuple('scaleValues', (
        'shift', 'scale', 'lower_lim', 'upper_lim', 'outlier_thresh'))):
    """Signal normalisation scaling parameters (tombo_helper.py:160)"""


class resquiggleParams(namedtuple('resquiggleParams', (
        'match_evalue', 'skip_pen', 'bandwidth', 'max_half_z_score', 'running_stat_width',
        'min_obs_per_base', 'raw_min_obs_per_base', 'mean_obs_per_event', 'z_shift',
        'stay_pen', 'use_t_test_seg', 'band_bound_thresh', 'start_bw', 'start_save_bw',
        'start_n_bases'))):
    """Re-squiggle parameters (tombo_helper.py:173)"""


resquiggleParams.__new__.__defaults__ = (None, None, None)


class stallParams(namedtuple('stallParams', (
        'window_size', 'threshold', 'min_consecutive_obs', 'edge_buffer', 'lower_pctl',
        'upper_pctl', 'mini_window_size', 'n_windows'))):
    """Parameters to identify RNA stalls (tombo_helper.py:207)"""


stallParams.__new__.__defaults__ = (None,) * 4


class startClipParams(namedtuple('startClipParams', ('bandwidth', 'num_genome_bases'))):
    """tombo_helper.py:219"""


class resquiggleResults(namedtuple('resquiggleResults', (
        'align_info', 'genome_loc', 'genome_seq', 'mean_q_score', 'raw_signal',
        'channel_info', 'read_start_rel_to_raw', 'segs', 'scale_values', 'sig_match_score',
        'norm_params_changed', 'start_clip_bases', 'stall_ints'))):
    """Re-squiggle results (tombo_helper.py:229)"""


resquiggleResults.__new__.__defaults__ = (None,) * 9


class dpResults(namedtuple('dpResults', (
        'read_start_rel_to_raw', 'segs', 'ref_means', 'ref_sds', 'genome_seq'))):
    """Dynamic programming results (tombo_helper.py:255)"""


class genomeLocation(namedtuple('genomeLocation', ('Start', 'Strand', 'Chrom'))):
    """tombo_helper.py:268"""


class sequenceData(namedtuple('sequenceData', ('seq', 'id', 'mean_q_score'))):
    """tombo_helper.py:277"""


class channelInfo(namedtuple('channelInfo', (
        'offset', 'range', 'digitisation', 'number', 'sampling_rate'))):
    """tombo_helper.py:286"""


class regionStats(namedtuple('regionStats', (
        'reg_frac_standard_base', 'reg_poss', 'chrm', 'strand', 'start', 'reg_cov', 'ctrl_cov',
        'valid_cov'))):
    """Region statistics (tombo_helper.py:299-313)"""


class groupStats(namedtuple('groupStats', (
        'reg_stats', 'reg_poss', 'chrm', 'strand', 'start', 'reg_cov', 'ctrl_cov'))):
    """Level-comparison region statistics (tombo_helper.py:315-328)"""


class seqSampleType(namedtuple('seqSampleType', ('name', 'rev_sig'))):
    """tombo_helper.py:330"""


# ---- sequence helpers ----------------------------------------------------------
def get_seq_kmers(seq, kmer_width, rev_strand=False):
    """tombo_helper.py:526-540"""
    seq_kmers = [seq[i:i + kmer_width] for i in range(len(seq) - kmer_width + 1)]
    if rev_strand:
        seq_kmers = seq_kmers[::-1]
    return seq_kmers


_COMP = {'A': 'T', 'C': 'G', 'G': 'C', 'T': 'A', '[': ']', ']': '['}
_COMP_BASES = dict(zip(map(ord, 'ACGT'), map(ord, 'TGCA')))


def rev_comp(seq):
    """tombo_helper.py:375-378 (other characters are kept as they are)"""
    return seq.translate(_COMP_BASES)[::-1]


class TomboMotif(object):
    """Sequence motif with a (1-based) modified position (tombo_helper.py:542-640):
    ``raw_motif``, ``motif_len``, ``motif_pat``, ``rev_comp_pat``, ``is_palindrome``,
    ``mod_pos``, ``mod_base``."""

    def _parse_motif(self, raw_motif, rev_comp_motif=False):
        conv = ''.join(SINGLE_LETTER_CODE[letter] for letter in raw_motif)
        if rev_comp_motif:
            conv = ''.join(_COMP[c] for c in conv[::-1])
        return re.compile(conv)

    def __init__(self, raw_motif, mod_pos=None):
        invalid = [c for c in raw_motif if c not in SINGLE_LETTER_CODE]
        if invalid:
            raise TomboError('Invalid characters in motif: ' + ', '.join(invalid))
        self.raw_motif = raw_motif
        self.motif_len = len(raw_motif)
        self.motif_pat = self._parse_motif(raw_motif)
        self.rev_comp_pat = self._parse_motif(raw_motif, True)
        self.is_palindrome = self.motif_pat.pattern == self.rev_comp_pat.pattern
        self.mod_pos = mod_pos
        if mod_pos is None:
            self.mod_base = None
        else:
            if not 0 < mod_pos <= self.motif_len:
                raise TomboError('Invalid modified position for motif.')
            self.mod_base = raw_motif[mod_pos - 1]
            if INVALID_BASES.match(self.mod_base):
                raise TomboError('Modified base within motif must be a single base.')


# ---- native wrappers (tombo_helper.py:76-102) -> CUDA -----------------------------
def valid_cpts_w_cap(raw_signal, min_base_obs, running_stat_width, num_cpts):
    st, cpts = _lib.get_context().valid_cpts_w_cap(
        raw_signal, min_base_obs, running_stat_width, num_cpts)
    _raise_status(st)
    return cpts


def valid_cpts_w_cap_t_test(raw_signal, min_base_obs, running_stat_width, num_cpts):
    st, cpts = _lib.get_context().valid_cpts_w_cap(
        raw_signal, min_base_obs, running_stat_width, num_cpts, t_test=True)
    _raise_status(st)
    return cpts


def banded_traceback(fwd_pass_tb, event_starts, band_pos, band_boundary_thresh=-1):
    st, tb = _lib.get_context().banded_traceback(
        fwd_pass_tb, event_starts, band_pos, band_boundary_thresh)
    _raise_status(st)
    return tb


def adaptive_banded_forward_pass(
        fwd_pass, fwd_pass_tb, event_starts, event_means, r_ref_means, r_ref_sds, z_shift,
        skip_pen, stay_pen, start_seq_pos, mask_fill_z_score, do_winsorize_z,
        max_half_z_score, return_z_scores=False):
    """In place on ``fwd_pass`` / ``fwd_pass_tb`` / ``event_starts`` like
    c_adaptive_banded_forward_pass (_c_dynamic_programming.pyx:314-412)."""
    if return_z_scores:
        raise NotImplementedError('return_z_scores is a plotting debug aid of the reference')
    st = _lib.get_context().adaptive_banded_forward_pass(
        fwd_pass, fwd_pass_tb, event_starts, event_means, r_ref_means, r_ref_sds, z_shift,
        skip_pen, stay_pen, start_seq_pos, mask_fill_z_score, do_winsorize_z,
        max_half_z_score)
    _raise_status(st)


# ---- FAST5 accessors: the I/O seam of compute_alt_model_read_stats -------------
def get_raw_read_slot(fast5_data):
    """tombo_helper.py:1593 -- HDF5 is outside the hot path; callers with h5py data
    use the reference layout, in-memory callers patch this accessor."""
    try:
        return next(iter(fast5_data['/Raw/Reads'].values()))
    except Exception:
        raise TomboError('Raw data is not found in /Raw/Reads/Read_[read#]')


def get_multiple_slots_read_centric(r_data, slot_names, corr_grp=None):
    """tombo_helper.py:1627-1660 (read-centric Events columns)."""
    try:
        if not hasattr(r_data, 'fn'):
            events = r_data['/Analyses/' + corr_grp + '/Events']
        else:
            import h5py
            with h5py.File(r_data.fn, 'r') as h5:
                events = h5['/'.join(('/Analyses', r_data.corr_group, 'Events'))][:]
        return [events[name] for name in slot_names]
    except Exception:
        return [None] * len(slot_names)


# ---- FAST5 Events table: the output seam of the resquiggle path (SURVEY 8(f)-3) ----
EVENTS_DTYPE = [(str('norm_mean'), 'f8'), (str('norm_stdev'), 'f8'), (str('start'), 'u4'),
                (str('length'), 'u4'), (str('base'), 'S1')]   # tombo_helper.py:2361-2364


def events_table(rsqgl_res, compute_sd=False, norm_means=None, norm_stds=None, device=0):
    """The per-base ``Events`` table the reference stores (tombo_helper.py:2347-2364):
    norm_mean, norm_stdev (NaN unless ``compute_sd``), start, length, base.  The means
    (and standard deviations) are the device's c_new_means / c_new_mean_stds unless the
    caller already holds them (``tb2_resquiggle_batch`` returns ``norm_mean``)."""
    segs = np.asarray(rsqgl_res.segs, dtype=np.int64)
    n = segs.shape[0] - 1
    if norm_means is None or (compute_sd and norm_stds is None):
        ctx = _lib.get_context(device)
        if compute_sd:
            norm_means, norm_stds = ctx.new_mean_stds(rsqgl_res.raw_signal, segs)
        else:
            norm_means = ctx.new_means(rsqgl_res.raw_signal, segs)
    if len(rsqgl_res.genome_seq) != n or len(norm_means) != n:
        raise TomboError('Error computing new events')
    ev = np.empty(n, dtype=EVENTS_DTYPE)
    ev['norm_mean'] = norm_means
    ev['norm_stdev'] = norm_stds if compute_sd else np.nan
    ev['start'] = segs[:-1]
    ev['length'] = np.diff(segs)
    ev['base'] = np.frombuffer(rsqgl_res.genome_seq.encode('ascii'), dtype='S1')
    return ev


def new_fast5_group_layout(rsqgl_res, norm_type, event_data, rna=False, alignVals=None,
                           old_segs=None):
    """What write_new_fast5_group stores under ``/Analyses/<corr_grp>/<subgroup>``
    (tombo_helper.py:2386-2443) as plain data: ``(attrs, alignment_attrs, datasets,
    events_attrs)``; ``datasets`` maps 'Alignment/<name>' / 'Events' to arrays."""
    sv = rsqgl_res.scale_values
    attrs = [('status', 'success'), ('rna', rna)]
    if rsqgl_res.sig_match_score is not None:
        attrs.append(('signal_match_score', rsqgl_res.sig_match_score))
    attrs += [('shift', sv.shift), ('scale', sv.scale), ('norm_type', norm_type)]
    for name, val in (('lower_lim', sv.lower_lim), ('upper_lim', sv.upper_lim),
                      ('outlier_threshold', sv.outlier_thresh)):
        if val is not None:
            attrs.append((name, val))
    gl = rsqgl_res.genome_loc
    aln = [('mapped_start', gl.Start), ('mapped_end', gl.Start + len(rsqgl_res.segs) - 1),
           ('mapped_strand', gl.Strand), ('mapped_chrom', gl.Chrom)]
    ai = rsqgl_res.align_info
    if ai is not None:
        aln += [('clipped_bases_start', ai.ClipStart), ('clipped_bases_end', ai.ClipEnd),
                ('num_insertions', ai.Insertions), ('num_deletions', ai.Deletions),
                ('num_matches', ai.Matches), ('num_mismatches', ai.Mismatches)]
    datasets = []
    if alignVals is not None:
        r_vals, g_vals = zip(*alignVals)
        datasets.append(('Alignment/read_alignment', np.array(r_vals, dtype='S1')))
        datasets.append(('Alignment/genome_alignment', np.array(g_vals, dtype='S1')))
    if old_segs is not None:
        datasets.append(('Alignment/read_segments', np.asarray(old_segs)))
    datasets.append(('Events', event_data))
    return attrs, aln, datasets, [('read_start_rel_to_raw', rsqgl_res.read_start_rel_to_raw)]


def _is_hdf5_like(obj):
    """an already-open HDF5 file object (h5py.File or a stand-in with its interface)"""
    return hasattr(obj, 'create_group') or (hasattr(obj, '__getitem__') and hasattr(obj, 'attrs'))


def write_new_fast5_group(fast5_data, corr_grp_slot, rsqgl_res, norm_type, compute_sd,
                          alignVals=None, old_segs=None, rna=False, norm_means=None,
                          norm_stds=None):
    """tombo_helper.py:2341-2460 over any h5py-like object.  Like the reference, anything
    that is not an open file object (str, bytes, os.PathLike ...) is opened here with h5py
    (h5py itself is outside this package's requirements) and closed again on every path."""
    try:
        event_data = events_table(rsqgl_res, compute_sd, norm_means, norm_stds)
    except TomboError:
        raise
    except Exception:
        raise TomboError('Error computing new events')          # tombo_helper.py:2364-2366
    attrs, aln, datasets, ev_attrs = new_fast5_group_layout(
        rsqgl_res, norm_type, event_data, rna, alignVals, old_segs)
    do_close = False
    if not _is_hdf5_like(fast5_data):
        try:
            import h5py
            fn = os.fsdecode(fast5_data) if isinstance(fast5_data, (bytes, os.PathLike)) else fast5_data
            fast5_data = h5py.File(fn, 'r+')
            do_close = True
        except Exception:
            raise TomboError('Error opening file for new group writing. This should have '
                             'been caught during the alignment phase. Check that there are '
                             'no other tombo processes or processes accessing these HDF5 '
                             'files running simultaneously.')
    try:
        try:
            corr_subgrp = fast5_data['/Analyses'][corr_grp_slot].create_group(
                rsqgl_res.align_info.Subgroup)
            for k, v in attrs:
                corr_subgrp.attrs[k] = v
            corr_alignment = corr_subgrp.create_group('Alignment')
            for k, v in aln:
                corr_alignment.attrs[k] = v
            for name, data in datasets:
                if name == 'Events':
                    ds = corr_subgrp.create_dataset('Events', data=data, compression='gzip')
                    for k, v in ev_attrs:
                        ds.attrs[k] = v
                else:
                    corr_alignment.create_dataset(name.split('/', 1)[1], data=data,
                                                  compression='gzip')
        except Exception:
            raise TomboError('Error writing resquiggle information back into fast5 file.')
    finally:
        if do_close:
            try:
                fast5_data.close()
            except Exception:
                raise TomboError('Error closing fast5 file after writing resquiggle information.')
