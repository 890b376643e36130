"""``tombo.tombo_stats`` surface of the resquiggle hot path, bound to the CUDA
library: k-mer models, signal normalisation, base means, sequence based rescaling,
parameter loading and per-read alternative-model log-likelihood ratios
(tombo_stats.py:203-573, 580-1123, 1505-1597, 2327-2370, 3888-4082).

Everything numeric runs in CUDA kernels through the C ABI (include/tombo_b200.h);
what the reference itself does in plain Python (parameter tuples, dict look-ups,
regex motif search, a two-line numpy score) stays plain Python here."""
import io
import itertools
import re

import numpy as np

from . import _lib
from . import tombo_helper as th
from ._default_parameters import (
    ALGN_PARAMS_TABLE, SEG_PARAMS_TABLE, RNA_SAMP_TYPE, DNA_SAMP_TYPE,
    MIN_EVENT_TO_SEQ_RATIO, OCLLHR_SCALE, OCLLHR_HEIGHT, OCLLHR_POWER, STALL_PARAMS,
    FM_OFFSET_DEFAULT, SMALLEST_PVAL, MEAN_PRIOR_CONST, SD_PRIOR_CONST, ALT_EST_BATCH,
    MAX_KMER_OBS, MIN_KMER_OBS_TO_EST)

__all__ = [
    'TomboModel', 'AltModel', 'normalize_raw_signal', 'compute_base_means',
    'get_read_seg_score', 'calc_kmer_fitted_shift_scale', 'load_resquiggle_parameters',
    'compute_num_events', 'get_dynamic_prog_params', 'identify_stalls',
    'compute_alt_model_read_stats', 'compute_alt_model_reads_stats', 'trim_seq_and_means', 'apply_per_read_thresh',
    'collate_reg_stats', 'calc_damp_fraction', 'calc_window_fishers_method',
    'compute_de_novo_read_stats', 'compute_sample_compare_read_stats',
    'compute_ks_tests', 'compute_u_tests', 'compute_t_tests', 'calc_window_means',
    'compute_group_reg_stats', 'get_reads_ref', 'compute_posterior_samp_dists',
    'parse_base_levels', 'est_kernel_density', 'write_kmer_densities_file',
    'parse_kmer_densities_file', 'isolate_alt_density']

# E|N(0,1)| = sqrt(2 / pi); the reference evaluates scipy.stats.halfnorm.expect()
# (tombo_stats.py:84), which returns this value (SURVEY.md 8c-2)
HALF_NORM_EXPECTED_VAL = float(np.sqrt(2.0 / np.pi))
STANDARD_MODEL_NAME = 'standard'
CONST_SD_MODEL = True                     # tombo_stats.py:112
SAMP_COMP_TXT, DE_NOVO_TXT, ALT_MODEL_TXT = 'sample_compare', 'de_novo', 'model_compare'   # :89-91
KS_TEST_TXT, U_TEST_TXT, T_TEST_TXT = 'ks_test', 'u_test', 't_test'                  # :95-97
KS_STAT_TEST_TXT, U_STAT_TEST_TXT, T_STAT_TEST_TXT = 'ks_stat_test', 'u_stat_test', 't_stat_test'
LEVEL_STATS_TXTS = (KS_TEST_TXT, U_TEST_TXT, T_TEST_TXT,
                    KS_STAT_TEST_TXT, U_STAT_TEST_TXT, T_STAT_TEST_TXT)               # :101-103
NORM_TYPES = ('none', 'pA', 'pA_raw', 'median', 'robust_median', 'median_const_scale')
_CODE = {'A': 0, 'C': 1, 'G': 2, 'T': 3}


def _kmer_code(kmer):
    idx = 0
    for b in kmer:
        idx = idx * 4 + _CODE[b]
    return idx


class TomboModel(object):
    """Canonical k-mer model (tombo_stats.py:580-919).  Built from ``kmer_ref`` (a
    list of ``(kmer, mean, sd)``) and ``central_pos``; model files need h5py and
    are outside the hot path."""

    def __init__(self, ref_fn=None, is_text_model=False, kmer_ref=None, central_pos=None,
                 seq_samp_type=None, reads_index=None, fast5_fns=None, minimal_startup=True):
        if kmer_ref is None:
            raise th.TomboError(
                'tombo_b200.TomboModel is initialised from kmer_ref=/central_pos= '
                '(model files are read by the reference with h5py)')
        assert central_pos is not None, (
            'central_pos must be provided is TomboModel is loaded with a kmer_ref')
        self.means, self.sds = {}, {}
        for kmer, kmer_mean, kmer_std in kmer_ref:
            try:
                kmer = kmer.decode()
            except AttributeError:
                pass
            self.means[kmer] = kmer_mean
            self.sds[kmer] = kmer_std
        self.central_pos = central_pos
        self.name = STANDARD_MODEL_NAME
        self.seq_samp_type = seq_samp_type
        self.kmer_width = len(next(k for k in self.means))
        self.inv_var = None
        if not minimal_startup:
            self.inv_var = dict((k, 1 / (s * s)) for k, s in self.sds.items())
        self._tables = None

    def tables(self):
        """dense (means, sds) indexed by the base-4 k-mer code (device layout)"""
        if self._tables is None:
            n = 4 ** self.kmer_width
            m, s = np.full(n, np.nan), np.full(n, np.nan)
            for k, v in self.means.items():
                if all(b in _CODE for b in k):
                    m[_kmer_code(k)] = v
                    s[_kmer_code(k)] = self.sds[k]
            self._tables = (m, s)
        return self._tables

    def reverse_sequence_copy(self):
        rev = TomboModel(kmer_ref=[(k[::-1], m, self.sds[k]) for k, m in self.means.items()],
                         central_pos=self.kmer_width - self.central_pos - 1,
                         seq_samp_type=self.seq_samp_type,
                         minimal_startup=self.inv_var is None)
        return rev

    def get_exp_levels_from_seq(self, seq, rev_strand=False):
        """tombo_stats.py:834-862"""
        seq_kmers = th.get_seq_kmers(seq, self.kmer_width, rev_strand)
        return self.get_exp_levels_from_kmers(seq_kmers)

    def get_exp_levels_from_kmers(self, seq_kmers):
        """tombo_stats.py:864-884"""
        try:
            ref_means = np.array([self.means[kmer] for kmer in seq_kmers])
            ref_sds = np.array([self.sds[kmer] for kmer in seq_kmers])
        except KeyError:
            raise th.TomboError('Invalid sequence encountered from genome sequence.')
        return ref_means, ref_sds

    def get_exp_levels_from_seq_with_gaps(self, reg_seq, rev_strand):
        """tombo_stats.py:886-918: expected levels of every k-mer of ``reg_seq``; NaN for
        k-mers that touch a non-ACGT base"""
        n = len(reg_seq) - self.kmer_width + 1
        ref_means, ref_sds = np.full(n, np.nan), np.full(n, np.nan)
        prev = 0
        for m in list(th.INVALID_BASE_RUNS.finditer(reg_seq)) + [None]:
            stop = len(reg_seq) if m is None else m.start()
            if stop - prev >= self.kmer_width:
                sm, ss = self.get_exp_levels_from_seq(reg_seq[prev:stop])
                ref_means[prev:stop - self.kmer_width + 1] = sm
                ref_sds[prev:stop - self.kmer_width + 1] = ss
            if m is not None:
                prev = m.end()
        if rev_strand:
            ref_means, ref_sds = ref_means[::-1], ref_sds[::-1]
        return ref_means, ref_sds


class AltModel(object):
    """Alternative-base k-mer model (tombo_stats.py:922-1123), from ``kmer_ref`` rows
    ``(kmer, pos, mean, sd)``."""

    def __init__(self, ref_fn=None, kmer_ref=None, central_pos=None, alt_base=None, name=None,
                 motif=None, minimal_startup=True):
        if kmer_ref is None:
            raise th.TomboError('tombo_b200.AltModel is initialised from kmer_ref=')
        assert central_pos is not None and alt_base is not None, (
            'central_pos and alt_base must be provided if AltModel is loaded with a kmer_ref')
        self.means, self.sds = {}, {}
        for kmer, pos, kmer_mean, kmer_std in kmer_ref:
            try:
                kmer = kmer.decode()
            except AttributeError:
                pass
            self.means[(kmer, pos)] = kmer_mean
            self.sds[(kmer, pos)] = kmer_std
        self.central_pos = central_pos
        self.alt_base = alt_base
        self.name = name
        if motif is None:
            self.motif = th.TomboMotif(self.alt_base, 1)
        else:
            assert isinstance(motif, th.TomboMotif) and motif.mod_pos is not None
            self.motif = motif
        self.kmer_width = len(next(kmer for kmer, pos in self.means))
        self.inv_var = None
        self._table = None

    def table(self):
        """dense alt means [code, pos] (NaN where absent) -- the device layout"""
        if self._table is None:
            t = np.full((4 ** self.kmer_width, self.kmer_width), np.nan)
            for (k, pos), v in self.means.items():
                t[_kmer_code(k), pos] = v
            self._table = t
        return self._table

    def get_exp_level(self, kmer, pos):
        return self.means.get((kmer, pos), np.nan)

    def get_exp_sd(self, kmer, pos):
        return self.sds.get((kmer, pos), np.nan)

    def get_exp_levels_from_kmers(self, seq_kmers, rev_strand=False):
        """tombo_stats.py:1096-1123"""
        pos_range = (range(self.kmer_width) if rev_strand
                     else range(self.kmer_width - 1, -1, -1))
        ref_means = np.array([self.get_exp_level(k, p) for k, p in zip(seq_kmers, pos_range)])
        ref_sds = np.array([self.get_exp_sd(k, p) for k, p in zip(seq_kmers, pos_range)])
        return ref_means, ref_sds


# ---------------------------------------------------------------------------
# signal normalisation (tombo_stats.py:203-233, 482-573)
# ---------------------------------------------------------------------------
def compute_base_means(all_raw_signal, base_starts):
    """c_new_means over ``base_starts`` (tombo_stats.py:203-215)"""
    return _lib.get_context().new_means(
        np.asarray(all_raw_signal).astype(np.float64), base_starts)


def normalize_raw_signal(
        all_raw_signal, read_start_rel_to_raw=0, read_obs_len=None, norm_type='median',
        outlier_thresh=None, channel_info=None, scale_values=None, event_means=None,
        model_means=None, model_inv_vars=None, const_scale=None):
    """tombo_stats.py:482-573 for the normalisation types the resquiggle path uses:
    ``median``, ``median_const_scale`` and provided ``scale_values``."""
    if read_obs_len is None:
        read_obs_len = all_raw_signal.shape[0] - read_start_rel_to_raw
    if norm_type not in NORM_TYPES and scale_values is None:
        raise th.TomboError(
            'Normalization type ' + norm_type + ' is not a valid option and shift or scale '
            'parameters were not provided.')
    raw_signal = all_raw_signal[read_start_rel_to_raw:read_start_rel_to_raw + read_obs_len]
    if scale_values is None and norm_type not in ('median', 'median_const_scale'):
        raise NotImplementedError(
            'norm_type ' + norm_type + ' is not on the resquiggle path (SURVEY.md 8a)')
    if scale_values is None and norm_type == 'median_const_scale':
        assert const_scale is not None
    st, norm, sv = _lib.get_context().normalize_raw_signal(
        np.asarray(raw_signal, dtype=np.float64), outlier_thresh=outlier_thresh,
        scale_values=scale_values,
        const_scale=const_scale if (scale_values is None and
                                    norm_type == 'median_const_scale') else None)
    if st == 100:
        raise FloatingPointError('divide by zero encountered in signal normalization')
    th._raise_status(st)
    none = lambda v: None if np.isnan(v) else v   # noqa: E731
    return norm, th.scaleValues(sv[0], sv[1], none(sv[2]), none(sv[3]), outlier_thresh)


def identify_stalls(all_raw_signal, stall_params=None, return_metric=False):
    """Mean-window stall detection (tombo_stats.py:269-368 with MEAN_STALL_PARAMS)."""
    if return_metric:
        raise NotImplementedError('return_metric is a plotting debug aid of the reference')
    if stall_params is not None:
        d = dict(STALL_PARAMS)
        given = dict((k, getattr(stall_params, k)) for k in d)
        if given != d:
            raise NotImplementedError('only the default mean-window stall parameters')
    ints = _lib.get_context().identify_stalls(np.asarray(all_raw_signal, dtype=np.float64))
    return [list(map(int, iv)) for iv in ints]


def calc_kmer_fitted_shift_scale(
        prev_shift, prev_scale, r_event_means, r_model_means, r_model_inv_vars=None,
        method='theil_sen', subsample_key=0):
    """Theil-Sen sequence based rescaling (tombo_stats.py:370-450).  Reads with more
    than MAX_POINTS_FOR_THEIL_SEN bases are sub-sampled with a keyed bijection
    (``subsample_key``) instead of the reference's unseeded np.random.choice."""
    if method != 'theil_sen':
        raise NotImplementedError('only method="theil_sen" is on the resquiggle path')
    st, out = _lib.get_context().theil_sen(
        prev_shift, prev_scale, r_event_means, r_model_means, subsample_key)
    th._raise_status(st)
    return out


def get_read_seg_score(r_means, r_ref_means, r_ref_sds):
    """tombo_stats.py:2327-2338 (a numpy one-liner in the reference too)"""
    return np.mean(np.abs((r_means - r_ref_means) / r_ref_sds))


def get_dynamic_prog_params(match_evalue):
    """tombo_stats.py:2364-2370"""
    return HALF_NORM_EXPECTED_VAL + match_evalue, match_evalue


def load_resquiggle_parameters(seq_samp_type, sig_aln_params=None, seg_params=None,
                               use_save_bandwidth=False):
    """tombo_stats.py:1505-1556"""
    if sig_aln_params is None:
        (match_evalue, skip_pen, bandwidth, save_bandwidth, max_half_z_score, band_bound_thresh,
         start_bw, start_save_bw, start_n_bases) = ALGN_PARAMS_TABLE[seq_samp_type.name]
    else:
        (match_evalue, skip_pen, bandwidth, save_bandwidth, max_half_z_score, band_bound_thresh,
         start_bw, start_save_bw, start_n_bases) = sig_aln_params
        bandwidth, save_bandwidth = int(bandwidth), int(save_bandwidth)
        band_bound_thresh, start_bw = int(band_bound_thresh), int(start_bw)
        start_save_bw, start_n_bases = int(start_save_bw), int(start_n_bases)
    if use_save_bandwidth:
        bandwidth = save_bandwidth
    if seg_params is None:
        (running_stat_width, min_obs_per_base, raw_min_obs_per_base,
         mean_obs_per_event) = SEG_PARAMS_TABLE[seq_samp_type.name]
    else:
        (running_stat_width, min_obs_per_base, raw_min_obs_per_base,
         mean_obs_per_event) = seg_params
    z_shift, stay_pen = get_dynamic_prog_params(match_evalue)
    return th.resquiggleParams(
        match_evalue, skip_pen, bandwidth, max_half_z_score, running_stat_width,
        min_obs_per_base, raw_min_obs_per_base, mean_obs_per_event, z_shift, stay_pen,
        seq_samp_type.name == RNA_SAMP_TYPE, band_bound_thresh, start_bw, start_save_bw,
        start_n_bases)


def compute_num_events(signal_len, seq_len, mean_obs_per_event,
                       min_event_to_seq_ratio=MIN_EVENT_TO_SEQ_RATIO):
    """tombo_stats.py:1558-1574"""
    return max(signal_len // mean_obs_per_event, int(seq_len * min_event_to_seq_ratio))


# ---------------------------------------------------------------------------
# per-read alternative-model statistics (tombo_stats.py:3888-4082)
# ---------------------------------------------------------------------------
def _slice_padded(seq, lo, hi):
    """``seq[lo:hi]`` where positions outside the string read as 'N'"""
    return 'N' * max(0, -lo) + seq[max(0, lo):max(0, min(len(seq), hi))] + 'N' * max(0, hi - len(seq))


def trim_seq_and_means(seq, means, r_start, reg_start, reg_end, strand, kmer_width,
                       central_pos, max_motif_bb, max_motif_ab):
    """Clip a read's sequence / base levels to a region (tombo_stats.py:3888-3970).

    Returns ``(kmers, means, r_start, motif_search_seq)``: the k-mers and levels of the
    positions that have a full k-mer inside ``[reg_start - (K-1), reg_end + (K-1))``, the
    genome position of the first testable base, and the sequence window motif searches
    run over (padded with 'N' where a motif would reach outside the read).

    Everything is expressed through two overhangs -- how far the read sticks out of the
    region on the genome's low and high side -- mapped to the read's 5' / 3' end by strand.
    Two slicing quirks of the reference are kept on purpose (they decide which reads raise):
    a zero-width trailing trim empties the array (``x[:-0]``)."""
    flank = kmer_width - 1
    low_over = max(0, reg_start - (r_start + flank))
    high_over = max(0, (r_start + means.shape[0] - flank) - reg_end)
    clip5, clip3 = (low_over, high_over) if strand == '+' else (high_over, low_over)
    if low_over > 0:
        r_start = reg_start - flank
    trimmed_seq = seq[clip5:max(0, len(seq) - clip3)]
    tail = clip3 + kmer_width - central_pos - 1
    trimmed_means = means[clip5 + central_pos:]
    trimmed_means = trimmed_means[:max(0, trimmed_means.shape[0] - tail)] if tail else trimmed_means[:0]
    if trimmed_means.shape[0] < kmer_width:
        raise th.TomboError('Read sequence too short in this region.')
    kmers = th.get_seq_kmers(trimmed_seq, kmer_width)
    if len(kmers) != trimmed_means.shape[0]:
        raise th.TomboError('Mismatching k-mer and mean levels.')
    # motif window: from max_motif_bb bases before the first testable base to
    # max_motif_ab bases after the last one
    lead = clip5 + flank - max_motif_bb
    trail = clip3 + flank - max_motif_ab
    window = _slice_padded(seq, lead, len(seq) - trail) if trail else ''
    return kmers, trimmed_means, r_start + flank, window


def compute_alt_model_read_stats(r_data, std_ref, alt_refs, use_standard_llhr=False,
                                 reg_data=None):
    """tombo_stats.py:3972-4082.  Read data arrive through
    ``tombo_helper.get_multiple_slots_read_centric`` / ``get_raw_read_slot`` (the
    FAST5 seam, :4013-4016); every site's k-mer window is scored on the GPU."""
    reg_start = reg_data.start if reg_data is not None else r_data.start
    reg_end = reg_data.end if reg_data is not None else r_data.end
    max_motif_bb = max([alt_ref.motif.mod_pos - 1 for _, alt_ref in alt_refs])
    max_motif_ab = max([alt_ref.motif.motif_len - alt_ref.motif.mod_pos
                        for _, alt_ref in alt_refs])
    r_means, r_seq = th.get_multiple_slots_read_centric(
        r_data, ['norm_mean', 'base'], r_data.corr_group)
    try:
        read_id = th.get_raw_read_slot(r_data).attrs.get('read_id')
    except Exception:
        read_id = getattr(r_data, 'read_id', None)
    if r_means is None or r_seq is None:
        raise th.TomboError('Read does not contain valid re-squiggled data.')
    r_seq = b''.join(r_seq).decode() if not isinstance(r_seq, str) else r_seq
    r_kmers, r_means, r_start, motif_search_seq = trim_seq_and_means(
        r_seq, np.asarray(r_means, dtype=np.float64), r_data.start, reg_start, reg_end,
        r_data.strand, std_ref.kmer_width, std_ref.central_pos, max_motif_bb, max_motif_ab)
    K = std_ref.kmer_width
    testable_len = r_means.shape[0] - K + 1
    r_ref_means, r_ref_sds = std_ref.get_exp_levels_from_kmers(r_kmers)
    r_ref_vars = np.square(r_ref_sds)
    ctx = _lib.get_context()
    all_poss, all_llhrs = {}, {}
    win = np.arange(K)
    for alt_name, alt_ref in alt_refs:
        search = motif_search_seq[max_motif_bb - (alt_ref.motif.mod_pos - 1):]
        trim_end = max_motif_ab - (alt_ref.motif.motif_len - alt_ref.motif.mod_pos)
        if trim_end > 0:
            search = search[:-trim_end]
        alt_poss = np.array([m.start() for m in alt_ref.motif.motif_pat.finditer(search)],
                            dtype=np.int64)
        if r_data.strand == '+':
            gen_poss = r_start + alt_poss
        else:
            gen_poss = r_start + testable_len - alt_poss - 1
        if alt_poss.shape[0] == 0:
            all_llhrs[alt_name], all_poss[alt_name] = np.array([]), np.array([])
            continue
        idx = alt_poss[:, None] + win[None, :]
        means_w = r_means[idx]
        ref_w = r_ref_means[idx]
        alt_w = np.array([alt_ref.get_exp_levels_from_kmers(r_kmers[p:p + K])[0]
                          for p in alt_poss])
        if CONST_SD_MODEL:
            mode = 1 if use_standard_llhr else 0
            llhrs = ctx.calc_llh_ratio_windows(mode, means_w, ref_w, alt_w, r_ref_vars[alt_poss],
                                               None, OCLLHR_SCALE, OCLLHR_HEIGHT, OCLLHR_POWER)
        else:
            if not use_standard_llhr:
                raise th.TomboError('Variable SD scaled likelihood ratio not implemented.')
            alt_v = np.array([np.square(alt_ref.get_exp_levels_from_kmers(
                r_kmers[p:p + K])[1]) for p in alt_poss])
            llhrs = ctx.calc_llh_ratio_windows(2, means_w, ref_w, alt_w, r_ref_vars[idx], alt_v)
        all_llhrs[alt_name] = llhrs
        all_poss[alt_name] = gen_poss
    return all_llhrs, all_poss, read_id


_BASE_CODE = np.full(256, 255, dtype=np.uint8)
_BASE_CODE[np.frombuffer(b'ACGT', dtype=np.uint8)] = np.arange(4, dtype=np.uint8)


def compute_alt_model_reads_stats(r_datas, std_ref, alt_refs, use_standard_llhr=False,
                                  reg_data=None, device=0):
    """Batched :func:`compute_alt_model_read_stats`: every read of ``r_datas`` (either strand)
    against every alt model of ``alt_refs`` (any ``TomboMotif``), clipped to ``reg_data``
    (None: whole reads), in one device call per alt model.  Read data arrive through the same
    FAST5 seam.  Returns, per read, ``(all_llhrs, all_poss, read_id)`` or the
    :class:`tombo_helper.TomboError` the reference would raise for that read.

    Two whole-read checks run before the region clip, where the reference would first clip
    and then look up levels: a read with a non-ACGT base anywhere fails with 'Invalid
    sequence encountered from genome sequence.' even if the region would clip that base
    away, and a read whose base and level counts differ fails with 'Mismatching k-mer and
    mean levels.' before it could be found too short.  Non-ACGT reference bases are outside
    what the device batch accepts; resquiggled reads always carry one level per base."""
    K, cpos = std_ref.kmer_width, std_ref.central_pos
    max_motif_bb = max([alt_ref.motif.mod_pos - 1 for _, alt_ref in alt_refs])
    max_motif_ab = max([alt_ref.motif.motif_len - alt_ref.motif.mod_pos
                        for _, alt_ref in alt_refs])
    out = [None] * len(r_datas)
    means, codes, starts, strands, ids, idx = [], [], [], [], [], []
    for i, r_data in enumerate(r_datas):
        r_means, r_seq = th.get_multiple_slots_read_centric(
            r_data, ['norm_mean', 'base'], r_data.corr_group)
        try:
            read_id = th.get_raw_read_slot(r_data).attrs.get('read_id')
        except Exception:
            read_id = getattr(r_data, 'read_id', None)
        if r_means is None or r_seq is None:
            out[i] = th.TomboError('Read does not contain valid re-squiggled data.')
            continue
        r_seq = b''.join(r_seq) if not isinstance(r_seq, str) else r_seq.encode()
        c = _BASE_CODE[np.frombuffer(r_seq, dtype=np.uint8)]
        if (c > 3).any():
            # non-ACGT bases: the reference fails the k-mer level look-up
            out[i] = th.TomboError('Invalid sequence encountered from genome sequence.')
            continue
        r_means = np.asarray(r_means, dtype=np.float64)
        if c.shape[0] != r_means.shape[0]:
            out[i] = th.TomboError('Mismatching k-mer and mean levels.')
            continue
        # the library's layout: nb + K - 1 codes, the read's bases cpos codes in
        means.append(r_means)
        codes.append(np.concatenate([np.zeros(cpos, np.uint8), c,
                                     np.zeros(K - 1 - cpos, np.uint8)]))
        starts.append(r_data.start)
        strands.append(0 if r_data.strand == '+' else 1)
        ids.append(read_id)
        idx.append(i)
    if not idx:
        return out
    nbs = np.array([m.shape[0] for m in means], dtype=np.int64)
    starts = np.array(starts, dtype=np.int64)
    if reg_data is not None:
        reg_start, reg_end = reg_data.start, reg_data.end
    else:
        # a region that contains every read leaves each one whole
        reg_start, reg_end = int(starts.min()), int((starts + nbs).max())
    norm_mean = np.concatenate(means)
    mean_off = np.concatenate([[0], np.cumsum(nbs)]).astype(np.int64)
    seq = np.concatenate(codes)
    seq_off = np.concatenate([[0], np.cumsum(nbs + K - 1)]).astype(np.int64)
    strands = np.array(strands, dtype=np.int8)
    ctx = _lib.get_context(device)
    _lib.ensure_model(ctx, std_ref)
    per_read = [({}, {}) for _ in idx]
    status = None
    for alt_name, alt_ref in alt_refs:
        ctx.set_alt_model(alt_ref.table(), alt_ref.kmer_width)
        llr, pos, off, status = ctx.alt_model_llr_motif_batch(
            norm_mean, mean_off, seq, seq_off, starts, strands,
            _lib.motif_struct(alt_ref.motif), max_motif_bb, max_motif_ab, reg_start, reg_end,
            use_standard_llhr, OCLLHR_SCALE, OCLLHR_HEIGHT, OCLLHR_POWER)
        for j in range(len(idx)):
            a, b = int(off[j]), int(off[j + 1])
            per_read[j][0][alt_name] = llr[a:b] if b > a else np.array([])
            per_read[j][1][alt_name] = pos[a:b] if b > a else np.array([])
    for j, i in enumerate(idx):
        if status[j] != 0:
            out[i] = th.TomboError(_lib.status_message(status[j]))
        else:
            out[i] = (per_read[j][0], per_read[j][1], ids[j])
    return out


# ---------------------------------------------------------------------------
# SURVEY 8(f)-1: per-position aggregation (tombo_stats.py:4084-4178, 2537-2552)
# ---------------------------------------------------------------------------
def _region_counts(stats, stat_locs, single_read_thresh, lower_thresh, stat_type, device=0):
    """dense-counter aggregation of (position, statistic) pairs on the device"""
    ctx = _lib.get_context(device)
    stat_locs = np.asarray(stat_locs, dtype=np.int64)
    lo, hi = int(stat_locs.min()), int(stat_locs.max())
    ctx.region_stats_begin(lo, hi - lo + 1)
    ctx.region_stats_add(stats, stat_locs, single_read_thresh, lower_thresh,
                         0 if stat_type == ALT_MODEL_TXT else 1)
    return ctx.region_stats_finalize()


def apply_per_read_thresh(reg_base_stats, single_read_thresh, lower_thresh, stat_type,
                          stat_locs, ctrl_cov=None):
    """tombo_stats.py:4084-4122 -> (reg_frac_std_base, reg_cov, ctrl_cov, valid_cov).
    ``reg_base_stats`` is the per-position list of statistic arrays the reference builds;
    thresholds and counts run on the device."""
    n_pos = len(reg_base_stats)
    lens = np.array([b.shape[0] for b in reg_base_stats], dtype=np.int64)
    flat = np.concatenate(reg_base_stats) if n_pos else np.zeros(0)
    agg = _region_counts(flat, np.repeat(np.arange(n_pos, dtype=np.int64), lens),
                         single_read_thresh, lower_thresh, stat_type) if flat.shape[0] else None
    frac = np.full(n_pos, np.nan)
    reg_cov = lens.copy()
    valid_cov = np.zeros(n_pos, dtype=np.int64)
    if agg is not None:
        frac[agg['pos']] = agg['frac']
        valid_cov[agg['pos']] = agg['valid_cov']
    if stat_type == SAMP_COMP_TXT:
        ctrl_cov = [ctrl_cov[pos] if ctrl_cov is not None and pos in ctrl_cov else 0
                    for pos in stat_locs]
    else:
        ctrl_cov = [0] * int(np.asarray(stat_locs).shape[0])
    return frac, reg_cov, ctrl_cov, valid_cov


def collate_reg_stats(stats, stat_locs, read_ids, per_read_q, reg_data, single_read_thresh,
                      lower_thresh, stat_type, stat_name, ctrl_cov):
    """tombo_stats.py:4124-4178 -> :class:`tombo_helper.regionStats`.  The reference sorts
    the region's (position, statistic) pairs and splits them per position; here the pairs
    go to dense per-position counters on the device (a counting sort) and come back as the
    covered positions in ascending order.  ``per_read_q`` (the per-read statistics writer)
    is outside the hot path and must be None."""
    if per_read_q is not None:
        raise NotImplementedError('per-read statistics blocks are written by the reference')
    stats = np.concatenate(stats)
    stat_locs = np.concatenate(stat_locs).astype(np.int64)
    keep = ~np.isnan(stats)
    if not keep.any():
        raise th.TomboError('No valid positions in this region.')
    agg = _region_counts(stats, stat_locs, single_read_thresh, lower_thresh, stat_type)
    locs_sorted = np.sort(stat_locs[keep])
    if stat_type == SAMP_COMP_TXT:
        cc = [ctrl_cov[pos] if ctrl_cov is not None and pos in ctrl_cov else 0
              for pos in locs_sorted]
    else:
        cc = [0] * int(locs_sorted.shape[0])
    return th.regionStats(agg['frac'], agg['pos'], reg_data.chrm, reg_data.strand,
                          reg_data.start, agg['cov'], cc, agg['valid_cov'])


def calc_damp_fraction(cov_damp_counts, fracs, valid_cov):
    """tombo_stats.py:2537-2552 (elementwise; the device evaluates the same expression inside
    tb2_region_stats_finalize for the fused path)"""
    non_mod_counts = np.round(fracs * valid_cov)
    return (non_mod_counts + cov_damp_counts['unmod']) / (
        valid_cov + sum(list(cov_damp_counts.values())))


# ---------------------------------------------------------------------------
# SURVEY 8(f)-2: de novo / sample-compare per-read tests (tombo_stats.py:2252-2271,
# 3675-3873)
# ---------------------------------------------------------------------------
def calc_window_fishers_method(pvals, lag):
    """tombo_stats.py:2252-2271 on the device (1-D input): Fisher's method over a moving
    window of 2 * lag + 1 p-values; NaN in the first / last ``lag`` positions."""
    assert lag > 0, 'Invalid p-value window provided.'
    pvals = np.asarray(pvals, dtype=np.float64)
    if pvals.ndim != 1:
        raise NotImplementedError('1-D p-value vectors only')
    if pvals.shape[-1] < (lag * 2) + 1:
        raise th.TomboError("P-values vector too short for Fisher's Method window compuation.")
    return _lib.get_context().window_fisher_pvals(
        pvals, None, None, np.array([0, pvals.shape[0]]), lag, False)


def _clip_to_region(r_means, r_seq, read_start, read_end, strand, reg_start, reg_end, lo_lag,
                    hi_lag):
    """keep the part of a read whose statistics fall inside [reg_start, reg_end): the read may
    stick out by its low / high lag (k-mer context + Fisher window)"""
    low_over = max(0, reg_start - (read_start + lo_lag))
    high_over = max(0, (read_end - hi_lag) - reg_end)
    clip5, clip3 = (low_over, high_over) if strand == '+' else (high_over, low_over)
    n = r_means.shape[0]
    r_means = r_means[clip5:max(clip5, n - clip3)] if clip3 or clip5 else r_means
    if r_seq is not None:
        r_seq = r_seq[clip5:max(clip5, len(r_seq) - clip3)] if clip3 or clip5 else r_seq
    if low_over:
        read_start = reg_start - lo_lag
    if high_over:
        read_end = reg_end + hi_lag
    return r_means, r_seq, read_start, read_end


def compute_de_novo_read_stats(r_data, std_ref, fm_offset=FM_OFFSET_DEFAULT, reg_data=None):
    """tombo_stats.py:3771-3873 -> ({'de_novo': p-values}, {'de_novo': positions}, read_id).
    Read data arrive through ``tombo_helper.get_multiple_slots_read_centric`` /
    ``get_raw_read_slot`` (the FAST5 seam); z-scores, p-values and the Fisher window run on
    the device."""
    reg_start = reg_data.start if reg_data is not None else r_data.start
    reg_end = reg_data.end if reg_data is not None else r_data.end
    dnstrm = std_ref.kmer_width - std_ref.central_pos - 1
    begin_lag, end_lag = (std_ref.central_pos, dnstrm) if r_data.strand == '+' else \
        (dnstrm, std_ref.central_pos)
    r_means, r_seq = th.get_multiple_slots_read_centric(r_data, ['norm_mean', 'base'],
                                                        r_data.corr_group)
    try:
        read_id = th.get_raw_read_slot(r_data).attrs.get('read_id')
    except Exception:
        read_id = getattr(r_data, 'read_id', None)
    if r_means is None or r_seq is None:
        raise th.TomboError('Read does not contain valid re-squiggled data.')
    r_seq = b''.join(r_seq).decode() if not isinstance(r_seq, str) else r_seq
    r_means, r_seq, read_start, read_end = _clip_to_region(
        np.asarray(r_means, dtype=np.float64), r_seq, r_data.start, r_data.end, r_data.strand,
        reg_start, reg_end, begin_lag + fm_offset, end_lag + fm_offset)
    if len(r_seq) < std_ref.kmer_width:
        raise th.TomboError('Read does not contain information in this region.')
    r_ref_means, r_ref_sds = std_ref.get_exp_levels_from_seq(r_seq, r_data.strand == '-')
    if r_data.strand == '-':
        r_means = r_means[::-1]
    r_means = r_means[begin_lag:r_means.shape[0] - end_lag] if end_lag else r_means[begin_lag:][:0]
    read_start += begin_lag
    read_end -= end_lag
    if fm_offset > 0 and r_means.shape[0] < 2 * fm_offset + 1:
        raise th.TomboError("P-values vector too short for Fisher's Method window compuation.")
    r_pvals = _lib.get_context().window_fisher_pvals(
        np.ascontiguousarray(r_means), r_ref_means, r_ref_sds, np.array([0, r_means.shape[0]]),
        fm_offset, True)
    return {DE_NOVO_TXT: r_pvals}, {DE_NOVO_TXT: np.arange(read_start, read_end)}, read_id


def compute_sample_compare_read_stats(r_data, ctrl_means, ctrl_sds, fm_offset=FM_OFFSET_DEFAULT,
                                      reg_data=None):
    """tombo_stats.py:3675-3769 -> ({'sample_compare': p-values}, {...: positions}, read_id);
    ``ctrl_means`` / ``ctrl_sds`` cover [reg_start - fm_offset, reg_end + fm_offset)."""
    reg_start = reg_data.start if reg_data is not None else r_data.start
    reg_end = reg_data.end if reg_data is not None else r_data.end
    got = th.get_multiple_slots_read_centric(r_data, ['norm_mean'], r_data.corr_group)
    r_means = got[0] if isinstance(got, (tuple, list)) else got
    try:
        read_id = th.get_raw_read_slot(r_data).attrs.get('read_id')
    except Exception:
        read_id = getattr(r_data, 'read_id', None)
    if r_means is None:
        raise th.TomboError('Read does not contain re-squiggled level means.')
    r_means, _, read_start, read_end = _clip_to_region(
        np.asarray(r_means, dtype=np.float64), None, r_data.start, r_data.end, r_data.strand,
        reg_start, reg_end, fm_offset, fm_offset)
    if r_data.strand == '-':
        r_means = r_means[::-1]
    a, b = read_start - reg_start + fm_offset, read_end - reg_start + fm_offset
    cm, cs = np.asarray(ctrl_means[a:b], dtype=np.float64), np.asarray(ctrl_sds[a:b], dtype=np.float64)
    with np.errstate(all='ignore'):
        if np.sum(~np.isnan(np.abs(r_means - cm) / cs)) == 0:
            raise th.TomboError('No valid z-scores in read.')
    if fm_offset > 0 and r_means.shape[0] < 2 * fm_offset + 1:
        raise th.TomboError("P-values vector too short for Fisher's Method window compuation.")
    r_pvals = _lib.get_context().window_fisher_pvals(
        np.ascontiguousarray(r_means), cm, cs, np.array([0, r_means.shape[0]]), fm_offset, False)
    r_poss = np.where(~np.isnan(r_pvals))[0]
    return {SAMP_COMP_TXT: r_pvals[r_poss]}, {SAMP_COMP_TXT: r_poss + read_start}, read_id


# ---------------------------------------------------------------------------
# level_sample_compare and control-sample reference levels (tombo_stats.py:2273-2287,
# 3572-3673, 4236-4393)
# ---------------------------------------------------------------------------
_LEVEL_TESTS = {KS_TEST_TXT: (0, False), U_TEST_TXT: (1, False), T_TEST_TXT: (2, False),
                KS_STAT_TEST_TXT: (0, True), U_STAT_TEST_TXT: (1, True),
                T_STAT_TEST_TXT: (2, True)}


def _ragged_reads(base_levels, reg_start):
    """positions x reads level matrix (``intervalData.get_base_levels``) -> ragged
    genome-ordered reads ``(levels, off, start)``: each column from its first to its last
    non-NaN level, in column (read) order"""
    bl = np.asarray(base_levels, dtype=np.float64)
    if bl.ndim != 2:
        raise th.TomboError('Base levels must be a positions x reads matrix.')
    valid = ~np.isnan(bl)
    cols = np.nonzero(valid.any(axis=0))[0]
    first = valid.argmax(axis=0)[cols]
    last = bl.shape[0] - valid[::-1].argmax(axis=0)[cols]
    lens = (last - first).astype(np.int64)
    levels = (np.concatenate([bl[f:l, c] for c, f, l in zip(cols, first, last)])
              if cols.shape[0] else np.zeros(0))
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return levels, off, (reg_start + first).astype(np.int64)


def _widened_levels(reg_data, fm_offset):
    return reg_data.copy().update(start=reg_data.start - fm_offset,
                                  end=reg_data.end + fm_offset).get_base_levels()


def _dense_level_tests(samp_base_levels, ctrl_base_levels, return_stat, test):
    samp = np.asarray(samp_base_levels, dtype=np.float64)
    ctrl = np.asarray(ctrl_base_levels, dtype=np.float64)
    n = samp.shape[0]
    out = np.full(n, np.nan)
    if n == 0:
        return out
    r = _lib.get_context().group_reg_stats(
        0, n, _ragged_reads(samp, 0), _ragged_reads(ctrl, 0), test, return_stat, 1, 0)
    out[r['pos']] = r['stat']
    return out


def compute_ks_tests(samp_base_levels, ctrl_base_levels, return_stat):
    """tombo_stats.py:4236-4260 on positions x reads matrices (NaN = missing).  A position
    where either sample has no level is NaN (the reference raises FloatingPointError)."""
    return _dense_level_tests(samp_base_levels, ctrl_base_levels, return_stat, 0)


def compute_u_tests(samp_base_levels, ctrl_base_levels, return_stat):
    """tombo_stats.py:4262-4297.  Tied levels: a sample level ranks before an equal
    control level (the reference's unstable argsort leaves that order undefined)."""
    return _dense_level_tests(samp_base_levels, ctrl_base_levels, return_stat, 1)


def compute_t_tests(samp_base_levels, ctrl_base_levels, return_stat):
    """tombo_stats.py:4299-4333.  Zero pooled variance, or one level in each sample, gives
    NaN (the reference raises FloatingPointError)."""
    return _dense_level_tests(samp_base_levels, ctrl_base_levels, return_stat, 2)


def calc_window_means(stats, lag):
    """tombo_stats.py:2273-2287 (host numpy, as in the reference; compute_group_reg_stats
    applies the same window on the device)"""
    assert lag > 0, 'Invalid window provided.'
    width = (lag * 2) + 1
    if stats.shape[-1] < width:
        raise th.TomboError("Statistics vector too short for window mean compuation.")
    m_stats = np.full(stats.shape, np.nan)
    m_stats[..., lag:-lag] = np.mean(np.lib.stride_tricks.sliding_window_view(
        stats, width, axis=-1), -1)
    return m_stats


def compute_group_reg_stats(reg_data, ctrl_reg_data, fm_offset, min_test_reads, stat_type):
    """tombo_stats.py:4335-4393 -> ``[(stat_type, tombo_helper.groupStats)]`` or ``[]``.
    Base levels come from ``reg_data.copy().update(...).get_base_levels()``; coverage, runs,
    the per-position test and the window all run on the device in one call.  The widened
    region holds at most 2^24 positions and each sample at most 2^30 - 1 reads (larger
    inputs raise ``_lib.TomboB200Error``); ``fm_offset`` has no other limit."""
    if stat_type not in _LEVEL_TESTS:
        raise NotImplementedError('Unrecognized test type.')
    test, return_stat = _LEVEL_TESTS[stat_type]
    start = reg_data.start - fm_offset
    size = reg_data.end - reg_data.start + 2 * fm_offset
    samp = _ragged_reads(_widened_levels(reg_data, fm_offset), start)
    ctrl = _ragged_reads(_widened_levels(ctrl_reg_data, fm_offset), start)
    r = _lib.get_context().group_reg_stats(start, size, samp, ctrl, test, return_stat,
                                           min_test_reads, fm_offset)
    if r['pos'].shape[0] == 0:
        return []
    return [(stat_type, th.groupStats(r['stat'], r['pos'], reg_data.chrm, reg_data.strand,
                                      reg_data.start, r['cov'], r['ctrl_cov']))]


def _prior_levels(ctrl_reg_data, std_ref, fm_offset):
    """compute_posterior_samp_dists :3575-3587: expected levels over the widened region"""
    dnstrm_bases = std_ref.kmer_width - std_ref.central_pos - 1
    plus = ctrl_reg_data.strand == '+'
    begin_lag = std_ref.central_pos if plus else dnstrm_bases
    end_lag = dnstrm_bases if plus else std_ref.central_pos
    reg_seq = ctrl_reg_data.copy().update(
        start=ctrl_reg_data.start - begin_lag - fm_offset,
        end=ctrl_reg_data.end + end_lag + fm_offset).add_seq().seq
    if ctrl_reg_data.strand == '-':
        reg_seq = th.rev_comp(reg_seq)
    return std_ref.get_exp_levels_from_seq_with_gaps(reg_seq, ctrl_reg_data.strand == '-')


def compute_posterior_samp_dists(ctrl_means, ctrl_sds, ctrl_cov, ctrl_reg_data, std_ref,
                                 prior_weights, min_test_reads, fm_offset):
    """tombo_stats.py:3572-3625: weighted means of the control levels and the model's
    expected levels (elementwise host numpy, as in the reference; get_reads_ref applies
    the same weights on the device)"""
    reg_ref_means, reg_ref_sds = _prior_levels(ctrl_reg_data, std_ref, fm_offset)
    post_ref_means = (((prior_weights[0] * reg_ref_means) + (ctrl_cov * ctrl_means)) /
                      (prior_weights[0] + ctrl_cov))
    post_ref_sds = (((prior_weights[1] * reg_ref_sds) + (ctrl_cov * ctrl_sds)) /
                    (prior_weights[1] + ctrl_cov))
    return post_ref_means, post_ref_sds


def get_reads_ref(reg_data, min_test_reads, fm_offset, std_ref=None, prior_weights=None,
                  est_mean=False):
    """tombo_stats.py:3627-3673 -> (means, sds, {position: coverage}).  Median (or mean)
    and standard deviation of the levels per position, the optional posterior with the
    model's expected levels, and the sd == 0 mask run on the device in one call.  The
    widened region holds at most 2^24 positions and at most 2^30 - 1 reads."""
    start = reg_data.start - fm_offset
    size = reg_data.end - reg_data.start + 2 * fm_offset
    reads = _ragged_reads(_widened_levels(reg_data, fm_offset), start)
    pm = ps = None
    weights = (0.0, 0.0)
    if std_ref is not None:
        weights = (MEAN_PRIOR_CONST, SD_PRIOR_CONST) if prior_weights is None else prior_weights
        pm, ps = _prior_levels(reg_data, std_ref, fm_offset)
    means, sds, cov = _lib.get_context().reads_ref_levels(
        start, size, reads, min_test_reads, est_mean, pm, ps, weights)
    if not (cov >= min_test_reads).any():
        return np.full(size, np.nan), np.full(size, np.nan), {}
    return means, sds, dict(zip(range(start, start + size), cov))


# ---------------------------------------------------------------------------
# alternative-model estimation (tombo_stats.py:1747-2071)
# ---------------------------------------------------------------------------
def _read_kmer_levels(r_data, kmer_width, central_pos):
    """one read's k-mer codes and levels in position order, paired as
    _parse_base_levels_worker pairs them (:1760-1772); None for a read without Events.
    K-mers with a non-ACGT base are dropped (the reference's worker dies on them)."""
    r_means, r_seq = th.get_multiple_slots_read_centric(
        r_data, ['norm_mean', 'base'], r_data.corr_group)
    if r_means is None:
        return None
    r_seq = b''.join(r_seq) if not isinstance(r_seq, str) else r_seq.encode()
    codes = _BASE_CODE[np.frombuffer(r_seq, dtype=np.uint8)]
    r_means = np.asarray(r_means, dtype=np.float64)
    dnstrm_bases = kmer_width - central_pos - 1
    # r_means[central_pos:-dnstrm_bases] is empty when dnstrm_bases == 0 (kept)
    levels = r_means[central_pos:-dnstrm_bases] if dnstrm_bases > 0 else r_means[:0]
    n = min(max(codes.shape[0] - kmer_width + 1, 0), levels.shape[0])
    kmer = np.zeros(n, dtype=np.int64)
    bad = np.zeros(n, dtype=bool)
    for j in range(kmer_width):
        c = codes[j:j + n]
        kmer = kmer * 4 + (c & 3)
        bad |= c > 3
    return kmer[~bad], levels[:n][~bad]


def parse_base_levels(all_reads, std_ref, parse_levels_batch_size, kmer_obs_thresh,
                      max_kmer_obs, min_kmer_obs_to_est, num_processes):
    """tombo_stats.py:1811-1884 -> ``{kmer: levels}`` for every ACGT k-mer, in
    ``itertools.product`` order, each a float64 array.

    Reads are taken in batches of ``parse_levels_batch_size``.  A k-mer that is complete
    (more than ``max_kmer_obs`` levels) when a batch starts gets nothing from that batch;
    every other k-mer gets all of the batch's levels, in read order, then position order --
    the order of the reference with one process (``num_processes`` is accepted; no process
    is started).  Parsing stops once the fewest levels among the k-mers still open exceed
    ``kmer_obs_thresh``, or when the reads run out.  Fewer than ``min_kmer_obs_to_est``
    levels for some k-mer raises :class:`tombo_helper.TomboError` with the reference's
    message; fewer than ``kmer_obs_thresh`` prints its warning."""
    kmer_width, central_pos = std_ref.kmer_width, std_ref.central_pos
    n_kmers = 4 ** kmer_width
    chunks = [[] for _ in range(n_kmers)]
    totals = np.zeros(n_kmers, dtype=np.int64)
    complete = np.zeros(n_kmers, dtype=bool)
    reads = iter(all_reads)
    while True:
        batch = list(itertools.islice(reads, parse_levels_batch_size))
        no_more_reads = len(batch) < parse_levels_batch_size
        open_kmers = ~complete
        if not open_kmers.any():
            # the reference takes min() of an empty list here
            raise th.TomboError('Every k-mer was complete before the last batch of reads; '
                                'kmer_obs_thresh must be below max_kmer_obs.')
        parsed = [p for p in (_read_kmer_levels(r, kmer_width, central_pos) for r in batch)
                  if p is not None]
        if parsed:
            kmers = np.concatenate([k for k, _ in parsed])
            levels = np.concatenate([lv for _, lv in parsed])
            keep = open_kmers[kmers]
            kmers, levels = kmers[keep], levels[keep]
            order = np.argsort(kmers, kind='stable')
            kmers, levels = kmers[order], levels[order]
            bounds = np.searchsorted(kmers, np.arange(n_kmers + 1))
            for k in np.nonzero(bounds[1:] > bounds[:-1])[0]:
                chunks[k].append(levels[bounds[k]:bounds[k + 1]])
            totals += bounds[1:] - bounds[:-1]
        complete |= open_kmers & (totals > max_kmer_obs)
        if totals[open_kmers].min() > kmer_obs_thresh or no_more_reads:
            break

    fewest_kmer_obs = int(totals.min())
    if fewest_kmer_obs < kmer_obs_thresh:
        if fewest_kmer_obs < min_kmer_obs_to_est:
            raise th.TomboError(
                'Too few minimal k-mer observations to continue to alternative estimation. '
                'Minimal k-mer has ' + str(fewest_kmer_obs) + ' total observations and ' +
                str(min_kmer_obs_to_est) + ' observations per k-mer are required.')
        th.warning_message(
            'Requested minimal k-mer observations not found in all reads. Continuing to '
            'estimation using a k-mer with ' + str(fewest_kmer_obs) + ' total observations')
    return dict((''.join(kmer), np.concatenate(c) if c else np.zeros(0))
                for kmer, c in zip(itertools.product('ACGT', repeat=kmer_width), chunks))


def write_kmer_densities_file(dens_fn, kmer_dens, save_x):
    """tombo_stats.py:1886-1893: tab-separated ``Kmer Signal Density`` rows"""
    rows = ('\t'.join(map(str, (kmer, x, y)))
            for kmer, dens_i in kmer_dens.items() for x, y in zip(save_x, dens_i))
    with io.open(dens_fn, 'wt') as fp:
        fp.write('Kmer\tSignal\tDensity\n')
        fp.write('\n'.join(rows) + '\n')


def parse_kmer_densities_file(dens_fn):
    """tombo_stats.py:1895-1912 -> ``{kmer: densities}`` in file order"""
    kmer_dens = {}
    with io.open(dens_fn) as fp:
        fp.readline()
        for line in fp:
            kmer, _, dens_i = line.split()
            kmer_dens.setdefault(kmer, []).append(float(dens_i))
    if len(set(len(d) for d in kmer_dens.values())) > 1:
        raise th.TomboError('Density file is valid.')
    return dict((kmer, np.array(d)) for kmer, d in kmer_dens.items())


def est_kernel_density(reads_index, std_ref, kmer_obs_thresh, density_basename, save_x,
                       kernel_dens_bw, num_processes, alt_or_stnd_name='alt',
                       parse_levels_batch_size=ALT_EST_BATCH, max_kmer_obs=MAX_KMER_OBS,
                       min_kmer_obs_to_est=MIN_KMER_OBS_TO_EST, device=0):
    """tombo_stats.py:1914-1939: shuffle the reads with numpy's global RNG (as the
    reference does, so one seed gives one order), group their levels by k-mer
    (:func:`parse_base_levels`), and fit every k-mer's Gaussian kernel density in one
    device call (tb2_kernel_densities): ``gaussian_kde(levels, kernel_dens_bw /
    levels.std(ddof=1)).evaluate(save_x)``.  Returns ``{kmer: density}`` and writes
    ``<density_basename>.<alt_or_stnd_name>_density.txt`` when a basename is given.  A
    k-mer whose levels the reference cannot fit raises :class:`tombo_helper.TomboError`."""
    all_reads = list(reads_index.iter_reads())
    np.random.shuffle(all_reads)
    base_levels = parse_base_levels(
        all_reads, std_ref, parse_levels_batch_size, kmer_obs_thresh, max_kmer_obs,
        min_kmer_obs_to_est, num_processes)
    kmers = list(base_levels)
    off = np.concatenate([[0], np.cumsum([base_levels[k].shape[0] for k in kmers])])
    dens, cho_cov, _ = _lib.get_context(device).kernel_densities(
        np.concatenate([base_levels[k] for k in kmers]), off, save_x, kernel_dens_bw)
    failed = np.nonzero(np.isnan(cho_cov))[0]
    if failed.shape[0]:
        raise th.TomboError(
            'Cannot fit a kernel density to the levels of k-mer ' + kmers[failed[0]] +
            ': fewer than 2 levels, a non-finite level or zero standard deviation.')
    kmer_dens = dict(zip(kmers, dens))
    if density_basename is not None:
        write_kmer_densities_file(
            density_basename + '.' + alt_or_stnd_name + '_density.txt', kmer_dens, save_x)
    return kmer_dens


def _isolate_alt_density(alt_dens, std_dens, alt_base, alt_frac_pctl, std_ref, save_x):
    """isolate_alt_density and the discrete decisions it took: ``offsets`` {kmer: grid
    points the alternative density moved}, ``peaks`` {kmer: (control peak, matched
    alternative peak)} for k-mers with one ``alt_base``"""
    save_x = np.asarray(save_x, dtype=np.float64)

    def dens_mean(dens):
        keep = dens > 1e-10
        return np.average(save_x[keep], weights=dens[keep])

    # mean shift alternative - control over the k-mers without alt_base, quadratic in the
    # control mean
    ctrl_means, shifts = [], []
    for kmer in std_dens:
        if alt_base not in kmer:
            ctrl_means.append(dens_mean(std_dens[kmer]))
            shifts.append(dens_mean(alt_dens[kmer]) - ctrl_means[-1])
    offset_fit = np.poly1d(np.polyfit(ctrl_means, shifts, 2))
    step = save_x[1] - save_x[0]
    offsets, shifted = {}, {}
    for kmer, dens in alt_dens.items():
        off = int(offset_fit(dens_mean(std_dens[kmer])) / step)
        offsets[kmer] = off
        shifted[kmer] = (np.concatenate([np.zeros(-off), dens[:off]]) if off < 0 else
                         np.concatenate([dens[off:], np.zeros(off)]))

    peaks, ratios = {}, []
    for kmer in std_dens:
        if kmer.count(alt_base) != 1:
            continue
        ctrl, alt = std_dens[kmer], shifted[kmer]
        ctrl_peak = np.argmax(ctrl)
        inner = alt[1:-1]
        alt_peaks = np.nonzero((inner > alt[:-2]) & (inner > alt[2:]))[0] + 1
        alt_peak = alt_peaks[np.argmin(abs(alt_peaks - ctrl_peak))]
        peaks[kmer] = (int(ctrl_peak), int(alt_peak))
        ratios.append(alt[alt_peak] / ctrl[ctrl_peak])
    std_frac = np.percentile(ratios, alt_frac_pctl)
    if std_frac >= 1:
        th.warning_message(
            'Alternative base incorporation rate estimate is approximately 0. Consider '
            'lowering --alt-fraction-percentile.')

    model_sd = np.mean(list(std_ref.sds.values()))
    alt_rows = []
    for kmer in std_ref.means:
        n_alt = kmer.count(alt_base)
        if n_alt == 0:
            continue
        # the control's share of this k-mer's observations: std_frac per alt_base
        diff_dens = shifted[kmer] - (std_dens[kmer] * std_frac**n_alt)
        diff_dens[diff_dens < 0] = 0
        alt_level = np.average(save_x, weights=diff_dens)
        alt_rows.extend((kmer, m.start(), alt_level, model_sd)
                        for m in re.finditer(alt_base, kmer))
    alt_ref = AltModel(kmer_ref=alt_rows, central_pos=std_ref.central_pos, alt_base=alt_base)
    return alt_ref, dict(offsets=offsets, peaks=peaks)


def isolate_alt_density(alt_dens, std_dens, alt_base, alt_frac_pctl, std_ref, save_x):
    """tombo_stats.py:1991-2071 (host numpy on the densities, as in the reference) ->
    :class:`AltModel` with one row per ``alt_base`` position of each k-mer of ``std_ref``"""
    return _isolate_alt_density(alt_dens, std_dens, alt_base, alt_frac_pctl, std_ref, save_x)[0]
