"""``tombo text_output browser_files`` for the read-derived file types (_text_output_commands.py):
coverage bedgraphs and per-position signal, signal SD, dwell and sample-difference wiggles.

Names mirror the reference.  The per-position work runs on the device:

* coverage is ``tb2_coverage_runs``, every (chromosome, strand) of a sample in one call;
* the signal, SD and dwell means are ``tb2_slot_sums_*``, fed one read's Events at a time, so
  a whole chromosome's Events are never held on the host.  Each position is the reference's
  sequential fp64 sum in read order (DESIGN.md §3 "Genome browser tracks").

The text is formatted on the host by array operations that give the characters of
``'{:d} {:.4f}'`` and ``'%d'``.  The statistics-file types (``fraction``,
``dampened_fraction``, ``valid_coverage``, ``statistic``) are not supported yet and raise
TomboError.  ``ctx`` is any object with ``coverage_runs`` and ``slot_means`` (default: the
device's shared context)."""
from __future__ import division

import io

import numpy as np

from . import _lib
from . import formats
from . import tombo_helper as th

OUT_HEADER = 'track type={0} name="{1}_{2}_{3}{4}" ' + 'description="{1} {2} {3}{5}"\n'
BG_TYPE = 'bedgraph'
WIG_TYPE = 'wig'
OUT_TYPES = {WIG_TYPE: 'wiggle_0', BG_TYPE: 'bedGraph'}
GROUP_NAME = 'sample'
CTRL_NAME = 'control'

COV_WIG_TYPE = 'coverage'
SIG_SLOT = 'norm_mean'
SD_SLOT = 'norm_stdev'
DWELL_SLOT = 'length'
SIG_WIG_TYPE = 'signal'
DIFF_WIG_TYPE = 'difference'
SD_WIG_TYPE = 'signal_sd'
DWELL_WIG_TYPE = 'dwell'

FRAC_WIG_TYPE = 'fraction'
DFRAC_WIG_TYPE = 'dampened_fraction'
STAT_WIG_TYPE = 'statistic'
VCOV_WIG_TYPE = 'valid_coverage'
STATS_WIG_TYPES = (FRAC_WIG_TYPE, DFRAC_WIG_TYPE, STAT_WIG_TYPE, VCOV_WIG_TYPE)
READ_WIG_TYPES = (SIG_WIG_TYPE, DIFF_WIG_TYPE, COV_WIG_TYPE, SD_WIG_TYPE, DWELL_WIG_TYPE)


# ---------------------------------------------------------------------------
# text: '{:d}' and '{:.4f}' over arrays
# ---------------------------------------------------------------------------
def _digits(x, width):
    """right-aligned ASCII digits of the non-negative int64 ``x`` in ``width`` columns, and the
    mask of the columns '{:d}' prints"""
    v = np.asarray(x, dtype=np.int64).copy()
    if v.size and (v.min() < 0 or v.max() >= 10 ** width):
        raise ValueError('integer outside the formatted width')
    d = np.empty((v.shape[0], width), dtype=np.uint8)
    keep = np.empty((v.shape[0], width), dtype=bool)
    for k in range(width - 1, -1, -1):
        d[:, k] = 48 + v % 10
        keep[:, k] = v > 0
        v //= 10
    keep[:, -1] = True
    return d, keep


def _const(n, text):
    c = np.frombuffer(text.encode(), dtype=np.uint8)
    return np.broadcast_to(c, (n, c.shape[0])), np.ones((n, c.shape[0]), dtype=bool)


def _fixed4(vals):
    """'{:.4f}' of each value as (columns, masks), and the rows left to Python's formatting:
    non-finite values, |x| >= 1e8, and values whose 4-digit rounding lies within 1e-3 of a
    half-unit tie, where the product x * 1e4 (relative error <= 2^-53, so absolute error below
    1.2e-4 here) could round the other way from the exact decimal value"""
    v = np.asarray(vals, dtype=np.float64)
    a = np.abs(v)
    with np.errstate(invalid='ignore', over='ignore'):
        y = a * 1e4
        frac = y - np.floor(y)
        slow = ~np.isfinite(v) | (a >= 1e8) | (np.abs(frac - 0.5) < 1e-3)
    q = np.where(slow, 0.0, np.rint(np.where(slow, 0.0, y))).astype(np.int64)
    n = v.shape[0]
    sign = np.full((n, 1), ord('-'), dtype=np.uint8), np.signbit(v)[:, None]
    ip = _digits(q // 10000, 9)
    fp = _digits(q % 10000, 4)
    return [sign, ip, _const(n, '.'), (fp[0], np.ones_like(fp[1]))], slow


def _rows(cols, slow, slow_text):
    """the rows of ``cols`` (each a (columns, mask) pair) as bytes, the ``slow`` rows replaced by
    ``slow_text(i)``"""
    data = np.concatenate([np.broadcast_to(c, m.shape) for c, m in cols], axis=1)
    mask = np.concatenate([m for _, m in cols], axis=1)
    flat = data[mask]
    if not np.any(slow):
        return flat.tobytes()
    ends = np.cumsum(mask.sum(axis=1))
    out, prev = [], 0
    for i in np.flatnonzero(slow):
        out.append(flat[prev:ends[i] - mask[i].sum()].tobytes())
        out.append(slow_text(i).encode())
        prev = ends[i]
    out.append(flat[prev:].tobytes())
    return b''.join(out)


def format_wig_lines(cs_poss, cs_vals):
    """'\\n'.join('{:d} {:.4f}'.format(p + 1, v)) + '\\n' as bytes"""
    cs_poss = np.asarray(cs_poss, dtype=np.int64)
    cs_vals = np.asarray(cs_vals, dtype=np.float64)
    n = cs_poss.shape[0]
    if n == 0:
        return b'\n'
    val_cols, slow = _fixed4(cs_vals)
    cols = [_digits(cs_poss + 1, 19), _const(n, ' ')] + val_cols + [_const(n, '\n')]
    return _rows(cols, slow, lambda i: '{:d} {:.4f}\n'.format(int(cs_poss[i]) + 1, float(cs_vals[i])))


def format_bedgraph_lines(chrm, cs_cov, cs_cov_starts):
    """the bedgraph text of write_cov_wig for one (chrm, strand) as bytes"""
    n = cs_cov.shape[0]
    cols = [_const(n, chrm + '\t'), _digits(cs_cov_starts[:-1], 19), _const(n, '\t'),
            _digits(cs_cov_starts[1:], 19), _const(n, '\t'), _digits(cs_cov, 19), _const(n, '\n')]
    return _rows(cols, np.zeros(n, dtype=bool), None)


# ---------------------------------------------------------------------------
# _text_output_commands.py
# ---------------------------------------------------------------------------
def open_browser_files(wig_base, group_text, type_name, out_type=WIG_TYPE):
    """the plus and minus strand files with their track headers (:64-79), opened for bytes"""
    group_w_dot = '' if group_text == '' else '.' + group_text
    group_w_us = '' if group_text == '' else '_' + group_text
    group_w_space = '' if group_text == '' else ' ' + group_text
    plus_wig_fp = io.open(wig_base + '.' + type_name + group_w_dot + '.plus.' + out_type, 'wb')
    minus_wig_fp = io.open(wig_base + '.' + type_name + group_w_dot + '.minus.' + out_type, 'wb')
    plus_wig_fp.write(OUT_HEADER.format(
        OUT_TYPES[out_type], wig_base, type_name, 'fwd_strand', group_w_us, group_w_space).encode())
    minus_wig_fp.write(OUT_HEADER.format(
        OUT_TYPES[out_type], wig_base, type_name, 'rev_strand', group_w_us, group_w_space).encode())
    return plus_wig_fp, minus_wig_fp


def _write_cs_data(wig_fp, chrm, cs_poss, cs_vals):
    """one variableStep block (:81-86)"""
    wig_fp.write('variableStep chrom={} span=1\n'.format(chrm).encode())
    wig_fp.write(format_wig_lines(cs_poss, cs_vals))


def filter_cs_nans(cs_vals):
    """(:230-233)"""
    valid_poss = np.where(~np.isnan(cs_vals))[0]
    return valid_poss, cs_vals[valid_poss]


def write_slot_mean_wig(reads_index, chrm_sizes, wig_base, group_name, wig_type, slot_name, ctx=None):
    """(:235-249)"""
    th.status_message('Parsing and outputting ' + group_name + ' ' + wig_type + '.')
    plus_fp, minus_fp = open_browser_files(wig_base, group_name, wig_type)
    with plus_fp, minus_fp:
        for chrm, strand, cs_vals, _ in th.iter_mean_slot_values(reads_index, chrm_sizes, slot_name, ctx=ctx):
            cs_poss, cs_vals = filter_cs_nans(cs_vals)
            _write_cs_data(plus_fp if strand == '+' else minus_fp, chrm, cs_poss, cs_vals)


def write_signal_and_diff_wigs(reads_index, ctrl_reads_index, chrm_sizes, wig_base, group_name,
                               write_sig, write_diff, ctx=None):
    """(:251-298): the sample's signal, the control's, and their difference where both are
    defined"""
    th.status_message('Parsing and outputting signal means and differences.')
    fps = []
    if write_sig:
        plus_sig1_fp, minus_sig1_fp = open_browser_files(wig_base, group_name, SIG_WIG_TYPE)
        fps += [plus_sig1_fp, minus_sig1_fp]
        if ctrl_reads_index is not None:
            plus_sig2_fp, minus_sig2_fp = open_browser_files(wig_base, CTRL_NAME, SIG_WIG_TYPE)
            fps += [plus_sig2_fp, minus_sig2_fp]
    if write_diff:
        plus_diff_fp, minus_diff_fp = open_browser_files(wig_base, '', DIFF_WIG_TYPE)
        fps += [plus_diff_fp, minus_diff_fp]
    try:
        for chrm, strand, means1, means2 in th.iter_mean_slot_values(
                reads_index, chrm_sizes, SIG_SLOT, ctrl_reads_index, ctx=ctx):
            if means1 is not None:
                poss1, vals1 = filter_cs_nans(means1)
                if write_sig:
                    _write_cs_data(plus_sig1_fp if strand == '+' else minus_sig1_fp, chrm, poss1, vals1)
            if means2 is not None:
                poss2, vals2 = filter_cs_nans(means2)
                if write_sig:
                    _write_cs_data(plus_sig2_fp if strand == '+' else minus_sig2_fp, chrm, poss2, vals2)
                if means1 is not None and write_diff:
                    valid = np.intersect1d(poss1, poss2, assume_unique=True)
                    _write_cs_data(plus_diff_fp if strand == '+' else minus_diff_fp, chrm, valid,
                                   means1[valid] - means2[valid])
    finally:
        for fp in fps:
            fp.close()


def write_cov_wig(reads_index, out_base, group_text, ctx=None):
    """(:300-320): one bedgraph line per coverage run, zero runs included"""
    th.status_message('Getting and writing ' + group_text + ' coverage bedgraphs.')
    plus_fp, minus_fp = open_browser_files(out_base, group_text, COV_WIG_TYPE, BG_TYPE)
    with plus_fp, minus_fp:
        for chrm, strand, cs_cov, cs_cov_starts in th.iter_coverage_regions(reads_index, ctx=ctx):
            (plus_fp if strand == '+' else minus_fp).write(format_bedgraph_lines(chrm, cs_cov, cs_cov_starts))


def write_all_browser_files(fast5s_dirs, ctrl_fast5s_dirs, corr_grp, bc_subgrps, stats_fn, wig_base,
                            wig_types, motif_descs=None, fasta_fn=None, ctx=None, device=0):
    """(:322-388) for the read-derived file types"""
    if any(t in wig_types for t in STATS_WIG_TYPES):
        raise th.TomboError('--file-types ' + ', '.join(t for t in STATS_WIG_TYPES if t in wig_types) +
                            ' (from a statistics file) are not supported yet.')
    ctx = ctx if ctx is not None else _lib.get_context(device)
    if fast5s_dirs is not None:
        reads_index = formats.load_reads_index(fast5s_dirs, corr_grp, bc_subgrps)
        if sum(len(x) for x in reads_index.values()) == 0:
            raise th.TomboError('No reads present in --fast5-basedirs.')
    group_name = '' if ctrl_fast5s_dirs is None else GROUP_NAME
    if ctrl_fast5s_dirs is not None:
        ctrl_reads_index = formats.load_reads_index(ctrl_fast5s_dirs, corr_grp, bc_subgrps)
        chrm_sizes = th.get_chrm_sizes(reads_index, ctrl_reads_index)
        if COV_WIG_TYPE in wig_types:
            write_cov_wig(ctrl_reads_index, wig_base, CTRL_NAME, ctx)
        if SD_WIG_TYPE in wig_types:
            write_slot_mean_wig(ctrl_reads_index, chrm_sizes, wig_base, CTRL_NAME, SD_WIG_TYPE, SD_SLOT, ctx)
        if DWELL_WIG_TYPE in wig_types:
            write_slot_mean_wig(ctrl_reads_index, chrm_sizes, wig_base, CTRL_NAME, DWELL_WIG_TYPE, DWELL_SLOT, ctx)
        if SIG_WIG_TYPE in wig_types or DIFF_WIG_TYPE in wig_types:
            write_signal_and_diff_wigs(reads_index, ctrl_reads_index, chrm_sizes, wig_base, group_name,
                                       SIG_WIG_TYPE in wig_types, DIFF_WIG_TYPE in wig_types, ctx)
    elif fast5s_dirs is not None:
        chrm_sizes = th.get_chrm_sizes(reads_index)
        if SIG_WIG_TYPE in wig_types:
            write_signal_and_diff_wigs(reads_index, None, chrm_sizes, wig_base, group_name,
                                       SIG_WIG_TYPE in wig_types, False, ctx)
    if COV_WIG_TYPE in wig_types:
        write_cov_wig(reads_index, wig_base, group_name, ctx)
    if SD_WIG_TYPE in wig_types:
        write_slot_mean_wig(reads_index, chrm_sizes, wig_base, group_name, SD_WIG_TYPE, SD_SLOT, ctx)
    if DWELL_WIG_TYPE in wig_types:
        write_slot_mean_wig(reads_index, chrm_sizes, wig_base, group_name, DWELL_WIG_TYPE, DWELL_SLOT, ctx)


def browser_files_main(args, ctx=None):
    """_browser_files_main (:427-463): the reference's argument checks, each a TomboError where
    the reference exits with the same message"""
    if any(t in args.file_types for t in READ_WIG_TYPES) and args.fast5_basedirs is None:
        raise th.TomboError('Must provide a fast5 basedir to output signal, difference, ' +
                            'coverage, signal_sd and/or length browser files.')
    if any(t in args.file_types for t in STATS_WIG_TYPES) and args.statistics_filename is None:
        raise th.TomboError('Must provide a statistics filename to output ' +
                            'fraction or valid coverage browser files.')
    if DIFF_WIG_TYPE in args.file_types and args.control_fast5_basedirs is None:
        raise th.TomboError('Must provide two sets of FAST5s to output difference wiggle files.')
    if args.control_fast5_basedirs is not None and args.fast5_basedirs is None:
        raise th.TomboError('Cannot provide a control FAST5 set of directories ' +
                            'without a sample set of FAST5 directories.')
    write_all_browser_files(
        args.fast5_basedirs, args.control_fast5_basedirs, args.corrected_group, args.basecall_subgroups,
        args.statistics_filename, args.browser_file_basename, args.file_types,
        getattr(args, 'motif_descriptions', None), getattr(args, 'genome_fasta', None), ctx=ctx)
