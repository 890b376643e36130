"""``tombo.resquiggle`` per-read API (resquiggle.py:345-1214) on the GPU: same
function names, arguments and return namedtuples as the reference; every function
is a batch of one over the batched C ABI, plus the batched entry point
:func:`resquiggle_reads` that the throughput numbers are quoted on (per-read
kernel launches are launch bound).

Mapping (mappy), FAST5 I/O and the multiprocessing plumbing of the reference
module (resquiggle.py:1221-2088) are outside the hot path; the worker's iterate /
rescue policy (:1492-1504, 1578-1588) is part of it and lives inside
tb2_resquiggle_batch.
"""
import numpy as np

from . import _lib
from . import tombo_helper as th
from . import tombo_stats as ts
from ._default_parameters import (
    EXTRA_SIG_FACTOR, DEL_FIX_WINDOW, MAX_DEL_FIX_WINDOW, MIN_EVENT_TO_SEQ_RATIO, MAX_RAW_CPTS,
    SIG_MATCH_THRESH, DNA_SAMP_TYPE, RNA_SAMP_TYPE, USE_RNA_EVENT_SCALE, RNA_SCALE_NUM_EVENTS,
    RNA_SCALE_MAX_FRAC_EVENTS, START_CLIP_PARAMS, OUTLIER_THRESH, MAX_SCALING_ITERS)

__all__ = [
    'resquiggle_read', 'resquiggle_reads', 'segment_signal', 'find_adaptive_base_assignment',
    'resolve_skipped_bases_with_raw', 'find_seq_start_in_events', 'find_static_base_assignment']

START_CLIP_PARAMS = th.startClipParams(*START_CLIP_PARAMS)
_LUT = np.full(256, 255, dtype=np.uint8)
for _i, _b in enumerate('ACGT'):
    _LUT[ord(_b)] = _i


def _seq_codes(seq):
    return _LUT[np.frombuffer(seq.encode(), dtype=np.uint8)]


def _ensure_model(ctx, std_ref):
    """upload the k-mer tables once per model object (_lib.ensure_model)"""
    _lib.ensure_model(ctx, std_ref)


# ---------------------------------------------------------------------------
def find_static_base_assignment(event_means, r_ref_means, r_ref_sds, rsqgl_params,
                                reg_id=None):
    """resquiggle.py:547-600 -> event to sequence mapping (``read_tb``)"""
    st, tb = _lib.get_context().find_static_base_assignment(
        event_means, r_ref_means, r_ref_sds, rsqgl_params)
    th._raise_status(st)
    return tb


def find_seq_start_in_events(event_means, r_ref_means, r_ref_sds, rsqgl_params, num_bases,
                             num_events, seq_samp_type=None, reg_id=None):
    """resquiggle.py:685-752 -> (start event, events per base)"""
    thresh = None if seq_samp_type is None else SIG_MATCH_THRESH[seq_samp_type.name]
    st, start_loc, epb = _lib.get_context().find_seq_start_in_events(
        event_means, r_ref_means, r_ref_sds, rsqgl_params, num_bases, num_events, thresh)
    th._raise_status(st)
    return start_loc, epb


def find_adaptive_base_assignment(
        valid_cpts, event_means, rsqgl_params, std_ref, genome_seq, start_clip_bases=None,
        start_clip_params=START_CLIP_PARAMS,
        seq_samp_type=th.seqSampleType(DNA_SAMP_TYPE, False), reg_id=None):
    """resquiggle.py:866-1050 -> :class:`tombo_helper.dpResults`"""
    if start_clip_bases is not None:
        raise NotImplementedError(
            'start_clip_bases is disabled in the reference (USE_START_CLIP_BASES=False, '
            'resquiggle.py:76)')
    dnstrm_bases = std_ref.kmer_width - std_ref.central_pos - 1
    r_ref_means, r_ref_sds = std_ref.get_exp_levels_from_seq(genome_seq)
    genome_seq = genome_seq[std_ref.central_pos:-dnstrm_bases]
    if len(genome_seq) != r_ref_means.shape[0]:
        raise th.TomboError('Discordant reference and seqeunce lengths.')
    st, segs, rsrtr, _ = _lib.get_context().find_adaptive_base_assignment(
        valid_cpts, event_means, rsqgl_params, r_ref_means, r_ref_sds,
        SIG_MATCH_THRESH[seq_samp_type.name])
    th._raise_status(st)
    return th.dpResults(read_start_rel_to_raw=rsrtr, segs=segs, ref_means=r_ref_means,
                        ref_sds=r_ref_sds, genome_seq=genome_seq)


def resolve_skipped_bases_with_raw(
        dp_res, norm_signal, rsqgl_params, max_raw_cpts=MAX_RAW_CPTS,
        del_fix_window=DEL_FIX_WINDOW, max_del_fix_window=MAX_DEL_FIX_WINDOW,
        extra_sig_factor=EXTRA_SIG_FACTOR):
    """resquiggle.py:402-540 -> deletion resolved base start positions"""
    if (del_fix_window, max_del_fix_window, extra_sig_factor) != (
            DEL_FIX_WINDOW, MAX_DEL_FIX_WINDOW, EXTRA_SIG_FACTOR):
        raise NotImplementedError('only the default deletion window constants are built in')
    st, segs = _lib.get_context().resolve_skipped_bases_with_raw(
        dp_res.segs, dp_res.ref_means, dp_res.ref_sds, norm_signal, rsqgl_params, max_raw_cpts)
    th._raise_status(st)
    return segs


def _remove_stall_cpts(stall_ints, valid_cpts):
    """Drop changepoints strictly inside a stall interval (tombo_stats.py:1576-1597).
    The reference walks the sorted intervals next to the sorted changepoints; with sorted,
    disjoint intervals that is an interval lookup: the only interval that can hold cpt is
    the first one whose end is >= cpt."""
    stall_ints = np.asarray(stall_ints, dtype=np.int64).reshape(-1, 2)
    if stall_ints.shape[0] == 0:
        return valid_cpts
    k = np.searchsorted(stall_ints[:, 1], valid_cpts, side='left')
    kc = np.minimum(k, stall_ints.shape[0] - 1)
    inside = (k < stall_ints.shape[0]) & (stall_ints[kc, 0] < valid_cpts) & \
        (valid_cpts < stall_ints[kc, 1])
    return valid_cpts[~inside]


def _rna_event_scale_values(raw, valid_cpts, outlier_thresh):
    """get_scale_values_from_events (tombo_stats.py:217-233): median / MAD of the first
    RNA_SCALE_NUM_EVENTS (at most RNA_SCALE_MAX_FRAC_EVENTS of all) event means."""
    n_ev = RNA_SCALE_NUM_EVENTS
    if valid_cpts.shape[0] * RNA_SCALE_MAX_FRAC_EVENTS < n_ev:
        n_ev = int(valid_cpts.shape[0] * RNA_SCALE_MAX_FRAC_EVENTS)
    ev_means = ts.compute_base_means(raw, valid_cpts[:n_ev])
    _, ev_sv = ts.normalize_raw_signal(ev_means, norm_type='median')
    return th.scaleValues(ev_sv.shift, ev_sv.scale, -outlier_thresh, outlier_thresh, None)


def segment_signal(map_res, num_events, rsqgl_params, outlier_thresh=None, const_scale=None):
    """resquiggle.py:1057-1120 -> (valid_cpts, norm_signal, scale_values).

    Two orders of the same two steps: RNA (t-test segmentation) finds changepoints on the
    raw signal and may derive the scaling from the events; DNA normalises first and
    segments the normalised signal.  Which normalisation runs is one precedence list:
    scale values carried by the read > ``const_scale`` > estimated from the signal."""
    raw = map_res.raw_signal
    rna = bool(rsqgl_params.use_t_test_seg)

    def changepoints(sig):
        find = th.valid_cpts_w_cap_t_test if rna else th.valid_cpts_w_cap
        cpts = find(sig.astype(np.float64) if rna else sig, rsqgl_params.min_obs_per_base,
                    rsqgl_params.running_stat_width, num_events)
        return cpts if map_res.stall_ints is None else _remove_stall_cpts(map_res.stall_ints, cpts)

    def normalise(event_cpts):
        if map_res.scale_values is not None:
            return ts.normalize_raw_signal(raw, scale_values=map_res.scale_values)
        if const_scale is not None:
            return ts.normalize_raw_signal(raw, norm_type='median_const_scale',
                                           outlier_thresh=outlier_thresh, const_scale=const_scale)
        if not rna:
            return ts.normalize_raw_signal(raw, norm_type='median', outlier_thresh=outlier_thresh)
        sv = _rna_event_scale_values(raw, event_cpts, outlier_thresh) if USE_RNA_EVENT_SCALE else None
        return ts.normalize_raw_signal(raw, scale_values=sv)

    if rna:
        valid_cpts = changepoints(raw)
        norm_signal, new_sv = normalise(valid_cpts)
    else:
        norm_signal, new_sv = normalise(None)
        valid_cpts = changepoints(norm_signal)
    return valid_cpts, norm_signal, new_sv


# ---------------------------------------------------------------------------
# batched driver shared by resquiggle_read / resquiggle_reads
# ---------------------------------------------------------------------------
def pack_reads(map_results):
    """Flat batch arrays of the C ABI (raw, raw_off, seq codes, seq_off); host only.

    A read whose ``raw_signal`` is None contributes an empty slice: the library reports
    TB2_ERR_NO_RAW for exactly that read ('Must have raw signal ...', resquiggle.py:1149)
    and the rest of the batch is unaffected, as in the reference where only that read's
    resquiggle_read raises."""
    n = len(map_results)
    raws = [np.zeros(0, dtype=np.int16) if mr.raw_signal is None else np.asarray(mr.raw_signal)
            for mr in map_results]
    all_int16 = all(r.dtype == np.int16 for r in raws)
    raw = np.concatenate([r if all_int16 else r.astype(np.float64) for r in raws]) if n else \
        np.zeros(0, dtype=np.float64)
    if raw.shape[0] == 0:
        raw = np.zeros(1, dtype=raw.dtype)     # the library wants a non-null buffer
    raw_off = np.zeros(n + 1, dtype=np.int64)
    raw_off[1:] = np.cumsum([r.shape[0] for r in raws])
    codes = [_seq_codes(mr.genome_seq) for mr in map_results]
    seq = np.concatenate(codes)
    seq_off = np.zeros(n + 1, dtype=np.int64)
    seq_off[1:] = np.cumsum([c.shape[0] for c in codes])
    return raw, raw_off, seq, seq_off


class LibraryError(Exception):
    """A per-read outcome that is NOT a TomboError in the reference: the reference's
    'Unexpected error' bucket (FloatingPointError etc., resquiggle.py:1589-1594) and this
    library's own limits (CUDA failure, compiled-in capacity).  The worker files these
    with is_tombo_error=False."""


_NON_TOMBO_STATUS = (100, 200, 201, 202)   # UNEXPECTED, CUDA, INVALID_ARG, CAPACITY


def _status_exception(st):
    msg = _lib.status_message(st)
    return LibraryError(msg) if st in _NON_TOMBO_STATUS else th.TomboError(msg)


def _run_batch(map_results, std_ref, rsqgl_params, save_params, outlier_thresh, max_raw_cpts,
               min_event_to_seq_ratio, const_scale, skip_seq_scaling, seq_samp_type,
               max_scaling_iters, worker_policy, subsample_seed, device):
    ctx = _lib.get_context(device)
    _ensure_model(ctx, std_ref)
    n = len(map_results)
    raw, raw_off, seq, seq_off = pack_reads(map_results)
    # worker_policy: RNA flip + stall detection + iterate + rescue happen in the
    # library; otherwise exactly one resquiggle_read call on the data as given
    is_rna_worker = worker_policy and seq_samp_type.name == RNA_SAMP_TYPE
    pol = _lib.make_policy(
        'RNA' if is_rna_worker else 'DNA', outlier_thresh=outlier_thresh,
        max_raw_cpts=max_raw_cpts, min_event_to_seq_ratio=min_event_to_seq_ratio,
        max_scaling_iters=max_scaling_iters if worker_policy else 1,
        skip_seq_scaling=skip_seq_scaling, const_scale=const_scale,
        subsample_seed=subsample_seed, rescue=bool(worker_policy and save_params is not None),
        sig_match_thresh=SIG_MATCH_THRESH[seq_samp_type.name])
    ctx.batch_upload(raw, raw_off, seq, seq_off, rsqgl_params, pol)
    sv_in = None
    if any(mr.scale_values is not None for mr in map_results):
        sv_in = np.full((n, 5), np.nan)
        for i, mr in enumerate(map_results):
            if mr.scale_values is not None:
                sv_in[i] = [np.nan if v is None else v for v in mr.scale_values]
    stalls = None
    if not is_rna_worker and any(mr.stall_ints is not None for mr in map_results):
        stalls = [[] if mr.stall_ints is None else list(mr.stall_ints) for mr in map_results]
    if sv_in is not None or stalls is not None:
        ctx.batch_set_read_inputs(sv_in, stalls)
    ctx.batch_compute(rsqgl_params, save_params, pol, want_norm_signal=True)
    res = ctx.batch_download(want_norm_signal=True)
    out = []
    k, cpos = std_ref.kmer_width, std_ref.central_pos
    for i, mr in enumerate(map_results):
        st = int(res['status'][i])
        if st != 0:
            out.append(_status_exception(st))
            continue
        a, b = res['seg_off'][i], res['seg_off'][i + 1]
        segs = res['segs'][a:b].copy()
        svr = res['scale_values'][i]
        ro = raw_off[i]
        out.append(mr._replace(
            read_start_rel_to_raw=int(res['read_start_rel_to_raw'][i]), segs=segs,
            genome_seq=mr.genome_seq[cpos:cpos + (b - a - 1)],
            raw_signal=res['norm_signal'][ro:ro + int(segs[-1])].copy(),
            scale_values=th.scaleValues(
                float(svr[0]), float(svr[1]), None if np.isnan(svr[2]) else float(svr[2]),
                None if np.isnan(svr[3]) else float(svr[3]), outlier_thresh),
            sig_match_score=float(res['sig_match_score'][i]),
            norm_params_changed=bool(res['flags'][i] & 1)))
    return out


def resquiggle_read(
        map_res, std_ref, rsqgl_params, outlier_thresh=None, all_raw_signal=None,
        max_raw_cpts=MAX_RAW_CPTS, min_event_to_seq_ratio=MIN_EVENT_TO_SEQ_RATIO,
        const_scale=None, skip_seq_scaling=False,
        seq_samp_type=th.seqSampleType(DNA_SAMP_TYPE, False), subsample_seed=0):
    """Raw signal to genome sequence assignment for one read (resquiggle.py:1122-1214):
    one call of the pipeline, no iteration, no rescue -- exactly the reference
    function.  Returns :class:`tombo_helper.resquiggleResults` (``raw_signal`` holds
    the trimmed, normalised signal) or raises :class:`tombo_helper.TomboError`."""
    if all_raw_signal is not None:
        map_res = map_res._replace(raw_signal=all_raw_signal)
    if map_res.raw_signal is None:
        raise th.TomboError('Must have raw signal in order to complete re-squiggle algorithm')
    res = _run_batch([map_res], std_ref, rsqgl_params, None, outlier_thresh, max_raw_cpts,
                     min_event_to_seq_ratio, const_scale, skip_seq_scaling, seq_samp_type, 1,
                     False, subsample_seed, 0)[0]
    if isinstance(res, Exception):
        raise res
    return res


def resquiggle_reads(
        map_results, std_ref, rsqgl_params, save_params=None, outlier_thresh=OUTLIER_THRESH,
        max_raw_cpts=MAX_RAW_CPTS, min_event_to_seq_ratio=MIN_EVENT_TO_SEQ_RATIO,
        const_scale=None, skip_seq_scaling=False,
        seq_samp_type=th.seqSampleType(DNA_SAMP_TYPE, False),
        max_scaling_iters=MAX_SCALING_ITERS, subsample_seed=0, device=0):
    """Batched resquiggle with the worker policy of the reference
    (_resquiggle_worker, resquiggle.py:1488-1597): RNA signal flip and stall
    detection, up to ``max_scaling_iters`` calls while the normalisation parameters
    change, one retry with ``save_params`` for reads that fail.

    ``map_results``: list of :class:`tombo_helper.resquiggleResults` holding
    ``genome_seq`` and ``raw_signal`` (as stored: RNA 3'->5').  Returns a list with a
    ``resquiggleResults`` per read, or the :class:`tombo_helper.TomboError` the
    reference would have reported for it.  The batch never aborts for one bad read."""
    if len(map_results) == 0:
        return []
    return _run_batch(list(map_results), std_ref, rsqgl_params, save_params, outlier_thresh,
                      max_raw_cpts, min_event_to_seq_ratio, const_scale, skip_seq_scaling,
                      seq_samp_type, max_scaling_iters, True, subsample_seed, device)
