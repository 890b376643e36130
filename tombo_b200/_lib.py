"""ctypes binding of libtombo_b200.so (the C ABI declared in include/tombo_b200.h).

There is no CPU fallback: importing works everywhere (so the ABI can be
inspected on a CPU box), but creating a context raises ``TomboB200Error`` when the
shared library is missing or no CUDA device is usable.
"""
import ctypes as C
import os
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libtombo_b200.so')

i64 = C.c_int64
f64 = C.c_double
P = C.POINTER


class TomboB200Error(RuntimeError):
    pass


class Params(C.Structure):
    """tb2_params == tombo_helper.resquiggleParams (tombo_helper.py:173-198)"""
    _fields_ = [('match_evalue', f64), ('skip_pen', f64), ('bandwidth', i64),
                ('max_half_z_score', f64), ('running_stat_width', i64),
                ('min_obs_per_base', i64), ('raw_min_obs_per_base', i64),
                ('mean_obs_per_event', i64), ('z_shift', f64), ('stay_pen', f64),
                ('use_t_test_seg', i64), ('band_bound_thresh', i64),
                ('start_bw', i64), ('start_save_bw', i64), ('start_n_bases', i64)]


class ScaleValues(C.Structure):
    _fields_ = [('shift', f64), ('scale', f64), ('lower_lim', f64),
                ('upper_lim', f64), ('outlier_thresh', f64)]


class Policy(C.Structure):
    _fields_ = [('outlier_thresh', f64), ('max_raw_cpts', i64),
                ('min_event_to_seq_ratio', f64), ('sig_match_thresh', f64),
                ('max_scaling_iters', i64), ('is_rna', i64),
                ('skip_seq_scaling', i64), ('const_scale', f64),
                ('subsample_seed', C.c_uint32), ('rescue', C.c_uint32)]


# tb2_acc_block: one statistics block of an accuracy labelling call, passed as a row of
# TB2_ACC_BLOCK_FIELDS int64 values
ACC_BLOCK_DTYPE = np.dtype([(name, np.int64) for name in (
    'seq_off', 'seq_len', 'seq_start', 'stat_off', 'n_stat', 'ctrl_off', 'n_ctrl', 'mod_off',
    'n_mod', 'unmod_off', 'n_unmod', 'strand')])


class Motif(C.Structure):
    """tb2_motif: a TomboMotif as IUPAC bit sets (A = 1, C = 2, G = 4, T = 8)"""
    _fields_ = [('len', C.c_int32), ('mod_pos', C.c_int32), ('mask', C.c_uint8 * 32)]


_IUPAC_BITS = {'A': 1, 'C': 2, 'G': 4, 'T': 8, 'B': 14, 'D': 13, 'H': 11, 'K': 12, 'M': 3,
               'N': 15, 'R': 5, 'S': 6, 'V': 7, 'W': 9, 'Y': 10}


def motif_struct(motif):
    """tombo_helper.TomboMotif (raw_motif, mod_pos) -> tb2_motif"""
    raw = motif.raw_motif
    if not 1 <= len(raw) <= 32 or motif.mod_pos is None:
        raise ValueError('motifs of 1 to 32 bases with a modified position only')
    m = Motif()
    m.len, m.mod_pos = len(raw), int(motif.mod_pos)
    for j, letter in enumerate(raw):
        m.mask[j] = _IUPAC_BITS[letter]
    return m


TB2_ERR_UNEXPECTED, TB2_ERR_INVALID_ARG = 100, 201

_lib = None
_lock = threading.Lock()

# (return type, argument types) of every function in include/tombo_b200.h, in its order; tb2_ctx * is
# an opaque handle.  tests/test_abi_cpu.py checks this table against the header.
_I, _CTX = C.c_int, C.c_void_p
pI, pI32, pI64, pF64 = P(C.c_int), P(C.c_int32), P(i64), P(f64)
pI8, pU8 = P(C.c_int8), P(C.c_uint8)
pPar, pPol, pSV, pMotif = P(Params), P(Policy), P(ScaleValues), P(Motif)
pU32 = P(C.c_uint32)
_PROTOS = {
    'tb2_abi_version': (_I, []),
    'tb2_device_count': (_I, []),
    'tb2_ctx_create': (_I, [_I, P(_CTX)]),
    'tb2_ctx_destroy': (None, [_CTX]),
    'tb2_status_message': (C.c_char_p, [_I]),
    'tb2_last_error': (C.c_char_p, [_CTX]),
    'tb2_launch_count': (i64, [_CTX]),
    'tb2_last_timing': (_I, [_CTX, pF64]),
    'tb2_host_alloc': (C.c_void_p, [C.c_size_t]),
    'tb2_host_free': (None, [C.c_void_p]),
    'tb2_set_model': (_I, [_CTX, pF64, pF64, _I, _I]),
    'tb2_set_alt_model': (_I, [_CTX, pF64, _I]),
    'tb2_new_means': (_I, [_CTX, pF64, i64, pI64, i64, pF64]),
    'tb2_new_mean_stds': (_I, [_CTX, pF64, i64, pI64, i64, pF64, pF64]),
    'tb2_normalize_raw_signal': (_I, [_CTX, pF64, i64, _I, f64, f64, pSV, pF64, pSV]),
    'tb2_identify_stalls': (_I, [_CTX, pF64, i64, pI64, i64, pI64]),
    'tb2_valid_cpts_w_cap': (_I, [_CTX, pF64, i64, i64, i64, i64, _I, pI64, pI]),
    'tb2_banded_forward_pass': (_I, [_CTX, pF64, pI64, i64, i64, f64, f64, pF64, pI64]),
    'tb2_banded_traceback': (_I, [_CTX, pI64, pI64, i64, i64, i64, i64, pI64, pI]),
    'tb2_adaptive_banded_forward_pass': (_I, [_CTX, pF64, pI64, pI64, i64, i64, pF64, i64, pF64,
                                              pF64, f64, f64, f64, i64, f64, _I, f64, pI]),
    'tb2_theil_sen': (_I, [_CTX, f64, f64, pF64, pF64, i64, C.c_uint32, pF64, pI]),
    'tb2_find_adaptive_base_assignment': (_I, [_CTX, pI64, i64, pF64, pPar, pF64, pF64, i64, f64,
                                               pI64, pI64, pI64, pI]),
    'tb2_find_static_base_assignment': (_I, [_CTX, pF64, i64, pF64, pF64, i64, pPar, pI64, pI]),
    'tb2_find_seq_start_in_events': (_I, [_CTX, pF64, i64, pF64, pF64, i64, pPar, i64, i64, _I,
                                          f64, pI64, pF64, pI]),
    'tb2_debug_div_check': (_I, [_CTX, C.c_uint64, _I, _I, P(C.c_uint64), pF64]),
    'tb2_debug_counters': (_I, [_CTX, P(C.c_ulonglong), _I]),
    'tb2_resolve_skipped_bases_with_raw': (_I, [_CTX, pI64, i64, pF64, pF64, pF64, i64, pPar, i64,
                                                pI64, pI]),
    'tb2_resquiggle_batch': (_I, [_CTX, i64, C.c_void_p, _I, pI64, pU8, pI64, pPar, pPar, pPol,
                                  pI64, pI64, pSV, pF64, pF64, pF64, pI32, pI32, pI32]),
    'tb2_pipeline_chunks': (_I, [_I, i64, pI64, _I]),
    'tb2_batch_upload': (_I, [_CTX, i64, C.c_void_p, _I, pI64, pU8, pI64, pPar, pPol]),
    'tb2_batch_set_read_inputs': (_I, [_CTX, pSV, pI64, pI64]),
    'tb2_batch_compute': (_I, [_CTX, pPar, pPar, pPol, _I]),
    'tb2_batch_download': (_I, [_CTX, pI64, pI64, pSV, pF64, pF64, pF64, pI32, pI32, pI32]),
    'tb2_alt_model_llr_batch': (_I, [_CTX, i64, pF64, pI64, pU8, pI64, pI64, _I, _I, f64, f64, f64,
                                     pF64, pI64, pI64]),
    'tb2_calc_llh_ratio_windows': (_I, [_CTX, _I, i64, _I, pF64, pF64, pF64, pF64, pF64, f64, f64,
                                        f64, pF64]),
    'tb2_timer_start': (_I, [_CTX]),
    'tb2_timer_stop': (_I, [_CTX, pF64]),
    'tb2_batch_alt_llr': (_I, [_CTX, pI64, _I, _I, f64, f64, f64, pI64]),
    'tb2_batch_llr_download': (_I, [_CTX, pF64, pI64, pI64]),
    'tb2_alt_model_llr_motif_batch': (_I, [_CTX, i64, pF64, pI64, pU8, pI64, pI64, pI8, pMotif, i64,
                                           i64, i64, i64, _I, f64, f64, f64, pF64, pI64, pI64,
                                           pI32]),
    'tb2_batch_alt_llr_motif': (_I, [_CTX, pI64, pI8, pMotif, i64, i64, i64, i64, _I, f64, f64, f64,
                                     pI32, pI64]),
    'tb2_region_stats_begin': (_I, [_CTX, i64, i64]),
    'tb2_region_stats_add': (_I, [_CTX, i64, pF64, pI64, f64, f64, _I]),
    'tb2_region_stats_add_batch_llr': (_I, [_CTX, f64, f64, _I]),
    'tb2_region_counts_get': (_I, [_CTX, pI32]),
    'tb2_region_counts_set': (_I, [_CTX, pI32]),
    'tb2_region_stats_finalize': (_I, [_CTX, f64, f64, i64, pI64, pF64, pF64, pI64, pI64, pI64]),
    'tb2_window_fisher_pvals': (_I, [_CTX, i64, pF64, pF64, pF64, pI64, i64, _I, pF64]),
    'tb2_de_novo_read_stats_batch': (_I, [_CTX, i64, pF64, pI64, pU8, pI64, pI64, i64, pF64, pI64,
                                          pI64]),
    'tb2_de_novo_region_stats': (_I, [_CTX, i64, pF64, pI64, pU8, pI64, pI64, pI8, i64, i64, i64,
                                      pF64, pI64, pI64, pI32]),
    'tb2_sample_compare_region_stats': (_I, [_CTX, i64, pF64, pI64, pI64, pI8, pF64, pF64, i64, i64,
                                             i64, pF64, pI64, pI64, pI32]),
    'tb2_batch_de_novo_region': (_I, [_CTX, pI64, pI8, i64, i64, i64, pF64, pI64, pI64, pI32]),
    'tb2_region_stats_add_tests': (_I, [_CTX, f64, f64]),
    'tb2_group_reg_stats': (_I, [_CTX, i64, i64, i64, pF64, pI64, pI64, i64, pF64, pI64, pI64, _I,
                                 _I, i64, i64, i64, pI64, pF64, pI64, pI64, pI64]),
    'tb2_reads_ref_levels': (_I, [_CTX, i64, i64, i64, pF64, pI64, pI64, i64, _I, pF64, pF64, f64,
                                  f64, pF64, pF64, pI64]),
    'tb2_kernel_densities': (_I, [_CTX, i64, pF64, pI64, i64, pF64, f64, pF64, pF64, pF64]),
    'tb2_kmer_level_summaries': (_I, [_CTX, i64, i64, pF64, pI64, pI64, i64, _I, pF64, pF64, pI64]),
    'tb2_kmer_medians': (_I, [_CTX, i64, i64, pI64, pF64, pF64, pI64, pF64, pF64]),
    'tb2_accuracy_reset': (_I, [_CTX]),
    'tb2_accuracy_count': (_I, [_CTX, _I, pI64]),
    'tb2_accuracy_download': (_I, [_CTX, _I, pF64, pU8]),
    'tb2_accuracy_load': (_I, [_CTX, _I, i64, pF64, pU8]),
    'tb2_accuracy_label_motif': (_I, [_CTX, i64, pI64, i64, pU8, i64, pU32, pF64, _I, pMotif, pI32,
                                      i64, i64, pI64]),
    'tb2_accuracy_label_truth': (_I, [_CTX, i64, pI64, i64, pU32, pF64, i64, pI64, i64, pI64, _I,
                                      pI64]),
    'tb2_accuracy_label_ctrl': (_I, [_CTX, i64, pI64, i64, pU8, i64, pU32, pF64, i64, pU32, pF64, _I,
                                     pMotif, pI32, pI64]),
    'tb2_accuracy_curve': (_I, [_CTX, _I, i64, pI64, pI64, pF64, pF64, pF64]),
    'tb2_accuracy_rates_ordered': (_I, [_CTX, i64, pU8, i64, pI64, pI64, pF64, pF64, pF64]),
    'tb2_stats_file_aggregate': (_I, [_CTX, i64, pI64, i64, i64, pU32, pF64, f64, f64, _I, f64, f64,
                                      pI64]),
    'tb2_stats_file_aggregate_download': (_I, [_CTX, pU32, pF64, pF64, pU32, pU32]),
    'tb2_most_signif_begin': (_I, [_CTX, _I, i64]),
    'tb2_most_signif_end': (_I, [_CTX]),
    'tb2_most_signif_reset': (_I, [_CTX]),
    'tb2_most_signif_add_rows': (_I, [_CTX, i64, pF64, pF64, pU32, pU32, pU32, pU32, C.c_uint32,
                                      C.c_uint8]),
    'tb2_most_signif_add_aggregate': (_I, [_CTX]),
    'tb2_most_signif_count': (_I, [_CTX, pI64]),
    'tb2_most_signif_get': (_I, [_CTX, pF64, pF64, pU32, pU32, pU32, pU32, pU32, pU8]),
    'tb2_dwell_percentiles': (_I, [_CTX, i64, pI64, pI64, _I, pF64, pF64]),
    'tb2_batch_read_filters': (_I, [_CTX, f64, _I, pF64, pF64, pI8, pF64]),
    'tb2_read_mid_coverage': (_I, [_CTX, i64, pI64, pI64, pI64, pI64]),
    'tb2_coverage_runs': (_I, [_CTX, i64, pI64, pI64, pI64, pI64, pI64, pI64]),
    'tb2_slot_sums_begin': (_I, [_CTX, i64]),
    'tb2_slot_sums_add': (_I, [_CTX, i64, pI64, pI64, pF64, pU8]),
    'tb2_slot_sums_means': (_I, [_CTX, pF64]),
}


def load():
    """Load the shared library (no device needed)."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise TomboB200Error(
                    'libtombo_b200.so is not built (run `python -c "import '
                    '__graft_entry__ as g; g.build()"` or make -C '
                    'tombo_b200/csrc); there is no CPU fallback')
            lib = C.CDLL(LIB_PATH)
            for name, (res, args) in _PROTOS.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    return _lib


def status_message(st):
    return load().tb2_status_message(int(st)).decode()


class PinnedArray(object):
    """numpy array backed by page-locked host memory (tb2_host_alloc)."""

    def __init__(self, shape, dtype):
        lib = load()
        self._lib = lib
        dt = np.dtype(dtype)
        n = int(np.prod(shape))
        self._p = lib.tb2_host_alloc(max(1, n * dt.itemsize))
        if not self._p:
            raise TomboB200Error('tb2_host_alloc failed (no CUDA device?)')
        buf = (C.c_char * (n * dt.itemsize)).from_address(self._p)
        self.array = np.frombuffer(buf, dtype=dt, count=n).reshape(shape)

    def free(self):
        if self._p:
            self.array = None
            self._lib.tb2_host_free(self._p)
            self._p = None


def as_f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def as_i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def ptr(a, ctype):
    return a.ctypes.data_as(P(ctype))


def _offsets(seq_off, k):
    """base_off / seg_off of a batch: sequences shorter than the k-mer map zero bases (the
    library clamps the same way), and each read has one more segment boundary than bases"""
    nb = np.maximum((seq_off[1:] - seq_off[:-1]) - (k - 1), 0)
    base_off = np.concatenate([[0], np.cumsum(nb)]).astype(np.int64)
    return base_off, base_off + np.arange(base_off.shape[0], dtype=np.int64)


def _batch_outputs(out, base_off, seg_off, n_samples, want_norm_signal):
    """the nine output pointers of tb2_resquiggle_batch / tb2_batch_download, into arrays of
    ``out`` that fit (new ones otherwise)"""
    n = base_off.shape[0] - 1

    def buf(name, shape, dt):
        a = out.get(name)
        if a is None or a.shape != tuple(np.atleast_1d(shape)) or a.dtype != dt:
            a = out[name] = np.empty(shape, dtype=dt)
        return a
    segs = buf('segs', int(seg_off[-1]), np.int64)
    rsrtr = buf('read_start_rel_to_raw', n, np.int64)
    sv = buf('scale_values', (n, 5), np.float64)
    score = buf('sig_match_score', n, np.float64)
    norm_mean = buf('norm_mean', int(base_off[-1]), np.float64)
    status = buf('status', n, np.int32)
    n_iters = buf('n_iters', n, np.int32)
    flags = buf('flags', n, np.int32)
    norm_sig = buf('norm_signal', n_samples, np.float64) if want_norm_signal else None
    return (ptr(segs, i64), ptr(rsrtr, i64), ptr(sv, ScaleValues), ptr(score, f64),
            ptr(norm_mean, f64), ptr(norm_sig, f64) if norm_sig is not None else None,
            ptr(status, C.c_int32), ptr(n_iters, C.c_int32), ptr(flags, C.c_int32))


def params_struct(p):
    mhz = p.max_half_z_score
    return Params(float(p.match_evalue), float(p.skip_pen), int(p.bandwidth),
                  float('nan') if mhz is None else float(mhz),
                  int(p.running_stat_width), int(p.min_obs_per_base),
                  int(p.raw_min_obs_per_base), int(p.mean_obs_per_event),
                  float(p.z_shift), float(p.stay_pen), int(bool(p.use_t_test_seg)),
                  int(p.band_bound_thresh), int(p.start_bw), int(p.start_save_bw),
                  int(p.start_n_bases))


class Context(object):
    """One CUDA context/stream (tb2_ctx).  Not thread safe; one per GPU/thread."""

    def __init__(self, device=0):
        lib = load()
        h = C.c_void_p()
        rc = lib.tb2_ctx_create(int(device), C.byref(h))
        if rc != 0 or not h:
            raise TomboB200Error(
                'cannot create a CUDA context on device %d (%s); tombo_b200 has '
                'no CPU fallback' % (device, status_message(rc)))
        self._h = h
        self.lib = lib
        self.device = device

    def close(self):
        if getattr(self, '_h', None):
            self.lib.tb2_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        if not self._h:
            raise TomboB200Error('context is closed')
        return self._h

    def check(self, rc):
        if rc != 0:
            msg = status_message(rc)
            err = self.lib.tb2_last_error(self.handle).decode()
            if err:
                msg += ': ' + err
            raise TomboB200Error('tombo_b200 call failed (%d): %s' % (rc, msg))

    def launch_count(self):
        return int(self.lib.tb2_launch_count(self.handle))

    def timer_start(self):
        self.check(self.lib.tb2_timer_start(self.handle))

    def timer_stop(self):
        """device milliseconds since timer_start (CUDA events on the library's stream)"""
        ms = f64(0.0)
        self.check(self.lib.tb2_timer_stop(self.handle, C.byref(ms)))
        return float(ms.value)

    def last_timing(self):
        """(compute ms, DP-kernel ms, DP launches, reads summed over DP launches)"""
        out = (f64 * 4)()
        self.lib.tb2_last_timing(self.handle, out)
        return tuple(out)

    # ---- staged batch API (resident inputs) --------------------------------
    def batch_upload(self, raw, raw_off, seq, seq_off, params, policy):
        raw = np.ascontiguousarray(raw)
        dtype = 1 if raw.dtype == np.int16 else 0
        if dtype == 0:
            raw = as_f64(raw)
        raw_off, seq_off = as_i64(raw_off), as_i64(seq_off)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        p = params if isinstance(params, Params) else params_struct(params)
        self.check(self.lib.tb2_batch_upload(self.handle, raw_off.shape[0] - 1,
                                             raw.ctypes.data_as(C.c_void_p), dtype,
                                             ptr(raw_off, i64), ptr(seq, C.c_uint8),
                                             ptr(seq_off, i64), C.byref(p), C.byref(policy)))
        self._base_off, self._seg_off = _offsets(seq_off, self.kmer_width)
        self._n_samples = int(raw_off[-1])

    def batch_compute(self, params, save_params, policy, want_norm_signal=False):
        p = params if isinstance(params, Params) else params_struct(params)
        sp = None
        if save_params is not None:
            sp = save_params if isinstance(save_params, Params) else params_struct(save_params)
        self.check(self.lib.tb2_batch_compute(self.handle, C.byref(p),
                                              C.byref(sp) if sp is not None else None,
                                              C.byref(policy), int(bool(want_norm_signal))))

    def batch_download(self, want_norm_signal=False, out=None):
        base_off, seg_off = self._base_off, self._seg_off
        if out is None:
            out = {}
        outs = _batch_outputs(out, base_off, seg_off, self._n_samples, want_norm_signal)
        self.check(self.lib.tb2_batch_download(self.handle, *outs))
        out['base_off'], out['seg_off'] = base_off, seg_off
        return out

    # ---- mirror API: _c_dynamic_programming.pyx ---------------------------
    def banded_forward_pass(self, z, event_starts, skip_pen, stay_pen):
        z = as_f64(z)
        es = as_i64(event_starts)
        nb, bw = z.shape
        fwd = np.empty((nb + 1, bw))
        tb = np.empty((nb + 1, bw), dtype=np.int64)
        self.check(self.lib.tb2_banded_forward_pass(self.handle, ptr(z, f64), ptr(es, i64), nb, bw,
                                                    skip_pen, stay_pen, ptr(fwd, f64),
                                                    ptr(tb, i64)))
        return fwd, tb

    def banded_traceback(self, tb, event_starts, band_pos, thresh=-1):
        tb = as_i64(tb)
        es = as_i64(event_starts)
        nb = tb.shape[0] - 1
        out = np.empty(nb + 1, dtype=np.int64)
        st = C.c_int(0)
        self.check(self.lib.tb2_banded_traceback(self.handle, ptr(tb, i64), ptr(es, i64), nb,
                                                 tb.shape[1], int(band_pos), int(thresh),
                                                 ptr(out, i64), C.byref(st)))
        return st.value, out

    def adaptive_banded_forward_pass(self, fwd, tb, event_starts, event_means,
                                     rm, rs, z_shift, skip_pen, stay_pen,
                                     start_seq_pos, mask_fill_z, do_winsorize,
                                     max_half_z):
        assert fwd.flags.c_contiguous and fwd.dtype == np.float64
        assert tb.flags.c_contiguous and tb.dtype == np.int64
        assert event_starts.flags.c_contiguous and event_starts.dtype == np.int64
        em, rm, rs = as_f64(event_means), as_f64(rm), as_f64(rs)
        st = C.c_int(0)
        self.check(self.lib.tb2_adaptive_banded_forward_pass(
            self.handle, ptr(fwd, f64), ptr(tb, i64), ptr(event_starts, i64), fwd.shape[0] - 1,
            fwd.shape[1], ptr(em, f64), em.shape[0], ptr(rm, f64), ptr(rs, f64), z_shift,
            skip_pen, stay_pen, int(start_seq_pos), mask_fill_z, int(bool(do_winsorize)),
            max_half_z, C.byref(st)))
        return st.value

    def find_adaptive_base_assignment(self, valid_cpts, event_means, params,
                                      rm, rs, sig_match_thresh=1.1):
        cp, em = as_i64(valid_cpts), as_f64(event_means)
        rm, rs = as_f64(rm), as_f64(rs)
        nb = rm.shape[0]
        segs = np.empty(nb + 1, dtype=np.int64)
        rsrtr = i64(0)
        dbg = np.zeros(3, dtype=np.int64)
        st = C.c_int(0)
        p = params if isinstance(params, Params) else params_struct(params)
        self.check(self.lib.tb2_find_adaptive_base_assignment(
            self.handle, ptr(cp, i64), cp.shape[0], ptr(em, f64), C.byref(p), ptr(rm, f64),
            ptr(rs, f64), nb, sig_match_thresh, ptr(segs, i64), C.byref(rsrtr), ptr(dbg, i64),
            C.byref(st)))
        return st.value, segs, rsrtr.value, dbg


    # ---- models -----------------------------------------------------------
    def set_model(self, means, sds, kmer_width, central_pos):
        means, sds = as_f64(means), as_f64(sds)
        assert means.shape[0] == 4 ** kmer_width == sds.shape[0]
        self._model_ref = self._model_digest = None     # ensure_model uploads next time
        self.check(self.lib.tb2_set_model(self.handle, ptr(means, f64), ptr(sds, f64),
                                          int(kmer_width), int(central_pos)))
        self.kmer_width, self.central_pos = kmer_width, central_pos

    def set_alt_model(self, alt_means, kmer_width):
        alt_means = as_f64(alt_means)
        assert alt_means.size == 4 ** kmer_width * kmer_width
        self.check(self.lib.tb2_set_alt_model(self.handle, ptr(alt_means, f64), int(kmer_width)))

    # ---- mirror API: _c_helper.pyx / tombo_stats.py ------------------------
    def new_means(self, sig, segs):
        sig, segs = as_f64(sig), as_i64(segs)
        out = np.empty(segs.shape[0] - 1)
        self.check(self.lib.tb2_new_means(self.handle, ptr(sig, f64), sig.shape[0], ptr(segs, i64),
                                          out.shape[0], ptr(out, f64)))
        return out

    def new_mean_stds(self, sig, segs):
        sig, segs = as_f64(sig), as_i64(segs)
        m = np.empty(segs.shape[0] - 1)
        sd = np.empty(segs.shape[0] - 1)
        self.check(self.lib.tb2_new_mean_stds(self.handle, ptr(sig, f64), sig.shape[0],
                                              ptr(segs, i64), m.shape[0], ptr(m, f64),
                                              ptr(sd, f64)))
        return m, sd

    def normalize_raw_signal(self, raw, outlier_thresh=None, scale_values=None,
                             const_scale=None):
        raw = as_f64(raw)
        norm = np.empty_like(raw)
        sv = ScaleValues()
        svi = None
        if scale_values is not None:
            svi = ScaleValues(*[float('nan') if v is None else float(v)
                                for v in scale_values])
        st = self.lib.tb2_normalize_raw_signal(
            self.handle, ptr(raw, f64), raw.shape[0], 0 if const_scale is None else 1,
            float('nan') if outlier_thresh is None else outlier_thresh,
            float('nan') if const_scale is None else const_scale,
            C.byref(svi) if svi is not None else None, ptr(norm, f64), C.byref(sv))
        if st >= 200:
            self.check(st)
        return st, norm, (sv.shift, sv.scale, sv.lower_lim, sv.upper_lim,
                          sv.outlier_thresh)

    def valid_cpts_w_cap(self, sig, min_base_obs, running_stat_width, num_cpts,
                         t_test=False):
        sig = as_f64(sig)
        out = np.empty(num_cpts, dtype=np.int64)
        st = C.c_int(0)
        self.check(self.lib.tb2_valid_cpts_w_cap(self.handle, ptr(sig, f64), sig.shape[0],
                                                 int(min_base_obs), int(running_stat_width),
                                                 int(num_cpts), int(bool(t_test)), ptr(out, i64),
                                                 C.byref(st)))
        return st.value, out

    def theil_sen(self, prev_shift, prev_scale, event_means, model_means, key=0):
        ev, md = as_f64(event_means), as_f64(model_means)
        out = np.empty(4)
        st = C.c_int(0)
        self.check(self.lib.tb2_theil_sen(self.handle, prev_shift, prev_scale, ptr(ev, f64),
                                          ptr(md, f64), ev.shape[0], int(key), ptr(out, f64),
                                          C.byref(st)))
        return st.value, tuple(out)

    def resolve_skipped_bases_with_raw(self, segs, rm, rs, norm, params,
                                       max_raw_cpts=200):
        segs, rm, rs, norm = as_i64(segs), as_f64(rm), as_f64(rs), as_f64(norm)
        out = np.empty_like(segs)
        st = C.c_int(0)
        p = params if isinstance(params, Params) else params_struct(params)
        self.check(self.lib.tb2_resolve_skipped_bases_with_raw(
            self.handle, ptr(segs, i64), segs.shape[0] - 1, ptr(rm, f64), ptr(rs, f64),
            ptr(norm, f64), norm.shape[0], C.byref(p),
            -1 if max_raw_cpts is None else int(max_raw_cpts), ptr(out, i64), C.byref(st)))
        return st.value, out

    def identify_stalls(self, raw):
        raw = as_f64(raw)
        cap = raw.shape[0] // 200 + 4
        out = np.empty(2 * cap, dtype=np.int64)
        n = i64(0)
        self.check(self.lib.tb2_identify_stalls(self.handle, ptr(raw, f64), raw.shape[0],
                                                ptr(out, i64), cap, C.byref(n)))
        return out[:2 * n.value].reshape(-1, 2).copy()

    def calc_llh_ratio_windows(self, mode, means, ref_means, alt_means, var_a, var_b=None,
                               scale_factor=4.0, height_factor=1.0, height_power=0.2):
        means, ref_means, alt_means = as_f64(means), as_f64(ref_means), as_f64(alt_means)
        var_a = as_f64(var_a)
        n, k = means.shape
        out = np.empty(n)
        vb = as_f64(var_b) if var_b is not None else None
        self.check(self.lib.tb2_calc_llh_ratio_windows(
            self.handle, int(mode), n, k, ptr(means, f64), ptr(ref_means, f64),
            ptr(alt_means, f64), ptr(var_a, f64), ptr(vb, f64) if vb is not None else None,
            scale_factor, height_factor, height_power, ptr(out, f64)))
        return out

    def find_static_base_assignment(self, event_means, rm, rs, params):
        em, rm, rs = as_f64(event_means), as_f64(rm), as_f64(rs)
        out = np.empty(rm.shape[0] + 1, dtype=np.int64)
        st = C.c_int(0)
        p = params if isinstance(params, Params) else params_struct(params)
        self.check(self.lib.tb2_find_static_base_assignment(
            self.handle, ptr(em, f64), em.shape[0], ptr(rm, f64), ptr(rs, f64), rm.shape[0],
            C.byref(p), ptr(out, i64), C.byref(st)))
        return st.value, out

    def find_seq_start_in_events(self, event_means, rm, rs, params, num_bases, num_events,
                                 sig_match_thresh=None):
        em, rm, rs = as_f64(event_means), as_f64(rm), as_f64(rs)
        st, sl, epb = C.c_int(0), i64(0), f64(0)
        p = params if isinstance(params, Params) else params_struct(params)
        self.check(self.lib.tb2_find_seq_start_in_events(
            self.handle, ptr(em, f64), em.shape[0], ptr(rm, f64), ptr(rs, f64), rm.shape[0],
            C.byref(p), int(num_bases), int(num_events), int(sig_match_thresh is not None),
            0.0 if sig_match_thresh is None else sig_match_thresh, C.byref(sl), C.byref(epb),
            C.byref(st)))
        return st.value, sl.value, epb.value

    def batch_set_read_inputs(self, scale_values=None, stall_ints=None):
        """scale_values: (n, 5) array with NaN shift where absent, or None;
        stall_ints: list (per read) of lists of (start, end), or None."""
        sv = None
        if scale_values is not None:
            sv = np.ascontiguousarray(scale_values, dtype=np.float64)
        flat = off = None
        if stall_ints is not None:
            off = np.zeros(len(stall_ints) + 1, dtype=np.int64)
            off[1:] = np.cumsum([len(s) for s in stall_ints])
            flat = np.zeros(max(1, int(off[-1])) * 2, dtype=np.int64)
            k = 0
            for s in stall_ints:
                for a, b in s:
                    flat[2 * k], flat[2 * k + 1] = a, b
                    k += 1
        self.check(self.lib.tb2_batch_set_read_inputs(
            self.handle, ptr(sv, ScaleValues) if sv is not None else None,
            ptr(flat, i64) if flat is not None else None,
            ptr(off, i64) if off is not None else None))

    # ---- the batched hot path ----------------------------------------------
    def resquiggle_batch(self, raw, raw_off, seq, seq_off, params, save_params,
                         policy, want_norm_signal=False, out=None):
        """tb2_resquiggle_batch.  raw: float64 or int16 flat array; seq: uint8
        base codes.  Returns a dict of numpy arrays (see include/tombo_b200.h)."""
        raw = np.ascontiguousarray(raw)
        if raw.dtype == np.int16:
            dtype = 1
        else:
            raw = as_f64(raw)
            dtype = 0
        raw_off, seq_off = as_i64(raw_off), as_i64(seq_off)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        base_off, seg_off = _offsets(seq_off, self.kmer_width)
        if out is None:
            out = {}
        outs = _batch_outputs(out, base_off, seg_off, raw.shape[0], want_norm_signal)
        p = params if isinstance(params, Params) else params_struct(params)
        sp = None
        if save_params is not None:
            sp = save_params if isinstance(save_params, Params) else params_struct(save_params)
        self.check(self.lib.tb2_resquiggle_batch(
            self.handle, raw_off.shape[0] - 1, raw.ctypes.data_as(C.c_void_p), dtype,
            ptr(raw_off, i64), ptr(seq, C.c_uint8), ptr(seq_off, i64), C.byref(p),
            C.byref(sp) if sp is not None else None, C.byref(policy), *outs))
        out['base_off'], out['seg_off'] = base_off, seg_off
        return out

    def alt_model_llr_batch(self, norm_mean, mean_off, seq, seq_off, read_start,
                            alt_base_code, use_standard_llhr=False,
                            scale_factor=4.0, height_factor=1.0, height_power=0.2):
        norm_mean, mean_off = as_f64(norm_mean), as_i64(mean_off)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        seq_off, read_start = as_i64(seq_off), as_i64(read_start)
        n = mean_off.shape[0] - 1
        cap = max(1, norm_mean.shape[0])
        llr = np.empty(cap)
        pos = np.empty(cap, dtype=np.int64)
        site_off = np.zeros(n + 1, dtype=np.int64)
        self.check(self.lib.tb2_alt_model_llr_batch(
            self.handle, n, ptr(norm_mean, f64), ptr(mean_off, i64), ptr(seq, C.c_uint8),
            ptr(seq_off, i64), ptr(read_start, i64), int(alt_base_code),
            int(bool(use_standard_llhr)), scale_factor, height_factor, height_power,
            ptr(llr, f64), ptr(pos, i64), ptr(site_off, i64)))
        tot = int(site_off[-1])
        return llr[:tot].copy(), pos[:tot].copy(), site_off


    # ---- per-read statistics on the resident batch / SURVEY 8(f) ----------
    def batch_alt_llr(self, read_start, alt_base_code, use_standard_llhr=False,
                      scale_factor=4.0, height_factor=1.0, height_power=0.2):
        """LLRs of the resident batch (after batch_compute); returns the site count"""
        read_start = as_i64(read_start)
        tot = i64(0)
        self.check(self.lib.tb2_batch_alt_llr(self.handle, ptr(read_start, i64), int(alt_base_code),
                                              int(bool(use_standard_llhr)), scale_factor,
                                              height_factor, height_power, C.byref(tot)))
        self._llr_total, self._llr_reads = int(tot.value), read_start.shape[0]
        return self._llr_total

    def alt_model_llr_motif_batch(self, norm_mean, mean_off, seq, seq_off, read_start, strand,
                                  motif, max_motif_bb, max_motif_ab, reg_start, reg_end,
                                  use_standard_llhr=False, scale_factor=4.0, height_factor=1.0,
                                  height_power=0.2):
        """tb2_alt_model_llr_motif_batch; motif is a Motif.  Returns (llr, pos, site_off,
        read_status)."""
        norm_mean, mean_off = as_f64(norm_mean), as_i64(mean_off)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        seq_off, read_start = as_i64(seq_off), as_i64(read_start)
        strand = np.ascontiguousarray(strand, dtype=np.int8)
        n = mean_off.shape[0] - 1
        cap = max(1, norm_mean.shape[0])
        llr = np.empty(cap)
        pos = np.empty(cap, dtype=np.int64)
        site_off = np.zeros(n + 1, dtype=np.int64)
        status = np.zeros(max(1, n), dtype=np.int32)
        self.check(self.lib.tb2_alt_model_llr_motif_batch(
            self.handle, n, ptr(norm_mean, f64), ptr(mean_off, i64), ptr(seq, C.c_uint8),
            ptr(seq_off, i64), ptr(read_start, i64), ptr(strand, C.c_int8), C.byref(motif),
            int(max_motif_bb), int(max_motif_ab), int(reg_start), int(reg_end),
            int(bool(use_standard_llhr)), scale_factor, height_factor, height_power,
            ptr(llr, f64), ptr(pos, i64), ptr(site_off, i64), ptr(status, C.c_int32)))
        tot = int(site_off[-1])
        return llr[:tot].copy(), pos[:tot].copy(), site_off, status[:n].copy()

    def batch_alt_llr_motif(self, read_start, strand, motif, max_motif_bb, max_motif_ab,
                            reg_start, reg_end, use_standard_llhr=False, scale_factor=4.0,
                            height_factor=1.0, height_power=0.2):
        """motif LLRs of the resident batch (after batch_compute); returns (site count,
        read_status).  batch_llr_download and region_stats_add_batch_llr read them."""
        read_start = as_i64(read_start)
        strand = np.ascontiguousarray(strand, dtype=np.int8)
        n = self._base_off.shape[0] - 1 if getattr(self, '_base_off', None) is not None else -1
        if read_start.shape != (n,) or strand.shape != (n,):
            raise ValueError('read_start and strand need one entry per read of the resident '
                             'batch (%d)' % n)
        status = np.zeros(max(1, n), dtype=np.int32)
        tot = i64(0)
        self.check(self.lib.tb2_batch_alt_llr_motif(
            self.handle, ptr(read_start, i64), ptr(strand, C.c_int8), C.byref(motif),
            int(max_motif_bb), int(max_motif_ab), int(reg_start), int(reg_end),
            int(bool(use_standard_llhr)), scale_factor, height_factor, height_power,
            ptr(status, C.c_int32), C.byref(tot)))
        self._llr_total, self._llr_reads = int(tot.value), read_start.shape[0]
        return self._llr_total, status[:read_start.shape[0]].copy()

    def batch_llr_download(self):
        llr = np.empty(max(1, self._llr_total))
        pos = np.empty(max(1, self._llr_total), dtype=np.int64)
        site_off = np.zeros(self._llr_reads + 1, dtype=np.int64)
        self.check(self.lib.tb2_batch_llr_download(self.handle, ptr(llr, f64), ptr(pos, i64),
                                                   ptr(site_off, i64)))
        return llr[:self._llr_total], pos[:self._llr_total], site_off

    def region_stats_begin(self, reg_start, reg_len):
        self.check(self.lib.tb2_region_stats_begin(self.handle, int(reg_start), int(reg_len)))
        self._reg_len = int(reg_len)

    def region_stats_add(self, stats, pos, single_read_thresh, lower_thresh=None, stat_type=0):
        stats, pos = as_f64(stats), as_i64(pos)
        self.check(self.lib.tb2_region_stats_add(
            self.handle, stats.shape[0], ptr(stats, f64), ptr(pos, i64), single_read_thresh,
            float('nan') if lower_thresh is None else lower_thresh, int(stat_type)))

    def region_stats_add_batch_llr(self, single_read_thresh, lower_thresh=None, stat_type=0):
        self.check(self.lib.tb2_region_stats_add_batch_llr(
            self.handle, single_read_thresh,
            float('nan') if lower_thresh is None else lower_thresh, int(stat_type)))

    def region_counts_get(self):
        cnt = np.zeros(3 * self._reg_len, dtype=np.int32)
        self.check(self.lib.tb2_region_counts_get(self.handle, ptr(cnt, C.c_int32)))
        return cnt

    def region_counts_set(self, counts):
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        assert cnt.shape[0] == 3 * self._reg_len
        self.check(self.lib.tb2_region_counts_set(self.handle, ptr(cnt, C.c_int32)))

    def region_stats_finalize(self, unmod_count=None, mod_count=None):
        cap = self._reg_len
        pos = np.empty(cap, dtype=np.int64)
        frac, damp = np.empty(cap), np.empty(cap)
        cov, valid = np.empty(cap, dtype=np.int64), np.empty(cap, dtype=np.int64)
        n = i64(0)
        self.check(self.lib.tb2_region_stats_finalize(
            self.handle, float('nan') if unmod_count is None else unmod_count,
            0.0 if mod_count is None else mod_count, cap, ptr(pos, i64), ptr(frac, f64),
            ptr(damp, f64), ptr(cov, i64), ptr(valid, i64), C.byref(n)))
        m = int(n.value)
        return dict(pos=pos[:m].copy(), frac=frac[:m].copy(), damp_frac=damp[:m].copy(),
                    cov=cov[:m].copy(), valid_cov=valid[:m].copy())

    def window_fisher_pvals(self, means, ref_means, ref_sds, seg_off, fm_offset, final_clamp):
        means = as_f64(means)
        seg_off = as_i64(seg_off)
        out = np.empty(max(1, means.shape[0]))
        if ref_means is None:            # `means` are p-values: Fisher window only
            prm = prs = None
        else:
            ref_means, ref_sds = as_f64(ref_means), as_f64(ref_sds)
            prm, prs = ptr(ref_means, f64), ptr(ref_sds, f64)
        self.check(self.lib.tb2_window_fisher_pvals(
            self.handle, seg_off.shape[0] - 1, ptr(means, f64), prm, prs, ptr(seg_off, i64),
            int(fm_offset), int(bool(final_clamp)), ptr(out, f64)))
        return out[:means.shape[0]]

    def group_reg_stats(self, reg_start, reg_len, samp, ctrl, test, return_stat, min_test_reads,
                        fm_offset):
        """tb2_group_reg_stats.  ``samp`` / ``ctrl`` are ragged genome-ordered reads
        ``(levels, off, start)``; ``test`` 0 = KS, 1 = U, 2 = t.  Returns a dict of the
        covered positions (ascending), their statistic and both coverages."""
        (sl, so, ss), (cl, co, cs) = [(as_f64(l), as_i64(o), as_i64(s)) for l, o, s in (samp, ctrl)]
        cap = int(reg_len)
        pos, stat = np.empty(cap, dtype=np.int64), np.empty(cap)
        cov, ccov = np.empty(cap, dtype=np.int64), np.empty(cap, dtype=np.int64)
        n = i64(0)
        self.check(self.lib.tb2_group_reg_stats(
            self.handle, int(reg_start), cap, so.shape[0] - 1, ptr(sl, f64), ptr(so, i64),
            ptr(ss, i64), co.shape[0] - 1, ptr(cl, f64), ptr(co, i64), ptr(cs, i64), int(test),
            int(bool(return_stat)), int(min_test_reads), int(fm_offset), cap, ptr(pos, i64),
            ptr(stat, f64), ptr(cov, i64), ptr(ccov, i64), C.byref(n)))
        m = int(n.value)
        return dict(pos=pos[:m].copy(), stat=stat[:m].copy(), cov=cov[:m].copy(),
                    ctrl_cov=ccov[:m].copy())

    def reads_ref_levels(self, reg_start, reg_len, reads, min_test_reads, est_mean=False,
                         prior_means=None, prior_sds=None, prior_weights=(0.0, 0.0)):
        """tb2_reads_ref_levels -> (means, sds, cov), each reg_len long"""
        lv, off, st = as_f64(reads[0]), as_i64(reads[1]), as_i64(reads[2])
        n = int(reg_len)
        means, sds, cov = np.empty(n), np.empty(n), np.empty(n, dtype=np.int64)
        pm = ps = None
        if prior_means is not None:
            prior_means, prior_sds = as_f64(prior_means), as_f64(prior_sds)
            if prior_means.shape[0] != n or prior_sds.shape[0] != n:
                raise ValueError('prior levels must cover the region')
            pm, ps = ptr(prior_means, f64), ptr(prior_sds, f64)
        self.check(self.lib.tb2_reads_ref_levels(
            self.handle, int(reg_start), n, off.shape[0] - 1, ptr(lv, f64), ptr(off, i64),
            ptr(st, i64), int(min_test_reads), int(bool(est_mean)), pm, ps,
            float(prior_weights[0]), float(prior_weights[1]), ptr(means, f64), ptr(sds, f64),
            ptr(cov, i64)))
        return means, sds, cov

    def de_novo_read_stats_batch(self, norm_mean, mean_off, seq, seq_off, read_start, fm_offset=1):
        norm_mean, mean_off = as_f64(norm_mean), as_i64(mean_off)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        seq_off, read_start = as_i64(seq_off), as_i64(read_start)
        n = mean_off.shape[0] - 1
        cap = max(1, norm_mean.shape[0])
        pv = np.empty(cap)
        pos = np.empty(cap, dtype=np.int64)
        stat_off = np.zeros(n + 1, dtype=np.int64)
        self.check(self.lib.tb2_de_novo_read_stats_batch(
            self.handle, n, ptr(norm_mean, f64), ptr(mean_off, i64), ptr(seq, C.c_uint8),
            ptr(seq_off, i64), ptr(read_start, i64), int(fm_offset), ptr(pv, f64), ptr(pos, i64),
            ptr(stat_off, i64)))
        t = int(stat_off[-1])
        return pv[:t].copy(), pos[:t].copy(), stat_off

    def de_novo_region_stats(self, norm_mean, mean_off, seq, seq_off, read_start, strand,
                             fm_offset, reg_start, reg_end):
        """tb2_de_novo_region_stats -> (pvals, pos, stat_off, read_status); the statistics
        also stay on the device for region_stats_add_tests"""
        norm_mean, mean_off = as_f64(norm_mean), as_i64(mean_off)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        seq_off, read_start = as_i64(seq_off), as_i64(read_start)
        strand = np.ascontiguousarray(strand, dtype=np.int8)
        n = mean_off.shape[0] - 1
        cap = max(1, norm_mean.shape[0])
        pv, pos = np.empty(cap), np.empty(cap, dtype=np.int64)
        stat_off = np.zeros(n + 1, dtype=np.int64)
        status = np.zeros(max(1, n), dtype=np.int32)
        self.check(self.lib.tb2_de_novo_region_stats(
            self.handle, n, ptr(norm_mean, f64), ptr(mean_off, i64), ptr(seq, C.c_uint8),
            ptr(seq_off, i64), ptr(read_start, i64), ptr(strand, C.c_int8), int(fm_offset),
            int(reg_start), int(reg_end), ptr(pv, f64), ptr(pos, i64), ptr(stat_off, i64),
            ptr(status, C.c_int32)))
        t = int(stat_off[-1])
        return pv[:t].copy(), pos[:t].copy(), stat_off, status[:n].copy()

    def sample_compare_region_stats(self, norm_mean, mean_off, read_start, strand, ctrl_means,
                                    ctrl_sds, fm_offset, reg_start, reg_end):
        """tb2_sample_compare_region_stats -> (pvals, pos, stat_off, read_status); ctrl_*
        cover [reg_start - fm_offset, reg_end + fm_offset)"""
        norm_mean, mean_off, read_start = as_f64(norm_mean), as_i64(mean_off), as_i64(read_start)
        strand = np.ascontiguousarray(strand, dtype=np.int8)
        ctrl_means, ctrl_sds = as_f64(ctrl_means), as_f64(ctrl_sds)
        if not ctrl_means.shape[0] == ctrl_sds.shape[0] == int(reg_end) - int(reg_start) + 2 * int(fm_offset):
            raise ValueError('control levels must cover [reg_start - fm_offset, reg_end + fm_offset)')
        n = mean_off.shape[0] - 1
        cap = max(1, norm_mean.shape[0])
        pv, pos = np.empty(cap), np.empty(cap, dtype=np.int64)
        stat_off = np.zeros(n + 1, dtype=np.int64)
        status = np.zeros(max(1, n), dtype=np.int32)
        self.check(self.lib.tb2_sample_compare_region_stats(
            self.handle, n, ptr(norm_mean, f64), ptr(mean_off, i64), ptr(read_start, i64),
            ptr(strand, C.c_int8), ptr(ctrl_means, f64), ptr(ctrl_sds, f64), int(fm_offset),
            int(reg_start), int(reg_end), ptr(pv, f64), ptr(pos, i64), ptr(stat_off, i64),
            ptr(status, C.c_int32)))
        t = int(stat_off[-1])
        return pv[:t].copy(), pos[:t].copy(), stat_off, status[:n].copy()

    def batch_de_novo_region(self, read_start, strand, fm_offset, reg_start, reg_end,
                             download=True):
        """de novo test of the resident batch (after batch_compute) -> (pvals, pos, stat_off,
        read_status); with download=False the statistics stay on the device only and
        (None, None, stat_off, read_status) is returned"""
        read_start = as_i64(read_start)
        strand = np.ascontiguousarray(strand, dtype=np.int8)
        n = self._base_off.shape[0] - 1 if getattr(self, '_base_off', None) is not None else -1
        if read_start.shape != (n,) or strand.shape != (n,):
            raise ValueError('read_start and strand need one entry per read of the resident '
                             'batch (%d)' % n)
        cap = max(1, int(self._base_off[-1]))
        pv = np.empty(cap) if download else None
        pos = np.empty(cap, dtype=np.int64) if download else None
        stat_off = np.zeros(n + 1, dtype=np.int64)
        status = np.zeros(max(1, n), dtype=np.int32)
        self.check(self.lib.tb2_batch_de_novo_region(
            self.handle, ptr(read_start, i64), ptr(strand, C.c_int8), int(fm_offset),
            int(reg_start), int(reg_end), ptr(pv, f64) if download else None,
            ptr(pos, i64) if download else None, ptr(stat_off, i64), ptr(status, C.c_int32)))
        t = int(stat_off[-1])
        if not download:
            return None, None, stat_off, status[:n].copy()
        return pv[:t].copy(), pos[:t].copy(), stat_off, status[:n].copy()

    def region_stats_add_tests(self, single_read_thresh, lower_thresh=None):
        """accumulate the last de novo / sample-compare region call into the open region"""
        self.check(self.lib.tb2_region_stats_add_tests(
            self.handle, single_read_thresh, float('nan') if lower_thresh is None else lower_thresh))

    def kernel_densities(self, levels, off, x, bw):
        """tb2_kernel_densities -> (densities (n_sets, len(x)), cho_cov, factor).  Set s is
        ``levels[off[s]:off[s + 1]]``; a set the reference cannot fit has NaN throughout."""
        levels, off, x = as_f64(levels), as_i64(off), as_f64(x)
        n = off.shape[0] - 1
        dens = np.empty((n, x.shape[0]))
        cho, factor = np.empty(n), np.empty(n)
        self.check(self.lib.tb2_kernel_densities(
            self.handle, n, ptr(levels, f64), ptr(off, i64), x.shape[0], ptr(x, f64),
            float(bw), ptr(dens, f64), ptr(cho, f64), ptr(factor, f64)))
        return dens, cho, factor

    def kmer_level_summaries(self, n_pos, reads, cov_thresh, est_mean=False):
        """tb2_kmer_level_summaries -> (levels, sds, cov), each n_pos long.  ``reads`` are
        ragged genome-ordered reads ``(levels, off, start)`` in positions 0 .. n_pos - 1;
        levels and sds are NaN where the coverage is not above ``cov_thresh``."""
        lv, off, st = as_f64(reads[0]), as_i64(reads[1]), as_i64(reads[2])
        n = int(n_pos)
        levels, sds, cov = np.empty(n), np.empty(n), np.empty(n, dtype=np.int64)
        self.check(self.lib.tb2_kmer_level_summaries(
            self.handle, n, off.shape[0] - 1, ptr(lv, f64), ptr(off, i64), ptr(st, i64),
            int(cov_thresh), int(bool(est_mean)), ptr(levels, f64), ptr(sds, f64), ptr(cov, i64)))
        return levels, sds, cov

    def kmer_medians(self, n_keys, keys, levels, sds):
        """tb2_kmer_medians -> (counts, median levels, median sds), each n_keys long (NaN
        medians for a key without observations)"""
        keys, levels, sds = as_i64(keys), as_f64(levels), as_f64(sds)
        if not keys.shape[0] == levels.shape[0] == sds.shape[0]:
            raise ValueError('keys, levels and sds must have one entry per observation')
        n = int(n_keys)
        cnt, med_lv, med_sd = np.empty(n, dtype=np.int64), np.empty(n), np.empty(n)
        self.check(self.lib.tb2_kmer_medians(
            self.handle, n, keys.shape[0], ptr(keys, i64), ptr(levels, f64), ptr(sds, f64),
            ptr(cnt, i64), ptr(med_lv, f64), ptr(med_sd, f64)))
        return cnt, med_lv, med_sd

    # accuracy of modified-base calls (csrc/accuracy.cu).  ``blocks`` is an ACC_BLOCK_DTYPE
    # array, ``seq`` the blocks' sequence codes, ``pos`` / ``stat`` their statistics.
    def _blocks(self, blocks):
        blocks = np.ascontiguousarray(blocks, dtype=ACC_BLOCK_DTYPE)
        return blocks, blocks.ctypes.data_as(pI64)

    def _label_args(self, pos, stat):
        pos = np.ascontiguousarray(pos, dtype=np.uint32)
        stat = as_f64(stat)
        if pos.shape != stat.shape:
            raise ValueError('pos and stat need one entry per statistic')
        return pos, stat

    def accuracy_reset(self):
        self.check(self.lib.tb2_accuracy_reset(self.handle))

    def accuracy_count(self, slot):
        n = i64(0)
        self.check(self.lib.tb2_accuracy_count(self.handle, int(slot), C.byref(n)))
        return int(n.value)

    def accuracy_download(self, slot):
        """(stats f64, labels bool) of a slot in append order"""
        n = self.accuracy_count(slot)
        st, lab = np.empty(max(1, n)), np.empty(max(1, n), dtype=np.uint8)
        self.check(self.lib.tb2_accuracy_download(self.handle, int(slot), ptr(st, f64),
                                                  ptr(lab, C.c_uint8)))
        return st[:n], lab[:n].view(bool)

    def accuracy_load(self, slot, stat, label):
        stat = as_f64(stat)
        label = np.ascontiguousarray(label, dtype=bool).view(np.uint8)
        if stat.shape != label.shape:
            raise ValueError('stat and label need the same length')
        self.check(self.lib.tb2_accuracy_load(self.handle, int(slot), stat.shape[0],
                                              ptr(stat, f64), ptr(label, C.c_uint8)))

    def accuracy_label_motif(self, blocks, seq, pos, stat, motifs, slots, bb, ab):
        """tb2_accuracy_label_motif -> counts (n_blocks, n_motifs)"""
        blocks, pb = self._blocks(blocks)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        pos, stat = self._label_args(pos, stat)
        ms = (Motif * len(motifs))(*motifs)
        sl = np.ascontiguousarray(slots, dtype=np.int32)
        cnt = np.zeros((max(1, blocks.shape[0]), len(motifs)), dtype=np.int64)
        rc = self.lib.tb2_accuracy_label_motif(
            self.handle, blocks.shape[0], pb, seq.shape[0], ptr(seq, C.c_uint8), pos.shape[0],
            ptr(pos, C.c_uint32), ptr(stat, f64), len(motifs), ms, ptr(sl, C.c_int32), int(bb),
            int(ab), ptr(cnt, i64))
        if rc == TB2_ERR_UNEXPECTED:
            # a window the reference slices empty or too short: window[bb] raises there
            raise IndexError('string index out of range')
        self.check(rc)
        return cnt[:blocks.shape[0]]

    def accuracy_label_truth(self, blocks, pos, stat, mod_locs, unmod_locs, slot=0):
        """tb2_accuracy_label_truth -> counts per block"""
        blocks, pb = self._blocks(blocks)
        pos, stat = self._label_args(pos, stat)
        mod_locs, unmod_locs = as_i64(mod_locs), as_i64(unmod_locs)
        cnt = np.zeros(max(1, blocks.shape[0]), dtype=np.int64)
        self.check(self.lib.tb2_accuracy_label_truth(
            self.handle, blocks.shape[0], pb, pos.shape[0], ptr(pos, C.c_uint32), ptr(stat, f64),
            mod_locs.shape[0], ptr(mod_locs, i64), unmod_locs.shape[0], ptr(unmod_locs, i64),
            int(slot), ptr(cnt, i64)))
        return cnt[:blocks.shape[0]]

    def accuracy_label_ctrl(self, blocks, seq, pos, stat, ctrl_pos, ctrl_stat, motifs, slots):
        """tb2_accuracy_label_ctrl -> counts (n_blocks, n_motifs)"""
        blocks, pb = self._blocks(blocks)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        pos, stat = self._label_args(pos, stat)
        ctrl_pos, ctrl_stat = self._label_args(ctrl_pos, ctrl_stat)
        ms = (Motif * len(motifs))(*motifs)
        sl = np.ascontiguousarray(slots, dtype=np.int32)
        cnt = np.zeros((max(1, blocks.shape[0]), len(motifs)), dtype=np.int64)
        self.check(self.lib.tb2_accuracy_label_ctrl(
            self.handle, blocks.shape[0], pb, seq.shape[0], ptr(seq, C.c_uint8), pos.shape[0],
            ptr(pos, C.c_uint32), ptr(stat, f64), ctrl_pos.shape[0], ptr(ctrl_pos, C.c_uint32),
            ptr(ctrl_stat, f64), len(motifs), ms, ptr(sl, C.c_int32), ptr(cnt, i64)))
        return cnt[:blocks.shape[0]]

    def accuracy_curve(self, slot, rate_idx, prec_idx):
        """tb2_accuracy_curve -> (tp_rate, fp_rate, precision)"""
        rate_idx, prec_idx = as_i64(rate_idx), as_i64(prec_idx)
        if rate_idx.shape != prec_idx.shape:
            raise ValueError('rate_idx and prec_idx need the same length')
        n = rate_idx.shape[0]
        tp, fp, prec = np.empty(n), np.empty(n), np.empty(n)
        rc = self.lib.tb2_accuracy_curve(
            self.handle, int(slot), n, ptr(rate_idx, i64), ptr(prec_idx, i64), ptr(tp, f64),
            ptr(fp, f64), ptr(prec, f64))
        if rc == TB2_ERR_INVALID_ARG and self.lib.tb2_last_error(self.handle) == b'NaN statistic':
            raise ValueError('NaN statistic: the order of the statistics is undefined')
        self.check(rc)
        return tp, fp, prec

    def accuracy_rates_ordered(self, labels, rate_idx, prec_idx):
        """tb2_accuracy_rates_ordered -> (tp_rate, fp_rate, precision)"""
        labels = np.ascontiguousarray(labels, dtype=bool).view(np.uint8)
        rate_idx, prec_idx = as_i64(rate_idx), as_i64(prec_idx)
        if rate_idx.shape != prec_idx.shape:
            raise ValueError('rate_idx and prec_idx need the same length')
        n = rate_idx.shape[0]
        tp, fp, prec = np.empty(n), np.empty(n), np.empty(n)
        self.check(self.lib.tb2_accuracy_rates_ordered(
            self.handle, labels.shape[0], ptr(labels, C.c_uint8), n, ptr(rate_idx, i64),
            ptr(prec_idx, i64), ptr(tp, f64), ptr(fp, f64), ptr(prec, f64)))
        return tp, fp, prec

    # ---- statistics files ---------------------------------------------------
    def stats_file_aggregate(self, blocks, region_size, pos, stat, single_read_thresh,
                             lower_thresh, stat_type, unmod_count, mod_count):
        """tb2_stats_file_aggregate -> row_off (n_blocks + 1); ``blocks`` rows are (start,
        stat_off, n_stat, chrm id, strand byte).  The rows stay on the device for
        stats_file_download and most_signif_add_aggregate."""
        blocks = as_i64(blocks).reshape(-1, 5)
        pos = np.ascontiguousarray(pos, dtype=np.uint32)
        stat = as_f64(stat)
        if pos.shape != stat.shape:
            raise ValueError('pos and stat need the same length')
        row_off = np.zeros(blocks.shape[0] + 1, dtype=np.int64)
        self.check(self.lib.tb2_stats_file_aggregate(
            self.handle, blocks.shape[0], ptr(blocks, i64), int(region_size), stat.shape[0],
            ptr(pos, C.c_uint32), ptr(stat, f64), float(single_read_thresh),
            float('nan') if lower_thresh is None else float(lower_thresh), int(stat_type),
            float(unmod_count), float(mod_count), ptr(row_off, i64)))
        return row_off

    def stats_file_download(self, n_rows):
        """the last aggregation's rows: (pos u4, damp_frac, frac, cov u4, valid_cov u4)"""
        out = (np.empty(n_rows, np.uint32), np.empty(n_rows), np.empty(n_rows),
               np.empty(n_rows, np.uint32), np.empty(n_rows, np.uint32))
        self.check(self.lib.tb2_stats_file_aggregate_download(
            self.handle, ptr(out[0], C.c_uint32), ptr(out[1], f64), ptr(out[2], f64),
            ptr(out[3], C.c_uint32), ptr(out[4], C.c_uint32)))
        return out

    def most_signif_begin(self, level, num_most_signif):
        """open this context's table; raises while another is open"""
        self.check(self.lib.tb2_most_signif_begin(self.handle, int(bool(level)), int(num_most_signif)))

    def most_signif_end(self):
        self.check(self.lib.tb2_most_signif_end(self.handle))

    def most_signif_reset(self):
        self.check(self.lib.tb2_most_signif_reset(self.handle))

    def most_signif_add_rows(self, key, pos, cov, control_cov, chrm, strand, frac=None,
                             valid_cov=None):
        """one block's rows; ``strand`` is the table's byte (b'+' / b'-')"""
        key = as_f64(key)
        n = key.shape[0]
        u4 = [np.ascontiguousarray(a, dtype=np.uint32) for a in (pos, cov, control_cov)]
        fr = as_f64(frac) if frac is not None else None
        vc = np.ascontiguousarray(valid_cov, dtype=np.uint32) if valid_cov is not None else None
        if any(a.shape[0] != n for a in u4 + [x for x in (fr, vc) if x is not None]):
            raise ValueError('row columns need the same length')
        sb = strand if isinstance(strand, int) else bytes(strand)[:1][0]
        self.check(self.lib.tb2_most_signif_add_rows(
            self.handle, n, ptr(key, f64), ptr(fr, f64) if fr is not None else None,
            ptr(u4[0], C.c_uint32), ptr(u4[1], C.c_uint32), ptr(u4[2], C.c_uint32),
            ptr(vc, C.c_uint32) if vc is not None else None, int(chrm), int(sb)))

    def most_signif_add_aggregate(self):
        self.check(self.lib.tb2_most_signif_add_aggregate(self.handle))

    def most_signif_count(self):
        n = i64(0)
        self.check(self.lib.tb2_most_signif_count(self.handle, C.byref(n)))
        return int(n.value)

    def most_signif_get(self):
        """the table in order: dict of columns (key, frac, pos, cov, control_cov, valid_cov,
        chrm, strand as S1)"""
        n = self.most_signif_count()
        c = dict(key=np.empty(n), frac=np.empty(n), pos=np.empty(n, np.uint32),
                 cov=np.empty(n, np.uint32), control_cov=np.empty(n, np.uint32),
                 valid_cov=np.empty(n, np.uint32), chrm=np.empty(n, np.uint32),
                 strand=np.empty(n, np.uint8))
        self.check(self.lib.tb2_most_signif_get(
            self.handle, ptr(c['key'], f64), ptr(c['frac'], f64), ptr(c['pos'], C.c_uint32),
            ptr(c['cov'], C.c_uint32), ptr(c['control_cov'], C.c_uint32),
            ptr(c['valid_cov'], C.c_uint32), ptr(c['chrm'], C.c_uint32),
            ptr(c['strand'], C.c_uint8)))
        c['strand'] = c['strand'].view('S1')
        return c

    # ---- read filters (read_filter.cu) -------------------------------------
    def dwell_percentiles(self, lens, len_off, pctl):
        """(n_reads, len(pctl)) array of np.percentile(lens[len_off[r]:len_off[r + 1]], p)"""
        lens, len_off, pctl = as_i64(lens), as_i64(len_off), as_f64(np.atleast_1d(pctl))
        n = len_off.shape[0] - 1
        out = np.empty((max(n, 0), pctl.shape[0]))
        self.check(self.lib.tb2_dwell_percentiles(self.handle, n, ptr(lens, i64), ptr(len_off, i64),
                                                  pctl.shape[0], ptr(pctl, f64), ptr(out, f64)))
        return out

    def batch_read_filters(self, sig_match_thresh, obs_filter=None, want_percentiles=False):
        """filter code of every read of the computed batch (-1 failed, 0 kept, 1 signal
        matching, 2 observations per base) and, with want_percentiles, the (n_reads,
        len(obs_filter)) percentiles of the successful reads"""
        pairs = list(obs_filter or [])
        pctl = as_f64([p for p, _ in pairs] or [0.0])
        thresh = as_f64([t for _, t in pairs] or [0.0])
        base_off = getattr(self, '_base_off', None)      # none before an upload: the call refuses
        n = 0 if base_off is None else base_off.shape[0] - 1
        code = np.empty(max(n, 1), dtype=np.int8)[:n]
        pout = np.empty((n, len(pairs))) if want_percentiles else None
        self.check(self.lib.tb2_batch_read_filters(
            self.handle, float(sig_match_thresh), len(pairs), ptr(pctl, f64), ptr(thresh, f64),
            ptr(code, C.c_int8), ptr(pout, f64) if pout is not None else None))
        return (code, pout) if want_percentiles else code

    def read_mid_coverage(self, grp_off, start, end):
        """coverage at each read's middle, per (chromosome, strand) group of reads"""
        grp_off, start, end = as_i64(grp_off), as_i64(start), as_i64(end)
        out = np.empty(start.shape[0], dtype=np.int64)
        self.check(self.lib.tb2_read_mid_coverage(self.handle, grp_off.shape[0] - 1, ptr(grp_off, i64),
                                                  ptr(start, i64), ptr(end, i64), ptr(out, i64)))
        return out

    # ---- genome browser tracks (browser_tracks.cu) -------------------------
    def coverage_runs(self, grp_off, start, end):
        """(run_off, run_start, run_cov): the coverage of each (chromosome, strand) group of
        reads as runs of equal value; group g's runs are run_off[g] .. run_off[g + 1], each
        starting at run_start (within the group) and lasting to the next start or max(end)"""
        grp_off, start, end = as_i64(grp_off), as_i64(start), as_i64(end)
        n_groups = grp_off.shape[0] - 1
        bound = 2 * start.shape[0] + max(n_groups, 0)      # at most 2 n_g + 1 runs per group
        run_off = np.zeros(max(n_groups, 0) + 1, dtype=np.int64)
        run_start = np.empty(max(bound, 1), dtype=np.int64)
        run_cov = np.empty(max(bound, 1), dtype=np.int64)
        self.check(self.lib.tb2_coverage_runs(self.handle, n_groups, ptr(grp_off, i64), ptr(start, i64),
                                              ptr(end, i64), ptr(run_off, i64), ptr(run_start, i64),
                                              ptr(run_cov, i64)))
        m = int(run_off[-1])
        return run_off, run_start[:m], run_cov[:m]

    def slot_means(self, chrm_len, batches):
        """per-position means over chrm_len positions of the values of ``batches``, an
        iterable of (start, val_off, vals, reverse) arrays added in order: read r of a batch
        holds vals[val_off[r]:val_off[r + 1]] from start[r] on, reversed when reverse[r].
        Each position's sum is the sequential fp64 sum of its values in read order; a
        position no read covers is NaN."""
        self.check(self.lib.tb2_slot_sums_begin(self.handle, int(chrm_len)))
        for start, val_off, vals, reverse in batches:
            start, val_off, vals = as_i64(start), as_i64(val_off), as_f64(vals)
            reverse = np.ascontiguousarray(reverse, dtype=np.uint8)
            self.check(self.lib.tb2_slot_sums_add(self.handle, start.shape[0], ptr(start, i64),
                                                  ptr(val_off, i64), ptr(vals, f64), ptr(reverse, C.c_uint8)))
        out = np.empty(max(int(chrm_len), 1))[:int(chrm_len)]
        self.check(self.lib.tb2_slot_sums_means(self.handle, ptr(out, f64)))
        return out


def make_policy(kind='DNA', outlier_thresh=5.0, max_raw_cpts=200,
                min_event_to_seq_ratio=1.1, max_scaling_iters=3,
                skip_seq_scaling=False, const_scale=None, subsample_seed=0,
                rescue=True, sig_match_thresh=None):
    if sig_match_thresh is None:
        sig_match_thresh = 1.1 if kind == 'DNA' else 2.0
    return Policy(float('nan') if outlier_thresh is None else outlier_thresh,
                  -1 if max_raw_cpts is None else max_raw_cpts,
                  min_event_to_seq_ratio, sig_match_thresh, max_scaling_iters,
                  int(kind == 'RNA'), int(bool(skip_seq_scaling)),
                  float('nan') if const_scale is None else const_scale,
                  subsample_seed, int(bool(rescue)))


def ensure_model(ctx, std_ref):
    """set ``std_ref`` (a TomboModel) as the context's canonical model, uploading the k-mer
    tables once per model object.  The context keeps a strong reference (an id() alone can
    be recycled after garbage collection) and a digest of the tables, so a model mutated in
    place is uploaded again.  Every Python entry point that sets a model on a shared
    context goes through here, so none of them can leave another one's cached model stale."""
    m, s = std_ref.tables()
    digest = hash((m.tobytes(), s.tobytes(), std_ref.kmer_width, std_ref.central_pos))
    if getattr(ctx, '_model_ref', None) is not std_ref or getattr(ctx, '_model_digest', None) != digest:
        ctx.set_model(m, s, std_ref.kmer_width, std_ref.central_pos)
        ctx._model_ref, ctx._model_digest = std_ref, digest


_default_ctx = {}


def get_context(device=0):
    """Process-wide default context per device (single-read API)."""
    ctx = _default_ctx.get(device)
    if ctx is None:
        ctx = _default_ctx[device] = Context(device)
    return ctx
