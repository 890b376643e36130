"""ctypes wrapper around oracle/liboracle.so (the C restatement in oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline leg.  Never by tombo_b200/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

i64 = C.c_int64
f64 = C.c_double
P = C.POINTER


class Params(C.Structure):
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
                ('max_scaling_iters', i64), ('tie_stable', i64), ('is_rna', i64),
                ('skip_seq_scaling', i64), ('const_scale', f64),
                ('subsample_seed', C.c_uint32)]


class ReadResult(C.Structure):
    _fields_ = [('read_start_rel_to_raw', i64), ('sv', ScaleValues),
                ('sig_match_score', f64), ('norm_params_changed', i64),
                ('n_norm', i64)]


def build(force=False):
    so = os.path.join(HERE, 'liboracle.so')
    src = [os.path.join(HERE, f) for f in ('oracle.c', 'oracle.h')]
    if (force or not os.path.exists(so) or
            any(os.path.getmtime(s) > os.path.getmtime(so) for s in src)):
        subprocess.check_call(['make', '-s', '-C', HERE, 'liboracle.so'])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.orc_status_message.restype = C.c_char_p
        for name in ('orc_median', 'orc_pairwise_sum', 'orc_np_mean',
                     'orc_calc_llh_ratio', 'orc_calc_llh_ratio_const_var',
                     'orc_calc_scaled_llh_ratio_const_var',
                     'orc_get_read_seg_score'):
            getattr(_LIB, name).restype = f64
        for name in ('orc_compute_num_events', 'orc_identify_stalls',
                     'orc_remove_stall_cpts', 'orc_perm_index'):
            getattr(_LIB, name).restype = i64
        _LIB.orc_subsample_key.restype = C.c_uint32
    return _LIB


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(P(f64))


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int64)
    return a, a.ctypes.data_as(P(i64))


def status_message(st):
    return lib().orc_status_message(int(st)).decode()


def params_from(p):
    """resquiggleParams-like (any object with the reference field names)."""
    mhz = p.max_half_z_score
    return Params(float(p.match_evalue), float(p.skip_pen), int(p.bandwidth),
                  float('nan') if mhz is None else float(mhz),
                  int(p.running_stat_width), int(p.min_obs_per_base),
                  int(p.raw_min_obs_per_base), int(p.mean_obs_per_event),
                  float(p.z_shift), float(p.stay_pen), int(bool(p.use_t_test_seg)),
                  int(p.band_bound_thresh), int(p.start_bw), int(p.start_save_bw),
                  int(p.start_n_bases))


def policy(kind='DNA', outlier_thresh=5.0, max_raw_cpts=200,
           min_event_to_seq_ratio=1.1, max_scaling_iters=3, tie_stable=1,
           skip_seq_scaling=False, const_scale=None, subsample_seed=0):
    return Policy(float('nan') if outlier_thresh is None else outlier_thresh,
                  -1 if max_raw_cpts is None else max_raw_cpts,
                  min_event_to_seq_ratio, 1.1 if kind == 'DNA' else 2.0,
                  max_scaling_iters, tie_stable, int(kind == 'RNA'),
                  int(skip_seq_scaling),
                  float('nan') if const_scale is None else const_scale,
                  subsample_seed)


# ---------------------------------------------------------------- helpers
def median(x):
    x, px = _d(x)
    return lib().orc_median(px, i64(x.shape[0]))


def np_mean(x):
    x, px = _d(x)
    return lib().orc_np_mean(px, i64(x.shape[0]))


def perm_index(i, n, key):
    """Keyed bijection on [0, n): the Theil-Sen sub-sample index i (stands in for
    np.random.choice(n, 1000, replace=False), tombo_stats.py:411-416)."""
    return int(lib().orc_perm_index(i64(i), i64(n), C.c_uint32(key)))


def linspace(start, stop, num):
    out = np.empty(max(num, 0))
    lib().orc_linspace(f64(start), f64(stop), i64(num), out.ctypes.data_as(P(f64)))
    return out


def new_means(sig, segs):
    sig, ps = _d(sig)
    segs, pg = _i(segs)
    out = np.empty(segs.shape[0] - 1)
    lib().orc_new_means(ps, pg, i64(out.shape[0]), out.ctypes.data_as(P(f64)))
    return out


def new_mean_stds(sig, segs):
    sig, ps = _d(sig)
    segs, pg = _i(segs)
    m = np.empty(segs.shape[0] - 1)
    s = np.empty(segs.shape[0] - 1)
    lib().orc_new_mean_stds(ps, pg, i64(m.shape[0]), m.ctypes.data_as(P(f64)),
                            s.ctypes.data_as(P(f64)))
    return m, s


def apply_outlier_thresh(sig, lo, hi):
    sig, ps = _d(sig)
    out = np.empty_like(sig)
    lib().orc_apply_outlier_thresh(ps, i64(sig.shape[0]), f64(lo), f64(hi),
                                   out.ctypes.data_as(P(f64)))
    return out


def valid_cpts_w_cap(sig, min_base_obs, w, num_cpts, t_test=False):
    sig, ps = _d(sig)
    out = np.empty(num_cpts, dtype=np.int64)
    fn = (lib().orc_valid_cpts_w_cap_t_test if t_test
          else lib().orc_valid_cpts_w_cap)
    st = fn(ps, i64(sig.shape[0]), i64(min_base_obs), i64(w), i64(num_cpts),
            C.c_int(1), out.ctypes.data_as(P(i64)))
    return st, out


def compute_slopes(ev, md, max_slope=1000.0):
    ev, pe = _d(ev)
    md, pm = _d(md)
    n = ev.shape[0]
    out = np.empty(n * (n - 1) // 2)
    lib().orc_compute_slopes(pe, pm, i64(n), f64(max_slope),
                             out.ctypes.data_as(P(f64)))
    return out


def calc_llh_ratio(m, rm, am, rv, av):
    m, a = _d(m); rm, b = _d(rm); am, c = _d(am); rv, d = _d(rv); av, e = _d(av)
    return lib().orc_calc_llh_ratio(a, b, c, d, e, i64(m.shape[0]))


def calc_llh_ratio_const_var(m, rm, am, cv):
    m, a = _d(m); rm, b = _d(rm); am, c = _d(am)
    return lib().orc_calc_llh_ratio_const_var(a, b, c, f64(cv), i64(m.shape[0]))


def calc_scaled_llh_ratio_const_var(m, rm, am, cv, sf, hf, hp):
    m, a = _d(m); rm, b = _d(rm); am, c = _d(am)
    return lib().orc_calc_scaled_llh_ratio_const_var(
        a, b, c, f64(cv), f64(sf), f64(hf), f64(hp), i64(m.shape[0]))


def base_z_scores(sig, ref_mean, ref_sd, do_winsorize=False, max_half_z=10.0):
    sig, ps = _d(sig)
    out = np.empty_like(sig)
    lib().orc_base_z_scores(ps, i64(sig.shape[0]), f64(ref_mean), f64(ref_sd),
                            C.c_int(int(do_winsorize)), f64(max_half_z),
                            out.ctypes.data_as(P(f64)))
    return out


def banded_forward_pass(z, event_starts, skip_pen, stay_pen):
    z, pz = _d(z)
    es, pe = _i(event_starts)
    nb, bw = z.shape
    fwd = np.empty((nb + 1, bw))
    tb = np.empty((nb + 1, bw), dtype=np.int64)
    lib().orc_banded_forward_pass(pz, pe, i64(nb), i64(bw), f64(skip_pen),
                                  f64(stay_pen), fwd.ctypes.data_as(P(f64)),
                                  tb.ctypes.data_as(P(i64)))
    return fwd, tb


def banded_traceback(tb, event_starts, band_pos, thresh=-1):
    tb, pt = _i(tb)
    es, pe = _i(event_starts)
    nb = tb.shape[0] - 1
    out = np.empty(nb + 1, dtype=np.int64)
    st = lib().orc_banded_traceback(pt, pe, i64(nb), i64(tb.shape[1]),
                                    i64(band_pos), i64(thresh),
                                    out.ctypes.data_as(P(i64)))
    return st, out


def adaptive_banded_forward_pass(fwd, tb, event_starts, event_means, rm, rs,
                                 z_shift, skip_pen, stay_pen, start_seq_pos,
                                 mask_fill_z, do_winsorize, max_half_z,
                                 return_z=False):
    """In-place on fwd / tb / event_starts like the reference."""
    assert fwd.flags.c_contiguous and tb.flags.c_contiguous
    assert fwd.dtype == np.float64 and tb.dtype == np.int64
    assert event_starts.dtype == np.int64
    em, pe = _d(event_means)
    rm, pr = _d(rm)
    rs, ps = _d(rs)
    nb, bw = fwd.shape[0] - 1, fwd.shape[1]
    zs = np.empty((nb - start_seq_pos, bw)) if return_z else None
    st = lib().orc_adaptive_banded_forward_pass(
        fwd.ctypes.data_as(P(f64)), tb.ctypes.data_as(P(i64)),
        event_starts.ctypes.data_as(P(i64)), i64(nb), i64(bw), pe,
        i64(em.shape[0]), pr, ps, f64(z_shift), f64(skip_pen), f64(stay_pen),
        i64(start_seq_pos), f64(mask_fill_z), C.c_int(int(do_winsorize)),
        f64(max_half_z), zs.ctypes.data_as(P(f64)) if return_z else None)
    return st, zs


def normalize_raw_signal(raw, outlier_thresh=None, scale_values=None,
                         const_scale=None):
    raw, pr = _d(raw)
    norm = np.empty_like(raw)
    sv = ScaleValues()
    svi = None
    if scale_values is not None:
        svi = ScaleValues(*[float('nan') if v is None else float(v)
                            for v in scale_values])
    st = lib().orc_normalize_raw_signal(
        pr, i64(raw.shape[0]), C.c_int(0 if const_scale is None else 1),
        f64(float('nan') if outlier_thresh is None else outlier_thresh),
        f64(float('nan') if const_scale is None else const_scale),
        C.byref(svi) if svi is not None else None,
        norm.ctypes.data_as(P(f64)), C.byref(sv))
    return st, norm, (sv.shift, sv.scale, sv.lower_lim, sv.upper_lim,
                      sv.outlier_thresh)


def theil_sen(prev_shift, prev_scale, ev, md, key=0):
    ev, pe = _d(ev)
    md, pm = _d(md)
    out = [f64(), f64(), f64(), f64()]
    st = lib().orc_theil_sen(f64(prev_shift), f64(prev_scale), pe, pm,
                             i64(ev.shape[0]), C.c_uint32(key),
                             *[C.byref(o) for o in out])
    return st, tuple(o.value for o in out)


def get_read_seg_score(means, rm, rs):
    means, a = _d(means); rm, b = _d(rm); rs, c = _d(rs)
    return lib().orc_get_read_seg_score(a, b, c, i64(means.shape[0]))


def identify_stalls(raw):
    raw, pr = _d(raw)
    cap = raw.shape[0] // 200 + 4
    out = np.empty(2 * cap, dtype=np.int64)
    n = lib().orc_identify_stalls(pr, i64(raw.shape[0]),
                                  out.ctypes.data_as(P(i64)), i64(cap))
    return out[:2 * n].reshape(-1, 2).copy()


def find_static_base_assignment(em, rm, rs, params):
    em, pe = _d(em); rm, pr = _d(rm); rs, ps = _d(rs)
    p = params_from(params)
    out = np.empty(rm.shape[0] + 1, dtype=np.int64)
    st = lib().orc_find_static_base_assignment(
        pe, i64(em.shape[0]), pr, ps, i64(rm.shape[0]), C.byref(p),
        out.ctypes.data_as(P(i64)))
    return st, out


def find_seq_start_in_events(em, rm, rs, params, num_bases, num_events,
                             sig_match_thresh=None):
    em, pe = _d(em); rm, pr = _d(rm); rs, ps = _d(rs)
    p = params_from(params)
    sl, epb = i64(), f64()
    st = lib().orc_find_seq_start_in_events(
        pe, i64(em.shape[0]), pr, ps, i64(rm.shape[0]), C.byref(p),
        i64(num_bases), i64(num_events),
        C.c_int(sig_match_thresh is not None),
        f64(0.0 if sig_match_thresh is None else sig_match_thresh),
        C.byref(sl), C.byref(epb))
    return st, sl.value, epb.value


def find_adaptive_base_assignment(cpts, em, params, rm, rs,
                                  sig_match_thresh=1.1):
    cpts, pc = _i(cpts)
    em, pe = _d(em); rm, pr = _d(rm); rs, ps = _d(rs)
    p = params_from(params)
    nb = rm.shape[0]
    segs = np.empty(nb + 1, dtype=np.int64)
    rsrtr = i64()
    dbg = np.zeros(3, dtype=np.int64)
    epb = f64()
    st = lib().orc_find_adaptive_base_assignment(
        pc, i64(cpts.shape[0]), pe, C.byref(p), pr, ps, i64(nb),
        f64(sig_match_thresh), segs.ctypes.data_as(P(i64)), C.byref(rsrtr),
        dbg.ctypes.data_as(P(i64)), C.byref(epb))
    return st, segs, rsrtr.value, dbg, epb.value


def resolve_skipped_bases_with_raw(segs, rm, rs, norm, params,
                                   max_raw_cpts=200):
    segs, pg = _i(segs)
    rm, pr = _d(rm); rs, ps = _d(rs); norm, pn = _d(norm)
    p = params_from(params)
    out = np.empty_like(segs)
    st = lib().orc_resolve_skipped_bases_with_raw(
        pg, i64(segs.shape[0] - 1), pr, ps, pn, i64(norm.shape[0]), C.byref(p),
        i64(-1 if max_raw_cpts is None else max_raw_cpts),
        out.ctypes.data_as(P(i64)))
    return st, out


def run_read(raw, rm, rs, params, save_params, pol, read_index=0,
             want_norm=False):
    """Full per-read policy (iterate + rescue).  Returns dict."""
    raw, praw = _d(raw)
    rm, pr = _d(rm); rs, ps = _d(rs)
    p, sp = params_from(params), params_from(save_params)
    nb = rm.shape[0]
    segs = np.empty(nb + 1, dtype=np.int64)
    norm = np.empty(raw.shape[0]) if want_norm else None
    res = ReadResult()
    info = np.zeros(4, dtype=np.int64)
    st = lib().orc_run_read(
        praw, i64(raw.shape[0]), pr, ps, i64(nb), C.byref(p), C.byref(sp),
        C.byref(pol), C.c_uint32(read_index), segs.ctypes.data_as(P(i64)),
        norm.ctypes.data_as(P(f64)) if want_norm else None, C.byref(res),
        info.ctypes.data_as(P(i64)))
    out = dict(status=st, message=status_message(st), calls=int(info[0]),
               rescued=bool(info[1]), n_iters=int(info[2]),
               first_status=int(info[3]))
    if st == 0:
        out.update(segs=segs, read_start_rel_to_raw=res.read_start_rel_to_raw,
                   shift=res.sv.shift, scale=res.sv.scale,
                   lower_lim=res.sv.lower_lim, upper_lim=res.sv.upper_lim,
                   sig_match_score=res.sig_match_score,
                   norm_params_changed=bool(res.norm_params_changed),
                   n_norm=res.n_norm)
        if want_norm:
            out['norm_signal'] = norm[:res.n_norm]
    return out


def resquiggle_read(raw, rm, rs, params, pol, scale_values=None,
                    first_call=True, stall_ints=None, key=0, want_norm=True):
    raw, praw = _d(raw)
    rm, pr = _d(rm); rs, ps = _d(rs)
    p = params_from(params)
    nb = rm.shape[0]
    segs = np.empty(nb + 1, dtype=np.int64)
    norm = np.empty(raw.shape[0])
    res = ReadResult()
    svi = None
    if scale_values is not None:
        svi = ScaleValues(*[float('nan') if v is None else float(v)
                            for v in scale_values])
    si, psi, nsi = None, None, 0
    if stall_ints is not None:
        si = np.ascontiguousarray(np.asarray(stall_ints, dtype=np.int64).reshape(-1))
        psi, nsi = si.ctypes.data_as(P(i64)), si.shape[0] // 2
        if nsi == 0:
            si = np.zeros(2, dtype=np.int64)
            psi = si.ctypes.data_as(P(i64))
    st = lib().orc_resquiggle_read(
        praw, i64(raw.shape[0]), pr, ps, i64(nb), C.byref(p), C.byref(pol),
        C.byref(svi) if svi is not None else None, C.c_int(int(first_call)),
        psi, i64(nsi), C.c_uint32(key), segs.ctypes.data_as(P(i64)),
        norm.ctypes.data_as(P(f64)), C.byref(res))
    out = dict(status=st, message=status_message(st))
    if st == 0:
        out.update(segs=segs, read_start_rel_to_raw=res.read_start_rel_to_raw,
                   scale_values=(res.sv.shift, res.sv.scale, res.sv.lower_lim,
                                 res.sv.upper_lim, res.sv.outlier_thresh),
                   sig_match_score=res.sig_match_score,
                   norm_params_changed=bool(res.norm_params_changed),
                   norm_signal=norm[:res.n_norm].copy())
    return out


# ---------------------------------------------------------------- batch checker
def levels_from_codes(codes, means, sds, k):
    """expected levels of one read from its base codes (dense 4^k tables)"""
    c = np.asarray(codes, dtype=np.int64)
    nb = c.shape[0] - k + 1
    kidx = np.zeros(max(nb, 0), dtype=np.int64)
    for j in range(k):
        kidx = kidx * 4 + c[j:j + nb]
    return means[kidx], sds[kidx]


def run_batch(raw, raw_off, seq, seq_off, means, sds, k, params, save_params, pol,
              indices=None, threads=None):
    """orc_run_read over reads `indices` of a flat batch (the C-ABI layout), on a thread
    pool (ctypes releases the GIL; oracle.c keeps no state between calls).  read_index =
    position in the batch, which keys the Theil-Sen sub-sampling like the library does.
    Returns {index: result dict}."""
    import os
    from multiprocessing.pool import ThreadPool
    lib()
    if indices is None:
        indices = range(raw_off.shape[0] - 1)
    indices = [int(i) for i in indices]
    if threads is None:
        try:
            threads = len(os.sched_getaffinity(0))
        except AttributeError:
            threads = os.cpu_count() or 1
    threads = max(1, min(threads, 64, len(indices)))

    def one(i):
        rm, rs = levels_from_codes(seq[seq_off[i]:seq_off[i + 1]], means, sds, k)
        r = np.asarray(raw[raw_off[i]:raw_off[i + 1]], dtype=np.float64)
        return i, run_read(r, rm, rs, params, save_params, pol, read_index=i)
    if threads == 1:
        return dict(one(i) for i in indices)
    with ThreadPool(threads) as tp:
        return dict(tp.imap_unordered(one, indices, chunksize=max(1, len(indices) // (threads * 8))))


def compare_batch(res, oracle_out):
    """bit-compare a tb2_resquiggle_batch result dict with run_batch output.  Returns a
    list of (read index, field) mismatches (empty = parity)."""
    bad = []
    for i, o in oracle_out.items():
        if int(res['status'][i]) != o['status']:
            bad.append((i, 'status %d != %d' % (int(res['status'][i]), o['status'])))
            continue
        if o['status'] != 0:
            continue
        a, b = int(res['seg_off'][i]), int(res['seg_off'][i + 1])
        if not np.array_equal(res['segs'][a:b], o['segs']):
            bad.append((i, 'segs'))
        if int(res['read_start_rel_to_raw'][i]) != o['read_start_rel_to_raw']:
            bad.append((i, 'read_start_rel_to_raw'))
        sv = res['scale_values'][i]
        for j, key in enumerate(('shift', 'scale', 'lower_lim', 'upper_lim')):
            if not (sv[j] == o[key] or (np.isnan(sv[j]) and np.isnan(o[key]))):
                bad.append((i, key))
        if res['sig_match_score'][i] != o['sig_match_score']:
            bad.append((i, 'sig_match_score'))
        if int(res['n_iters'][i]) != o['n_iters']:
            bad.append((i, 'n_iters'))
        if bool(res['flags'][i] & 2) != o['rescued']:
            bad.append((i, 'rescued'))
        if bool(res['flags'][i] & 1) != o['norm_params_changed']:
            bad.append((i, 'norm_params_changed'))
    return bad
