"""ctypes driver of tests/emul/libemul_dp.so: the device source of the banded-DP kernel
run on the host (TEST INFRASTRUCTURE ONLY -- see cuda_emul.h)."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(REPO, 'tombo_b200', 'csrc')
_LIB = None


def build():
    so = os.path.join(HERE, 'libemul_dp.so')
    srcs = [os.path.join(HERE, f) for f in ('emul_dp.cpp', 'cuda_emul.cpp', 'cuda_emul.h')]
    srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    srcs.append(os.path.join(REPO, 'include', 'tombo_b200.h'))
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(['g++', '-O1', '-g', '-std=c++17', '-ffp-contract=off', '-fPIC',
                               '-shared', '-o', so, os.path.join(HERE, 'emul_dp.cpp'),
                               os.path.join(HERE, 'cuda_emul.cpp')])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.emul_tb_words.restype = C.c_size_t
        _LIB.emul_tb_words.argtypes = [C.c_longlong] * 3
        _LIB.emul_row_cells.argtypes = [C.c_longlong]
        _LIB.emul_abs_chunk.argtypes = [C.c_longlong]
        _LIB.emul_abs_ms_chunk.argtypes = [C.c_longlong]
        _LIB.emul_wpl_of.argtypes = [C.c_int]
    return _LIB


def plan(p, n_em, nb):
    """host capacity plan of one read (mirrors plan_align in csrc/dp_kernels.cu)"""
    L = lib()
    mask_len = min(nb, n_em) // 4
    w_static = max(1, n_em - mask_len)
    bw, sbw, snb, ssbw = int(p.bandwidth), int(p.start_bw), int(p.start_n_bases), int(p.start_save_bw)
    is_short = n_em < sbw + snb or nb < snb
    w_main = w_static if is_short else max(sbw, bw)
    smem_cells = L.emul_row_cells(w_main)
    if not is_short and 528 < bw <= 1616:   # three chunks per lane (dp_row2.cuh)
        smem_cells = max(smem_cells, 3 * (13 if bw <= 1236 else 17) * 16)
    elif not is_short and bw > 1616:        # lane-chunk engine rows (dp_row.cuh)
        smem_cells = max(smem_cells, L.emul_row_cells(bw))
    tb = L.emul_tb_words(nb, w_static, n_em)
    grow = L.emul_row_cells(max(1, n_em))
    if not is_short:
        tb = max(tb, L.emul_tb_words(nb, bw, n_em + bw), L.emul_tb_words(snb, sbw, snb),
                 L.emul_tb_words(snb, ssbw, snb))
        grow = max(grow, L.emul_row_cells(ssbw))
    return smem_cells, tb, grow, is_short


def align_batch(reads, params, sig_match_thresh=1.1, klass=0, n_blocks=1, smem_cells=None):
    """reads: list of (cpts int array, em, rm, rs).  Runs k_align<klass> on the host
    emulation.  Returns list of dict(status, segs, rsrtr, dbg, starts, read_tb)."""
    from tombo_b200 import _lib
    L = lib()
    n = len(reads)
    ev_off = np.zeros(n + 1, dtype=np.int64)
    base_off = np.zeros(n + 1, dtype=np.int64)
    for i, (cp, em, rm, rs) in enumerate(reads):
        ev_off[i + 1] = ev_off[i] + cp.shape[0] + 1
        base_off[i + 1] = base_off[i] + rm.shape[0]
    cpts = np.zeros(ev_off[-1], dtype=np.int32)
    emf = np.zeros(ev_off[-1], dtype=np.float64)
    rmf = np.zeros(base_off[-1]); rsf = np.zeros(base_off[-1])
    n_cpts = np.zeros(n, dtype=np.int32)
    nev = np.zeros(n, dtype=np.int32)
    sc, tbw, grow = 32, 32, 32
    for i, (cp, em, rm, rs) in enumerate(reads):
        cpts[ev_off[i]:ev_off[i] + cp.shape[0]] = cp
        emf[ev_off[i]:ev_off[i] + em.shape[0]] = em
        rmf[base_off[i]:base_off[i + 1]] = rm
        rsf[base_off[i]:base_off[i + 1]] = rs
        n_cpts[i] = cp.shape[0]
        nev[i] = cp.shape[0]
        a, b, c, _ = plan(params, cp.shape[0] - 1, rm.shape[0])
        sc, tbw, grow = max(sc, a), max(tbw, b), max(grow, c)
    if smem_cells is not None:
        sc = smem_cells
    segs = np.zeros(base_off[-1] + n, dtype=np.int32)
    rsrtr = np.zeros(n, dtype=np.int32)
    status = np.zeros(n, dtype=np.int32)
    dbg = np.zeros(3 * n, dtype=np.int32)
    starts = np.zeros(base_off[-1] + 8, dtype=np.int32)
    read_tb = np.zeros(base_off[-1] + n + 8, dtype=np.int32)
    ps = _lib.params_struct(params)

    def ptr(a, t):
        return a.ctypes.data_as(C.POINTER(t))
    L.emul_align_batch(
        C.c_int(klass), C.c_int(n), ptr(cpts, C.c_int), ptr(emf, C.c_double),
        ptr(ev_off, C.c_longlong), ptr(n_cpts, C.c_int), ptr(nev, C.c_int), ptr(rmf, C.c_double),
        ptr(rsf, C.c_double), ptr(base_off, C.c_longlong), ptr(segs, C.c_int), ptr(rsrtr, C.c_int),
        ptr(status, C.c_int), ptr(dbg, C.c_int), C.byref(ps), C.c_double(sig_match_thresh),
        C.c_int(sc), C.c_longlong(tbw), C.c_int(grow), C.c_int(n_blocks), ptr(starts, C.c_int),
        ptr(read_tb, C.c_int))
    out = []
    for i in range(n):
        bo, nb = int(base_off[i]), int(base_off[i + 1] - base_off[i])
        out.append(dict(status=int(status[i]), segs=segs[bo + i:bo + i + nb + 1].astype(np.int64),
                        rsrtr=int(rsrtr[i]), dbg=dbg[3 * i:3 * i + 3].copy(),
                        starts=starts[bo:bo + nb].copy(),
                        read_tb=read_tb[bo + i:bo + i + nb + 1].copy()))
    return out


# ---------------------------------------------------------------- stage kernels
_LIB_STAGE = None


def stage_lib():
    global _LIB_STAGE
    if _LIB_STAGE is None:
        so = os.path.join(HERE, 'libemul_stage.so')
        srcs = [os.path.join(HERE, f) for f in ('emul_stage.cpp', 'cuda_emul.cpp', 'cuda_emul.h')]
        srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(['g++', '-O1', '-g', '-std=c++17', '-ffp-contract=off', '-fPIC',
                                   '-shared', '-o', so, os.path.join(HERE, 'emul_stage.cpp'),
                                   os.path.join(HERE, 'cuda_emul.cpp')])
        _LIB_STAGE = C.CDLL(so)
    return _LIB_STAGE


def resolve(segs_dp, rm, rs, norm, params, max_raw_cpts=200, cap_doubles=1 << 15,
            big_cap_doubles=1 << 22):
    """k_resolve on one read -> (status, segs)"""
    from tombo_b200 import _lib
    L = stage_lib()
    segs_dp = np.ascontiguousarray(segs_dp, dtype=np.int32)
    rm, rs, norm = (np.ascontiguousarray(a, dtype=np.float64) for a in (rm, rs, norm))
    nb = rm.shape[0]
    out = np.zeros(nb + 1, dtype=np.int32)
    st = C.c_int(0)
    ps = _lib.params_struct(params)
    L.emul_resolve(segs_dp.ctypes.data_as(C.POINTER(C.c_int)), C.c_int(nb),
                   rm.ctypes.data_as(C.POINTER(C.c_double)), rs.ctypes.data_as(C.POINTER(C.c_double)),
                   norm.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(norm.shape[0]), C.byref(ps),
                   C.c_longlong(-1 if max_raw_cpts is None else max_raw_cpts),
                   C.c_longlong(cap_doubles), C.c_longlong(big_cap_doubles),
                   out.ctypes.data_as(C.POINTER(C.c_int)), C.byref(st))
    return st.value, out.astype(np.int64)


def theil_sen(prev_shift, prev_scale, bm, rm, key=0):
    """k_theil_sen on one read -> (status, (shift, scale, shift_corr, scale_corr))"""
    L = stage_lib()
    bm, rm = (np.ascontiguousarray(a, dtype=np.float64) for a in (bm, rm))
    out = np.zeros(4)
    st = C.c_int(0)
    L.emul_theil_sen(bm.ctypes.data_as(C.POINTER(C.c_double)), rm.ctypes.data_as(C.POINTER(C.c_double)),
                     C.c_int(bm.shape[0]), C.c_double(prev_shift), C.c_double(prev_scale),
                     C.c_uint(key), out.ctypes.data_as(C.POINTER(C.c_double)), C.byref(st))
    return st.value, tuple(out.tolist())


def select2(values, k):
    """tb2_block_select2 on the host: (value of rank k, value of rank k + 1)"""
    L = stage_lib()
    v = np.ascontiguousarray(values, dtype=np.float64)
    out = np.zeros(2)
    L.emul_select2(v.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(v.shape[0]), C.c_int(k),
                   out.ctypes.data_as(C.POINTER(C.c_double)))
    return float(out[0]), float(out[1])


def segment(raw, params, num_events, outlier_thresh=5.0, const_scale=None, scale_values=None,
            thresh_with_sv=False, stall_ints=None):
    """k_normalize -> k_cumsum -> k_cpts -> k_event_means on one read ->
    (status, norm, (shift, scale, lower, upper, outlier_thresh), sorted cpts, event means).
    scale_values: supplied 5-tuple (None -> NaN); thresh_with_sv: winsorise them by
    outlier_thresh (the normalize_raw_signal mirror); stall_ints: (start, end) pairs, clamped
    to [-1, n + 1] as tb2_batch_set_read_inputs does"""
    from tombo_b200 import _lib
    L = stage_lib()
    raw = np.ascontiguousarray(raw, dtype=np.float64)
    dp = C.POINTER(C.c_double)
    svi = si = None
    if scale_values is not None:
        svi = np.array([np.nan if v is None else float(v) for v in scale_values])
    if stall_ints is not None:
        si = np.clip(np.asarray(stall_ints, dtype=np.int64).reshape(-1), -1, raw.shape[0] + 1)
        si = np.ascontiguousarray(np.append(si, [0, 0]), dtype=np.int32)
    extra = (svi.ctypes.data_as(dp) if svi is not None else None, C.c_int(int(bool(thresh_with_sv))),
             si.ctypes.data_as(C.POINTER(C.c_int)) if si is not None else None,
             C.c_int(0 if si is None else (si.shape[0] - 2) // 2))
    n = raw.shape[0]
    norm = np.zeros(n)
    sv = np.zeros(5)
    cp = np.zeros(num_events + 8, dtype=np.int32)
    em = np.zeros(num_events + 8)
    ncp, st = C.c_int(0), C.c_int(0)
    ps = _lib.params_struct(params)
    L.emul_segment(raw.ctypes.data_as(dp), C.c_int(n), C.byref(ps), C.c_int(num_events),
                   C.c_double(float('nan') if outlier_thresh is None else outlier_thresh),
                   C.c_double(float('nan') if const_scale is None else const_scale),
                   norm.ctypes.data_as(dp), sv.ctypes.data_as(dp), cp.ctypes.data_as(C.POINTER(C.c_int)),
                   C.byref(ncp), em.ctypes.data_as(dp), C.byref(st), *extra)
    k = ncp.value
    return st.value, norm, tuple(sv.tolist()), cp[:k].astype(np.int64), em[:max(k - 1, 0)]


def stalls(raw, stall_cap=64):
    """k_stalls on one read -> (status, (n, 2) interval array)"""
    L = stage_lib()
    raw = np.ascontiguousarray(raw, dtype=np.float64)
    ints = np.zeros(2 * stall_cap, dtype=np.int32)
    k, st = C.c_int(0), C.c_int(0)
    L.emul_stalls(raw.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(raw.shape[0]), C.c_int(stall_cap),
                  ints.ctypes.data_as(C.POINTER(C.c_int)), C.byref(k), C.byref(st))
    return st.value, ints[:2 * min(k.value, stall_cap)].reshape(-1, 2).astype(np.int64), k.value


def finalize(norm, segs, rm, rs, shc, scc, rescale=True):
    """k_finalize on one read -> (per-base means, re-normalised signal, sig_match_score)"""
    L = stage_lib()
    norm, rm, rs = (np.ascontiguousarray(a, dtype=np.float64) for a in (norm, rm, rs))
    segs = np.ascontiguousarray(segs, dtype=np.int32)
    nb = rm.shape[0]
    bm, sig, score = np.zeros(nb), np.zeros(norm.shape[0]), C.c_double(0)
    dp = C.POINTER(C.c_double)
    st = L.emul_finalize(norm.ctypes.data_as(dp), C.c_int(norm.shape[0]), segs.ctypes.data_as(C.POINTER(C.c_int)),
                         C.c_int(nb), rm.ctypes.data_as(dp), rs.ctypes.data_as(dp), C.c_double(shc),
                         C.c_double(scc), C.c_int(1 if rescale else 0), bm.ctypes.data_as(dp),
                         sig.ctypes.data_as(dp), C.byref(score))
    assert st == 0
    return bm, sig, score.value
