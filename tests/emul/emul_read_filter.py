"""ctypes driver of tests/emul/libemul_read_filter.so: the read filters' device source run on
the host (TEST INFRASTRUCTURE ONLY -- see cuda_emul.h).  EmulContext has the read-filter
surface of tombo_b200._lib.Context, so tombo_b200.filters runs over it unchanged."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(REPO, 'tombo_b200', 'csrc')
_LIB = None


def lib():
    """builds into a temporary directory when the tree is not writable"""
    global _LIB
    if _LIB is None:
        srcs = [os.path.join(HERE, f) for f in ('emul_read_filter.cpp', 'cuda_emul.cpp', 'cuda_emul.h')]
        srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
        srcs.append(os.path.join(REPO, 'include', 'tombo_b200.h'))
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix='emul_rf_')
        so = os.path.join(out_dir, 'libemul_read_filter.so')
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(['g++', '-O1', '-g', '-std=c++17', '-ffp-contract=off', '-fPIC',
                                   '-shared', '-o', so, srcs[0], srcs[1]])
        _LIB = C.CDLL(so)
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class EmulContext(object):
    def dwell_percentiles(self, lens, len_off, pctl):
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        off = np.ascontiguousarray(len_off, dtype=np.int64)
        pctl = np.ascontiguousarray(np.atleast_1d(pctl), dtype=np.float64)
        n = off.shape[0] - 1
        assert n >= 0 and np.all(np.diff(off) > 0) and off[0] == 0
        out = np.empty((n, pctl.shape[0]))
        if n:
            lib().emul_rf_pctl(C.c_int(n), _p(lens, C.c_longlong), _p(off, C.c_longlong),
                               C.c_int(pctl.shape[0]), _p(pctl, C.c_double), _p(out, C.c_double))
        return out

    def batch_read_filters_on(self, segs_list, scores, ok, sig_match_thresh, obs_filter=None):
        """the resident-batch kernel over host arrays: (codes, percentiles)"""
        n = len(segs_list)
        pairs = list(obs_filter or [])
        pctl = np.array([p for p, _ in pairs] or [0.0], dtype=np.float64)
        pth = np.array([t for _, t in pairs] or [0.0], dtype=np.float64)
        nb = np.array([len(s) - 1 for s in segs_list], dtype=np.int64)
        base_off = np.concatenate([[0], np.cumsum(nb)]).astype(np.int64)
        segs = np.ascontiguousarray(np.concatenate([np.asarray(s, dtype=np.int64) for s in segs_list]))
        status = np.array([0 if g else 1 for g in ok], dtype=np.int32)
        score = np.ascontiguousarray(scores, dtype=np.float64)
        code = np.empty(n, dtype=np.int8)
        pout = np.empty((n, len(pairs)))
        lib().emul_rf_batch(C.c_int(n), _p(segs, C.c_longlong), _p(base_off, C.c_longlong),
                            _p(status, C.c_int), _p(score, C.c_double), C.c_double(sig_match_thresh),
                            C.c_int(len(pairs)), _p(pctl, C.c_double), _p(pth, C.c_double),
                            _p(code, C.c_int8), _p(pout, C.c_double))
        return code, pout

    def read_mid_coverage(self, grp_off, start, end):
        """the host placement of tb2_read_mid_coverage, then its kernels"""
        grp_off, start, end = (np.asarray(a, dtype=np.int64) for a in (grp_off, start, end))
        assert np.all(end > start) and np.all(start >= 0)
        a_s, a_e = start.copy(), end.copy()
        base = 0
        for g in range(grp_off.shape[0] - 1):
            a, b = grp_off[g], grp_off[g + 1]
            if b > a:
                a_s[a:b] += base
                a_e[a:b] += base
                base += int(end[a:b].max()) + 1
        out = np.empty(start.shape[0], dtype=np.int64)
        if start.shape[0]:
            lib().emul_rf_mid(C.c_longlong(start.shape[0]), _p(np.ascontiguousarray(a_s), C.c_longlong),
                              _p(np.ascontiguousarray(a_e), C.c_longlong), C.c_longlong(base),
                              _p(out, C.c_longlong))
        return out
