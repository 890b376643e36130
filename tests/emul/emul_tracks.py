"""ctypes driver of tests/emul/libemul_tracks.so: the genome browser tracks' device source run
on the host (TEST INFRASTRUCTURE ONLY -- see cuda_emul.h).  EmulContext has the
coverage_runs / slot_means surface of tombo_b200._lib.Context, so tombo_b200.text_output runs
over it unchanged; the host placement and checks restate browser_tracks.cu's."""
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
        srcs = [os.path.join(HERE, f) for f in ('emul_tracks.cpp', 'cuda_emul.cpp', 'cuda_emul.h')]
        srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
        srcs.append(os.path.join(REPO, 'include', 'tombo_b200.h'))
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix='emul_bt_')
        so = os.path.join(out_dir, 'libemul_tracks.so')
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(['g++', '-O1', '-g', '-std=c++17', '-ffp-contract=off', '-fPIC',
                                   '-shared', '-o', so, srcs[0], srcs[1]])
        _LIB = C.CDLL(so)
        _LIB.emul_bt_runs.restype = C.c_longlong
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class EmulContext(object):
    def coverage_runs(self, grp_off, start, end):
        grp_off, start, end = (np.ascontiguousarray(a, dtype=np.int64) for a in (grp_off, start, end))
        assert np.all(end > start) and np.all(start >= 0)
        n_groups = grp_off.shape[0] - 1
        a_s, a_e = start.copy(), end.copy()
        base = np.zeros(n_groups + 1, dtype=np.int64)
        for g in range(n_groups):
            a, b = grp_off[g], grp_off[g + 1]
            base[g + 1] = base[g]
            if b > a:
                a_s[a:b] += base[g]
                a_e[a:b] += base[g]
                base[g + 1] += int(end[a:b].max()) + 1
        bound = 2 * start.shape[0] + n_groups
        run_off = np.zeros(n_groups + 1, dtype=np.int64)
        rs, rc = np.empty(max(bound, 1), np.int64), np.empty(max(bound, 1), np.int64)
        if start.shape[0] == 0:
            return run_off, rs[:0], rc[:0]
        m = lib().emul_bt_runs(C.c_longlong(start.shape[0]), _p(a_s, C.c_longlong), _p(a_e, C.c_longlong),
                               C.c_longlong(n_groups), _p(base, C.c_longlong), _p(run_off, C.c_longlong),
                               _p(rs, C.c_longlong), _p(rc, C.c_longlong))
        return run_off, rs[:m], rc[:m]

    def slot_means(self, chrm_len, batches):
        sums = np.zeros(chrm_len)
        cov = np.zeros(chrm_len, dtype=np.int32)
        for start, val_off, vals, reverse in batches:
            start, val_off = np.asarray(start, np.int64), np.asarray(val_off, np.int64)
            nv = np.diff(val_off)
            if np.any(nv < 0) or np.any(start < 0) or np.any(start + nv > chrm_len):
                raise ValueError('slot sums: a read\'s values run outside [0, chrm_len)')
            if nv.sum() == 0:
                continue
            has = nv > 0
            kmin, kmax = int(start[has].min()), int((start + nv - 1)[has].max())
            off = np.ascontiguousarray(val_off - val_off[0])
            v = np.ascontiguousarray(np.asarray(vals, np.float64)[val_off[0]:val_off[-1]])
            rev = np.ascontiguousarray(reverse, dtype=np.uint8)
            st = np.ascontiguousarray(start)
            if lib().emul_bt_add(C.c_longlong(st.shape[0]), _p(st, C.c_longlong), _p(off, C.c_longlong),
                                 _p(rev, C.c_uint8), _p(v, C.c_double), C.c_longlong(kmin), C.c_longlong(kmax),
                                 _p(sums, C.c_double), _p(cov, C.c_int)):
                raise ValueError('slot sums: coverage above 2^31 - 1 at a position')
        out = np.empty(chrm_len)
        if chrm_len:
            lib().emul_bt_means(_p(sums, C.c_double), _p(cov, C.c_int), C.c_longlong(chrm_len), _p(out, C.c_double))
        return out
