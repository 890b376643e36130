"""ctypes driver of tests/emul/libemul_stats_file.so: the statistics-file kernels' device
source run on the host (TEST INFRASTRUCTURE ONLY -- see cuda_emul.h).  EmulContext has the
tb2_stats_file_* / tb2_most_signif_* surface of tombo_b200._lib.Context, so the writers and
aggregate_per_read_stats run over it unchanged."""
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
        srcs = [os.path.join(HERE, f) for f in ('emul_stats_file.cpp', 'cuda_emul.cpp', 'cuda_emul.h')]
        srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
        srcs.append(os.path.join(REPO, 'include', 'tombo_b200.h'))
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix='emul_sf_')
        so = os.path.join(out_dir, 'libemul_stats_file.so')
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(['g++', '-O1', '-g', '-std=c++17', '-ffp-contract=off', '-fPIC',
                                   '-shared', '-o', so, srcs[0], srcs[1]])
        _LIB = C.CDLL(so)
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class EmulContext(object):
    """``smem`` picks the aggregation's shared-memory counters; otherwise global counters with
    ``per`` blocks a launch (the chunking of the fallback path)"""

    def __init__(self, smem=True, per=1 << 20):
        self.smem, self.per = smem, per

    def stats_file_aggregate(self, blocks, region_size, pos, stat, thresh, lower, stat_type,
                             unmod, mod):
        blocks = np.ascontiguousarray(blocks, dtype=np.int64).reshape(-1, 5)
        pos = np.ascontiguousarray(pos, dtype=np.uint32)
        stat = np.ascontiguousarray(stat, dtype=np.float64)
        off = np.zeros(blocks.shape[0] + 1, dtype=np.int64)
        err = lib().emul_sf_aggregate(
            C.c_longlong(blocks.shape[0]), _p(blocks, C.c_longlong), C.c_longlong(region_size),
            _p(pos, C.c_uint32), _p(stat, C.c_double), C.c_double(thresh),
            C.c_double(np.nan if lower is None else lower), C.c_int(int(stat_type == 0)),
            C.c_double(unmod), C.c_double(mod), C.c_int(int(self.smem)), C.c_longlong(self.per),
            _p(off, C.c_longlong))
        if err:
            raise ValueError('position outside its block')
        return off

    def stats_file_download(self, n):
        out = (np.empty(n, np.uint32), np.empty(n), np.empty(n), np.empty(n, np.uint32),
               np.empty(n, np.uint32))
        lib().emul_sf_download(_p(out[0], C.c_uint32), _p(out[1], C.c_double), _p(out[2], C.c_double),
                               _p(out[3], C.c_uint32), _p(out[4], C.c_uint32))
        return out

    def most_signif_begin(self, level, n):
        self._level = bool(level)
        lib().emul_ms_begin(C.c_int(int(self._level)), C.c_longlong(n))

    def most_signif_end(self):
        pass

    def most_signif_add_rows(self, key, pos, cov, control_cov, chrm, strand, frac=None,
                             valid_cov=None):
        key = np.ascontiguousarray(key, dtype=np.float64)
        u = [np.ascontiguousarray(a, dtype=np.uint32) for a in (pos, cov, control_cov)]
        fr = np.ascontiguousarray(frac, dtype=np.float64) if frac is not None else None
        vc = np.ascontiguousarray(valid_cov, dtype=np.uint32) if valid_cov is not None else None
        sb = strand if isinstance(strand, int) else bytes(strand)[0]
        lib().emul_ms_add_rows(C.c_longlong(key.shape[0]), _p(key, C.c_double),
                               _p(fr, C.c_double) if fr is not None else None, _p(u[0], C.c_uint32),
                               _p(u[1], C.c_uint32), _p(u[2], C.c_uint32),
                               _p(vc, C.c_uint32) if vc is not None else None, C.c_uint(int(chrm)),
                               C.c_ubyte(sb))

    def most_signif_add_aggregate(self):
        lib().emul_ms_add_aggregate()

    def most_signif_get(self):
        lib().emul_ms_count.restype = C.c_longlong
        n = lib().emul_ms_count()
        K = 4 if self._level else 5
        w = np.zeros((K, n), dtype=np.uint64)
        lib().emul_ms_words(_p(w, C.c_uint64))
        c = dict(key=w[0].view(np.float64))
        if self._level:
            c.update(pos=(w[1] >> 32).astype(np.uint32), cov=(w[1] & 0xffffffff).astype(np.uint32),
                     control_cov=(w[2] >> 32).astype(np.uint32), chrm=(w[2] & 0xffffffff).astype(np.uint32),
                     strand=w[3].astype(np.uint8))
        else:
            c.update(frac=w[1].view(np.float64), pos=(w[2] >> 32).astype(np.uint32),
                     cov=(w[2] & 0xffffffff).astype(np.uint32), control_cov=(w[3] >> 32).astype(np.uint32),
                     valid_cov=(w[3] & 0xffffffff).astype(np.uint32), chrm=(w[4] >> 8).astype(np.uint32),
                     strand=(w[4] & 255).astype(np.uint8))
        c['strand'] = c['strand'].view('S1')
        return c
