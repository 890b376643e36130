"""ctypes driver of tests/emul/libemul_motif.so: the motif LLR kernel's and the offsets
kernel's device source run on the host (TEST INFRASTRUCTURE ONLY -- see cuda_emul.h)."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(REPO, 'tombo_b200', 'csrc')
_LIB = None


def lib():
    """builds into a temporary directory when the tree is not writable"""
    global _LIB
    if _LIB is None:
        import tempfile
        srcs = [os.path.join(HERE, f) for f in ('emul_motif.cpp', 'cuda_emul.cpp', 'cuda_emul.h')]
        srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
        srcs.append(os.path.join(REPO, 'include', 'tombo_b200.h'))
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix='emul_motif_')
        so = os.path.join(out_dir, 'libemul_motif.so')
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(['g++', '-O1', '-g', '-std=c++17', '-ffp-contract=off', '-fPIC',
                                   '-shared', '-o', so, srcs[0], srcs[1]])
        _LIB = C.CDLL(so)
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def can_overlap(mask):
    m = np.ascontiguousarray(mask, dtype=np.uint8)
    return bool(lib().emul_motif_can_overlap(_p(m, C.c_uint8), C.c_int(m.shape[0])))


def llr_motif(norm_mean, mean_off, seq, seq_off, read_start, strand, K, cpos, kmeans, ksds, alt,
              mask, mod_pos, max_ab, reg_start, reg_end, mode=1, sf=4.0, hf=1.0, hp=0.2):
    """k_llr_motif count / scan / fill on the host -> (llr, pos, site_off, status)"""
    f64, i64 = C.c_double, C.c_longlong
    norm_mean = np.ascontiguousarray(norm_mean, dtype=np.float64)
    mean_off, seq_off, read_start = (np.ascontiguousarray(a, dtype=np.int64)
                                     for a in (mean_off, seq_off, read_start))
    seq = np.ascontiguousarray(seq, dtype=np.uint8)
    strand = np.ascontiguousarray(strand, dtype=np.int8)
    kmeans, ksds, alt = (np.ascontiguousarray(a, dtype=np.float64) for a in (kmeans, ksds, alt))
    mask = np.ascontiguousarray(mask, dtype=np.uint8)
    n = mean_off.shape[0] - 1
    cap = max(1, norm_mean.shape[0])
    llr, pos = np.zeros(cap), np.zeros(cap, dtype=np.int64)
    off, st = np.zeros(n + 1, dtype=np.int64), np.zeros(max(1, n), dtype=np.int32)
    lib().emul_llr_motif(
        C.c_int(n), _p(norm_mean, f64), _p(mean_off, i64), _p(seq, C.c_uint8), _p(seq_off, i64),
        _p(read_start, i64), _p(strand, C.c_int8), C.c_int(K), C.c_int(cpos), _p(kmeans, f64),
        _p(ksds, f64), _p(alt, f64), C.c_int(1 if mode == 1 else 0), f64(sf), f64(hf), f64(hp),
        C.c_int(mask.shape[0]), C.c_int(mod_pos), _p(mask, C.c_uint8), i64(max_ab), i64(reg_start),
        i64(reg_end), _p(llr, f64), _p(pos, i64), _p(off, i64), _p(st, C.c_int32))
    t = int(off[-1])
    return llr[:t], pos[:t], off, st[:n]


def scan_offsets(cnt, in_place=False):
    """k_scan_offsets on the host: int32 or uint64 counts -> int64 offsets (n + 1).  in_place
    (uint64 only) scans a buffer of n + 1 entries that holds the counts, as accuracy does."""
    cnt = np.ascontiguousarray(cnt)
    n = cnt.shape[0]
    u64 = cnt.dtype == np.uint64
    assert u64 or cnt.dtype == np.int32
    if in_place:
        assert u64
        buf = np.zeros(n + 1, dtype=np.uint64)
        buf[:n] = cnt
        lib().emul_scan_offsets(C.c_int(1), _p(buf, C.c_uint64), _p(buf, C.c_longlong), C.c_longlong(n))
        return buf.view(np.int64)
    off = np.full(n + 1, -1, dtype=np.int64)
    lib().emul_scan_offsets(C.c_int(1 if u64 else 0), _p(cnt, C.c_uint64 if u64 else C.c_int32),
                            _p(off, C.c_longlong), C.c_longlong(n))
    return off
