"""Harness that imports the UNMODIFIED reference built by oracle/build_ref.py
(oracle/_ref/) and drives its resquiggle hot path on in-memory synthetic reads.

TEST INFRASTRUCTURE ONLY (oracle/): used by tests/golden/make_golden.py, by the
CPU tests that pin oracle/ against the reference, and by bench.py's
cpu_baseline / --impl reference leg.  Never imported by tombo_b200/.

Shims (SURVEY.md section 8c-2), all harness side, no reference edits:
  * ``numpy.NAN`` alias (numpy 2 removed it; tombo_stats.py:307,313);
  * ``h5py`` / ``mappy`` replaced by MagicMock (FAST5 / minimap2 are outside
    the path; resquiggle.py:14-26, tombo_stats.py:16);
  * ``scipy.stats.halfnorm.expect`` evaluated under ``np.errstate(ignore)``
    because tombo_helper.py:18 sets ``np.seterr(all='raise')`` before
    tombo_stats.py:84 runs scipy's quadrature.
  * optional: ``np.argsort`` pinned to ``kind='stable'`` inside _c_helper for
    the int16 (tied-score) parity set (SURVEY.md section 8c-7).
  * ``np.random.choice`` inside tombo_stats replaced by the keyed sub-sampler of
    tombo_b200.synthetic (the reference's draw is from the unseeded global RNG).
"""
import os
import sys
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REF_DIR = os.path.join(HERE, '_ref')

_mods = None


def available():
    sys.path.insert(0, HERE)
    try:
        import build_ref
        return build_ref.is_built()
    finally:
        sys.path.remove(HERE)


def load_reference():
    """Import tombo.{tombo_helper,tombo_stats,resquiggle} from oracle/_ref."""
    global _mods
    if _mods is not None:
        return _mods
    if not available():
        raise RuntimeError('oracle/_ref is not built (run oracle/build_ref.py '
                           'where /root/reference exists)')
    if not hasattr(np, 'NAN'):
        np.NAN = np.nan
    for name in ('h5py', 'mappy'):
        if name not in sys.modules or not isinstance(
                sys.modules[name], mock.MagicMock):
            sys.modules[name] = mock.MagicMock()
    import scipy.stats as st
    orig_expect = st.halfnorm.expect

    def _expect(*a, **k):
        with np.errstate(all='ignore'):
            return orig_expect(*a, **k)
    st.halfnorm.expect = _expect
    import warnings
    sys.path.insert(0, REF_DIR)
    old_err = np.geterr()
    try:
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            import tombo.tombo_helper as th
            import tombo.tombo_stats as ts
            import tombo.resquiggle as rsq
            import tombo._c_helper as ch
            import tombo._c_dynamic_programming as cdp
    finally:
        sys.path.remove(REF_DIR)
        st.halfnorm.expect = orig_expect
    # the reference sets np.seterr(all='raise') globally at import; keep that
    # only while reference code runs (see ref_errstate below)
    np.seterr(**old_err)
    _mods = dict(th=th, ts=ts, rsq=rsq, ch=ch, cdp=cdp)
    return _mods


class ref_errstate(object):
    """Reference code runs with np.seterr(all='raise') (tombo_helper.py:18)."""

    def __enter__(self):
        self._old = np.seterr(all='raise')

    def __exit__(self, *a):
        np.seterr(**self._old)


class stable_argsort(object):
    """Pin np.argsort to kind='stable' (tie rule for the int16 parity set)."""

    def __enter__(self):
        self._orig = np.argsort

        def _stable(a, *args, **kw):
            kw['kind'] = 'stable'
            return self._orig(a, *args, **kw)
        np.argsort = _stable

    def __exit__(self, *a):
        np.argsort = self._orig


class keyed_choice(object):
    """Replace np.random.choice by the keyed sub-sampler while the reference
    runs one resquiggle_read call."""

    def __init__(self, key):
        self.key = key

    def __enter__(self):
        sys.path.insert(0, REPO)
        from tombo_b200.synthetic import theil_sen_subsample
        sys.path.remove(REPO)
        self._orig = np.random.choice
        key = self.key

        def _choice(n, size, replace=False):
            assert not replace
            return theil_sen_subsample(int(n), int(size), key)
        np.random.choice = _choice

    def __exit__(self, *a):
        np.random.choice = self._orig


def make_models(kmer_ref, central_pos, alt_rows=None, alt_base='C'):
    m = load_reference()
    std_ref = m['ts'].TomboModel(kmer_ref=kmer_ref, central_pos=central_pos)
    alt_ref = None
    if alt_rows is not None:
        alt_ref = m['ts'].AltModel(kmer_ref=alt_rows, central_pos=central_pos,
                                   alt_base=alt_base, name='5mC')
    return std_ref, alt_ref


def make_params(kind='DNA', sig_aln_params=None, seg_params=None):
    m = load_reference()
    th, ts = m['th'], m['ts']
    sst = th.seqSampleType(kind, kind == 'RNA')
    p = ts.load_resquiggle_parameters(sst, sig_aln_params, seg_params)
    sp = ts.load_resquiggle_parameters(sst, sig_aln_params, seg_params,
                                       use_save_bandwidth=True)
    return sst, p, sp


def make_map_res(raw, genome_seq, read_id='r'):
    th = load_reference()['th']
    return th.resquiggleResults(
        align_info=th.alignInfo(read_id, 'BaseCalled_template', 0, 0, 0, 0,
                                len(genome_seq), 0),
        genome_loc=th.genomeLocation(0, '+', 'chr'),
        genome_seq=genome_seq, mean_q_score=10.0, raw_signal=raw)


def run_read(raw, genome_seq, std_ref, sst, params, save_params,
             outlier_thresh=5.0, max_scaling_iters=3, key_seed=0,
             read_index=0, stable_ties=False, const_scale=None,
             skip_seq_scaling=False, scale_values=None, stall_ints=None,
             max_raw_cpts=None, min_event_to_seq_ratio=None):
    """The worker's per-read policy, restated from resquiggle.py:1492-1530 and
    1575-1595 (adjust_map_res, run_rsqgl_iters, rescue with save_params).
    ``scale_values`` / ``stall_ints`` go into the initial map_res; for RNA,
    adjust_map_res overwrites the stalls with identify_stalls.  ``max_raw_cpts`` and
    ``min_event_to_seq_ratio`` are passed to every resquiggle_read call when given
    (None: the reference's defaults).

    Returns ``(res, err, info)``: the final resquiggleResults or None, the
    TomboError/other message or None, and a dict with the call count.
    """
    m = load_reference()
    th, ts, rsq = m['th'], m['ts'], m['rsq']
    sys.path.insert(0, REPO)
    from tombo_b200.synthetic import subsample_key
    sys.path.remove(REPO)
    map_res = make_map_res(raw, genome_seq)._replace(scale_values=scale_values,
                                                     stall_ints=stall_ints)
    info = dict(calls=0, rescued=False)
    call_kw = {}
    if max_raw_cpts is not None:
        call_kw['max_raw_cpts'] = max_raw_cpts
    if min_event_to_seq_ratio is not None:
        call_kw['min_event_to_seq_ratio'] = min_event_to_seq_ratio

    def one_call(mr, prm, **kw):
        key = subsample_key(key_seed, read_index, info['calls'])
        info['calls'] += 1
        kw.update(call_kw)
        with keyed_choice(key):
            return rsq.resquiggle_read(mr, std_ref, prm, outlier_thresh,
                                       seq_samp_type=sst, **kw)

    def run_iters(mr, prm, all_raw):
        res = one_call(mr, prm, const_scale=const_scale,
                       skip_seq_scaling=skip_seq_scaling)
        n_iters = 1
        while n_iters < max_scaling_iters and res.norm_params_changed:
            res = one_call(mr._replace(scale_values=res.scale_values), prm,
                           all_raw_signal=all_raw)
            n_iters += 1
        info['n_iters'] = n_iters
        return res

    ctxs = [ref_errstate()]
    if stable_ties:
        ctxs.append(stable_argsort())
    for c in ctxs:
        c.__enter__()
    try:
        try:
            if sst.name == 'RNA':
                map_res = map_res._replace(raw_signal=map_res.raw_signal[::-1])
                map_res = map_res._replace(stall_ints=ts.identify_stalls(
                    map_res.raw_signal, rsq.DEFAULT_STALL_PARAMS))
            all_raw = map_res.raw_signal
            try:
                res = run_iters(map_res, params, all_raw)
            except Exception as e:   # noqa  (reference: bare except)
                info['rescued'] = True
                info['first_error'] = str(e)
                res = run_iters(map_res, save_params, all_raw)
        except th.TomboError as e:
            return None, str(e), info
        except Exception as e:
            return None, 'UNEXPECTED: ' + repr(e), info
    finally:
        for c in reversed(ctxs):
            c.__exit__(None, None, None)
    return res, None, info
