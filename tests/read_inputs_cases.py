"""Caller-supplied per-read inputs of resquiggle_read: map_res.scale_values and
map_res.stall_ints (resquiggle.py:1079-1118).  The case lists shared by the host-emulation
tests and the GPU tests, and a plain restatement of remove_stall_cpts."""
import numpy as np

NORM_THRESHOLDS = (5.0, 0.5)    # 0.5 MAD: most samples are clipped


def remove_stall_cpts(stall_ints, cpts):
    """tombo_stats.py:1576-1597 as written: walk the intervals in list order next to the
    ascending changepoints; test each one against the first interval whose end is >= it,
    or the last interval when there is none"""
    if len(stall_ints) == 0:
        return np.asarray(cpts)
    it = iter(stall_ints)
    cur = next(it)
    keep = []
    for i, c in enumerate(cpts):
        while c > cur[1]:
            try:
                cur = next(it)
            except StopIteration:
                break
        if not (cur[0] < c < cur[1]):
            keep.append(i)
    return np.asarray(cpts)[keep]


def norm_signal(n, seed, integer):
    """a heavy-tailed DAC-like signal of n samples, integer-valued if asked"""
    raw = 480 + 60 * np.random.RandomState(seed).standard_t(5, n)
    return np.round(raw) if integer else raw


def norm_scale_values(raw):
    """(name, scale_values) for normalize_raw_signal: the signal's own median / MAD with
    finite limits, and a shifted and scaled copy with None limits"""
    raw = np.asarray(raw, dtype=np.float64)
    med = float(np.median(raw))
    mad = float(np.median(np.abs(raw - med)))
    return [('own_finite', (med, mad, -4.0, 4.0, None)),
            ('shifted_none', (med + 3.7, mad * 1.13, None, None, None))]


def stall_lists(n, cpts):
    """name -> stall list of a read of n samples whose sorted changepoints are cpts.
    'unsorted', 'overlapping' and 'nested_*' are lists identify_stalls never returns; on
    them 'inside any interval' and the reference's walk disagree"""
    def a(f):
        return int(n * f)
    c = [int(x) for x in cpts]
    return {
        'sorted': [(a(.1), a(.2)), (a(.4), a(.5))],
        'unsorted': [(a(.4), a(.5)), (a(.1), a(.2))],
        'overlapping': [(a(.2), a(.5)), (a(.1), a(.3))],
        'nested_inner_first': [(a(.2), a(.3)), (a(.1), a(.9))],
        'nested_outer_first': [(a(.1), a(.6)), (a(.2), a(.3))],
        'endpoints': [(c[10], c[20]), (c[30], c[31]), (c[40], c[40])],   # strict comparisons
        'empty': [],
        'huge': [(-2 ** 40, c[5]), (c[len(c) // 2], 2 ** 40)],           # int64 beyond int32
    }


# ---------------------------------------------------------------- tests/golden/rsqgl_inputs.npz
def golden():
    import golden_util as gu
    return gu.load('rsqgl_inputs')


def golden_norm_cases(g):
    """(raw, outlier_thresh, scale_values, expected norm, expected five values with None)"""
    out = []
    for i in range(g['nm_n'].shape[0]):
        raw = norm_signal(int(g['nm_n'][i]), int(g['nm_seed'][i]), int(g['nm_int'][i]))
        t = None if np.isnan(g['nm_t'][i]) else float(g['nm_t'][i])
        sv = tuple(None if np.isnan(v) else float(v) for v in g['nm_sv'][i])
        e = tuple(None if g['nm_out_none'][i][j] else float(g['nm_out'][i][j]) for j in range(5))
        out.append((raw, t, sv, g['nm_norm'][g['nm_off'][i]:g['nm_off'][i + 1]], e))
    return out


def golden_cases(g, RP):
    """one dict per resquiggle case: the regenerated read, its inputs and parameters, and what
    the reference returned ('expected': message, segs, rsrtr, five scale values with None,
    score, changed, calls, rescued, n_iters)"""
    import golden_util as gu
    from tombo_b200 import synthetic as syn
    out = []
    for i in range(g['c_call'].shape[0]):
        kind = str(g['c_kind'][i])
        kmer_ref, cpos = syn.make_kmer_ref(kind, 0)
        plant = g['c_plant'][i]
        kw = {} if plant[0] < 0 else dict(stall=(int(plant[0]), int(plant[1])))
        r = syn.make_read(kmer_ref, cpos, int(g['c_nbases'][i]), int(g['c_seed'][i]), kind=kind, **kw)
        assert float(np.sum(np.asarray(r.raw, dtype=np.float64))) == float(g['raw_checksum'][i]), \
            'synthetic generator drifted from the golden inputs'
        aln = g['c_aln'][i]
        aln = gu.RNA_ALN if np.isnan(aln[0]) else tuple(
            float(a) if j in (0, 1, 4) else int(a) for j, a in enumerate(aln))
        rna = bool(g['c_rna_params'][i])
        seg = gu.RNA_SEG if rna else gu.DNA_SEG
        sv = tuple(None if np.isnan(v) else float(v) for v in g['c_sv'][i]) if g['c_has_sv'][i] else None
        a, b = g['c_stall_off'][i], g['c_stall_off'][i + 1]
        si = [(int(x), int(y)) for x, y in g['c_stalls'][a:b]] if g['c_has_stalls'][i] else None
        s = g['o_scalars'][i]
        msg = str(g['o_messages'][i])
        e = dict(message=msg, calls=int(s[8]), rescued=bool(s[9]))
        if not msg:
            sa, sb = g['o_seg_off'][i], g['o_seg_off'][i + 1]
            e.update(segs=g['o_segs'][sa:sb], scale_values=tuple(
                None if g['o_none'][i][j] else float(s[j]) for j in range(5)),
                sig_match_score=float(s[5]), read_start_rel_to_raw=int(s[6]),
                norm_params_changed=bool(s[7]), n_iters=int(s[10]))
        cs = float(g['c_const_scale'][i])
        out.append(dict(
            call=int(g['c_call'][i]), kind=kind, kmer_ref=kmer_ref, cpos=cpos, read=r,
            rp=RP(aln, seg, rna=rna), sp=RP(aln, seg, rna=rna, save=True),
            skip=bool(g['c_skip'][i]), const_scale=None if np.isnan(cs) else cs,
            scale_values=sv, stall_ints=si, group=int(g['c_group'][i]),
            read_index=int(g['c_read_index'][i]), expected=e))
    return out


def same_message(status, message, expected):
    """a status / message against the reference's: its TomboError text, or its
    'Unexpected error' bucket (any other exception) for status 100"""
    if expected.startswith('UNEXPECTED'):
        return status == 100
    return status != 0 and message == expected
