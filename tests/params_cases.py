"""Resquiggle at caller-chosen parameters: the parameter points of tests/golden/rsqgl_params.npz
(what Tombo's --signal-align-parameters, --segmentation-parameters, --outlier-threshold,
--max-scaling-iterations, --skip-sequence-rescaling and --fixed-scale let a user set, plus
per-k-mer model sds and int16 raw), and the helpers the CPU and GPU tests replay them with.

Each point changes one thing from the DNA or RNA defaults unless its name says otherwise.
The bandwidth points sit on both sides of every boundary where the device's adaptive-band
engine changes (engine_of restates tb2_abs_chunk_host / tb2_abs_ms_chunk_host of
tombo_b200/csrc/kernels.h and the lane-chunk move-word widths of dp_align.cuh)."""
import numpy as np

DNA_ALN = (4.2, 4.2, 300, 1500, 20.0, 40, 750, 2500, 250)     # ALGN_PARAMS_TABLE['DNA']
RNA_ALN = (6, 4, 500, 1500, 20.0, 50, 1000, 3000, 250)
DNA_SEG, RNA_SEG = (5, 3, 1, 5), (12, 6, 2, 15)
ALN_FIELDS = ('match_evalue', 'skip_pen', 'bandwidth', 'save_bandwidth', 'max_half_z_score',
              'band_bound_thresh', 'start_bw', 'start_save_bw', 'start_n_bases')
SEG_FIELDS = ('running_stat_width', 'min_obs_per_base', 'raw_min_obs_per_base',
              'mean_obs_per_event')
POLICY = dict(outlier_thresh=5.0, max_scaling_iters=3, skip_seq_scaling=False, const_scale=None,
              max_raw_cpts=200, min_event_to_seq_ratio=1.1)
MAX_BAND = 8192          # TB2_MAX_CHUNK (256) cells per lane * 32 lanes


def engine_of(W):
    """(engine, width) the device runs an adaptive band of W cells on: ('reg', chunk) for
    the register engine (kernels.h tb2_abs_chunk_host), ('ms', chunk) for three chunks per
    lane (tb2_abs_ms_chunk_host), ('lane', move words per lane) for the lane-chunk engine
    (kernels.h tb2_tb_words: wpl 1-5, then 8 and 16), ('capacity', None) beyond 8192"""
    if W <= 218:
        return 'reg', 7
    if W <= 311:
        return 'reg', 10
    if W <= 404:
        return 'reg', 13
    if W <= 528:
        return 'reg', 17
    if W <= 95 * 13 + 1:
        return 'ms', 13
    if W <= 95 * 17 + 1:
        return 'ms', 17
    if W > MAX_BAND:
        return 'capacity', None
    wpl = ((W + 31) // 32 + 15) // 16
    return 'lane', wpl if wpl <= 5 else (8 if wpl <= 8 else 16)


def adaptive_nbases(W):
    """bases of a synthetic DNA read (~1.8 events per base) long enough for the start search
    (start_bw + start_n_bases = 1000 events) and for an adaptive band of W events after it"""
    return max(700, int(W / 1.6) + 300)


def _pt(name, kind='DNA', aln=None, seg=None, nbases=(444, 444, 900, 1300, 300, 700),
        pol=None, sd_range=None, int16=False, stable=None, stall=None, **aln_seg):
    """one point; ``stable`` pins the reference's changepoint argsort to the stable tie rule
    (DESIGN.md, tie rule) where the signal has exact ties: int16 raw, and winsorising limits
    tight enough that many samples are clipped to the same value"""
    aln = list(DNA_ALN if kind == 'DNA' else RNA_ALN) if aln is None else list(aln)
    seg = list(DNA_SEG if kind == 'DNA' else RNA_SEG) if seg is None else list(seg)
    for k, v in aln_seg.items():
        if k in ALN_FIELDS:
            aln[ALN_FIELDS.index(k)] = v
        else:
            seg[SEG_FIELDS.index(k)] = v
    p = dict(POLICY)
    p.update(pol or {})
    return dict(name=name, kind=kind, aln=tuple(aln), seg=tuple(seg), nbases=list(nbases),
                pol=p, sd_range=sd_range, int16=int16,
                stable=int16 if stable is None else stable, stall=stall or {})


def _bw_point(W):
    nb = adaptive_nbases(W)
    n_long = 3 if W >= 2048 else 4
    return _pt('bw_%d' % W, bandwidth=W, nbases=[nb] * n_long + [nb + 150, 444])


BOUNDARY_BWS = (218, 219, 311, 312, 404, 405, 528, 529, 1236, 1237, 1616, 1617, 2048, 2049,
                4096, 4097, 8192)
RNA_LONG = (270, 270, 400, 600, 900)


def points():
    P = [_bw_point(W) for W in BOUNDARY_BWS + (333,)]
    # a save bandwidth on the lane-chunk engine: planted stalls leave the 150 band
    P.append(_pt('save_bw_2100', bandwidth=150, save_bandwidth=2100, nbases=[2000] * 4 + [2300],
                 stall={0: (700, 4000), 1: (900, 4000), 2: (500, 4000), 4: (1100, 4000)}))
    P += [_pt('mhz_none', max_half_z_score=None), _pt('mhz_1', max_half_z_score=1.0),
          _pt('mhz_3', max_half_z_score=3.0)]
    P += [_pt('me0_sp4.2', match_evalue=0.0), _pt('me4.2_sp0', skip_pen=0.0),
          _pt('me2_sp10', match_evalue=2.0, skip_pen=10.0),
          _pt('me8_sp1', match_evalue=8.0, skip_pen=1.0),
          _pt('me6_sp4_rna_values', match_evalue=6, skip_pen=4)]
    P += [_pt('bbt_0', band_bound_thresh=0), _pt('bbt_1', band_bound_thresh=1),
          _pt('bbt_half_bw_m1', band_bound_thresh=300 // 2 - 1)]
    P += [_pt('start_bw_lt_n_bases', start_bw=150, start_n_bases=250),
          _pt('start_n_bases_30', start_n_bases=30, start_bw=300),
          _pt('start_n_bases_60', start_n_bases=60),
          _pt('start_save_bw_lt_start_bw', start_save_bw=500, start_bw=750,
              nbases=(444, 444, 900, 1300, 700, 2000)),
          _pt('start_bw_static_long', start_bw=4000, nbases=(900, 1300, 1800, 2000, 444))]
    P += [_pt('rsw_%d' % w, running_stat_width=w) for w in (2, 8, 30)]
    P += [_pt('min_obs_%d' % m, min_obs_per_base=m) for m in (1, 4, 6, 10)]
    # few enough events requested that six samples per base still segment
    P.append(_pt('min_obs_6_mean_obs_12', min_obs_per_base=6, mean_obs_per_event=12))
    P += [_pt('raw_min_obs_%d' % m, raw_min_obs_per_base=m) for m in (2, 3)]
    P += [_pt('mean_obs_%d' % m, mean_obs_per_event=m) for m in (1, 3, 12)]
    P += [_pt('rna_raw_min_obs_1', kind='RNA', raw_min_obs_per_base=1, nbases=RNA_LONG),
          _pt('rna_rsw8_min_obs4', kind='RNA', running_stat_width=8, min_obs_per_base=4,
              nbases=RNA_LONG)]
    P += [_pt('outlier_none', pol=dict(outlier_thresh=None)),
          _pt('outlier_1', pol=dict(outlier_thresh=1.0), stable=True),
          _pt('outlier_2.5', pol=dict(outlier_thresh=2.5), stable=True)]
    P += [_pt('iters_%d' % n, pol=dict(max_scaling_iters=n)) for n in (1, 2, 5)]
    # without sequence rescaling, and with a tight model (sd 0.03-0.06) so that z-scores beyond
    # 20 occur and None differs from the default clamp
    P += [_pt('skip_seq_scaling_mhz_none', max_half_z_score=None,
              pol=dict(skip_seq_scaling=True), sd_range=(0.03, 0.06),
              nbases=(444, 444, 900, 1300, 300, 700, 600, 800)),
          _pt('const_scale_dna', pol=dict(const_scale=57.0)),
          _pt('max_raw_cpts_8', pol=dict(max_raw_cpts=8)),
          _pt('event_ratio_2', pol=dict(min_event_to_seq_ratio=2.0))]
    P += [_pt('model_sd_dna', sd_range=(0.1, 0.4)),
          _pt('model_sd_rna', kind='RNA', sd_range=(0.1, 0.4), nbases=RNA_LONG)]
    P += [_pt('int16_mhz_1', max_half_z_score=1.0, int16=True),
          _pt('int16_me0_sp0', match_evalue=0.0, skip_pen=0.0, int16=True)]
    # the widest changepoint bit sets (min_obs_per_base 10) on reads that segment: RNA dwells
    P.append(_pt('rna_min_obs_10', kind='RNA', min_obs_per_base=10, nbases=RNA_LONG))
    return P


# load_resquiggle_parameters on float tuples as the CLI parses them (type=float)
LOAD_PARAM_CASES = [
    ('DNA', (4.2, 4.2, 333.7, 1500.2, 20.0, 40.9, 750.5, 2500.1, 250.9), None),
    ('DNA', (0.0, 10.5, 2100.0, 2100.0, None, 0.0, 150.0, 500.0, 30.0), (2, 10, 3, 12)),
    ('RNA', (6.0, 4.0, 500.5, 1500.0, 1.0, 50.0, 1000.0, 3000.0, 250.0), (8, 4, 1, 15)),
    ('RNA', None, None),
    ('DNA', None, (30, 1, 2, 1)),
]


# ---------------------------------------------------------------- replaying the golden
def golden():
    import golden_util as gu
    return gu.load('rsqgl_params')


def _none(v):
    return None if np.isnan(v) else float(v)


def point_of(g, j, RP):
    """the parameters of golden point j: RP(params), RP(save params), kind, oracle-style policy
    keywords, sd_range, int16"""
    kind = str(g['p_kind'][j])
    a = g['p_aln'][j]
    aln = tuple(_none(v) if i == 4 else (float(v) if i in (0, 1) else int(v))
                for i, v in enumerate(a))
    seg = tuple(int(v) for v in g['p_seg'][j])
    pol = dict(outlier_thresh=_none(g['p_outlier'][j]), max_scaling_iters=int(g['p_iters'][j]),
               skip_seq_scaling=bool(g['p_skip'][j]), const_scale=_none(g['p_const_scale'][j]),
               max_raw_cpts=int(g['p_max_raw_cpts'][j]),
               min_event_to_seq_ratio=float(g['p_ev_ratio'][j]))
    sdr = None if np.isnan(g['p_sd_range'][j][0]) else tuple(float(v) for v in g['p_sd_range'][j])
    rna = kind == 'RNA'
    return dict(name=str(g['p_name'][j]), kind=kind, aln=aln, seg=seg,
                rp=RP(aln, seg, rna=rna), sp=RP(aln, seg, rna=rna, save=True), pol=pol,
                sd_range=sdr, int16=bool(g['p_int16'][j]))


def reads_of_point(g, j):
    """the regenerated reads of golden point j (checked against the stored checksums) and the
    model they were drawn from"""
    from tombo_b200 import synthetic as syn
    pt = dict(kind=str(g['p_kind'][j]))
    sdr = None if np.isnan(g['p_sd_range'][j][0]) else tuple(g['p_sd_range'][j])
    kmer_ref, cpos = syn.make_kmer_ref(pt['kind'], 0, sd_range=sdr)
    reads = []
    for i in range(int(g['p_read_off'][j]), int(g['p_read_off'][j + 1])):
        kw = dict(kind=pt['kind'], int16=bool(g['p_int16'][j]))
        if g['r_stall'][i][0] >= 0:
            kw['stall'] = (int(g['r_stall'][i][0]), int(g['r_stall'][i][1]))
        r = syn.make_read(kmer_ref, cpos, int(g['r_nbases'][i]), int(g['r_seed'][i]), **kw)
        assert float(np.sum(np.asarray(r.raw, dtype=np.float64))) == float(g['raw_checksum'][i]), \
            'synthetic generator drifted from the golden inputs'
        reads.append(r)
    return kmer_ref, cpos, reads


def expected(g, i):
    """what the reference returned for golden read i (global read index)"""
    s = g['scalars'][i]
    a, b = int(g['seg_off'][i]), int(g['seg_off'][i + 1])
    return dict(message=str(g['messages'][i]), segs=g['segs'][a:b].astype(np.int64), shift=s[0],
                scale=s[1], lower_lim=s[2], upper_lim=s[3], sig_match_score=s[4],
                read_start_rel_to_raw=int(s[5]) if not np.isnan(s[5]) else None,
                calls=int(s[6]), rescued=bool(s[7]), n_iters=int(s[8]),
                norm_params_changed=bool(s[9]))
