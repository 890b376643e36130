"""Cases of tests/golden/roc.npz (accuracy of modified-base calls) and a vectorised numpy
restatement of the reference's labelling (_compute_motif_stats, _compute_ground_truth_stats,
_compute_ctrl_motif_stats tombo_stats.py:2406-2535) and of prep_accuracy_rates with
compute_accuracy_rates (_plot_commands.py:60-82, tombo_stats.py:2377-2404).

Inputs are rebuilt from recorded seeds: a two-chromosome genome, per-read or per-site
statistics blocks of several sizes on both strands, ground-truth locations and control
statistics.  The objects follow the protocol the reference iterates: ``stats`` yields
``(chrm, strand, start, end, block_stats)`` and has ``_stat_slot``; ``genome_index.get_seq``;
``ctrl_stats.get_reg_stats``."""
import re

import numpy as np

PER_READ_DT = np.dtype([('pos', 'u4'), ('stat', 'f8'), ('read_id', 'u4')])
PER_SITE_DT = np.dtype([('pos', 'u4'), ('frac', 'f8'), ('damp_frac', 'f8'), ('valid_cov', 'u4')])
ROC_PLOT_POINTS = 1000
CHRMS = (('chr1', 520), ('chr2', 340))
COMP = {'A': 'T', 'C': 'G', 'G': 'C', 'T': 'A'}
IUPAC = {'A': 'A', 'C': 'C', 'G': 'G', 'T': 'T', 'B': '[CGT]', 'D': '[AGT]', 'H': '[ACT]',
         'K': '[GT]', 'M': '[AC]', 'N': '[ACGT]', 'R': '[AG]', 'S': '[CG]', 'V': '[ACG]',
         'W': '[AT]', 'Y': '[CT]'}
IUPAC_SETS = {k: set(v.strip('[]')) for k, v in IUPAC.items()}


class Genome(object):
    def __init__(self, seqs):
        self.seqs = dict(seqs)
        self.calls = []

    def get_seq(self, chrm, start, end, error_end=False):
        self.calls.append((chrm, int(start), int(end)))
        return self.seqs[chrm][start:end]


class Stats(object):
    """blocks in iteration order; ``pulled`` counts the blocks handed out"""

    def __init__(self, blocks, stat_slot):
        self.blocks = blocks
        self._stat_slot = stat_slot
        self.pulled = 0

    def __iter__(self):
        for b in self.blocks:
            self.pulled += 1
            yield b


class CtrlStats(object):
    def __init__(self, blocks, none_every=0):
        self.by_key = {(c, s, st, en): bs for c, s, st, en, bs in blocks}
        self.none_every = none_every
        self.calls = []

    def get_reg_stats(self, chrm, strand, start, end):
        self.calls.append((chrm, strand, int(start), int(end)))
        if self.none_every and len(self.calls) % self.none_every == 0:
            return None
        return self.by_key.get((chrm, strand, start, end))


def make_genome(seed):
    rs = np.random.RandomState(seed)
    seqs = []
    for chrm, n in CHRMS:
        s = ''.join(rs.choice(list('ACGT'), n, p=[0.25, 0.3, 0.3, 0.15]))
        s = s[:40] + 'NNN' + s[43:]                   # a non-ACGT run (code 4)
        seqs.append((chrm, s))
    return Genome(seqs)


def _stat_values(rs, n):
    """tie-heavy: quarters, with -0.0, +0.0, -inf and +inf sprinkled in"""
    v = np.round(rs.normal(0, 1.5, n) * 4) / 4
    k = rs.randint(0, 12, n)
    v[k == 0] = -0.0
    v[k == 1] = 0.0
    v[k == 2] = np.inf
    v[k == 3] = -np.inf
    return v


def make_blocks(seed, per_site=False, margin=(4, 4), sizes=(37, 60, 101), cov=2.0):
    """blocks over both chromosomes and strands, statistics at positions in
    [margin[0], len - margin[1]) so no window fails (the edge cases add their own)"""
    rs = np.random.RandomState(seed)
    out = []
    for chrm, n in CHRMS:
        for strand in ('+', '-'):
            start, k = 0, 0
            while start < n:
                end = min(n, start + sizes[k % len(sizes)])
                k += 1
                poss = np.arange(max(start, margin[0]), min(end, n - margin[1]))
                if per_site:
                    keep = poss[rs.rand(poss.shape[0]) < 0.8]
                    b = np.zeros(keep.shape[0], dtype=PER_SITE_DT)
                    b['pos'] = keep
                    b['damp_frac'] = _stat_values(rs, keep.shape[0])
                    b['frac'] = b['damp_frac']
                    b['valid_cov'] = 5
                else:
                    reps = rs.poisson(cov, poss.shape[0])
                    pos = np.repeat(poss, reps)
                    b = np.zeros(pos.shape[0], dtype=PER_READ_DT)
                    b['pos'] = pos
                    b['stat'] = _stat_values(rs, pos.shape[0])
                    b['read_id'] = rs.randint(0, 50, pos.shape[0])
                    b = b[rs.permutation(b.shape[0])]      # blocks are not position-sorted
                out.append((chrm, strand, start, end, b))
                start = end
    return out


def make_locs(seed, genome):
    """ground truth: (chrm1, '-') has no mod entry, one position is in both sets, and some
    locations lie outside every chromosome's range"""
    rs = np.random.RandomState(seed)
    mod, unmod = {}, {}
    for chrm, n in CHRMS:
        for strand in ('+', '-'):
            poss = rs.choice(n, n // 3, replace=False)
            m, u = np.sort(poss[: n // 8]), np.sort(poss[n // 8:])
            if (chrm, strand) != ('chr1', '-'):
                mod[(chrm, strand)] = np.concatenate([m, [n + 5, n + 90]])
            unmod[(chrm, strand)] = np.concatenate([u, [m[0]] if m.shape[0] else []]).astype(np.int64)
    return mod, unmod


# ---- cases ----------------------------------------------------------------------------
# path, motif descriptions, per-site, seeds (genome, stats, ctrl/locs), stats_per_block,
# total_stats_limit, rng seed for the subsampling, ctrl get_reg_stats None every k calls
CASES = [
    dict(name='motif_read', path='motif', descs='CG:1:cpg::GATC:2:dam', per_site=False, seed=11),
    dict(name='motif_site', path='motif', descs='CCWGG:2:dcm', per_site=True, seed=12),
    dict(name='motif_spb', path='motif', descs='CG:1:cpg::GATC:2:dam', per_site=False, seed=13,
         stats_per_block=5, rng_seed=2024),
    dict(name='motif_limit', path='motif', descs='CG:1:cpg::GATC:2:dam', per_site=False, seed=14,
         total_stats_limit=700),
    dict(name='motif_allc', path='motif', descs='C:1:allc::CG:1:cpg', per_site=True, seed=15),
    dict(name='motif_minus_end', path='motif', descs='GATC:3:g3', per_site=False, seed=16,
         edge='minus_end_shift'),
    dict(name='motif_err_start', path='motif', descs='CG:1:cpg::GATC:2:dam', per_site=False, seed=17,
         edge='plus_start'),
    dict(name='motif_err_end', path='motif', descs='GATC:3:g3', per_site=False, seed=18,
         edge='minus_end_short'),
    dict(name='truth_read', path='truth', per_site=False, seed=21),
    dict(name='truth_site', path='truth', per_site=True, seed=22),
    dict(name='truth_allfalse', path='truth', per_site=False, seed=23, no_mod=True),
    dict(name='ctrl_read', path='ctrl', descs='CG:1:cpg::GATC:2:dam::CC:1:cc', per_site=False,
         seed=31, none_every=4),
    dict(name='ctrl_limit', path='ctrl', descs='CG:1:cpg::CC:1:cc', per_site=False, seed=32,
         total_stats_limit=500),
    dict(name='ctrl_alltrue', path='ctrl', descs='GATC:2:dam', per_site=True, seed=33, none_every=1),
]


def parse_descs(th, descs):
    """the case's motif descriptions through ``th.parse_motif_descs``"""
    return th.parse_motif_descs(descs)


def build_case(c):
    """(stats, genome, extra) of a case; extra is the ctrl stats or the ground truth"""
    genome = make_genome(c['seed'])
    blocks = make_blocks(c['seed'] + 100, per_site=c['per_site'])
    slot = 'damp_frac' if c['per_site'] else 'stat'
    edge = c.get('edge')
    if edge:
        # one more block at the chromosome edge, first in iteration order
        n = dict(CHRMS)['chr2']
        if edge == 'plus_start':
            pos, strand, start, end = [3, 0, 5], '+', 0, 10
        elif edge == 'minus_end_short':
            pos, strand, start, end = [n - 4, n - 1], '-', n - 10, n
        else:
            pos, strand, start, end = [n - 2, n - 3, n - 2, n - 5], '-', n - 10, n
        b = np.zeros(len(pos), dtype=PER_READ_DT)
        b['pos'] = pos
        b['stat'] = [0.5, -0.25, 1.0, 0.0][:len(pos)]
        blocks = [('chr2', strand, start, end, b)] + blocks
    extra = None
    if c['path'] == 'ctrl':
        ctrl_blocks = make_blocks(c['seed'] + 200, per_site=c['per_site'], cov=1.5)
        extra = CtrlStats(ctrl_blocks, c.get('none_every', 0))
    elif c['path'] == 'truth':
        mod, unmod = make_locs(c['seed'] + 300, genome)
        extra = ({} if c.get('no_mod') else mod, unmod, 'truth')
    return Stats(blocks, slot), genome, extra


# ---- restatement ------------------------------------------------------------------------
def _codes(s):
    t = np.full(256, 4, dtype=np.int64)
    for i, b in enumerate('ACGT'):
        t[ord(b)] = i
    return t[np.frombuffer(s.encode(), dtype=np.uint8)]


def _class_bits(letter):
    return np.array([b in IUPAC_SETS[letter] for b in 'ACGT'] + [False])


def motif_stats(stats, motif_descs, genome_index, stats_per_block=None, total_stats_limit=None):
    """_compute_motif_stats vectorised per block -> ({name: (stats, labels)}, error or None)"""
    names = list(dict.fromkeys(n for _, n in motif_descs))
    out = {n: ([], []) for n in names}
    bb = max(m.mod_pos for m, _ in motif_descs) - 1
    ab = max(m.motif_len - m.mod_pos for m, _ in motif_descs)
    total = 0
    for chrm, strand, start, end, bs in stats:
        seq_start = max(start - bb, 0) if strand == '+' else max(start - ab, 0)
        seq_end = end + ab if strand == '+' else end + bb
        codes = _codes(genome_index.get_seq(chrm, seq_start, seq_end, error_end=False))
        L = codes.shape[0]
        if stats_per_block is not None and bs.shape[0] > stats_per_block:
            bs = bs[np.random.choice(bs.shape[0], stats_per_block, replace=False)]
        total += bs.shape[0]
        r = bs['pos'].astype(np.int64) - seq_start
        lo, hi = (r - bb, r + ab + 1) if strand == '+' else (r - ab, r + bb + 1)
        wend = np.minimum(hi, L)
        wlen = np.maximum(wend - lo, 0)
        if np.any((lo < 0) | (wlen <= bb)):
            return None, 'IndexError'

        def win(k):                     # window character k of every statistic (4 outside)
            k = np.asarray(k)
            ok = k < wlen
            if strand == '+':
                idx = np.where(ok, lo + k, 0)
                c = codes[idx]
            else:
                idx = np.where(ok, wend - 1 - k, 0)
                c = codes[idx]
                c = np.where(c < 4, 3 - c, c)
            return np.where(ok, c, 4)
        base = win(bb)
        keep = np.zeros((bs.shape[0], len(motif_descs)), dtype=bool)
        lab = np.zeros_like(keep)
        for m, (motif, _) in enumerate(motif_descs):
            keep[:, m] = base == 'ACGT'.index(motif.mod_base)
            hit = np.ones(bs.shape[0], dtype=bool)
            s = bb - motif.mod_pos + 1
            for j, letter in enumerate(motif.raw_motif):
                hit &= _class_bits(letter)[win(s + j)]
            lab[:, m] = hit
        vals = bs[stats._stat_slot]
        for name in names:
            cols = [m for m, (_, n) in enumerate(motif_descs) if n == name]
            k, l = keep[:, cols], lab[:, cols]
            out[name][0].append(np.repeat(vals, k.sum(1)))
            out[name][1].append(l[k])
        if total_stats_limit is not None and total >= total_stats_limit:
            break
    return {n: (np.concatenate(v[0]) if v[0] else np.zeros(0),
                np.concatenate(v[1]) if v[1] else np.zeros(0, dtype=bool)) for n, v in out.items()}, None


def truth_stats(stats, ground_truth_locs):
    mod_locs, unmod_locs, mod_name = ground_truth_locs
    st, lab = [], []
    for chrm, strand, start, end, bs in stats:
        m = np.asarray(mod_locs.get((chrm, strand), []), dtype=np.int64)
        u = np.asarray(unmod_locs.get((chrm, strand), []), dtype=np.int64)
        m, u = m[(m >= start) & (m < end)], u[(u >= start) & (u < end)]
        sel = np.isin(bs['pos'], np.concatenate([m, u]))
        st.append(bs[stats._stat_slot][sel])
        lab.append(np.isin(bs['pos'][sel], m))
    return {mod_name: (np.concatenate(st) if st else np.zeros(0),
                       np.concatenate(lab) if lab else np.zeros(0, dtype=bool))}


def _rc_pattern(raw):
    return ''.join(IUPAC[COMP.get(x, x)] if x in 'ACGT' else
                   '[' + ''.join(sorted(COMP[b] for b in IUPAC_SETS[x])) + ']'
                   for x in raw[::-1])


def ctrl_stats_of(stats, ctrl_stats, motif_descs, genome_index, total_stats_limit=None):
    names = list(dict.fromkeys(n for _, n in motif_descs))
    out = {n: ([], []) for n in names}
    bb = max(m.mod_pos for m, _ in motif_descs) - 1
    ab = max(m.motif_len - m.mod_pos for m, _ in motif_descs)
    total = 0
    for chrm, strand, start, end, bs in stats:
        seq_start = max(start - bb, 0) if strand == '+' else max(start - ab, 0)
        seq_end = end + ab if strand == '+' else end + bb
        reg_seq = genome_index.get_seq(chrm, seq_start, seq_end, error_end=False)
        cbs = ctrl_stats.get_reg_stats(chrm, strand, start, end)
        for motif, name in motif_descs:
            if strand == '+':
                pat = ''.join(IUPAC[x] for x in motif.raw_motif)
                sites = [m.start() + motif.mod_pos - 1 for m in re.finditer(pat, reg_seq)]
            else:
                sites = [m.start() + motif.motif_len - motif.mod_pos
                         for m in re.finditer(_rc_pattern(motif.raw_motif), reg_seq)]
            sites = np.array(sites, dtype=np.int64) + seq_start
            sel = np.isin(bs['pos'], sites)
            out[name][0].append(bs[stats._stat_slot][sel])
            out[name][1].append(np.ones(int(sel.sum()), dtype=bool))
            total += int(sel.sum())
            if cbs is not None:
                csel = np.isin(cbs['pos'], sites)
                out[name][0].append(cbs[stats._stat_slot][csel])
                out[name][1].append(np.zeros(int(csel.sum()), dtype=bool))
                total += int(csel.sum())
        if total_stats_limit is not None and total >= total_stats_limit:
            break
    return {n: (np.concatenate(v[0]) if v[0] else np.zeros(0),
                np.concatenate(v[1]) if v[1] else np.zeros(0, dtype=bool)) for n, v in out.items()}


def ordered_labels(st, lab):
    """Python's (stat, bool) tuple order: stat ascending (-0.0 == 0.0), False before True"""
    return np.asarray(lab, dtype=bool)[np.lexsort((lab, st))]


def accuracy_rates(ordered, num_plot_points=ROC_PLOT_POINTS):
    """compute_accuracy_rates in the reference's numpy expressions"""
    with np.errstate(invalid='ignore', divide='ignore'):
        tp_cumsum = np.cumsum(ordered)
        tp_rate = tp_cumsum / tp_cumsum[-1]
        fp_cumsum = np.cumsum(np.logical_not(ordered))
        fp_rate = fp_cumsum / fp_cumsum[-1]
        precision = tp_cumsum / np.arange(1, len(ordered) + 1, dtype=float)
    n = tp_rate.shape[0]
    return (tp_rate[np.linspace(0, n - 1, num_plot_points).astype(np.int64)],
            fp_rate[np.linspace(0, n - 1, num_plot_points).astype(np.int64)],
            precision[np.linspace(0, n - 1, num_plot_points + 1).astype(np.int64)][1:])


def auc(tp_rate, fp_rate):
    return np.sum(tp_rate[:-1] * (fp_rate[1:] - fp_rate[:-1]))


def mean_ap(tp_rate, precision):
    return np.sum(np.diff(np.concatenate([[0, ], tp_rate, [1, ]]), ) *
                  np.concatenate([[0, ], precision, [1, ]])[:-1])


def curve(st, lab, num_plot_points=ROC_PLOT_POINTS):
    tp, fp, prec = accuracy_rates(ordered_labels(st, lab), num_plot_points)
    return tp, fp, prec, auc(tp, fp), mean_ap(tp, prec)


def run_case(c, th):
    """restated labelling of case ``c`` -> ({name: (stats, labels)}, error or None)"""
    stats, genome, extra = build_case(c)
    if c['path'] == 'truth':
        return truth_stats(stats, extra), None
    descs = parse_descs(th, c['descs'])
    if c['path'] == 'ctrl':
        return ctrl_stats_of(stats, extra, descs, genome, c.get('total_stats_limit')), None
    if c.get('rng_seed') is not None:
        np.random.seed(c['rng_seed'])
    return motif_stats(stats, descs, genome, c.get('stats_per_block'), c.get('total_stats_limit'))
