"""Plain numpy / scipy restatement of the per-read tests behind compute_reg_stats (helper
module of test_reg_stats_cpu.py / test_reg_stats_gpu.py and the golden generator, no pytest
here): the de novo clip / k-mer lookup / z / p / Fisher path (compute_de_novo_read_stats
tombo_stats.py:3771-3873) and the sample-compare path (:3675-3769), written step by step
with the reference's own slicing.  Also the synthetic region data the goldens are built from.
"""
import numpy as np
from scipy import stats

SMALLEST_PVAL = 1e-50
NO_INFO = 'Read does not contain information in this region.'
FISHER_SHORT = "P-values vector too short for Fisher's Method window compuation."
NO_VALID_Z = 'No valid z-scores in read.'
INVALID_SEQ = 'Invalid sequence encountered from genome sequence.'
STATUS_MSG = {0: '', 23: NO_INFO, 24: FISHER_SHORT, 25: NO_VALID_Z, 203: INVALID_SEQ}


class CaseError(Exception):
    pass


def window_fisher(pvals, lag):
    """calc_window_fishers_method :2252-2271"""
    width = lag * 2 + 1
    if pvals.shape[-1] < width:
        raise CaseError(FISHER_SHORT)
    with np.errstate(invalid='ignore'):
        pvals = np.maximum(pvals, SMALLEST_PVAL)
    log_sums = np.lib.stride_tricks.sliding_window_view(np.log(pvals), width).sum(-1)
    f = np.full(pvals.shape, np.nan)
    with np.errstate(invalid='ignore'):
        f[lag:-lag] = stats.chi2.sf(log_sums * -2, width * 2)
    return f


def de_novo(means, bases, start, end, strand, kmer_means, kmer_sds, K, cpos, fm, reg_start,
            reg_end):
    """one read -> (p-values, positions); bases are read-centric codes (0..3, other = invalid);
    kmer_means / kmer_sds are indexed by the base-4 k-mer code"""
    dn = K - cpos - 1
    begin_lag, end_lag = (cpos, dn) if strand == '+' else (dn, cpos)
    r_means, r_seq = np.asarray(means, dtype=np.float64), np.asarray(bases)
    if start + begin_lag + fm < reg_start:
        clip = reg_start - (start + begin_lag + fm)
        start = reg_start - begin_lag - fm
        r_means, r_seq = (r_means[clip:], r_seq[clip:]) if strand == '+' else \
            (r_means[:-clip], r_seq[:-clip])
    if end - end_lag - fm > reg_end:
        clip = (end - end_lag - fm) - reg_end
        end = reg_end + end_lag + fm
        r_means, r_seq = (r_means[:-clip], r_seq[:-clip]) if strand == '+' else \
            (r_means[clip:], r_seq[clip:])
    if len(r_seq) < K:
        raise CaseError(NO_INFO)
    n = len(r_seq) - K + 1
    if (r_seq > 3).any():
        raise CaseError(INVALID_SEQ)
    codes = np.zeros(n, dtype=np.int64)
    for j in range(K):
        codes = codes * 4 + r_seq[j:j + n]
    if strand == '-':
        codes = codes[::-1]
        r_means = r_means[::-1]
    ref_m, ref_s = kmer_means[codes], kmer_sds[codes]
    if np.isnan(ref_m).any():
        raise CaseError(INVALID_SEQ)
    r_means = r_means[begin_lag:-end_lag] if end_lag else r_means[:0]
    start += begin_lag
    end -= end_lag
    with np.errstate(all='ignore'):
        p = stats.norm.cdf(-(np.abs(r_means - ref_m) / ref_s)) * 2.0
    if fm > 0:
        p = window_fisher(p, fm)
    with np.errstate(invalid='ignore'):
        p = np.maximum(p, SMALLEST_PVAL)
    return p, np.arange(start, end)


def sample_compare(means, start, end, strand, ctrl_means, ctrl_sds, fm, reg_start, reg_end):
    """one read -> (non-NaN p-values, positions); ctrl_* cover [reg_start - fm, reg_end + fm)"""
    r_means = np.asarray(means, dtype=np.float64)
    if start + fm < reg_start:
        clip = reg_start - (start + fm)
        start = reg_start - fm
        r_means = r_means[clip:] if strand == '+' else r_means[:-clip]
    if end - fm > reg_end:
        clip = (end - fm) - reg_end
        end = reg_end + fm
        r_means = r_means[:-clip] if strand == '+' else r_means[clip:]
    if strand == '-':
        r_means = r_means[::-1]
    a, b = start - reg_start + fm, end - reg_start + fm
    with np.errstate(all='ignore'):
        z = np.abs(r_means - ctrl_means[a:b]) / ctrl_sds[a:b]
    if np.sum(~np.isnan(z)) == 0:
        raise CaseError(NO_VALID_Z)
    with np.errstate(all='ignore'):
        p = stats.norm.cdf(-z) * 2.0
    if fm > 0:
        p = window_fisher(p, fm)
    keep = np.where(~np.isnan(p))[0]
    return p[keep], keep + start


def near_threshold(v, thresh, lower, llr=False, rel=1e-6):
    """a statistic within rel of a threshold (counts could flip under a 1e-7 tolerance)"""
    v = np.asarray(v, dtype=np.float64)
    v = v[~np.isnan(v)]
    ts = [thresh] + ([] if lower is None else [lower]) + ([-thresh] if llr else [])
    return any(bool((np.abs(v - t) <= rel * abs(t)).any()) for t in ts)


def golden_read(g, i):
    """read i of tests/golden/reg_stats.npz as a dict (start, end, strand, means, bases)"""
    a, b = int(g['reads_off'][i]), int(g['reads_off'][i + 1])
    return dict(start=int(g['reads_start'][i]), end=int(g['reads_end'][i]),
                strand='+-'[int(g['reads_strand'][i])], means=g['reads_means'][a:b],
                bases=g['reads_bases'][a:b].astype(np.int64))


def golden_settings(g, k):
    """(stat_type, region index, fm_offset, min_test_reads, thresh, lower, prior) of call k"""
    st, reg, fm, mtr, thresh, lower, prior = [str(x) for x in g['q%d_settings' % k]]
    return (st, int(reg), int(fm), int(mtr), float(thresh),
            None if lower == 'None' else float(lower), prior == '1')


def golden_results(g, k):
    """the reference's per-read results of call k: one (message, p-values, positions) per read
    of the region, ('', ...) for a read without error"""
    src = int(g['q%d_same_as' % k]) if 'q%d_same_as' % k in g else k
    msgs, off = g['q%d_read_msgs' % src], g['q%d_res_off' % src]
    pv, pos = g['q%d_res_pvals' % src], g['q%d_res_pos' % src]
    return [(str(m), pv[off[j]:off[j + 1]], pos[off[j]:off[j + 1]]) for j, m in enumerate(msgs)]


def golden_block(g, k):
    """the per-read block collate_reg_stats queues for de novo / sample-compare call k:
    (positions, statistics, read indices) of the non-NaN results in read order"""
    pos, stat, read = [], [], []
    for i, (msg, pv, ps) in zip(g['q%d_reads' % k], golden_results(g, k)):
        if msg:
            continue
        keep = ~np.isnan(pv)
        pos.append(ps[keep])
        stat.append(pv[keep])
        read.append(np.full(int(keep.sum()), i, dtype=np.int64))
    if not pos:
        return np.zeros(0, np.int64), np.zeros(0), np.zeros(0, np.int64)
    return np.concatenate(pos), np.concatenate(stat), np.concatenate(read)


def _rev_comp(codes):
    return (3 - codes)[::-1]


def make_dataset(seed, kmer_ref, cpos, regions):
    """(genome, sample reads, control reads, regions).  Reads are dicts with start, end,
    strand, read-centric means and base codes; levels follow the model with a shift at a
    few positions, so some p-values are small.  Every region gets reads on both strands that
    are clipped at the start, at the end, at both ends, not at all, reach it only through the
    lag margins, or are too short in it."""
    rs = np.random.RandomState(seed)
    K = len(kmer_ref[0][0])
    kmeans = np.full(4 ** K, np.nan)
    for k, m, _ in kmer_ref:
        c = 0
        for b in k:
            c = c * 4 + 'ACGT'.index(b)
        kmeans[c] = m
    glen = max(e for _, e in regions) + 400
    genome = rs.randint(0, 4, glen)
    shift = np.zeros(glen)
    shift[rs.choice(glen, glen // 25, replace=False)] = rs.choice([-1.5, 1.5], glen // 25)

    def read(a, b, strand, noise, ctrl=False):
        g = genome[a:b]
        bases = g if strand == '+' else _rev_comp(g)
        nb = b - a
        m = rs.normal(0.0, noise, nb)
        n = nb - K + 1
        if n > 0:
            codes = np.zeros(n, dtype=np.int64)
            for j in range(K):
                codes = codes * 4 + bases[j:j + n]
            m[cpos:cpos + n] += kmeans[codes]
        # genome-ordered shift at the modified positions (sample reads only)
        gs = np.zeros(nb) if ctrl else shift[a:b]
        m += gs if strand == '+' else gs[::-1]
        return dict(start=a, end=b, strand=strand, means=m, bases=bases.astype(np.int64))

    reads, ctrl = [], []
    for s, e in regions:
        for _ in range(16):
            a = int(rs.randint(s - 120, e + 20))
            b = a + int(rs.randint(3, 160))
            reads.append(read(a, b, '+-'[rs.randint(2)], 0.25))
        for strand in '+-':
            reads.append(read(s - 200, e + 200, strand, 0.25))     # clipped at both ends
            reads.append(read(s + 10, e - 10, strand, 0.25))       # whole
            reads.append(read(s - 50, s + 40, strand, 0.25))       # clipped at the start
            reads.append(read(e - 40, e + 50, strand, 0.25))       # clipped at the end
            reads.append(read(s - 30, s + 2, strand, 0.25))        # reaches it through the lags
            reads.append(read(e - 1, e + 30, strand, 0.25))
            reads.append(read(s + 5, s + 5 + K - 1, strand, 0.25))  # too short
        for _ in range(8):
            a = int(rs.randint(s - 60, s + 20))
            b = int(rs.randint(max(a + 30, e - 20), e + 60))
            ctrl.append(read(a, b, '+-'[rs.randint(2)], 0.25, ctrl=True))
    gstr = ''.join('ACGT'[c] for c in genome)
    return gstr, reads, ctrl, regions
