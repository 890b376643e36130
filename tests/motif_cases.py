"""Plain restatement of compute_alt_model_read_stats for motif models, both strands and a
region (helper module of test_motif_llr_cpu.py / test_motif_llr_gpu.py, no pytest here).

It follows the reference's own string slicing step by step (trim_seq_and_means
tombo_stats.py:3888-3970, the per-model search window and re.finditer :4040-4050), on reads
in the library's layout: read r has nb per-base means and nb + K - 1 base codes, its nb
read-centric bases S at codes cpos .. cpos + nb - 1.  The per-site scores are
stats_cases.score_window, so stats_cases.llr_bound holds the device to them.

Seeded case families for the site finder and the region clip are at the end."""
import re

import numpy as np

import stats_cases as sc

SINGLE_LETTER_CODE = {
    'A': 'A', 'C': 'C', 'G': 'G', 'T': 'T', 'B': '[CGT]', 'D': '[AGT]', 'H': '[ACT]',
    'K': '[GT]', 'M': '[AC]', 'N': '[ACGT]', 'R': '[AG]', 'S': '[CG]', 'V': '[ACG]',
    'W': '[AT]', 'Y': '[CT]'}                 # tombo_helper.py SINGLE_LETTER_CODE
TOO_SHORT = 22                               # TB2_ERR_READ_TOO_SHORT_IN_REGION
TOO_SHORT_MSG = 'Read sequence too short in this region.'
# (raw motif, mod_pos, alternative base) of every family the tests run
MOTIFS = [('C', 1, 'C'), ('A', 1, 'A'), ('CG', 1, 'C'), ('GATC', 2, 'A'), ('CCWGG', 2, 'C'),
          ('AA', 1, 'A'), ('NNNNNNCG', 7, 'C'), ('CNNNNN', 1, 'C')]


def motif_bounds(motifs):
    """(max_motif_bb, max_motif_ab) of one call's models (:4002-4006)"""
    return (max(p - 1 for _, p in motifs), max(len(m) - p for m, p in motifs))


def read_sites(S, means, r_start, strand, reg_start, reg_end, K, cpos, motif, mod_pos,
               max_bb, max_ab):
    """one read, one model: (status, alt_pos list, genome positions, trimmed means, trimmed
    k-mer codes).  S: the read's bases as a string; strand '+' or '-'."""
    nb = means.shape[0]
    r_end = r_start + nb
    clip5 = clip3 = 0
    if r_start + K - 1 < reg_start:
        if strand == '+':
            clip5 = reg_start - (r_start + K - 1)
        else:
            clip3 = reg_start - (r_start + K - 1)
        r_start = reg_start - (K - 1)
    if r_end - K + 1 > reg_end:
        if strand == '+':
            clip3 = r_end - K + 1 - reg_end
        else:
            clip5 = r_end - K + 1 - reg_end
    seq = S[clip5:]
    if clip3 > 0:
        seq = seq[:-clip3]
    m = means[clip5 + cpos:]
    m = m[:-(clip3 + K - cpos - 1)]
    if m.shape[0] < K:
        return TOO_SHORT, [], [], None, None
    codes = sc.kmer_codes(np.array(['ACGT'.index(b) for b in seq], dtype=np.int64), K)
    assert codes.shape[0] == m.shape[0]
    r_start += K - 1
    mss = S
    lead = clip5 + K - 1 - max_bb
    mss = mss[lead:] if lead >= 0 else 'N' * -lead + mss
    trail = clip3 + K - 1 - max_ab
    mss = mss[:-trail] if trail >= 0 else mss + 'N' * -trail
    testable_len = m.shape[0] - K + 1
    search = mss[max_bb - (mod_pos - 1):]
    te = max_ab - (len(motif) - mod_pos)
    if te > 0:
        search = search[:-te]
    pat = re.compile(''.join(SINGLE_LETTER_CODE[c] for c in motif))
    alt_pos = [x.start() for x in pat.finditer(search)]
    if strand == '+':
        gpos = [r_start + a for a in alt_pos]
    else:
        gpos = [r_start + testable_len - a - 1 for a in alt_pos]
    return 0, alt_pos, gpos, m, codes


def motif_llr_reads(norm_mean, mean_off, seq, seq_off, read_start, strand, motif, mod_pos,
                    max_bb, max_ab, reg_start, reg_end, kmeans, ksds, alt, K, cpos, mode,
                    sf=4.0, hf=1.0, hp=0.2):
    """tb2_alt_model_llr_motif_batch restated: strand[r] 0 '+', 1 '-', -1 skip.
    Returns (llr, pos, site_off, S, status)."""
    llr, pos, s_all, off, status = [], [], [], [0], []
    for r in range(mean_off.shape[0] - 1):
        nb = int(mean_off[r + 1] - mean_off[r])
        if strand[r] < 0:
            status.append(0)
            off.append(off[-1])
            continue
        S = ''.join('ACGT'[c & 3] for c in seq[seq_off[r] + cpos:seq_off[r] + cpos + nb])
        st, alt_pos, gpos, m, codes = read_sites(
            S, norm_mean[mean_off[r]:mean_off[r + 1]], int(read_start[r]),
            '+' if strand[r] == 0 else '-', reg_start, reg_end, K, cpos, motif, mod_pos,
            max_bb, max_ab)
        status.append(st)
        for a, g in zip(alt_pos, gpos):
            w = codes[a:a + K]
            sd = float(ksds[w[0]])
            v, s = sc.score_window(mode, m[a:a + K], kmeans[w], alt[w, K - 1 - np.arange(K)],
                                   sd * sd, sf=sf, hf=hf, hp=hp)
            llr.append(v)
            s_all.append(s)
            pos.append(g)
        off.append(off[-1] + len(alt_pos))
    return (np.array(llr, dtype=np.float64), np.array(pos, dtype=np.int64),
            np.array(off, dtype=np.int64), np.array(s_all, dtype=np.float64),
            np.array(status, dtype=np.int32))


def motif_sites(S, r_start, strand, reg_start, reg_end, K, cpos, motif, mod_pos, max_bb, max_ab):
    """(status, genome positions) of one read; the levels do not matter to the site finder"""
    st, _, gpos, _, _ = read_sites(S, np.zeros(len(S)), r_start, strand, reg_start, reg_end,
                                   K, cpos, motif, mod_pos, max_bb, max_ab)
    return st, gpos


def alt_table(kmer_ref, base):
    """(4^K, K) alternative means of the synthetic model for `base`
    (synthetic.make_alt_kmer_ref(kmer_ref, base, seed=1)); NaN where a k-mer has no `base`
    at that position"""
    from tombo_b200 import synthetic as syn
    K = len(kmer_ref[0][0])
    alt = np.full((4 ** K, K), np.nan)
    for km, pos, m, _ in syn.make_alt_kmer_ref(kmer_ref, base, seed=1):
        idx = 0
        for b in km:
            idx = idx * 4 + 'ACGT'.index(b)
        alt[idx, pos] = m
    return alt


def iupac_mask(motif):
    bits = {'A': 1, 'C': 2, 'G': 4, 'T': 8}
    return [sum(bits[b] for b in SINGLE_LETTER_CODE[c].strip('[]')) for c in motif]


# ---------------------------------------------------------------------------
# seeded case families
# ---------------------------------------------------------------------------
def rand_bases(rs, n, motif_rich=None):
    """n read bases; motif_rich plants copies of that (concrete) motif, runs of A included"""
    s = rs.randint(0, 4, n)
    if motif_rich:
        for _ in range(max(1, n // 12)):
            p = rs.randint(0, max(1, n - len(motif_rich)))
            for j, c in enumerate(motif_rich):
                if p + j < n:
                    s[p + j] = 'ACGT'.index(c)
        if rs.uniform() < 0.5 and n > 8:
            p = rs.randint(0, n - 8)
            s[p:p + rs.randint(2, 9)] = 0          # homopolymer run of A
    return s.astype(np.uint8)


def concrete(motif, rs):
    """one sequence that matches an IUPAC motif"""
    return ''.join(rs.choice(list(SINGLE_LETTER_CODE[c].strip('[]'))) for c in motif)


def layout(reads, K, cpos, rs):
    """[(bases, means, start, strand)] -> library arrays; flank codes are random (the
    library must read them as 'N')"""
    nm, mo, sq, so, st, sd = [], [0], [], [0], [], []
    for b, m, start, strand in reads:
        codes = np.concatenate([rs.randint(0, 4, cpos), b, rs.randint(0, 4, K - 1 - cpos)])
        sq.append(codes.astype(np.uint8))
        nm.append(np.asarray(m, dtype=np.float64))
        mo.append(mo[-1] + b.shape[0])
        so.append(so[-1] + codes.shape[0])
        st.append(start)
        sd.append(strand)
    return (np.concatenate(nm) if nm else np.zeros(0), np.array(mo, dtype=np.int64),
            np.concatenate(sq) if sq else np.zeros(0, np.uint8), np.array(so, dtype=np.int64),
            np.array(st, dtype=np.int64), np.array(sd, dtype=np.int8))


def level_means(bases, kmeans, K, cpos, rs, noise=0.3):
    """per-base levels near the model: base i's k-mer starts cpos bases before it (bases
    outside the read are drawn at random)"""
    nb = bases.shape[0]
    ext = np.concatenate([rs.randint(0, 4, cpos), bases, rs.randint(0, 4, K - 1 - cpos)])
    return kmeans[sc.kmer_codes(ext.astype(np.int64), K)][:nb] + rs.normal(0, noise, nb)


def sweep_reads(n, K, cpos, kmeans, seed, nb_lo=1, nb_hi=400, motif=None):
    """n seeded reads of mixed strands (about one in ten skipped) with starts in [0, 5000)"""
    rs = np.random.RandomState(seed)
    reads = []
    for _ in range(n):
        nb = int(rs.randint(nb_lo, nb_hi))
        b = rand_bases(rs, nb, concrete(motif, rs) if motif else None)
        u = rs.uniform()
        strand = -1 if u < 0.1 else (0 if u < 0.55 else 1)
        reads.append((b, level_means(b, kmeans, K, cpos, rs), int(rs.randint(0, 5000)), strand))
    return layout(reads, K, cpos, rs)
