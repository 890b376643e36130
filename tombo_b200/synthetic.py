"""Synthetic k-mer models and reads for parity tests and the benchmark.

Definition follows SURVEY.md section 8(d):

* DNA model: all 4**6 6-mers, ``central_pos=2``; level ~ N(0, 1.4826**2) so
  that the level MAD over random sequence is ~1 (Tombo models live in
  median/MAD-normalised units), sd = 0.2 for every k-mer (one global SD).
* RNA model: all 4**5 5-mers, ``central_pos=1``, sd = 0.25.
* Alt (5mC) model: every (kmer, pos) with ``kmer[pos] == 'C'``;
  level = canonical + N(0, 0.3**2), same sd, ``alt_base='C'``.
* Read: uniform random ACGT of ``B + K - 1`` bases; dwell per base
  ``min_obs + Geometric(1 / (mean_dwell - min_obs))``; sample = level +
  sd * N(0, 1); a leader of N(0, 1) samples is prepended; raw = signal * scale +
  offset.  The primary parity set keeps raw as float64 (tie free), the secondary
  set rounds to int16 (see ``tie_rule`` in DESIGN.md).

Everything is drawn from ``numpy.random.RandomState`` (frozen legacy stream) so a
seed pins the data on every machine.  Only numpy is needed.
"""
from __future__ import annotations

import itertools
from collections import namedtuple

import numpy as np

DNA_KMER, DNA_CENTRAL = 6, 2
RNA_KMER, RNA_CENTRAL = 5, 1

SynthRead = namedtuple(
    'SynthRead', ('raw', 'genome_seq', 'true_starts', 'leader', 'seed'))


def all_kmers(k):
    return [''.join(p) for p in itertools.product('ACGT', repeat=k)]


def make_kmer_ref(kind='DNA', seed=0):
    """Return ``(kmer_ref, central_pos)`` with ``kmer_ref`` a list of
    ``(kmer, mean, sd)`` tuples suitable for ``TomboModel(kmer_ref=...)``."""
    rs = np.random.RandomState(seed)
    if kind == 'DNA':
        k, cpos, sd = DNA_KMER, DNA_CENTRAL, 0.2
    elif kind == 'RNA':
        k, cpos, sd = RNA_KMER, RNA_CENTRAL, 0.25
    else:
        raise ValueError(kind)
    kmers = all_kmers(k)
    means = rs.normal(0.0, 1.4826, len(kmers))
    return [(km, float(m), sd) for km, m in zip(kmers, means)], cpos


def make_alt_kmer_ref(kmer_ref, alt_base='C', seed=1, delta_sd=0.3):
    """Alternative-base model rows ``(kmer, pos, mean, sd)`` for every k-mer
    position holding ``alt_base``."""
    rs = np.random.RandomState(seed)
    rows = []
    for km, m, sd in kmer_ref:
        for pos, b in enumerate(km):
            if b == alt_base:
                rows.append((km, pos, float(m + rs.normal(0.0, delta_sd)), sd))
    return rows


def kmer_table(kmer_ref):
    """Dense level tables indexed by the base-4 k-mer code (A=0,C=1,G=2,T=3)."""
    k = len(kmer_ref[0][0])
    means = np.full(4 ** k, np.nan)
    sds = np.full(4 ** k, np.nan)
    code = {'A': 0, 'C': 1, 'G': 2, 'T': 3}
    for km, m, sd in kmer_ref:
        idx = 0
        for b in km:
            idx = idx * 4 + code[b]
        means[idx] = m
        sds[idx] = sd
    return means, sds


def make_read(kmer_ref, central_pos, n_bases, seed, kind='DNA', leader=None,
              scale=None, offset=480.0, int16=False, stall=None):
    """One synthetic read.  ``stall=(base_idx, n_extra)`` plants ``n_extra``
    additional samples on one base (drives the adaptive band off the path, used
    to exercise the save-bandwidth rescue)."""
    rs = np.random.RandomState(seed)
    k = len(kmer_ref[0][0])
    means, sds = kmer_table(kmer_ref)
    if kind == 'DNA':
        min_obs, mean_dwell = 3, 9
        leader = 150 if leader is None else leader
        scale = 60.0 if scale is None else scale
    else:
        min_obs, mean_dwell = 6, 30
        leader = 300 if leader is None else leader
        scale = 100.0 if scale is None else scale
    codes = rs.randint(0, 4, n_bases + k - 1)
    seq = ''.join('ACGT'[c] for c in codes)
    kidx = np.zeros(n_bases, dtype=np.int64)
    for j in range(k):
        kidx = kidx * 4 + codes[j:j + n_bases]
    dwell = min_obs + rs.geometric(1.0 / (mean_dwell - min_obs), n_bases)
    if stall is not None:
        dwell[stall[0]] += stall[1]
    lev = np.repeat(means[kidx], dwell)
    sd = np.repeat(sds[kidx], dwell)
    sig = lev + sd * rs.normal(0.0, 1.0, lev.shape[0])
    lead = rs.normal(0.0, 1.0, leader)
    sig = np.concatenate([lead, sig])
    raw = sig * scale + offset
    if int16:
        raw = np.round(raw).astype(np.int16)
    true_starts = leader + np.concatenate([[0], np.cumsum(dwell)])
    if kind == 'RNA':
        # RNA signal is stored 3'->5'; the worker flips it before resquiggle
        raw = raw[::-1].copy()
    return SynthRead(raw, seq, true_starts, leader, seed)


def make_reads(kmer_ref, central_pos, n_reads, n_bases, seed0=1000, **kw):
    if np.isscalar(n_bases):
        n_bases = [int(n_bases)] * n_reads
    return [make_read(kmer_ref, central_pos, int(nb), seed0 + i, **kw)
            for i, nb in enumerate(n_bases)]


def bases_for_samples(n_samples, kind='DNA'):
    """Mapped bases giving ~n_samples raw samples (excluding the leader)."""
    return max(8, int(round(n_samples / (9.0 if kind == 'DNA' else 30.0))))


# --------------------------------------------------------------------------
# Fast vectorised bulk generator (benchmark sized sets, e.g. 100k reads)
# --------------------------------------------------------------------------
def make_read_batch(kmer_ref, n_reads, n_bases, seed, kind='DNA', int16=False,
                    leader=None, scale=None, offset=480.0, stall_every=0, stall_extra=0):
    """Generate ``n_reads`` reads at once.

    Returns ``(raw_flat, raw_off, seq_codes_flat, seq_off)``: raw signal
    concatenated (float64 or int16), int64 offsets (n_reads+1), base codes
    (uint8, A=0..T=3) concatenated with ``B + K - 1`` codes per read, and their
    offsets.  ``n_bases`` may be a scalar or an int array of per-read sizes.
    """
    rs = np.random.RandomState(seed)
    k = len(kmer_ref[0][0])
    means, sds = kmer_table(kmer_ref)
    if kind == 'DNA':
        min_obs, mean_dwell = 3, 9
        leader = 150 if leader is None else leader
        scale = 60.0 if scale is None else scale
    else:
        min_obs, mean_dwell = 6, 30
        leader = 300 if leader is None else leader
        scale = 100.0 if scale is None else scale
    nb = np.broadcast_to(np.asarray(n_bases, dtype=np.int64), (n_reads,))
    seq_len = nb + k - 1
    seq_off = np.concatenate([[0], np.cumsum(seq_len)]).astype(np.int64)
    codes = rs.randint(0, 4, int(seq_off[-1])).astype(np.uint8)
    base_off = np.concatenate([[0], np.cumsum(nb)]).astype(np.int64)
    # position of every base's first k-mer code in the flat code array
    read_of_base = np.repeat(np.arange(n_reads), nb)
    first = seq_off[read_of_base] + (np.arange(base_off[-1]) -
                                     base_off[read_of_base])
    kidx = np.zeros(int(base_off[-1]), dtype=np.int64)
    for j in range(k):
        kidx = kidx * 4 + codes[first + j]
    dwell = min_obs + rs.geometric(1.0 / (mean_dwell - min_obs),
                                   int(base_off[-1]))
    if stall_every and stall_extra:
        sel = np.arange(stall_every - 1, n_reads, stall_every)
        dwell[base_off[sel] + nb[sel] // 2] += int(stall_extra)
    sig_per_read = np.add.reduceat(dwell, base_off[:-1]) + leader
    raw_off = np.concatenate([[0], np.cumsum(sig_per_read)]).astype(np.int64)
    total = int(raw_off[-1])
    sig = rs.normal(0.0, 1.0, total)
    # scatter levels: sample i of base b -> level[b] + sd[b] * noise
    base_sig_start = raw_off[read_of_base] + leader + (
        np.cumsum(dwell) - dwell - np.repeat(
            (np.cumsum(dwell) - dwell)[base_off[:-1]], nb))
    lev = np.zeros(total)
    sdv = np.ones(total)
    idx = np.repeat(base_sig_start, dwell) + (
        np.arange(int(dwell.sum())) - np.repeat(np.cumsum(dwell) - dwell, dwell))
    lev[idx] = np.repeat(means[kidx], dwell)
    sdv[idx] = np.repeat(sds[kidx], dwell)
    raw = (lev + sdv * sig) * scale + offset
    if kind == 'RNA':
        # stored reversed per read
        out = np.empty_like(raw)
        for r in range(n_reads):
            out[raw_off[r]:raw_off[r + 1]] = raw[raw_off[r]:raw_off[r + 1]][::-1]
        raw = out
    if int16:
        raw = np.round(raw).astype(np.int16)
    return raw, raw_off, codes, seq_off


def codes_to_seq(codes):
    return ''.join('ACGT'[c] for c in codes)


def seq_to_codes(seq):
    lut = np.full(256, 255, dtype=np.uint8)
    for i, b in enumerate('ACGT'):
        lut[ord(b)] = i
    return lut[np.frombuffer(seq.encode(), dtype=np.uint8)]


# --------------------------------------------------------------------------
# Theil-Sen sub-sampling (reads with > MAX_POINTS_FOR_THEIL_SEN bases)
# --------------------------------------------------------------------------
# The reference draws ``np.random.choice(n, 1000, replace=False)`` from the
# unseeded global RNG (tombo_stats.py:411-416): it is not reproducible.  This
# framework pins the draw to a keyed bijection on [0, n) that is cheap on both
# host and device; the oracle harness injects the same indices into the
# reference (SURVEY.md section 7, hard part 5).
_M32 = 0xFFFFFFFF


def _mix32(x):
    x &= _M32
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & _M32
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & _M32
    x ^= x >> 16
    return x


def subsample_key(seed, read_index, call_index):
    return _mix32(_mix32(seed ^ 0x9E3779B9) + _mix32(read_index * 2654435761 + 1)
                  + call_index * 0x632BE5AB)


def perm_index(i, n, key):
    """Keyed bijection on [0, n) (4-round Feistel + cycle walking)."""
    bits = max(2, int(n - 1).bit_length())
    half = (bits + 1) // 2
    mask = (1 << half) - 1
    x = i
    while True:
        left, right = x >> half, x & mask
        for rnd in range(4):
            f = _mix32(right ^ key ^ ((rnd * 0x9E3779B9) & _M32)) & mask
            left, right = right, left ^ f
        x = (left << half) | right
        if x < n:
            return x


def theil_sen_subsample(n, n_points, key):
    """Indices standing in for ``np.random.choice(n, n_points, False)``."""
    return np.array([perm_index(i, n, key) for i in range(n_points)],
                    dtype=np.int64)


def make_event_model(kmer_width, seed=0, sd=0.2):
    """A ``kmer_ref`` of all ``4**kmer_width`` k-mers with levels ~ N(0, 1) and one sd."""
    rs = np.random.RandomState(seed)
    kmers = all_kmers(kmer_width)
    return [(km, float(m), sd) for km, m in zip(kmers, rs.normal(0.0, 1.0, len(kmers)))]


def make_event_read(kmer_ref, central_pos, n_bases, seed, alt_base=None, alt_frac=0.0,
                    alt_shift=0.0, noise_sd=0.15, shift=0.0):
    """One resquiggled read as its Events columns ``(norm_mean, base)``: uniform random
    bases; the level of base b is the model level of the k-mer centred on it (``central_pos``
    bases before b) plus ``alt_shift`` per modified base in that k-mer, plus
    N(0, noise_sd**2), plus ``shift`` for every base.  With ``alt_base``, each such base is modified with probability
    ``alt_frac``.  Bases without a whole k-mer around them get the noise only."""
    rs = np.random.RandomState(seed)
    k = len(kmer_ref[0][0])
    means, _ = kmer_table(kmer_ref)
    codes = rs.randint(0, 4, n_bases)
    mod = np.zeros(n_bases, dtype=bool)
    if alt_base is not None:
        mod = (codes == 'ACGT'.index(alt_base)) & (rs.uniform(size=n_bases) < alt_frac)
    level = rs.normal(0.0, noise_sd, n_bases) + shift
    nk = max(n_bases - k + 1, 0)
    kidx = np.zeros(nk, dtype=np.int64)
    n_mod = np.zeros(nk)
    for j in range(k):
        kidx = kidx * 4 + codes[j:j + nk]
        n_mod += mod[j:j + nk]
    level[central_pos:central_pos + nk] += means[kidx] + alt_shift * n_mod
    base = np.frombuffer(codes_to_seq(codes).encode(), dtype='S1')
    return level, base
