"""One context serves the resident batch and every single-read mirror.  The mirrors work
in buffers of their own, so a resident batch, its LLRs and the region counters come out
bit for bit the same whatever mirror calls run in between, and the mirrors return what
they return on a fresh context."""
import numpy as np
import pytest

from tombo_b200 import _lib, synthetic as syn

pytestmark = pytest.mark.gpu

ALN = (4.2, 4.2, 200, 1500, 20.0, 40, 750, 2500, 250)
K = 6
REG_START, REG_LEN = 10000, 4000


@pytest.fixture(scope='module')
def model():
    kmer_ref, cpos = syn.make_kmer_ref('DNA', 0)
    means, sds = syn.kmer_table(kmer_ref)
    alt = np.full((4 ** K, K), np.nan)
    code = {'A': 0, 'C': 1, 'G': 2, 'T': 3}
    for km, pos, m, _ in syn.make_alt_kmer_ref(kmer_ref, 'C', seed=1):
        idx = 0
        for b in km:
            idx = idx * 4 + code[b]
        alt[idx, pos] = m
    return kmer_ref, cpos, means, sds, alt


def _context(model):
    _, cpos, means, sds, alt = model
    c = _lib.Context(0)
    c.set_model(means, sds, K, cpos)
    c.set_alt_model(alt, K)
    return c


@pytest.fixture(scope='module')
def batch(model):
    """mixed lengths: 120-base reads run the static-band k_align class, 900-base reads the
    general one"""
    kmer_ref = model[0]
    n = 300
    n_bases = np.where(np.arange(n) % 3 == 0, 900, 120)
    raw, raw_off, seq, seq_off = syn.make_read_batch(kmer_ref, n, n_bases, 41)
    raw[raw_off[7]:raw_off[8]] = 480.0          # one hopeless read
    read_start = REG_START + (np.arange(n, dtype=np.int64) * 37) % 3000
    return raw, raw_off, seq, seq_off, read_start


def _levels(genome_seq, means, sds):
    codes = syn.seq_to_codes(genome_seq).astype(np.int64)
    nb = codes.shape[0] - K + 1
    kidx = np.zeros(nb, dtype=np.int64)
    for j in range(K):
        kidx = kidx * 4 + codes[j:j + nb]
    return means[kidx], sds[kidx]


def _ragged(rs, n_reads, reg_len, shift):
    lv, off, start = [], [0], []
    for _ in range(n_reads):
        m = int(rs.randint(50, 400))
        lv.append(rs.normal(shift, 1.0, m))
        off.append(off[-1] + m)
        start.append(int(rs.randint(0, reg_len - 30)))
    return np.concatenate(lv), np.array(off, dtype=np.int64), np.array(start, dtype=np.int64)


def _if_ok(st, *arrays):
    """outputs that a call writes only on success"""
    return [st] + (list(arrays) if st == 0 else [])


def _run_mirrors(ctx, model, rp, batch_res, batch_in, n_theil_sen):
    """every single-read and per-call entry point once; returns their outputs"""
    kmer_ref, cpos, means, sds, _ = model
    out = []
    rs = np.random.RandomState(7)
    read = syn.make_read(kmer_ref, cpos, 1500, 23000)
    rm, rsd = _levels(read.genome_seq, means, sds)
    # stage mirrors
    st, norm, sv = ctx.normalize_raw_signal(read.raw, outlier_thresh=5.0)
    out += [st, norm, np.array(sv)]
    ne = max(read.raw.shape[0] // rp.mean_obs_per_event, int(rm.shape[0] * 1.1))
    st, cpts = ctx.valid_cpts_w_cap(norm, rp.min_obs_per_base, rp.running_stat_width, ne)
    assert st == 0
    em = ctx.new_means(norm, cpts)
    out += [cpts, em]
    # more points than the resident batch has bases
    ev, md = rs.normal(0, 1.4826, n_theil_sen), rs.normal(0, 1.4826, n_theil_sen)
    st, ts = ctx.theil_sen(480.0, 60.0, ev, md, 12345)
    out += [st, np.array(ts)]
    nb = 300
    dwell = 3 + rs.geometric(1 / 6.0, nb)
    dwell[rs.choice(np.arange(5, nb - 5), 12, replace=False)] = 0
    segs = np.concatenate([[0], np.cumsum(dwell)]).astype(np.int64)
    srm = rs.normal(0, 1.4826, nb)
    snorm = np.repeat(srm, dwell) + 0.2 * rs.normal(0, 1, segs[-1])
    out += _if_ok(*ctx.resolve_skipped_bases_with_raw(segs, srm, np.full(nb, 0.2), snorm, rp))
    stall = read.raw.copy()
    stall[3000:3600] = stall[3000] + rs.normal(0, 3, 600)
    out.append(ctx.identify_stalls(stall))
    # DP mirrors
    out += _if_ok(*ctx.find_static_base_assignment(em[:700], rm[:330], rsd[:330], rp))
    out += list(ctx.find_seq_start_in_events(em, rm, rsd, rp, 250, 750, 1.1))
    st, a_segs, rsrtr, dbg = ctx.find_adaptive_base_assignment(cpts, em, rp, rm, rsd)
    out += _if_ok(st, a_segs) + [rsrtr, dbg]
    # banded passes: seed rows of a static pass, then the adaptive rows (test_dp_gpu.py)
    nba, bw, n_ev, ssp = 300, 200, 650, 51
    arm, arsd = rs.normal(0, 1.4826, nba), np.full(nba, 0.2)
    per = np.maximum(1, rs.poisson(n_ev / nba, nba))
    aem = (np.repeat(arm, per) + rs.normal(0, 0.2, per.sum()))[:n_ev]
    z_shift = 4.2 + float(np.sqrt(2 / np.pi))
    es0 = (np.arange(ssp) * (n_ev / nba)).astype(np.int64)
    z0 = np.full((ssp, bw), -15.0)
    for r in range(ssp):
        seg = aem[es0[r]:es0[r] + bw]
        z0[r, :seg.shape[0]] = z_shift - np.minimum(20.0, np.abs(seg - arm[r]) / arsd[r])
    f_seed, t_seed = ctx.banded_forward_pass(z0, es0, 4.2, 4.2)
    out += [f_seed, t_seed]
    fwd, tb = np.zeros((nba + 1, bw)), np.zeros((nba + 1, bw), dtype=np.int64)
    es = np.zeros(nba, dtype=np.int64)
    fwd[:ssp + 1], tb[:ssp + 1], es[:ssp] = f_seed, t_seed, es0
    out.append(ctx.adaptive_banded_forward_pass(fwd, tb, es, aem, arm, arsd, z_shift, 4.2, 4.2,
                                                ssp, -15.0, True, 20.0))
    out += [fwd, tb, es]
    # statistics
    out += list(ctx.new_mean_stds(norm, cpts))
    w = rs.normal(0, 1, (500, K))
    out.append(ctx.calc_llh_ratio_windows(0, w, w + 0.1, w - 0.2, np.full(500, 0.04)))
    seg_off = np.array([0, 200, 700, 1000], dtype=np.int64)
    out.append(ctx.window_fisher_pvals(em[:1000], rm[:1000], rsd[:1000], seg_off, 1, 1))
    samp, ctrl = _ragged(rs, 40, 2000, 0.0), _ragged(rs, 30, 2000, 0.3)
    out += list(ctx.group_reg_stats(5000, 2000, samp, ctrl, 0, False, 5, 1).values())
    out += list(ctx.reads_ref_levels(5000, 2000, samp, 5))
    _, _, seq, seq_off, read_start = batch_in
    out += list(ctx.alt_model_llr_batch(batch_res['norm_mean'], batch_res['base_off'], seq,
                                        seq_off, read_start, 1))
    out += list(ctx.de_novo_read_stats_batch(batch_res['norm_mean'], batch_res['base_off'], seq,
                                             seq_off, read_start))
    return out


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _assert_same_download(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert _same_bits(got[k], want[k]), k


def test_single_read_calls_leave_the_resident_batch_intact(model, batch, RPcls):
    raw, raw_off, seq, seq_off, read_start = batch
    rp, sp = RPcls(ALN), RPcls(ALN, save=True)
    pol = _lib.make_policy('DNA')
    ctx = _context(model)
    try:
        ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
        ctx.batch_compute(rp, sp, pol)
        base = {k: v.copy() for k, v in ctx.batch_download().items()}
        ok = base['status'] == 0
        assert not ok[7] and ok[0::3].sum() >= 50 and ok[1::3].sum() >= 50   # both classes
        ctx.batch_alt_llr(read_start, 1)
        llr_base = [a.copy() for a in ctx.batch_llr_download()]
        assert llr_base[0].shape[0] > 0
        # region counters of a run without interleaved calls
        ctx.region_stats_begin(REG_START, REG_LEN)
        ctx.region_stats_add_batch_llr(2.5, -1.5, 0)
        counts_ref = ctx.region_counts_get()
        fin_ref = ctx.region_stats_finalize(2, 0)
        assert fin_ref['pos'].shape[0] > 0
        ctx.region_stats_begin(REG_START, REG_LEN)
        ctx.region_stats_add_batch_llr(2.5, -1.5, 0)

        mirrors = _run_mirrors(ctx, model, rp, base, batch, int(base['base_off'][-1]) + 1000)

        _assert_same_download(ctx.batch_download(), base)
        ctx.batch_alt_llr(read_start, 1)
        for got, want in zip(ctx.batch_llr_download(), llr_base):
            assert _same_bits(got, want)
        assert _same_bits(ctx.region_counts_get(), counts_ref)
        fin = ctx.region_stats_finalize(2, 0)
        assert sorted(fin) == sorted(fin_ref)
        for k in fin_ref:
            assert _same_bits(fin[k], fin_ref[k]), k
        # "may be repeated on one upload"
        ctx.batch_compute(rp, sp, pol)
        _assert_same_download(ctx.batch_download(), base)
    finally:
        ctx.close()
    # the mirrors do not see the batch either
    fresh = _context(model)
    try:
        alone = _run_mirrors(fresh, model, rp, base, batch, int(base['base_off'][-1]) + 1000)
    finally:
        fresh.close()
    assert len(alone) == len(mirrors)
    for i, (a, b) in enumerate(zip(mirrors, alone)):
        assert _same_bits(a, b), i
