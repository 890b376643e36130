// emul_stage.cpp -- TEST INFRASTRUCTURE ONLY: the stage kernels' device source
// (tombo_b200/csrc/stage_kernels.cuh) run on the host through tests/emul/cuda_emul.h, one
// read at a time, for comparison with the oracle in the CPU test-suite.
#include "cuda_emul.h"
#include "../../tombo_b200/csrc/stage_kernels.cuh"
#include <vector>

extern "C" {

// k_resolve on one read (resolve_skipped_bases_with_raw resquiggle.py:402-540)
int emul_resolve(const int *segs_dp, int nb, const double *rm, const double *rs, const double *norm,
                 int n_norm, const tb2_params *p, long long max_raw_cpts, long long cap_doubles,
                 long long big_cap_doubles, int *segs_out, int *status_out)
{
    BatchView b;
    memset(&b, 0, sizeof(b));
    long long raw_off[2] = {0, n_norm}, base_off[2] = {0, nb};
    ReadState st;
    memset(&st, 0, sizeof(st));
    st.active = 1; st.status = TB2_OK; st.rsrtr = 0;
    std::vector<int> starts(nb + 8), read_tb(nb + 8), sd(segs_dp, segs_dp + nb + 1), so(nb + 1);
    std::vector<double> n2(norm, norm + n_norm), rmv(rm, rm + nb), rsv(rs, rs + nb);
    b.n_reads = 1; b.raw_off = raw_off; b.base_off = base_off;
    b.norm = n2.data(); b.rm = rmv.data(); b.rs = rsv.data();
    b.starts = starts.data(); b.read_tb = read_tb.data();
    b.segs_dp = sd.data(); b.segs = so.data(); b.st = &st;
    StagePolicy pol;
    memset(&pol, 0, sizeof(pol));
    pol.max_raw_cpts = max_raw_cpts;
    std::vector<double> pool((size_t)cap_doubles * 4 + 8), big((size_t)big_cap_doubles + 8);
    int counter[4] = {0, 0, 0, 0};
    emul::launch(emul::Idx3{1, 1, 1}, 128, 0, [&]() {
        k_resolve(b, *p, pol, pool.data(), (size_t)cap_doubles, counter, big.data(),
                  (unsigned long long)big_cap_doubles, (unsigned long long *)(counter + 2));
    });
    for (int i = 0; i <= nb; ++i) segs_out[i] = so[i];
    *status_out = st.status;
    return 0;
}

// k_theil_sen on one read (calc_kmer_fitted_shift_scale tombo_stats.py:370-450)
int emul_theil_sen(const double *bm, const double *rm, int nb, double prev_shift, double prev_scale,
                   unsigned int key, double *out4 /* shift, scale, shc, scc */, int *status_out)
{
    BatchView b;
    memset(&b, 0, sizeof(b));
    long long base_off[2] = {0, nb};
    ReadState st;
    memset(&st, 0, sizeof(st));
    st.active = 1; st.status = TB2_OK;
    st.sv.shift = prev_shift; st.sv.scale = prev_scale;
    std::vector<double> bmv(bm, bm + nb), rmv(rm, rm + nb);
    b.n_reads = 1; b.base_off = base_off; b.bm = bmv.data(); b.rm = rmv.data(); b.st = &st;
    StagePolicy pol;
    memset(&pol, 0, sizeof(pol));
    pol.outlier_thresh = 5.0; pol.subsample_seed = key; pol.literal_key = 1;
    emul::launch(emul::Idx3{1, 1, 1}, ST_THREADS, sizeof(TsSmem), [&]() { k_theil_sen(b, pol, 0); });
    out4[0] = st.sv.shift; out4[1] = st.sv.scale; out4[2] = st.shc; out4[3] = st.scc;
    *status_out = st.status;
    return 0;
}

// k_normalize -> k_cumsum / k_cpts -> k_event_means on one read (first call of
// segment_signal resquiggle.py:1052-1117: normalize_raw_signal tombo_stats.py:482-573,
// c_valid_cpts_w_cap(_t_test) _c_helper.pyx:89-202, c_new_means _c_helper.pyx:59-71,
// remove_stall_cpts tombo_stats.py:1576-1597).  sv_in5 (may be NULL): supplied scale values;
// thresh_with_sv: winsorise them by outlier_thresh as tb2_normalize_raw_signal does.
// stalls (may be NULL): n_stalls (start, end) pairs, as tb2_batch_set_read_inputs stores them.
int emul_segment(const double *raw, int n, const tb2_params *p, int num_events, double outlier_thresh,
                 double const_scale, double *norm_out, double *sv_out5, int *cpts_out, int *n_cpts_out,
                 double *em_out, int *status_out, const double *sv_in5, int thresh_with_sv,
                 const int *stalls, int n_stalls)
{
    BatchView b;
    memset(&b, 0, sizeof(b));
    long long raw_off[2] = {0, n}, ev_off[2] = {0, (long long)num_events + 8};
    ReadState st;
    memset(&st, 0, sizeof(st));
    st.active = 1; st.status = TB2_OK; st.num_events = num_events;
    std::vector<double> rawf(raw, raw + n), norm((size_t)n + 8), cs((size_t)n + 16), scores((size_t)n + 8);
    std::vector<unsigned char> cstate((size_t)2 * n + 1024);
    std::vector<int> cpts((size_t)num_events + 16);
    std::vector<double> em((size_t)num_events + 16);
    b.n_reads = 1; b.max_raw = n; b.raw_off = raw_off; b.ev_off = ev_off;
    b.rawf = rawf.data(); b.norm = norm.data(); b.cs = cs.data(); b.scores = scores.data();
    b.cstate = cstate.data(); b.cpts = cpts.data(); b.em = em.data(); b.st = &st;
    if (sv_in5) {
        st.use_sv = 1;
        st.sv.shift = sv_in5[0]; st.sv.scale = sv_in5[1];
        st.sv.lower_lim = sv_in5[2]; st.sv.upper_lim = sv_in5[3]; st.sv.outlier_thresh = sv_in5[4];
    }
    std::vector<int> si;
    if (stalls) {
        si.assign(stalls, stalls + 2 * n_stalls);
        si.resize((size_t)2 * n_stalls + 2);
        b.stall_ints = si.data(); b.stall_cap = std::max(1, n_stalls); st.n_stalls = n_stalls;
    }
    StagePolicy pol;
    memset(&pol, 0, sizeof(pol));
    pol.outlier_thresh = outlier_thresh; pol.const_scale = const_scale;
    pol.thresh_with_sv = thresh_with_sv;
    emul::launch(emul::Idx3{1, 1, 1}, ST_THREADS, 0, [&]() { k_normalize(b, pol, 1); });
    if (st.status == TB2_OK) {
        if (!p->use_t_test_seg)
            emul::launch(emul::Idx3{1, 1, 1}, CS_WARPS * 32, 0, [&]() { k_cumsum(b, 0); });
        const long long nw = ((long long)n + 32) / 32;
        long long words = (4 + std::max(0, (int)p->min_obs_per_base - 1)) * nw;   // tb2_launch_cpts
        if (words * 4 > 48 * 1024) words = 0;
        emul::launch(emul::Idx3{1, 1, 1}, ST_THREADS, (size_t)words * 4, [&]() { k_cpts(b, *p, 0, (int)words); });
    }
    if (st.status == TB2_OK)
        emul::launch(emul::Idx3{1, 1, 1}, ST_THREADS, 0, [&]() { k_event_means(b); });
    for (int i = 0; i < n; ++i) norm_out[i] = norm[i];
    sv_out5[0] = st.sv.shift; sv_out5[1] = st.sv.scale; sv_out5[2] = st.sv.lower_lim;
    sv_out5[3] = st.sv.upper_lim; sv_out5[4] = st.sv.outlier_thresh;
    *n_cpts_out = st.n_cpts;
    for (int i = 0; i < st.n_cpts && i < num_events + 8; ++i) cpts_out[i] = cpts[i];
    for (int i = 0; i + 1 < st.n_cpts && i < num_events + 8; ++i) em_out[i] = em[i];
    *status_out = st.status;
    return 0;
}

// k_stalls on one read (identify_stalls, mean-window method, tombo_stats.py:269-368)
int emul_stalls(const double *raw, int n, int stall_cap, int *ints_out /* 2 * stall_cap */, int *n_out,
                int *status_out)
{
    BatchView b;
    memset(&b, 0, sizeof(b));
    long long raw_off[2] = {0, n};
    ReadState st;
    memset(&st, 0, sizeof(st));
    st.active = 1; st.status = TB2_OK;
    std::vector<double> rawf(raw, raw + n), cs((size_t)n + 16), scores((size_t)n + 8);
    std::vector<unsigned char> cstate((size_t)2 * n + 1024);
    std::vector<int> ints((size_t)2 * stall_cap + 8);
    b.n_reads = 1; b.max_raw = n; b.raw_off = raw_off;
    b.rawf = rawf.data(); b.cs = cs.data(); b.scores = scores.data(); b.cstate = cstate.data();
    b.stall_ints = ints.data(); b.stall_cap = stall_cap; b.st = &st;
    emul::launch(emul::Idx3{1, 1, 1}, ST_THREADS, 0, [&]() { k_stalls(b); });
    *n_out = st.n_stalls;
    for (int i = 0; i < 2 * stall_cap; ++i) ints_out[i] = ints[i];
    *status_out = st.status;
    return 0;
}

// k_finalize on one read: final re-normalisation, per-base means, sig_match_score
// (resquiggle.py:1190-1199, get_read_seg_score tombo_stats.py:2327-2338)
int emul_finalize(const double *norm, int n_norm, const int *segs, int nb, const double *rm,
                  const double *rs, double shc, double scc, int rescale, double *bm_out,
                  double *norm_sig_out, double *score_out)
{
    BatchView b;
    memset(&b, 0, sizeof(b));
    long long raw_off[2] = {0, n_norm}, base_off[2] = {0, nb};
    ReadState st;
    memset(&st, 0, sizeof(st));
    st.active = 1; st.status = TB2_OK; st.rsrtr = 0; st.n_norm = n_norm; st.shc = shc; st.scc = scc;
    std::vector<double> nv(norm, norm + n_norm), rmv(rm, rm + nb), rsv(rs, rs + nb), bm((size_t)nb + 8),
        tmp((size_t)nb + 8);
    std::vector<int> sg(segs, segs + nb + 1);
    b.n_reads = 1; b.raw_off = raw_off; b.base_off = base_off; b.norm = nv.data(); b.segs = sg.data();
    b.rm = rmv.data(); b.rs = rsv.data(); b.bm = bm.data(); b.tmp_b = tmp.data(); b.st = &st;
    StagePolicy pol;
    memset(&pol, 0, sizeof(pol));
    pol.skip_seq_scaling = rescale ? 0 : 1;
    emul::launch(emul::Idx3{1, 1, 1}, ST_THREADS, 0, [&]() { k_finalize(b, pol, 1, bm_out, norm_sig_out); });
    *score_out = st.score;
    return st.status;
}

// tb2_block_select2 (select.cuh) on one array: values of ascending rank k and k + 1
void emul_select2(const double *v, int n, int k, double *out2)
{
    static SelectSmem sm;
    emul::launch(emul::Idx3{1, 1, 1}, TB2_SEL_THREADS, 0, [&]() {
        double a = 0, b = 0;
        auto f = [&](int i) { return v[i]; };
        tb2_block_select2(f, PredAll(), n, k, true, &a, &b, sm);
        if (threadIdx.x == 0) { out2[0] = a; out2[1] = b; }
    });
}

void emul_ts_counters(unsigned long long *out8, int reset)
{
    for (int i = 0; i < 8; ++i) out8[i] = g_tb2_counters[i];
    if (reset) for (int i = 0; i < 8; ++i) g_tb2_counters[i] = 0;
}
}
