// emul_dp.cpp -- TEST INFRASTRUCTURE ONLY: runs the device source of the banded-DP
// assignment kernel (tombo_b200/csrc/dp_align_kernel.cuh, the file nvcc compiles for
// sm_90a) on the host through tests/emul/cuda_emul.h, so the CPU test-suite can compare
// the kernel's logic with the oracle.  Not part of libtombo_b200.so.
#include "cuda_emul.h"
#include "../../tombo_b200/csrc/dp_align_kernel.cuh"
#include <vector>

extern "C" {

// one batch through k_align<klass>; all arrays are host arrays in the AlignBatch layout
// (stride 1).  n_blocks CTAs of 4 warps pull reads from the shared counter.
int emul_align_batch(int klass, int n_reads, const int *cpts, const double *em,
                     const long long *ev_off, const int *n_cpts, const int *num_events,
                     const double *rm, const double *rs, const long long *base_off,
                     int *segs /* sum(nb) + n */, int *rsrtr, int *status, int *dbg,
                     const tb2_params *params, double sig_match_thresh, int smem_cells,
                     long long tb_words, int grow_cells, int n_blocks, int *starts_out,
                     int *read_tb_out)
{
    AlignBatch b;
    b.n_reads = n_reads;
    b.order = nullptr;
    b.cpts = cpts; b.em = em; b.ev_off = ev_off; b.n_cpts = n_cpts; b.num_events = num_events;
    b.rm = rm; b.rs = rs; b.base_off = base_off;
    const long long nbt = base_off[n_reads];
    std::vector<int> starts((size_t)nbt + 8), read_tb((size_t)nbt + n_reads + 8);
    b.starts = starts.data(); b.read_tb = read_tb.data(); b.segs = segs;
    b.rsrtr = rsrtr; b.status = status; b.active = nullptr; b.stride = 1; b.dbg = dbg;
    b.params = *params;
    b.sig_match_thresh = sig_match_thresh;
    AlignLaunchCfg cfg;
    cfg.smem_cells = smem_cells; cfg.tb_words = (size_t)tb_words; cfg.grow_cells = grow_cells;
    cfg.klass = klass;
    const size_t slots = (size_t)n_blocks * ALIGN_WARPS;
    std::vector<uint32_t> tb_pool(slots * cfg.tb_words + 64);
    std::vector<double> grow_pool(slots * 2 * (size_t)grow_cells + 8);
    int counter = 0;
    const size_t smem = (size_t)ALIGN_WARPS * (2 * (size_t)cfg.smem_cells + TB2_WF_RING) * sizeof(double);
    emul::launch(emul::Idx3{(unsigned)n_blocks, 1, 1}, ALIGN_WARPS * 32, smem, [&]() {
        if (klass == 1) k_align<1>(b, cfg, tb_pool.data(), grow_pool.data(), &counter);
        else if (klass == 2) k_align<2>(b, cfg, tb_pool.data(), grow_pool.data(), &counter);
        else k_align<0>(b, cfg, tb_pool.data(), grow_pool.data(), &counter);
    });
    if (starts_out) memcpy(starts_out, starts.data(), (size_t)nbt * sizeof(int));
    if (read_tb_out) memcpy(read_tb_out, read_tb.data(), ((size_t)nbt + n_reads) * sizeof(int));
    return 0;
}

size_t emul_tb_words(long long rows, long long W, long long drift) { return tb2_tb_words(rows, W, drift); }
int emul_row_cells(long long W) { return tb2_row_cells(W); }
// the adaptive-band engine choice of the device source (kernels.h, dp_align.cuh), for the
// tests that place parameter points on either side of each boundary
int emul_abs_chunk(long long W) { return tb2_abs_chunk_host(W); }
int emul_abs_ms_chunk(long long W) { return tb2_abs_ms_chunk_host(W); }
int emul_wpl_of(int chunk) { return tb2_wpl_of(chunk); }
}

// tuning counters of the adaptive engines (meaningful when built with -DTB2_DP_COUNTERS)
extern "C" void emul_dp_counters(unsigned long long *out8, int reset)
{
    for (int i = 0; i < 8; ++i) out8[i] = g_tb2_dp_counters[i];
    if (reset) for (int i = 0; i < 8; ++i) g_tb2_dp_counters[i] = 0;
}
