// emul_motif.cpp -- TEST INFRASTRUCTURE ONLY: the motif LLR kernel's device source
// (tombo_b200/csrc/motif_llr.cuh) run on the host through tests/emul/cuda_emul.h, the way
// tb2_alt_model_llr_motif_batch launches it (count pass, scan, fill pass).
#include "cuda_emul.h"
#include "../../include/tombo_b200.h"
#include "../../tombo_b200/csrc/motif_llr.cuh"
#include <vector>

extern "C" {

int emul_motif_can_overlap(const unsigned char *mask, int len) { return motif_can_overlap(mask, len) ? 1 : 0; }

void emul_llr_motif(int n, const double *norm_mean, const long long *mean_off, const unsigned char *seq,
                    const long long *seq_off, const long long *read_start, const signed char *strand, int K,
                    int cpos, const double *kmeans, const double *ksds, const double *alt, int use_std,
                    double sf, double hf, double hp, int len, int mod_pos, const unsigned char *mask,
                    long long max_ab, long long reg_start, long long reg_end, double *llr_out,
                    long long *pos_out, long long *site_off, int *read_status)
{
    MotifArgs a;
    memset(&a, 0, sizeof(a));
    a.s.n_reads = n; a.s.K = K; a.s.cpos = cpos; a.s.alt_code = -1; a.s.use_std = use_std;
    a.s.sf = sf; a.s.hf = hf; a.s.hp = hp;
    a.s.norm_mean = norm_mean; a.s.mean_off = mean_off; a.s.seq_off = seq_off;
    a.s.read_start = read_start; a.s.seq = seq;
    a.s.kmeans = kmeans; a.s.ksds = ksds; a.s.alt = alt;
    a.m.len = len; a.m.mod_pos = mod_pos;
    for (int j = 0; j < len; ++j) a.m.mask[j] = mask[j];
    a.m.overlap = motif_can_overlap(a.m.mask, len) ? 1 : 0;
    a.strand = strand; a.max_ab = max_ab; a.reg_start = reg_start; a.reg_end = reg_end;
    a.read_status = read_status;
    std::vector<int> cnt((size_t)n + 1);
    if (n == 0) { site_off[0] = 0; return; }
    emul::launch(emul::Idx3{(unsigned)n, 1, 1}, 256, 0,
                 [&]() { k_llr_motif<false>(a, cnt.data(), nullptr, nullptr, nullptr); });
    site_off[0] = 0;
    for (int r = 0; r < n; ++r) site_off[r + 1] = site_off[r] + cnt[r];
    emul::launch(emul::Idx3{(unsigned)n, 1, 1}, 256, 0,
                 [&]() { k_llr_motif<true>(a, nullptr, site_off, llr_out, pos_out); });
}
}
