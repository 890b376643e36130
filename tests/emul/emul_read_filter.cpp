// emul_read_filter.cpp -- TEST INFRASTRUCTURE ONLY: the device source of the read filters
// (tombo_b200/csrc/read_filter.cuh) run on the host through tests/emul/cuda_emul.h, launched
// as tb2_dwell_percentiles, tb2_batch_read_filters and tb2_read_mid_coverage launch it.
#include "cuda_emul.h"
#include "../../include/tombo_b200.h"
#include "../../tombo_b200/csrc/read_filter.cuh"
#include <algorithm>
#include <vector>

extern "C" {

void emul_rf_pctl(int n, const long long *lens, const long long *off, int n_pctl, const double *pctl,
                  double *out)
{
    emul::launch(emul::Idx3{(unsigned)n, 1, 1}, TB2_SEL_THREADS, 0,
                 [&]() { k_rf_dwell_pctl(lens, off, n_pctl, pctl, out); });
}

// segs at base_off[r] + r; status of read r at status[r] (stride 1)
void emul_rf_batch(int n, const long long *segs, const long long *base_off, const int *status,
                   const double *score, double thresh, int n_pctl, const double *pctl,
                   const double *pthresh, signed char *code, double *pout)
{
    emul::launch(emul::Idx3{(unsigned)n, 1, 1}, TB2_SEL_THREADS, 0, [&]() {
        k_rf_batch(segs, base_off, status, 1, score, thresh, n_pctl, pctl, pthresh, code, pout);
    });
}

// abs_start / abs_end already placed in the concatenated coverage arrays of total length len
void emul_rf_mid(long long n, const long long *as, const long long *ae, long long len, long long *out)
{
    std::vector<int> cov((size_t)len, 0);
    const long long n_tiles = (len + RF_TILE - 1) / RF_TILE;
    std::vector<long long> tsum((size_t)n_tiles), toff((size_t)n_tiles + 1);
    const unsigned g = (unsigned)std::max<long long>(1, (n + 255) / 256);
    emul::launch(emul::Idx3{g, 1, 1}, 256, 0, [&]() { k_rf_cov_diff(as, ae, n, cov.data()); });
    emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RF_NT, 0, [&]() { k_rf_tile_sum(cov.data(), len, tsum.data()); });
    emul::launch(emul::Idx3{1, 1, 1}, 1024, 0, [&]() { k_scan_offsets<long long>(tsum.data(), toff.data(), n_tiles); });
    emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RF_NT, 0, [&]() { k_rf_tile_scan(cov.data(), len, toff.data()); });
    emul::launch(emul::Idx3{g, 1, 1}, 256, 0, [&]() { k_rf_mid(as, ae, n, cov.data(), out); });
}

}
