// emul_tracks.cpp -- TEST INFRASTRUCTURE ONLY: the device source of the genome browser tracks
// (tombo_b200/csrc/browser_tracks.cuh, with the coverage kernels of read_filter.cuh and the
// radix sort of radix_sort.cuh) run on the host through tests/emul/cuda_emul.h, launched as
// tb2_coverage_runs and tb2_slot_sums_add / _means launch them.
#include "cuda_emul.h"
#include "../../include/tombo_b200.h"

// __match_any_sync over a full warp (the radix sort's scatter), as emul_stats_file.cpp has it
inline unsigned __match_any_sync(unsigned m, int v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)(uint32_t)v, 0, all);
    unsigned r = 0;
    for (int l = 0; l < 32; ++l) r |= (uint32_t)all[l] == (uint32_t)v ? 1u << l : 0u;
    return r;
}

#include "../../tombo_b200/csrc/read_filter.cuh"
#include "../../tombo_b200/csrc/browser_tracks.cuh"
#include <algorithm>
#include <vector>

namespace {

unsigned grid(long long n, int nt) { return (unsigned)std::max<long long>(1, (n + nt - 1) / nt); }

void scan(int *x, long long len)
{
    const long long n_tiles = (len + RF_TILE - 1) / RF_TILE;
    std::vector<long long> tsum((size_t)n_tiles), toff((size_t)n_tiles + 1);
    emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RF_NT, 0, [&]() { k_rf_tile_sum(x, len, tsum.data()); });
    emul::launch(emul::Idx3{1, 1, 1}, 1024, 0, [&]() { k_scan_offsets<long long>(tsum.data(), toff.data(), n_tiles); });
    emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RF_NT, 0, [&]() { k_rf_tile_scan(x, len, toff.data()); });
}

}  // namespace

extern "C" {

// abs_start / abs_end already placed in the concatenated coverage arrays; base[g] is group g's
// first entry (n_groups + 1 entries); returns the run count
long long emul_bt_runs(long long n, const long long *as, const long long *ae, long long n_groups,
                       const long long *base, long long *run_off, long long *run_start, long long *run_cov)
{
    const long long len = base[n_groups];
    std::vector<int> cov((size_t)len, 0), flag((size_t)len, 0);
    emul::launch(emul::Idx3{grid(n, 256), 1, 1}, 256, 0, [&]() { k_rf_cov_diff(as, ae, n, cov.data()); });
    scan(cov.data(), len);
    emul::launch(emul::Idx3{grid(len, 256), 1, 1}, 256, 0, [&]() { k_bt_run_flags(cov.data(), len, flag.data()); });
    emul::launch(emul::Idx3{grid(n_groups, 256), 1, 1}, 256, 0, [&]() { k_bt_run_ends(base, n_groups, flag.data()); });
    scan(flag.data(), len);
    emul::launch(emul::Idx3{grid(len, 256), 1, 1}, 256, 0, [&]() {
        k_bt_run_scatter(cov.data(), flag.data(), len, base, n_groups, run_start, run_cov);
    });
    emul::launch(emul::Idx3{grid(n_groups + 1, 256), 1, 1}, 256, 0,
                 [&]() { k_bt_run_off(flag.data(), base, n_groups, run_off); });
    return run_off[n_groups];
}

// one tb2_slot_sums_add on sums / cov (offsets rebased to 0, kmin the least start of a read
// with values, kmax its last position); returns the overflow flag
int emul_bt_add(long long n_reads, const long long *start, const long long *off, const unsigned char *rev,
                const double *vals, long long kmin, long long kmax, double *sums, int *cov)
{
    const long long total = off[n_reads];
    const long long n_tiles = (total + RADIX_TILE - 1) / RADIX_TILE;
    std::vector<unsigned long long> key[2] = {std::vector<unsigned long long>((size_t)total),
                                              std::vector<unsigned long long>((size_t)total)};
    std::vector<double> val[2] = {std::vector<double>((size_t)total), std::vector<double>((size_t)total)};
    std::vector<unsigned long long> gh((size_t)BT_DIGITS * 256, 0), toff((size_t)256 * n_tiles);
    std::vector<unsigned int> th((size_t)256 * n_tiles);
    emul::launch(emul::Idx3{std::min<unsigned>(grid(total, 256), 7), 1, 1}, 256, 0, [&]() {
        k_bt_entries(vals, off, start, rev, n_reads, total, kmin, key[0].data(), val[0].data(), gh.data());
    });
    int cur = 0;
    for (int d = 0; d < BT_DIGITS && (kmax - kmin) >> (8 * d); ++d) {
        const unsigned long long *ph = gh.data() + (size_t)d * 256;
        if (std::any_of(ph, ph + 256, [&](unsigned long long c) { return c == (unsigned long long)total; })) continue;
        emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RADIX_NT, 0, [&]() {
            k_radix_tile_hist(key[cur].data(), val[cur].data(), total, 8 * d, th.data(), n_tiles);
        });
        emul::launch(emul::Idx3{256, 1, 1}, RADIX_NT, 0,
                     [&]() { k_radix_tile_scan(th.data(), n_tiles, gh.data() + (size_t)d * 256, toff.data()); });
        emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RADIX_NT, 0, [&]() {
            k_radix_scatter_pass(key[cur].data(), val[cur].data(), key[1 - cur].data(), val[1 - cur].data(), total,
                                 8 * d, toff.data(), n_tiles);
        });
        cur ^= 1;
    }
    int overflow = 0;
    emul::launch(emul::Idx3{grid(total, 256), 1, 1}, 256, 0, [&]() {
        k_bt_accumulate(key[cur].data(), val[cur].data(), total, kmin, sums, cov, &overflow);
    });
    return overflow;
}

void emul_bt_means(const double *sums, const int *cov, long long n, double *out)
{
    emul::launch(emul::Idx3{grid(n, 256), 1, 1}, 256, 0, [&]() { k_bt_means(sums, cov, n, out); });
}

}
