// emul_stats_file.cpp -- TEST INFRASTRUCTURE ONLY: the device source of the statistics-file
// kernels (tombo_b200/csrc/stats_file.cuh, radix_sort.cuh) run on the host through
// tests/emul/cuda_emul.h, launched in the order tb2_stats_file_aggregate and the
// tb2_most_signif_* calls launch them, with the same host decisions (sf_reduce_before_add,
// sf_live_digits, sf_pack_row).
#include "cuda_emul.h"
#include "../../include/tombo_b200.h"

// __match_any_sync over a full warp: the lanes holding the caller's value
inline unsigned __match_any_sync(unsigned m, int v)
{
    emul::check_mask(m);
    uint64_t all[32];
    emul::xchg((uint64_t)(uint32_t)v, 0, all);
    unsigned r = 0;
    for (int l = 0; l < 32; ++l) r |= (uint32_t)all[l] == (uint32_t)v ? 1u << l : 0u;
    return r;
}

#include "../../tombo_b200/csrc/stats_file.cuh"
#include <algorithm>
#include <vector>

namespace {
unsigned grid_of(long long n) { return (unsigned)std::max<long long>(1, (n + 255) / 256); }

struct Table {
    int kind = 0, K = 5, nf = 2;
    long long N = 0, n = 0, cap = 0, sorted = 0;
    std::vector<unsigned long long> raw;
};
Table T;
// last aggregation, packed
std::vector<tb2_sf_block> A_blk;
std::vector<long long> A_off;
std::vector<unsigned> A_pos, A_cov, A_valid;
std::vector<double> A_damp, A_frac;

void reserve(long long need)
{
    if (need <= T.cap) return;
    const long long cap = std::max(need + need / 4, 2 * T.N);
    std::vector<unsigned long long> nb((size_t)T.K * cap);
    for (int w = 0; w < T.K; ++w)
        std::copy(T.raw.begin() + (size_t)w * T.cap, T.raw.begin() + (size_t)w * T.cap + T.n, nb.begin() + (size_t)w * cap);
    T.raw.swap(nb);
    T.cap = cap;
}

// table_reduce: histograms, the live digits of each word least significant first, the radix
// passes over (key, row index), the gather of the first N
void reduce()
{
    if (T.n == T.sorted && T.n <= T.N) return;
    const long long n = T.n, m = std::min(T.n, T.N), cap = T.cap;
    const long long n_tiles = (n + RADIX_TILE - 1) / RADIX_TILE;
    std::vector<unsigned long long> gh((size_t)MAXW * 8 * 256, 0), key[2], toff((size_t)256 * n_tiles);
    std::vector<unsigned> idx[2], th((size_t)256 * n_tiles);
    for (int c = 0; c < 2; ++c) { key[c].resize(n); idx[c].resize(n); }
    const unsigned long long *raw = T.raw.data();
    emul::launch(emul::Idx3{std::min<unsigned>(grid_of(n), 4), 1, 1}, 256, 0,
                 [&]() { k_sf_hist(raw, cap, n, T.K, T.nf, gh.data()); });
    int cur = 0;
    bool any = false;
    for (int w = T.K - 1; w >= 0; --w) {
        bool live[8];
        if (!sf_live_digits(gh.data(), n, w, live)) continue;
        emul::launch(emul::Idx3{grid_of(n), 1, 1}, 256, 0, [&]() {
            k_sf_word_keys(raw + (size_t)w * cap, w < T.nf, any ? idx[cur].data() : nullptr, n, key[cur].data(),
                           any ? nullptr : idx[cur].data());
        });
        any = true;
        for (int d = 0; d < 8; ++d) {
            if (!live[d]) continue;
            emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RADIX_NT, 0,
                         [&]() { k_radix_tile_hist(key[cur].data(), idx[cur].data(), n, 8 * d, th.data(), n_tiles); });
            emul::launch(emul::Idx3{256, 1, 1}, RADIX_NT, 0, [&]() {
                k_radix_tile_scan(th.data(), n_tiles, gh.data() + (size_t)(w * 8 + d) * 256, toff.data());
            });
            emul::launch(emul::Idx3{(unsigned)n_tiles, 1, 1}, RADIX_NT, 0, [&]() {
                k_radix_scatter_pass(key[cur].data(), idx[cur].data(), key[1 - cur].data(), idx[1 - cur].data(), n,
                                     8 * d, toff.data(), n_tiles);
            });
            cur ^= 1;
        }
    }
    std::vector<unsigned long long> out((size_t)T.K * cap);
    emul::launch(emul::Idx3{grid_of(m), 1, 1}, 256, 0,
                 [&]() { k_sf_gather(raw, out.data(), cap, T.K, any ? idx[cur].data() : nullptr, m); });
    T.raw.swap(out);
    T.n = T.sorted = m;
}
}  // namespace

extern "C" {

// tb2_stats_file_aggregate's launches: shared-memory counters (smem = 1) or global counters
// cut to `per` blocks a launch; row_off (n_blocks + 1) out; returns the error flag
int emul_sf_aggregate(long long n_blocks, const long long *blocks, long long R, const unsigned *pos,
                      const double *stat, double thresh, double lower, int llr, double unmod, double mod, int smem,
                      long long per, long long *row_off)
{
    const tb2_sf_block *blk = (const tb2_sf_block *)blocks;
    std::vector<long long> ub(n_blocks + 1, 0), cnt(n_blocks + 1, 0);
    for (long long b = 0; b < n_blocks; ++b) ub[b + 1] = ub[b] + std::min<long long>(blk[b].n_stat, R);
    const long long U = ub[n_blocks] + 1;
    std::vector<unsigned> upos(U), ucov(U), uvalid(U);
    std::vector<double> udamp(U), ufrac(U);
    std::vector<int> gcnt(smem ? 1 : (size_t)per * 3 * R);
    int err = 0;
    AggArgs a;
    memset(&a, 0, sizeof(a));
    a.blk = blk; a.pos = pos; a.stat = stat; a.R = R;
    a.thresh = thresh; a.lower = lower; a.unmod = unmod; a.mod = mod; a.llr = llr;
    a.ub = ub.data(); a.gcnt = gcnt.data();
    a.o_pos = upos.data(); a.o_damp = udamp.data(); a.o_frac = ufrac.data(); a.o_cov = ucov.data();
    a.o_valid = uvalid.data(); a.n_rows = cnt.data(); a.err = &err;
    if (smem && n_blocks) {
        emul::launch(emul::Idx3{(unsigned)n_blocks, 1, 1}, AGG_NT, (size_t)R * 12, [&]() { k_sf_aggregate<true>(a); });
    } else {
        for (long long b0 = 0; b0 < n_blocks; b0 += per) {
            a.blk0 = (int)b0;
            emul::launch(emul::Idx3{(unsigned)std::min(per, n_blocks - b0), 1, 1}, AGG_NT, 0,
                         [&]() { k_sf_aggregate<false>(a); });
        }
    }
    emul::launch(emul::Idx3{1, 1, 1}, 1024, 0, [&]() { k_scan_offsets(cnt.data(), row_off, n_blocks); });
    const long long rows = row_off[n_blocks] + 1;
    A_blk.assign(blk, blk + n_blocks);
    A_off.assign(row_off, row_off + n_blocks + 1);
    A_pos.resize(rows); A_cov.resize(rows); A_valid.resize(rows); A_damp.resize(rows); A_frac.resize(rows);
    if (n_blocks)
        emul::launch(emul::Idx3{(unsigned)n_blocks, 1, 1}, 256, 0, [&]() {
            k_sf_pack_rows(ub.data(), row_off, upos.data(), udamp.data(), ufrac.data(), ucov.data(), uvalid.data(),
                           A_pos.data(), A_damp.data(), A_frac.data(), A_cov.data(), A_valid.data());
        });
    return err;
}

void emul_sf_download(unsigned *pos, double *damp, double *frac, unsigned *cov, unsigned *valid)
{
    const size_t n = (size_t)A_off.back();
    std::copy(A_pos.begin(), A_pos.begin() + n, pos);
    std::copy(A_damp.begin(), A_damp.begin() + n, damp);
    std::copy(A_frac.begin(), A_frac.begin() + n, frac);
    std::copy(A_cov.begin(), A_cov.begin() + n, cov);
    std::copy(A_valid.begin(), A_valid.begin() + n, valid);
}

void emul_ms_begin(int kind, long long N)
{
    T = Table();
    T.kind = kind; T.K = kind == 0 ? 5 : 4; T.nf = kind == 0 ? 2 : 1; T.N = N;
}

void emul_ms_add_rows(long long n, const double *key, const double *frac, const unsigned *pos, const unsigned *cov,
                      const unsigned *ctrl, const unsigned *valid, unsigned chrm, unsigned char strand)
{
    if (n == 0) return;
    if (sf_reduce_before_add(T.n, n, T.cap, T.N)) reduce();
    reserve(T.n + n);
    for (long long i = 0; i < n; ++i)
        sf_pack_row(T.kind, key[i], frac ? frac[i] : 0.0, pos[i], cov[i], ctrl[i], valid ? valid[i] : 0, chrm, strand,
                    T.raw.data() + T.n + i, T.cap);
    T.n += n;
}

void emul_ms_add_aggregate()
{
    const long long n = A_off.back();
    if (n == 0) return;
    if (sf_reduce_before_add(T.n, n, T.cap, T.N)) reduce();
    reserve(T.n + n);
    emul::launch(emul::Idx3{(unsigned)A_blk.size(), 1, 1}, 256, 0, [&]() {
        k_sf_table_from_agg(A_blk.data(), A_off.data(), A_pos.data(), A_damp.data(), A_frac.data(), A_cov.data(),
                            A_valid.data(), T.raw.data(), T.cap, T.n);
    });
    T.n += n;
}

// the table in order as raw words, word-major with stride n (count first)
long long emul_ms_count()
{
    reduce();
    return T.n;
}

void emul_ms_words(unsigned long long *out)
{
    for (int w = 0; w < T.K; ++w)
        std::copy(T.raw.begin() + (size_t)w * T.cap, T.raw.begin() + (size_t)w * T.cap + T.n, out + (size_t)w * T.n);
}
}
