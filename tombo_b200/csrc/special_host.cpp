// special_host.cpp -- the functions of special.cuh compiled for the host (same source,
// -ffp-contract=off), so tests can compare them with scipy on dense grids without a GPU.
#include <stdint.h>
#include "special.cuh"

extern "C" {
double tb2_host_kolmogorov_sf(double y) { return tb2_kolmogorov_sf(y); }
double tb2_host_t_two_sided_p(double df, double t) { return tb2_t_two_sided_p(df, t); }
double tb2_host_chi2_sf_even(double y, int k) { return tb2_chi2_sf_even(y, k); }
double tb2_host_div12(uint64_t hi, uint64_t lo)
{
    return tb2_div12(((unsigned __int128)hi << 64) | lo);
}
}
