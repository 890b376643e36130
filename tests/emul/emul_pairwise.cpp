// emul_pairwise.cpp -- TEST INFRASTRUCTURE ONLY: warp_pairwise_sum (tombo_b200/csrc/common.cuh)
// run on the host through tests/emul/cuda_emul.h, for tests/test_warp_pairwise_sum_cpu.py.
#include "cuda_emul.h"
#include "../../tombo_b200/csrc/common.cuh"

extern "C" {

// warp_pairwise_sum of v[0 .. n) by one warp
void emul_warp_pairwise_sum(const double *v, int n, double *out)
{
    emul::launch(emul::Idx3{1, 1, 1}, 32, 0, [&]() {
        const double s = warp_pairwise_sum([v](int i) { return v[i]; }, n);
        if (threadIdx.x == 0) *out = s;
    });
}

}  // extern "C"
