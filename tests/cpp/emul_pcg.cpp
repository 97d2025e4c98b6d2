// tests/cpp/emul_pcg.cpp -- fiber emulation (cuda_fiber.h) of k_pcg alone (csrc/seam.cu, kernel text unchanged) on
// hand-built systems: the CSR arrays k_matrix would produce (diagonal first, column | weight class << 31), grid = 1.
// seam_kernels.inc is generated from seam.cu by tests/test_emul_pcg.py (or tests/golden/make_pcg_emul.py).
#include "cuda_fiber.h"

#include <vector>

#include "seam_kernels.inc"

using namespace b2;

extern "C" {

// rhs and x are [3][R]; status gets iterations[3], residual bits[3], loop iterations.  Returns 0, -1 if the launch hung.
int emul_pcg(uint32_t R, const uint32_t *csr_ptr, const uint32_t *csr_enc, const float *diag_val, const float *inv_diag,
             const float *rhs, uint32_t max_iters, float *x, uint32_t *status /* 16 */)
{
    std::vector<float> r(3 * (size_t)R), t(3 * (size_t)R);
    std::vector<float4> p(R);
    std::vector<double> partials(2 * 8, 0.0);
    for (int i = 0; i < 16; ++i) status[i] = 0;
    Pcg q{R, csr_ptr, csr_enc, diag_val, inv_diag, rhs, x, r.data(), t.data(), p.data(), partials.data(), status, max_iters, 0.0001f};
    return emul::launch(1, PCG_THREADS, [&] { k_pcg(q); }) ? 0 : -1;
}

}  // extern "C"
