// CPU harness around the Gaussianization pair math of zuko_b200/csrc/bijector_grad.cuh (what
// uni_bwd_kernel runs on the GPU), compiled by g++ from tests/test_gf_host.py.
#include <stdint.h>

#include "../../zuko_b200/csrc/bijector_grad.cuh"

extern "C" {

// x, y, gy, gl, gx: (n) pairs; phi, gphi: (n, 2K) rows (shift[K], scale[K]), or one shared row when phi_ld == 0
void gauss_backward_pairs(const float* x, const float* y, const float* phi, int64_t phi_ld, const float* gy,
                          const float* gl, int64_t n, int K, float* gx, float* gphi) {
    for (int64_t i = 0; i < n; ++i)
        zk::bijgrad::gauss_backward_pair(phi + i * phi_ld, K, x[i], y[i], gy[i], gl[i], gx[i], gphi + i * 2 * K);
}
}
