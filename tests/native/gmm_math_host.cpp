// CPU harness around the Gaussian mixture row math of zuko_b200/csrc/gmm_math.cuh (what gmm_log_prob_kernel,
// gmm_backward_kernel and gmm_sample_kernel run on the GPU), compiled by g++ from tests/test_gmm_host.py.
#include <stdint.h>

#include <vector>

#include "../../zuko_b200/csrc/gmm_math.cuh"

extern "C" {

// phi: (B, P) rows, or one row read by every sample when ldphi == 0
void gmm_log_prob_rows(const float* x, const float* phi, int64_t ldphi, int64_t B, int D, int K, int cov, int tied,
                       float eps, float* out) {
    const zk::gmm::Layout l = zk::gmm::make_layout(D, K, cov, tied);
    std::vector<float> v(D), t(K);
    for (int64_t b = 0; b < B; ++b) out[b] = zk::gmm::row_log_prob(x + b * D, phi + b * ldphi, l, eps, v.data(), 1, t.data(), 1);
}

// gx (B, D), gphi (B, P) per-row gradients of sum(g * log_prob)
void gmm_backward_rows(const float* x, const float* phi, int64_t ldphi, int64_t B, int D, int K, int cov, int tied,
                       float eps, const float* g, float* gx, float* gphi) {
    const zk::gmm::Layout l = zk::gmm::make_layout(D, K, cov, tied);
    std::vector<float> v(D), w(D), t(K);
    for (int64_t b = 0; b < B; ++b)
        zk::gmm::row_backward(x + b * D, phi + b * ldphi, l, eps, g[b], gx + b * D, gphi + b * l.total, v.data(), 1,
                              w.data(), 1, t.data(), 1);
}

void gmm_sample_rows(const float* phi, int64_t ldphi, const float* u, const float* z, int64_t B, int D, int K, int cov,
                     int tied, float eps, float* x) {
    const zk::gmm::Layout l = zk::gmm::make_layout(D, K, cov, tied);
    for (int64_t b = 0; b < B; ++b) zk::gmm::row_sample(phi + b * ldphi, l, eps, u[b], z + b * D, x + b * D);
}

int gmm_select_component(const float* logits, int K, float u) { return zk::gmm::select_component(logits, K, u); }

int gmm_params_per_row(int D, int K, int cov, int tied) { return zk::gmm::make_layout(D, K, cov, tied).total; }

}  // extern "C"
