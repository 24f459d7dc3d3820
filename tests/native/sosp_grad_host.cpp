// CPU harness around the sum-of-squares polynomial pair math of zuko_b200/csrc/sosp_math.cuh (what
// uni_kernel, uni_bwd_kernel and ar_inverse_kernel run on the GPU) and its host Gauss-Legendre routine,
// compiled by g++ from tests/test_sospf_host.py.  Only the runtime-shape instantiation runs here.
#include <stdint.h>

#include "../../zuko_b200/csrc/sosp_math.cuh"

using zk::sosp::Const;

extern "C" {

void sosp_nodes(int n, double* t, double* w) { zk::sosp::gauss_legendre01(n, t, w); }

// x, y, ladj: (n) pairs; phi: (n, P) rows (a[K][L+1], constant), or one shared row when phi_ld == 0
void sosp_forward_pairs(const float* x, const float* phi, int64_t phi_ld, int64_t n, int K, int L, float* y, float* ladj) {
    const Const c = zk::sosp::make_const(K, L, 10.f, 1e-3f, 25);
    for (int64_t i = 0; i < n; ++i) {
        float gx;
        y[i] = zk::sosp::forward<0>(phi + i * phi_ld, c, x[i], gx);
        ladj[i] = logf(gx);
    }
}

void sosp_inverse_pairs(const float* y, const float* phi, int64_t phi_ld, int64_t n, int K, int L, float* x) {
    const Const c = zk::sosp::make_const(K, L, 10.f, 1e-3f, 25);
    for (int64_t i = 0; i < n; ++i) x[i] = zk::sosp::inverse<0>(phi + i * phi_ld, c, y[i]);
}

// gphi: (n, P) per-pair gradients; the default shape also runs the compile-time instantiation
void sosp_backward_pairs(const float* x, const float* phi, int64_t phi_ld, const float* gy, const float* gl, int64_t n,
                         int K, int L, float* gx, float* gphi) {
    const Const c = zk::sosp::make_const(K, L, 10.f, 1e-3f, 25);
    const int P = K * (L + 1) + 1;
    for (int64_t i = 0; i < n; ++i) {
        if (K == zk::sosp::kDefK && L == zk::sosp::kDefL)
            zk::sosp::backward_pair<zk::sosp::kDefK>(phi + i * phi_ld, c, x[i], gy[i], gl[i], gx[i], gphi + i * P);
        else
            zk::sosp::backward_pair<0>(phi + i * phi_ld, c, x[i], gy[i], gl[i], gx[i], gphi + i * P);
    }
}

// the kernels rewrite a per-sample parameter block in place: gphi == phi
void sosp_backward_in_place(const float* x, float* phi, const float* gy, const float* gl, int64_t n, int K, int L,
                            float* gx) {
    const Const c = zk::sosp::make_const(K, L, 10.f, 1e-3f, 25);
    const int P = K * (L + 1) + 1;
    for (int64_t i = 0; i < n; ++i) zk::sosp::backward_pair<0>(phi + i * P, c, x[i], gy[i], gl[i], gx[i], phi + i * P);
}
}
