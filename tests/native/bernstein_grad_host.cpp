// CPU harness around the bounded Bernstein pair math of zuko_b200/csrc/bernstein_math.cuh (what
// uni_kernel, uni_bwd_kernel and ar_inverse_kernel run on the GPU), compiled by g++ from
// tests/test_bpf_host.py.  The default degree also runs the compile-time instantiation.
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "../../zuko_b200/csrc/bernstein_math.cuh"

using zk::bern::Const;

namespace {

int steps(float bound, float eps) { return (int)ceil(log2(2.0 * (double)bound / (double)eps)); }

template <int PT, class F>
float with_pair(const float* u, const Const& c, F f) {
    float w[PT > 0 ? PT : 1], mx, rs;
    zk::bern::softmax<PT>(u, c, w, mx, rs);
    constexpr int MT = PT > 0 ? zk::bern::order_of(PT) : 0;
    return f([&](int j) { return zk::bern::delta<PT>(u, w, c, mx, rs, j); },
             std::integral_constant<int, MT>());
}

}  // namespace

extern "C" {

// x, y, ladj: (n) pairs; phi: (n, P) rows, or one shared row when phi_ld == 0
void bern_forward_pairs(const float* x, const float* phi, int64_t phi_ld, int64_t n, int degree, float bound, float eps,
                        float* y, float* ladj) {
    const Const c = zk::bern::make_const(degree, bound, eps, steps(bound, eps));
    for (int64_t i = 0; i < n; ++i) {
        float fp = 0.f;
        auto run = [&](auto dl, auto mt) { return zk::bern::forward<decltype(mt)::value>(c, x[i], dl, &fp); };
        y[i] = degree == zk::bern::kDefDegree ? with_pair<zk::bern::kDefP>(phi + i * phi_ld, c, run)
                                              : with_pair<0>(phi + i * phi_ld, c, run);
        ladj[i] = logf(fp);
    }
}

void bern_inverse_pairs(const float* y, const float* phi, int64_t phi_ld, int64_t n, int degree, float bound, float eps,
                        float* x) {
    const Const c = zk::bern::make_const(degree, bound, eps, steps(bound, eps));
    for (int64_t i = 0; i < n; ++i) {
        auto run = [&](auto dl, auto mt) { return zk::bern::inverse<decltype(mt)::value>(c, y[i], dl); };
        x[i] = degree == zk::bern::kDefDegree ? with_pair<zk::bern::kDefP>(phi + i * phi_ld, c, run)
                                              : with_pair<0>(phi + i * phi_ld, c, run);
    }
}

// gphi: (n, P) per-pair gradients
void bern_backward_pairs(const float* x, const float* phi, int64_t phi_ld, const float* gy, const float* gl, int64_t n,
                         int degree, float bound, float eps, float* gx, float* gphi) {
    const Const c = zk::bern::make_const(degree, bound, eps, 0);
    const int P = degree + 1;
    for (int64_t i = 0; i < n; ++i) {
        if (degree == zk::bern::kDefDegree)
            zk::bern::backward_pair<zk::bern::kDefP>(phi + i * phi_ld, c, x[i], gy[i], gl[i], gx[i], gphi + i * P);
        else
            zk::bern::backward_pair<0>(phi + i * phi_ld, c, x[i], gy[i], gl[i], gx[i], gphi + i * P);
    }
}

// the kernels rewrite a per-sample parameter block in place: gphi == phi (runtime-degree path)
void bern_backward_in_place(const float* x, float* phi, const float* gy, const float* gl, int64_t n, int degree,
                            float bound, float eps, float* gx) {
    const Const c = zk::bern::make_const(degree, bound, eps, 0);
    const int P = degree + 1;
    for (int64_t i = 0; i < n; ++i)
        zk::bern::backward_pair<0>(phi + i * P, c, x[i], gy[i], gl[i], gx[i], phi + i * P);
}
}
