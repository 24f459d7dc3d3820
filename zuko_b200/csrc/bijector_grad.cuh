// zuko_b200 — reverse-mode math of the univariate bijectors, per (sample, dim) pair.
//
// Host/device code (plain IEEE fp32, no MUFU approximations): the same functions are compiled by
// g++ into a CPU harness (tests/native/bijector_grad_host.cpp) so that the derivation is checked
// against the gradient oracle without a GPU, and by nvcc into uni_bwd_kernel (backward.cu).
//
// Formulation (same as the forward kernel, bijector_math.cuh): with soft-clipped logits
// u_i = sc(w_i), softmax numerators e_i = exp(u_i), S = sum e_i,
//     bin width  dx = 2B e_k / S,   left knot  x0 = -B + 2B sum_{i<k} e_i / S
// (heights likewise), d_j = exp(sc(r_{j-1})) for interior knots and 1 at both ends.  x0 and dx are
// independent functions of the softmax outputs W_i = e_i / S, so
//     dL/dW_i = 2B (G_x0 [i < k] + G_dx [i == k]),
//     dL/du_i = W_i (dL/dW_i - sum_j W_j dL/dW_j),   sum_j W_j dL/dW_j = G_x0 (x0 + B) + G_dx dx.
// Reference ops being differentiated: zuko/transforms.py:480-490 (constructor), 499-523 (bin
// search), 556-567 (spline and log-derivative); 435-446 (affine).
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define ZK_HD __host__ __device__ __forceinline__
#else
#define ZK_HD inline
#endif

namespace zk {
namespace bijgrad {

// soft clip v / (1 + |v| a) and its derivative 1 / (1 + |v| a)^2
ZK_HD float sc(float v, float a) { return v / fmaf(fabsf(v), a, 1.0f); }
ZK_HD float dsc(float v, float a) {
    const float d = fmaf(fabsf(v), a, 1.0f);
    return 1.0f / (d * d);
}

// FAST = true (device only, zk_set_fast_math(1)): MUFU reciprocal / ex2 instead of IEEE division / expf — the
// same approximations the forward kernels use (bijector_math.cuh); ~1e-6 relative on values bounded by the soft
// clip, against a 5e-5 bar on the gradients.  Host builds (tests/native) always take the IEEE forms.
template <bool FAST>
ZK_HD float rcp_(float v) {
#if defined(__CUDA_ARCH__)
    if constexpr (FAST) return __fdividef(1.0f, v);
#endif
    return 1.0f / v;
}
template <bool FAST>
ZK_HD float div_(float a, float b) {
#if defined(__CUDA_ARCH__)
    if constexpr (FAST) return __fdividef(a, b);
#endif
    return a / b;
}
template <bool FAST>
ZK_HD float exp_(float v) {
#if defined(__CUDA_ARCH__)
    if constexpr (FAST) return __expf(v);
#endif
    return expf(v);
}

// soft clip u = v / (1 + |v| a) and its derivative d = 1 / (1 + |v| a)^2 from ONE reciprocal
template <bool FAST = false>
ZK_HD void sc_parts(float v, float a, float& u, float& d) {
    const float r = rcp_<FAST>(fmaf(fabsf(v), a, 1.0f));
    u = v * r;
    d = r * r;
}

// One (sample, dim) pair of MonotonicRQSTransform.call_and_ladj, reverse mode.
//   p   : the pair's P = 3K-1 raw parameters (widths, heights, derivatives)
//   gy  : dL/dy, gl : dL/dladj (of this pair's log-derivative)
//   gx  : dL/dx (direct dependence only), gp : dL/dp (P values; may alias p)
// The softmax numerators / soft-clip derivatives of the 2K width / height parameters are recomputed
// in each of the three sweeps (1 reciprocal + 1 exp per parameter and sweep).  Keeping them in
// registers instead (kCacheNumerators) costs registers (92 instead of 64 per thread at K = 8), which
// halves the resident warps of this latency-bound kernel; the code path is kept for reference, both
// give bit-identical results.
constexpr bool kCacheNumerators = false;

template <int KT_, bool FAST = false>
ZK_HD void rqs_backward_pair(const float* p, int Krt, float x, float gy, float gl, float bound,
                             float aw, float ad, float& gx, float* gp) {
    constexpr int KT = kCacheNumerators ? KT_ : 0;  // 0 = recompute path
    const int K = KT_ > 0 ? KT_ : Krt;
    const int P = 3 * K - 1;
    constexpr int KA = KT > 0 ? KT : 1;
    float ew[KA], eh[KA], dw[KA], dh[KA];
    float sw = 0.f, sh = 0.f;
    for (int k = 0; k < K; ++k) {
        float u0, d0_, u1, d1_;
        sc_parts<FAST>(p[k], aw, u0, d0_);
        sc_parts<FAST>(p[K + k], aw, u1, d1_);
        const float e0 = exp_<FAST>(u0), e1 = exp_<FAST>(u1);
        if constexpr (KT > 0) {
            ew[k] = e0; eh[k] = e1; dw[k] = d0_; dh[k] = d1_;
        }
        sw += e0;
        sh += e1;
    }
    const float gxs = div_<FAST>(2.f * bound, sw);  // numerator -> width
    const float gys = div_<FAST>(2.f * bound, sh);
    // bin search on the horizontal knots (strict <, transforms.py:521-523)
    float cw = 0.f, ch = 0.f, xl = -bound, yl = -bound;
    int kb = 0;
    float x0 = -bound, y0 = -bound, ewk = 0.f, ehk = 0.f, cwk = 0.f, chk = 0.f;
    for (int j = 0; j < K; ++j) {
        float e0, e1;
        if constexpr (KT > 0) {
            e0 = ew[j];
            e1 = eh[j];
        } else {
            float u, d;
            sc_parts<FAST>(p[j], aw, u, d);
            e0 = exp_<FAST>(u);
            sc_parts<FAST>(p[K + j], aw, u, d);
            e1 = exp_<FAST>(u);
        }
        const bool take = (j == 0) || (xl < x);
        if (take) {
            kb = j; x0 = xl; y0 = yl; ewk = e0; ehk = e1; cwk = cw; chk = ch;
        }
        cw += e0;
        ch += e1;
        xl = fmaf(cw, gxs, -bound);
        yl = fmaf(ch, gys, -bound);
    }
    const bool inside = (-bound < x) && !(xl < x);
    if (!inside) {  // identity outside the domain: dy/dx = 1, ladj = 0 (transforms.py:567)
        gx = gy;
        for (int i = 0; i < P; ++i) gp[i] = 0.f;
        return;
    }
    const float dx = ewk * gxs, dy = ehk * gys;
    float ur0 = 0.f, dr0 = 0.f, ur1 = 0.f, dr1 = 0.f;  // soft-clipped derivatives of the bin's two knots
    if (kb > 0) sc_parts<FAST>(p[2 * K + kb - 1], ad, ur0, dr0);
    if (kb < K - 1) sc_parts<FAST>(p[2 * K + kb], ad, ur1, dr1);
    const float d0 = (kb > 0) ? exp_<FAST>(ur0) : 1.f;  // pad (1, 1) with 0 -> exp(0) = 1
    const float d1 = (kb < K - 1) ? exp_<FAST>(ur1) : 1.f;
    const float rdx = rcp_<FAST>(dx);
    const float s = dy * rdx;
    const float z = (x - x0) * rdx;
    const float omz = 1.f - z;
    const float q = z * omz;
    const float t = d0 + d1 - 2.f * s;
    const float num = fmaf(s * z, z, d0 * q);
    const float den = fmaf(t, q, s);
    const float m = 2.f * s * q + d0 * omz * omz + d1 * z * z;
    const float rden = rcp_<FAST>(den), rm = rcp_<FAST>(m);
    const float rden2 = rden * rden;
    // y = y0 + dy num / den,  ladj = 2 log s + log m - 2 log den
    const float dy_dz = dy * s * m * rden2;  // (num_z den - num den_z) = s m
    const float dy_ds = dy * (z * z * den - num * (1.f - 2.f * q)) * rden2;
    const float dy_dd0 = dy * q * (den - num) * rden2;
    const float dy_dd1 = -dy * num * q * rden2;
    const float dl_ds = div_<FAST>(2.f, s) + 2.f * q * rm - 2.f * (1.f - 2.f * q) * rden;
    const float dl_dz = (2.f * s * (1.f - 2.f * z) - 2.f * d0 * omz + 2.f * d1 * z) * rm -
                        2.f * t * (1.f - 2.f * z) * rden;
    const float dl_dd0 = omz * omz * rm - 2.f * q * rden;
    const float dl_dd1 = z * z * rm - 2.f * q * rden;
    const float Gs = gy * dy_ds + gl * dl_ds;
    const float Gz = gy * dy_dz + gl * dl_dz;
    const float Gd0 = gy * dy_dd0 + gl * dl_dd0;
    const float Gd1 = gy * dy_dd1 + gl * dl_dd1;
    gx = Gz * rdx;
    const float Gdy = fmaf(gy * num, rden, Gs * rdx);  // s = dy / dx
    const float Gdx = -(Gs * s + Gz * z) * rdx;        // s, z both carry 1 / dx
    const float Gx0 = -Gz * rdx;
    const float Gy0 = gy;
    // sum_j W_j dL/dW_j, divided by 2B
    const float dotw = div_<FAST>(Gx0 * (cwk * gxs) + Gdx * dx, 2.f * bound);
    const float doth = div_<FAST>(Gy0 * (chk * gys) + Gdy * dy, 2.f * bound);
    const float gd0 = Gd0 * d0 * dr0, gd1 = Gd1 * d1 * dr1;  // gradients of the two raw derivative parameters
    for (int i = 0; i < K; ++i) {
        float e0, e1, c0, c1;
        if constexpr (KT > 0) {
            e0 = ew[i]; e1 = eh[i]; c0 = dw[i]; c1 = dh[i];
        } else {
            float u;
            sc_parts<FAST>(p[i], aw, u, c0);
            e0 = exp_<FAST>(u);
            sc_parts<FAST>(p[K + i], aw, u, c1);
            e1 = exp_<FAST>(u);
        }
        const float selw = (i < kb ? Gx0 : 0.f) + (i == kb ? Gdx : 0.f);
        const float selh = (i < kb ? Gy0 : 0.f) + (i == kb ? Gdy : 0.f);
        gp[i] = e0 * gxs * (selw - dotw) * c0;
        gp[K + i] = e1 * gys * (selh - doth) * c1;
    }
    for (int j = 0; j < K - 1; ++j) gp[2 * K + j] = (j == kb - 1 ? gd0 : 0.f) + (j == kb ? gd1 : 0.f);
}

// MonotonicAffineTransform (transforms.py:435-446): p = (shift, unconstrained log-scale)
ZK_HD void affine_backward_pair(const float* p, float x, float gy, float gl, float ad, float& gx,
                                float* gp) {
    const float a = p[1];
    const float e = expf(sc(a, ad));
    gx = gy * e;
    gp[0] = gy;
    gp[1] = fmaf(gy * x, e, gl) * dsc(a, ad);
}

// GaussianizationTransform (transforms.py:834-875): p = (b[K] shifts, a[K] log-scales), y = f(x)
// supplied by the caller (erfinv has no host form in the C++ library; the kernel evaluates it with
// the forward math of bijector_math.cuh, the CPU harness reads it from the goldens).  With
// s_k = exp(a_k), u_k = s_k x + b_k, t_k = a_k - u_k^2/2, L = logsumexp_k t_k, w_k = exp(t_k - L):
//     dy/db_k = exp(y^2/2 + log(c/K) - u_k^2/2) =: e_k,   dy/da_k = e_k s_k x,   dy/dx = J = exp(ladj)
//     ladj = y^2/2 + log(c/K) + L:
//     dladj/dx = y J - sum_k w_k u_k s_k,  dladj/db_k = y e_k - w_k u_k,  dladj/da_k = y e_k s_k x + w_k (1 - u_k s_k x)
template <bool FAST = false>
ZK_HD void gauss_backward_pair(const float* p, int K, float x, float y, float gy, float gl, float& gx,
                               float* gp) {
    float mx = -INFINITY;
    for (int k = 0; k < K; ++k) {
        const float u = fmaf(exp_<FAST>(p[K + k]), x, p[k]);
        mx = fmaxf(mx, fmaf(-0.5f * u, u, p[K + k]));
    }
    float se = 0.f;
    for (int k = 0; k < K; ++k) {
        const float u = fmaf(exp_<FAST>(p[K + k]), x, p[k]);
        se += exp_<FAST>(fmaf(-0.5f * u, u, p[K + k]) - mx);
    }
    const float L = mx + logf(se);
    const float h = fmaf(0.5f * y, y, logf((1.f - 1e-6f) / (float)K));  // y^2/2 + log(c/K)
    const float G = fmaf(gl, y, gy);                                     // gy + gl y
    float acc = 0.f;  // sum_k w_k u_k s_k
    for (int k = 0; k < K; ++k) {
        const float a = p[K + k];
        const float s = exp_<FAST>(a);
        const float u = fmaf(s, x, p[k]);
        const float t = fmaf(-0.5f * u, u, a);
        const float w = exp_<FAST>(t - L);
        const float e = exp_<FAST>(h + t - a);
        const float us = u * s;
        acc = fmaf(w, us, acc);
        gp[k] = fmaf(G, e, -gl * w * u);
        gp[K + k] = fmaf(G * e * s, x, gl * w * fmaf(-us, x, 1.f));
    }
    gx = fmaf(G, exp_<FAST>(h + L), -gl * acc);
}

}  // namespace bijgrad
}  // namespace zk
