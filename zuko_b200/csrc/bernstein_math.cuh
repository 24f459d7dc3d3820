// zuko_b200 — per-pair math of the bounded Bernstein polynomial bijector of BPF
// (BoundedBernsteinTransform, zuko/transforms.py:640-831; zuko/flows/polynomial.py:79-117).  Host/device
// code without CUDA headers: nvcc compiles it into uni_kernel, uni_bwd_kernel and ar_inverse_kernel,
// g++ into the CPU harness tests/native/bernstein_grad_host.cpp.
//
// A pair's P = degree + 1 parameters u are constrained to M + 1 = P + 5 rising coefficients
//     theta = cumsum([-B, db, db, softmax(u) dw, db, db]),   db = 2B / (P + 4),  dw = 2B - 4 db,
// whose M non-negative differences are Delta_1 .. Delta_M.  (Degree 0 keeps the reference's shape
// quirk: `ones_like(diffs[..., :2])` has one entry when P = 1, so theta = cumsum([-B, db, dw, db]),
// M = 3, and the polynomial ends at B - 2 db.)  With t = (x + B) / 2B (IEEE division in
// both math modes, so that the branch tests below pick the reference's branch):
//     eps < t < 1 - eps:  y = sum_i theta_i b_{i,M}(t) = -B + sum_i C_i b_{i,M}(t),  C_i = sum_{j<=i} Delta_j
//                         f'(x) = (M / 2B) sum_k Delta_{k+1} b_{k,M-1}(t)
//     t <= eps:           y = 2B (t - eps) - B          (f' = 1: ladj = 0)
//     t >= 1 - eps:       y = 2B (t - 1 + eps) + B
// so outside [-B, B] the map is x -+ 2B eps, not the identity.  The inverse returns the two linear
// branches exactly for y <= -B and y >= B, and otherwise bisects on [-B, B] with the full f.
//
// The Bernstein basis comes from the ratio recurrence b_{k+1,n} = b_{k,n} s (n - k) / (k + 1),
// s = t / (1 - t), started at b_{0,n} = (1 - t)^n: every term and every sum is non-negative.  For
// t > 1/2 the pair is evaluated mirrored, at 1 - t (exact there) with the differences reversed:
// y(t; Delta) = theta_M - B - y(1 - t; reversed Delta), so the recurrence always starts from the larger end.
#pragma once

#include <math.h>

#include "sosp_math.cuh"  // zk::bisect

#if defined(__CUDACC__)
#define ZK_BERN_HD __host__ __device__ __forceinline__
#else
#define ZK_BERN_HD inline
#endif

namespace zk {
namespace bern {

constexpr int kDefDegree = 16;          // BPF's default degree: the compile-time shape
constexpr int kDefP = kDefDegree + 1;   // 17 parameters per pair
constexpr int kMaxM = 64;               // runtime shapes: M = degree + 5 <= 64
constexpr int kMaxDegree = kMaxM - 5;   // 59
ZK_BERN_HD constexpr int ends_of(int P) { return P >= 2 ? 2 : 1; }     // fixed differences at each end
ZK_BERN_HD constexpr int order_of(int P) { return P + 2 * ends_of(P); }  // M
constexpr int kDefM = kDefP + 4;  // 21

// Everything a kernel needs besides the pair's parameters.
struct Const {
    int P = 0, M = 0;   // parameters per pair, polynomial order
    int iters = 0;      // bisection steps of the inverse
    float bound = 5.f, two_b = 10.f;
    float eps = 1e-6f, one_m_eps = 1.f - 1e-6f;  // branch thresholds on t; 1 - eps rounded from double
    float db = 0.f, dw = 0.f;                    // 2B / (P + 4) and 2B - 4 db
    float scale = 0.f;                           // M / 2B: f' per unit of the degree M - 1 sum
    float top = 5.f;                             // theta_M: B, or B - 2 db for degree 0
};

inline Const make_const(int degree, float bound, float eps, int iters) {
    Const c;
    c.P = degree + 1;
    c.M = order_of(c.P);
    c.iters = iters;
    c.bound = bound;
    c.two_b = (float)(2.0 * bound);
    c.eps = eps;
    c.one_m_eps = (float)(1.0 - (double)eps);
    c.db = (float)(2.0 * bound / (c.P + 4));
    c.dw = (float)(2.0 * bound - 4.0 * (2.0 * bound / (c.P + 4)));
    c.scale = (float)(c.M / (2.0 * bound));
    c.top = (float)(bound - (c.P >= 2 ? 0.0 : 2.0 * (2.0 * bound / (c.P + 4))));
    return c;
}

// Single-rounding fp32 operations that nvcc must not contract into FMAs: the linear branches and t
// reproduce the reference's fp32 expressions operation by operation.
ZK_BERN_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
ZK_BERN_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
ZK_BERN_HD float div_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
ZK_BERN_HD float t_of(const Const& c, float x) { return div_rn(add_rn(x, c.bound), c.two_b); }  // (x + B) / 2B

// The scaled softmax of a pair, Delta_{e+1} .. Delta_{M-e} (e = ends_of(P)): PT > 0 writes all PT of them to w; PT == 0
// returns the max and dw / sum so that delta() can form each one on the fly from u.  expf in both math modes:
// MUFU ex2 put a three-layer flow's z 1.1e-5 off its fp64 value, beyond the 1e-5 bar.
template <int PT>
ZK_BERN_HD void softmax(const float* u, const Const& c, float* w, float& mx, float& rs) {
    const int P = PT > 0 ? PT : c.P;
    mx = u[0];
#pragma unroll
    for (int p = 1; p < P; ++p) mx = fmaxf(mx, u[p]);
    float s = 0.f;
#pragma unroll
    for (int p = 0; p < P; ++p) {
        const float e = expf(u[p] - mx);
        if constexpr (PT > 0) w[p] = e;
        s += e;
    }
    rs = c.dw / s;
    if constexpr (PT > 0) {
#pragma unroll
        for (int p = 0; p < P; ++p) w[p] *= rs;
    }
}

// Delta_j, 1 <= j <= M, of a pair prepared by softmax<PT>
template <int PT>
ZK_BERN_HD float delta(const float* u, const float* w, const Const& c, float mx, float rs, int j) {
    const int M = PT > 0 ? order_of(PT) : c.M;
    const int e = PT > 0 ? ends_of(PT) : ends_of(c.P);
    if (j <= e || j > M - e) return c.db;
    if constexpr (PT > 0) return w[j - e - 1];
    return expf(u[j - e - 1] - mx) * rs;
}

ZK_BERN_HD float fmx(float a, float b, float c) { return fmaf(a, b, c); }
ZK_BERN_HD double fmx(double a, double b, double c) { return fma(a, b, c); }

// Scalar of the basis recurrences: fp64.  In fp32 the chain of M roundings drifts: 0.61 of the 1e-5
// value bar for one degree-16 pair, 1.5x it at degree 40, and past it in three-layer degree-16 flows.
template <int N>
using Real = double;

template <class T>
ZK_BERN_HD T ipow(T v, int n) {
    T r = 1;
#pragma unroll
    for (int e = n; e > 0; e >>= 1) {
        if (e & 1) r *= v;
        v *= v;
    }
    return r;
}

// For tt <= 1/2 (the caller mirrors), with Delta_j = dl(j):
//     sy = sum_i C_i b_{i,M}(tt)            (y = -B + sy)
//     sd = sum_k Delta_{k+1} b_{k,M-1}(tt)  (f' = scale sd)
// The degree M - 1 basis runs the ratio recurrence; each degree M value is one de Casteljau step of
// two neighbours, b_{i,M} = (1 - tt) b_{i,M-1} + tt b_{i-1,M-1}.
template <int MT, class Delta>
ZK_BERN_HD void sums(const Const& c, float t32, Delta dl, float& sy32, float& sd32) {
    using T = Real<MT>;
    const int M = MT > 0 ? MT : c.M;
    const T tt = t32, omt = T(1) - tt;
    const T s = tt / omt;
    T b = ipow(omt, M - 1);  // b_{0,M-1}
    T prev = 0, C = 0, sy = 0, sd = 0;
#pragma unroll
    for (int i = 0; i < M; ++i) {
        sy = fmx(fmx(omt, b, tt * prev), C, sy);
        const T d = dl(i + 1);
        sd = fmx(d, b, sd);
        C += d;
        prev = b;
        b *= s * (T(M - 1 - i) / T(i + 1));
    }
    sy32 = (float)fmx(tt * prev, C, sy);  // b_{M,M} = tt b_{M-1,M-1}
    sd32 = (float)sd;
}

// y = f(x); dfdx = f'(x) when the caller asks for it (1 in the linear branches)
template <int MT, class Delta>
ZK_BERN_HD float forward(const Const& c, float x, Delta dl, float* dfdx) {
    const float t = t_of(c, x);
    if (t <= c.eps) {
        if (dfdx) *dfdx = 1.f;
        return add_rn(mul_rn(c.two_b, add_rn(t, -c.eps)), -c.bound);
    }
    if (t >= c.one_m_eps) {
        if (dfdx) *dfdx = 1.f;
        return add_rn(mul_rn(c.two_b, add_rn(add_rn(t, -1.f), c.eps)), c.bound);
    }
    const int M = MT > 0 ? MT : c.M;
    const bool rev = t > 0.5f;
    float sy, sd;
    sums<MT>(c, rev ? 1.f - t : t, [&](int j) { return rev ? dl(M + 1 - j) : dl(j); }, sy, sd);
    if (dfdx) *dfdx = c.scale * sd;
    return rev ? c.top - sy : sy - c.bound;
}

// x = f^-1(y): the linear branches for y <= -B and y >= B, else the reference's bisection of the full f
template <int MT, class Delta>
ZK_BERN_HD float inverse(const Const& c, float y, Delta dl) {
    if (y <= -c.bound) {
        const float t = add_rn(div_rn(add_rn(y, c.bound), c.two_b), c.eps);
        return add_rn(mul_rn(2.f * t, c.bound), -c.bound);
    }
    if (y >= c.bound) {
        const float t = add_rn(add_rn(div_rn(add_rn(y, -c.bound), c.two_b), -c.eps), 1.f);
        return add_rn(mul_rn(2.f * t, c.bound), -c.bound);
    }
    return bisect(c.bound, c.iters, [&](float m) { return forward<MT>(c, m, dl, nullptr) < y; });
}

// Reverse mode of one pair, given dL/dy = gy and dL/dladj = gl, inside (-B, B):
//     dL/dx       = gy f' + gl f'' / f'
//     dL/dDelta_j = gy S_j + gl (M / 2B) b_{j-1,M-1} / f',   S_j = sum_{i>=j} b_{i,M}
//     dL/du_p     = Delta_{p+e+1} (dL/dDelta_{p+e+1} - sigma),  sigma = sum_q Delta_{q+e+1} dL/dDelta_{q+e+1} / dw
// (softmax through the scale dw).  In the linear branches dL/dx = gy and the parameters get 0.
// Three O(M) passes over the basis (degree M - 2 by recurrence, M - 1 and M by de Casteljau steps):
// f' and f'', then sigma, then the parameter gradients.  gp may alias u: u_p is read only in the
// last pass, right before gp[p] is written.
template <int PT>
ZK_BERN_HD void backward_pair(const float* u, const Const& c, float x, float gy, float gl, float& gx, float* gp) {
    const int P = PT > 0 ? PT : c.P;
    const int M = order_of(P), e = ends_of(P);
    const float t = t_of(c, x);
    if (t <= c.eps || t >= c.one_m_eps) {
        gx = gy;
#pragma unroll
        for (int p = 0; p < P; ++p) gp[p] = 0.f;
        return;
    }
    float w[PT > 0 ? PT : 1];
    float mx, rs;
    softmax<PT>(u, c, w, mx, rs);
    auto dl = [&](int j) { return delta<PT>(u, w, c, mx, rs, j); };
    using T = Real<PT>;
    const bool rev = t > 0.5f;
    const T tt = rev ? 1.f - t : t;
    const T omt = T(1) - tt;
    const T s = tt / omt;
    const T b0 = ipow(omt, M - 2);  // b_{0,M-2}
    // pass 1: sd = sum_k Delta'_{k+1} b_{k,M-1}, sdd = sum_k (Delta'_{k+2} - Delta'_{k+1}) b_{k,M-2}
    T sd = 0, sdd = 0;
    {
        T b2 = b0, p2 = 0;
        float dprev = rev ? dl(M) : dl(1);
#pragma unroll
        for (int i = 0; i < M; ++i) {
            const T b1 = fmx(omt, b2, tt * p2);  // b_{i,M-1}
            sd = fmx(T(dprev), b1, sd);
            if (i < M - 1) {
                const float dnext = rev ? dl(M - 1 - i) : dl(i + 2);
                sdd = fmx(T(dnext - dprev), b2, sdd);
                dprev = dnext;
            }
            p2 = b2;
            b2 = (i < M - 2) ? b2 * (s * (T(M - 2 - i) / T(i + 1))) : T(0);
        }
    }
    const float sgn = rev ? -1.f : 1.f;
    const float fp = c.scale * (float)sd;
    const float fpp = sgn * c.scale * ((float)(M - 1) / c.two_b) * (float)sdd;
    gx = fmaf(gy, fp, gl * fpp / fp);
    const float gys = gy * sgn, gls = gl / (float)sd;
    // passes 2 and 3: dL/dDelta'_j = gys S'_j + gls b_{j-1,M-1}, S'_j = 1 - sum_{i<j} b_{i,M}, for the
    // middle indices e < j <= M - e (Delta'_j = Delta_J, J = M + 1 - j when mirrored)
    float sigma = 0.f;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
        T b2 = b0, p2 = 0, p1 = 0, H = 0;
#pragma unroll
        for (int i = 0; i <= M; ++i) {
            const T b1 = fmx(omt, b2, tt * p2);  // b_{i,M-1} (0 at i = M)
            const T bm = fmx(omt, b1, tt * p1);  // b_{i,M}
            if (i > e && i <= M - e) {
                const float g = fmaf(gys, (float)(T(1) - H), gls * (float)p1);  // p1 = b_{i-1,M-1}
                const float d = rev ? dl(M + 1 - i) : dl(i);  // Delta_J: reads u[J - e - 1] before gp[J - e - 1] is written
                if (pass == 0) {
                    sigma = fmaf(d, g, sigma);
                } else {
                    gp[(rev ? M + 1 - i : i) - e - 1] = d * (g - sigma);
                }
            }
            H += bm;
            p1 = b1;
            p2 = b2;
            b2 = (i < M - 2) ? b2 * (s * (T(M - 2 - i) / T(i + 1))) : T(0);
        }
        if (pass == 0) sigma /= c.dw;
    }
}

}  // namespace bern
}  // namespace zk
