// zuko_b200 — per-pair math of the sum-of-squares polynomial bijector: SOSPolynomialTransform followed
// by AdditiveTransform (ShiftedSOSPTransform, zuko/flows/polynomial.py:23-28; transforms.py:878-963,
// utils.py:118-363).  Host/device code in plain fp32 FMAs: nvcc compiles it into uni_kernel,
// uni_bwd_kernel and ar_inverse_kernel, g++ into the CPU harness tests/native/sosp_grad_host.cpp.
//
// A pair's P = K (L + 1) + 1 parameters are a[K][L + 1] (row-major) then the additive constant.  With
// v = u / B:
//     p_k(u) = 1 + sum_j a_kj v^j,      g(u) = (1/K) sum_k p_k(u)^2 + slope
//     y = x sum_i w_i g(t_i x) + constant        (n = L + 1 Gauss-Legendre nodes on [0, 1]: exact for
//                                                 g of degree 2L, as in GaussLegendre.quadrature)
//     ladj = log g(x)                            (UnconstrainedMonotonicTransform.call_and_ladj)
// The inverse subtracts the constant and bisects on [-B, B] (MonotonicTransform._inverse).
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define ZK_SOSP_HD __host__ __device__ __forceinline__
#else
#define ZK_SOSP_HD inline
#endif

namespace zk {

// The reference's bisection (utils.py:159-183): `iters` halvings of [-bound, bound] on the test
// below(m) = "f(m) < y"; returns the midpoint of the final interval.  A y beyond the range of f
// therefore returns +-(bound - half the final interval).
template <class Below>
ZK_SOSP_HD float bisect(float bound, int iters, Below below) {
    float lo = -bound, hi = bound;
    for (int it = 0; it < iters; ++it) {
        const float m = 0.5f * (lo + hi);
        const bool b = below(m);
        lo = b ? m : lo;
        hi = b ? hi : m;
    }
    return 0.5f * (lo + hi);
}

namespace sosp {

constexpr int kMaxNodes = 16;  // degree L <= 15
constexpr int kDefK = 3;       // SOSPF defaults (polynomials, degree): P = 16, the compile-time shape
constexpr int kDefL = 4;
constexpr int kDefP = kDefK * (kDefL + 1) + 1;

// Everything a kernel needs besides the pair's parameters.  The quadrature is pre-scaled on the host:
// tb_i = t_i / B turns a node into v directly, wk_i = w_i / K folds the mean over the polynomials in.
struct Const {
    int K = 0, L = 0;  // polynomials, degree
    int iters = 0;     // bisection steps of the inverse
    float bound = 10.f, inv_bound = 0.1f, slope = 1e-3f, inv_k = 1.f;
    float tb[kMaxNodes] = {};
    float wk[kMaxNodes] = {};
};

// n-point Gauss-Legendre nodes and weights on [-1, 1] (Newton on P_n from the Chebyshev-like initial
// guesses, ascending, symmetrised like numpy.polynomial.legendre.leggauss), mapped to [0, 1]:
// t = (x + 1) / 2, w = w / 2 (GaussLegendre.nodes).  Host only, double precision.
inline void gauss_legendre01(int n, double* t, double* w) {
    const double pi = 3.14159265358979323846;
    double x[kMaxNodes], wt[kMaxNodes];
    for (int i = 0; i < n; ++i) {
        double z = -cos(pi * (i + 0.75) / (n + 0.5));
        double dp = 1.0;
        for (int it = 0; it < 100; ++it) {
            double p0 = 1.0, p1 = z;  // P_0, P_1
            for (int k = 2; k <= n; ++k) {
                const double p2 = ((2 * k - 1) * z * p1 - (k - 1) * p0) / k;
                p0 = p1;
                p1 = p2;
            }
            dp = n * (z * p1 - p0) / (z * z - 1.0);  // P_n'(z)
            const double dz = p1 / dp;
            z -= dz;
            if (fabs(dz) <= 1e-15) {  // quadratic convergence: z is now exact to rounding
                p0 = 1.0, p1 = z;
                for (int k = 2; k <= n; ++k) {
                    const double p2 = ((2 * k - 1) * z * p1 - (k - 1) * p0) / k;
                    p0 = p1;
                    p1 = p2;
                }
                dp = n * (z * p1 - p0) / (z * z - 1.0);
                break;
            }
        }
        x[i] = z;
        wt[i] = 2.0 / ((1.0 - z * z) * dp * dp);
    }
    for (int i = 0; i < n; ++i) {
        const double xs = 0.5 * (x[i] - x[n - 1 - i]), ws = 0.5 * (wt[i] + wt[n - 1 - i]);
        t[i] = 0.5 * (xs + 1.0);
        w[i] = 0.5 * ws;
    }
}

inline Const make_const(int K, int L, float bound, float slope, int iters) {
    Const c;
    c.K = K; c.L = L; c.iters = iters; c.bound = bound; c.slope = slope;
    c.inv_bound = (float)(1.0 / bound);
    c.inv_k = (float)(1.0 / K);
    double t[kMaxNodes], w[kMaxNodes];
    gauss_legendre01(L + 1, t, w);
    for (int i = 0; i <= L; ++i) {
        c.tb[i] = (float)(t[i] / bound);
        c.wk[i] = (float)(w[i] / K);
    }
    return c;
}

// KT > 0: the compile-time default shape (kDefK, kDefL), every loop unrolled and the caller's
// parameters in registers; KT == 0: K and L from `c`, the node loops unrolled to kMaxNodes with a
// guard so that the node tables are only ever indexed by constants.
#define ZK_SOSP_SHAPE                   \
    const int K = KT > 0 ? kDefK : c.K; \
    const int L = KT > 0 ? kDefL : c.L; \
    const int n = L + 1;                \
    (void)K
template <int KT>
constexpr int kNodeSlots = KT > 0 ? kDefL + 1 : kMaxNodes;  // unrolled node loop length

// sum_k p_k(v)^2, each p_k by Horner in v
template <int KT>
ZK_SOSP_HD float sq_sum(const float* a, const Const& c, float v) {
    ZK_SOSP_SHAPE;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float* ak = a + k * n;
        float h = ak[L];
#pragma unroll
        for (int j = L - 1; j >= 0; --j) h = fmaf(h, v, ak[j]);
        const float p = 1.f + h;
        s = fmaf(p, p, s);
    }
    return s;
}

// g(x), the derivative of the forward map
template <int KT>
ZK_SOSP_HD float g(const float* a, const Const& c, float x) {
    return fmaf(sq_sum<KT>(a, c, x * c.inv_bound), c.inv_k, c.slope);
}

// x sum_i w_i g(t_i x): the forward map without its constant
template <int KT>
ZK_SOSP_HD float integral(const float* a, const Const& c, float x) {
    ZK_SOSP_SHAPE;
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < kNodeSlots<KT>; ++i)
        if (i < n) acc = fmaf(c.wk[i], sq_sum<KT>(a, c, c.tb[i] * x), acc);
    return x * (acc + c.slope);
}

// y = f(x) and g(x) (the caller takes its log: ladj)
template <int KT>
ZK_SOSP_HD float forward(const float* a, const Const& c, float x, float& gx) {
    ZK_SOSP_SHAPE;
    gx = g<KT>(a, c, x);
    return integral<KT>(a, c, x) + a[K * n];
}

// x = f^-1(y): y - constant, then the bisection on [-B, B]
template <int KT>
ZK_SOSP_HD float inverse(const float* a, const Const& c, float y) {
    ZK_SOSP_SHAPE;
    const float t = y - a[K * n];
    return bisect(c.bound, c.iters, [&](float m) { return integral<KT>(a, c, m) < t; });
}

// Reverse mode of one pair, given dL/dy = gy and dL/dladj = gl:
//     dy/dx = g(x),  dy/dconstant = 1,  dy/da_kj = x sum_i w_i (2/K) p_k(t_i x) (t_i x / B)^j
//     dladj/dx = g'(x) / g(x),  dladj/da_kj = (2/K) p_k(x) (x / B)^j / g(x)
// (GaussLegendre.backward gives dy/dx = g(x), not the derivative of the quadrature.)  gp may alias a:
// every row is read before it is written, and no row is read after it was written.
template <int KT>
ZK_SOSP_HD void backward_pair(const float* a, const Const& c, float x, float gy, float gl, float& gx, float* gp) {
    ZK_SOSP_SHAPE;
    constexpr int NU = kNodeSlots<KT>;
    const float v = x * c.inv_bound;
    float s = 0.f, ds = 0.f;  // sum_k p_k^2, sum_k p_k dp_k/dv
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float* ak = a + k * n;
        float h = ak[L], dh = 0.f;
#pragma unroll
        for (int j = L - 1; j >= 0; --j) {
            dh = fmaf(dh, v, h);
            h = fmaf(h, v, ak[j]);
        }
        const float p = 1.f + h;
        s = fmaf(p, p, s);
        ds = fmaf(p, dh, ds);
    }
    const float gv = fmaf(s, c.inv_k, c.slope);
    const float rg = 1.f / gv;
    gx = fmaf(gy, gv, gl * (2.f * ds * c.inv_k * c.inv_bound) * rg);
    const float cy = 2.f * gy * x;            // dy/da_kj = cy' sum_i wk_i p_k(v_i) v_i^j
    const float cl = 2.f * gl * c.inv_k * rg;  // dladj/da_kj = cl' p_k(x) v^j
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float* ak = a + k * n;
        float q[NU], vi[NU], pw[NU];
#pragma unroll
        for (int i = 0; i < NU; ++i) {
            vi[i] = 0.f;
            q[i] = 0.f;
            pw[i] = 1.f;
            if (i < n) {
                vi[i] = c.tb[i] * x;
                float h = ak[L];
#pragma unroll
                for (int j = L - 1; j >= 0; --j) h = fmaf(h, vi[i], ak[j]);
                q[i] = c.wk[i] * (1.f + h);
            }
        }
        float h = ak[L];
#pragma unroll
        for (int j = L - 1; j >= 0; --j) h = fmaf(h, v, ak[j]);
        const float px = cl * (1.f + h);
        float pv = 1.f;
#pragma unroll
        for (int j = 0; j < n; ++j) {
            float acc = 0.f;
#pragma unroll
            for (int i = 0; i < NU; ++i) {
                if (i < n) {
                    acc = fmaf(q[i], pw[i], acc);
                    pw[i] *= vi[i];
                }
            }
            gp[k * n + j] = fmaf(cy, acc, px * pv);
            pv *= v;
        }
    }
    gp[K * n] = gy;
}

#undef ZK_SOSP_SHAPE

}  // namespace sosp
}  // namespace zk
