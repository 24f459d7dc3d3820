// zuko_b200 — per-row math of the Gaussian mixture model (zuko/mixtures.py:25-99 with Mixture,
// zuko/distributions.py:216-290).  Host/device code without CUDA headers: nvcc compiles it into the
// kernels of gmm.cu, g++ into the CPU harness tests/native/gmm_math_host.cpp.
//
// A row's parameters phi come in the reference's unpack order (mixtures.py:160-189), L = 1 if tied else K:
//     logits (K) | loc (K, D) | diag (L, Dd) | tril (L, D (D - 1) / 2)      (tril: full covariance only)
// with Dd = 1 for a spherical covariance, D otherwise.  Component k's scale matrix L_k is lower
// triangular with L_ii = exp(diag_i) + eps and, for a full covariance, tril scattered below the diagonal
// in torch.tril_indices(D, D, -1) order (row-major: (1,0), (2,0), (2,1), ...; entry (i, j) at
// i (i - 1) / 2 + j).  Diagonal and spherical covariances are the same matrices without the tril.
//     v_k = L_k^-1 (x - mu_k)                         forward substitution
//     log p_k(x) = -1/2 (D log 2 pi + |v_k|^2) - sum_i log L_k,ii
//     t_k = log_softmax(logits)_k + log p_k(x),   log p(x) = logsumexp_k t_k
// Reverse mode of log p(x) for an upstream gradient g, with r_k = g softmax(t)_k and w_k = L_k^-T v_k:
//     dx = -sum_k r_k w_k,   dmu_k = r_k w_k,   dlogits = r - g softmax(logits)
//     dL_k = r_k (w_k v_k^T - diag(1 / L_k,ii)) on the lower triangle,   ddiag_i = dL_ii exp(diag_i)
// (spherical: ddiag sums dL_ii over i; tied: the covariance gradients sum over k).
// Sampling from a uniform u and a standard normal z: the component is the first k whose fixed-order
// running sum of softmax(logits) exceeds u (when rounding leaves u at or above the sum of the first K - 1,
// the last component whose fp32 weight is positive: a zero weight is never drawn), and x = mu_k + L_k z.
//
// Per-row vectors (v, w, t) live behind a stride so the kernels can keep them in shared memory, one
// column per thread.
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define ZK_GMM_HD __host__ __device__ __forceinline__
#else
#define ZK_GMM_HD inline
#endif

namespace zk {
namespace gmm {

constexpr int kMaxD = 64;  // features covered by the kernels
constexpr int kMaxK = 32;  // components covered by the kernels
constexpr float kLog2Pi = 1.8378770664093453f;

enum { kFull = 0, kDiagonal = 1, kSpherical = 2 };  // ZK_COV_*

// offsets of a phi row
struct Layout {
    int D = 0, K = 0, cov = kFull, tied = 0;
    int nd = 0, nt = 0;          // diag / tril entries per covariance
    int loc = 0, diag = 0, tril = 0, total = 0;
};

ZK_GMM_HD Layout make_layout(int D, int K, int cov, int tied) {
    Layout l;
    l.D = D; l.K = K; l.cov = cov; l.tied = tied;
    l.nd = (cov == kSpherical) ? 1 : D;
    l.nt = (cov == kFull) ? D * (D - 1) / 2 : 0;
    const int L = tied ? 1 : K;
    l.loc = K;
    l.diag = K + K * D;
    l.tril = l.diag + L * l.nd;
    l.total = l.tril + L * l.nt;
    return l;
}

ZK_GMM_HD int tril_index(int i, int j) { return i * (i - 1) / 2 + j; }

// logsumexp over n values a[0], a[s], ... (max first, then the sum of the shifted exponentials, as torch)
ZK_GMM_HD float lse(const float* a, int s, int n) {
    float m = a[0];
    for (int k = 1; k < n; ++k) m = fmaxf(m, a[k * s]);
    if (isinf(m)) return m;
    float acc = 0.f;
    for (int k = 0; k < n; ++k) acc += expf(a[k * s] - m);
    return m + logf(acc);
}

// L_ii of component k's covariance parameters dg (nd entries)
ZK_GMM_HD float scale_at(const float* dg, const Layout& l, int i, float eps) {
    return expf(dg[l.cov == kSpherical ? 0 : i]) + eps;
}

// v = L^-1 (x - mu); returns log p_k(x)
ZK_GMM_HD float component_log_density(const float* x, const float* mu, const float* dg, const float* tl,
                                      const Layout& l, float eps, float* v, int vs) {
    float sq = 0.f, logdet = 0.f;
    for (int i = 0; i < l.D; ++i) {
        float e = x[i] - mu[i];
        if (l.cov == kFull)
            for (int j = 0; j < i; ++j) e -= tl[tril_index(i, j)] * v[j * vs];
        const float s = scale_at(dg, l, i, eps);
        const float vi = e / s;
        v[i * vs] = vi;
        sq += vi * vi;
        logdet += logf(s);
    }
    return -0.5f * ((float)l.D * kLog2Pi + sq) - logdet;
}

// w = L^-T v (back substitution)
ZK_GMM_HD void solve_transpose(const float* v, int vs, const float* dg, const float* tl, const Layout& l,
                               float eps, float* w, int ws) {
    for (int i = l.D - 1; i >= 0; --i) {
        float e = v[i * vs];
        if (l.cov == kFull)
            for (int j = i + 1; j < l.D; ++j) e -= tl[tril_index(j, i)] * w[j * ws];
        w[i * ws] = e / scale_at(dg, l, i, eps);
    }
}

ZK_GMM_HD const float* cov_diag(const float* phi, const Layout& l, int k) { return phi + l.diag + (l.tied ? 0 : k) * l.nd; }
ZK_GMM_HD const float* cov_tril(const float* phi, const Layout& l, int k) { return phi + l.tril + (l.tied ? 0 : k) * l.nt; }

// log p(x) of one row; t[k * ts] receives t_k
ZK_GMM_HD float row_log_prob(const float* x, const float* phi, const Layout& l, float eps, float* v, int vs,
                             float* t, int ts) {
    const float zl = lse(phi, 1, l.K);
    for (int k = 0; k < l.K; ++k)
        t[k * ts] = (phi[k] - zl) +
                    component_log_density(x, phi + l.loc + k * l.D, cov_diag(phi, l, k), cov_tril(phi, l, k), l, eps, v, vs);
    return lse(t, ts, l.K);
}

// Reverse mode of row_log_prob for the upstream gradient g.  Writes gx (D, may be null) and the row's
// gradient gphi (l.total entries, never aliasing phi); returns log p(x).
ZK_GMM_HD float row_backward(const float* x, const float* phi, const Layout& l, float eps, float g, float* gx,
                             float* gphi, float* v, int vs, float* w, int ws, float* t, int ts) {
    const float out = row_log_prob(x, phi, l, eps, v, vs, t, ts);
    const float zl = lse(phi, 1, l.K);
    if (gx)
        for (int i = 0; i < l.D; ++i) gx[i] = 0.f;
    if (l.tied)
        for (int i = l.diag; i < l.total; ++i) gphi[i] = 0.f;
    for (int k = 0; k < l.K; ++k) {
        const float rk = expf(t[k * ts] - out);
        const float r = g * rk;
        gphi[k] = g * (rk - expf(phi[k] - zl));
        const float* mu = phi + l.loc + k * l.D;
        const float* dg = cov_diag(phi, l, k);
        const float* tl = cov_tril(phi, l, k);
        component_log_density(x, mu, dg, tl, l, eps, v, vs);
        solve_transpose(v, vs, dg, tl, l, eps, w, ws);
        float* gmu = gphi + l.loc + k * l.D;
        float* gdg = gphi + l.diag + (l.tied ? 0 : k) * l.nd;
        float* gtl = gphi + l.tril + (l.tied ? 0 : k) * l.nt;
        float sph = 0.f;
        for (int i = 0; i < l.D; ++i) {
            const float wi = w[i * ws], vi = v[i * vs];
            gmu[i] = r * wi;
            if (gx) gx[i] -= r * wi;
            const float s = scale_at(dg, l, i, eps);
            const float dL = r * (wi * vi - 1.f / s);
            if (l.cov == kSpherical) {
                sph += dL;
            } else {
                const float d = dL * expf(dg[i]);
                gdg[i] = l.tied ? gdg[i] + d : d;
            }
            if (l.cov == kFull)
                for (int j = 0; j < i; ++j) {
                    const float d2 = r * wi * v[j * vs];
                    float& o = gtl[tril_index(i, j)];
                    o = l.tied ? o + d2 : d2;
                }
        }
        if (l.cov == kSpherical) {
            const float d = sph * expf(dg[0]);
            gdg[0] = l.tied ? gdg[0] + d : d;
        }
    }
    return out;
}

// the component u selects; never one whose fp32 weight is zero (for u >= 0 the running sum only passes
// u at a positive weight, and the fallback is the last positive weight, not component K - 1)
ZK_GMM_HD int select_component(const float* logits, int K, float u) {
    const float zl = lse(logits, 1, K);
    float c = 0.f;
    int last = 0;
    for (int k = 0; k < K; ++k) {
        const float p = expf(logits[k] - zl);
        if (p > 0.f) last = k;
        c += p;
        if (k < K - 1 && u < c) return k;
    }
    return last;
}

// x = mu_k + L_k z for the component u selects
ZK_GMM_HD void row_sample(const float* phi, const Layout& l, float eps, float u, const float* z, float* x) {
    const int k = select_component(phi, l.K, u);
    const float* mu = phi + l.loc + k * l.D;
    const float* dg = cov_diag(phi, l, k);
    const float* tl = cov_tril(phi, l, k);
    for (int i = 0; i < l.D; ++i) {
        float acc = mu[i];
        if (l.cov == kFull)
            for (int j = 0; j < i; ++j) acc += tl[tril_index(i, j)] * z[j];
        x[i] = acc + scale_at(dg, l, i, eps) * z[i];
    }
}

}  // namespace gmm
}  // namespace zk
