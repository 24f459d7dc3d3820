// zuko_b200 — activation functions of the conditioner (zuko/nn.py:160-192, 258-318: any
// `activation()` module between the linear layers; the engine implements torch's defaults of the
// element-wise ones below).  Internal codes: 0 = none, 1 = ReLU, >= 2 = ZK_ACT_* of the C ABI.
#pragma once

#include <math.h>

#include "../../include/zuko_b200.h"

#if defined(__CUDACC__)
#define ZK_ACT_HD __host__ __device__ __forceinline__
#else
#define ZK_ACT_HD inline
#endif

namespace zk {

ZK_ACT_HD float act_apply(float v, int act) {
    switch (act) {
        case 1: return fmaxf(v, 0.f);                                  // torch.nn.ReLU
        case ZK_ACT_ELU: return v > 0.f ? v : expm1f(v);               // ELU(alpha=1)
        case ZK_ACT_TANH: return tanhf(v);                             // Tanh
        case ZK_ACT_SILU: return v / (1.f + expf(-v));                 // SiLU
        case ZK_ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));  // GELU(approximate='none')
        case ZK_ACT_LEAKY_RELU: return v > 0.f ? v : 0.01f * v;        // LeakyReLU(0.01)
        case ZK_ACT_SOFTPLUS: return v > 20.f ? v : log1pf(expf(v));   // Softplus(beta=1, threshold=20)
        case ZK_ACT_SIGMOID: return 1.f / (1.f + expf(-v));            // Sigmoid
        default: return v;
    }
}

// the same over N values with ONE switch outside the loops (inside an unrolled epilogue a per-element
// switch multiplies the code size and slows the epilogue through the instruction cache)
template <int N>
ZK_ACT_HD void act_apply_n(float (&v)[N], int act) {
    switch (act) {
        case 1:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = fmaxf(v[i], 0.f);
            break;
        case ZK_ACT_ELU:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = v[i] > 0.f ? v[i] : expm1f(v[i]);
            break;
        case ZK_ACT_TANH:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = tanhf(v[i]);
            break;
        case ZK_ACT_SILU:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = v[i] / (1.f + expf(-v[i]));
            break;
        case ZK_ACT_GELU:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = 0.5f * v[i] * (1.f + erff(v[i] * 0.70710678118654752f));
            break;
        case ZK_ACT_LEAKY_RELU:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = v[i] > 0.f ? v[i] : 0.01f * v[i];
            break;
        case ZK_ACT_SOFTPLUS:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = v[i] > 20.f ? v[i] : log1pf(expf(v[i]));
            break;
        case ZK_ACT_SIGMOID:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = 1.f / (1.f + expf(-v[i]));
            break;
        default: break;
    }
}

#if defined(__CUDACC__)
// MUFU forms for the fast-math kernels (zk_set_fast_math(1), the default): ex2 / rcp / lg2 approximations,
// absolute error ~1e-7 on activations of magnitude O(1) — far inside the 1e-5 bar on log_prob that the
// split-bf16 products set.  GELU keeps erff (no cheap form at that accuracy); ReLU / LeakyReLU are exact.
template <int N>
__device__ __forceinline__ void act_apply_n_fast(float (&v)[N], int act) {
    auto ex2 = [](float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; };
    auto rcp = [](float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; };
    auto lg2 = [](float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; };
    constexpr float kL2E = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
    switch (act) {
        case ZK_ACT_ELU:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = v[i] > 0.f ? v[i] : ex2(v[i] * kL2E) - 1.f;
            break;
        case ZK_ACT_TANH:  // 1 - 2 / (1 + e^{2 v}); e^{2 v} saturates cleanly to 0 / inf
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = 1.f - 2.f * rcp(1.f + ex2(v[i] * (2.f * kL2E)));
            break;
        case ZK_ACT_SILU:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = v[i] * rcp(1.f + ex2(-v[i] * kL2E));
            break;
        case ZK_ACT_SOFTPLUS:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = v[i] > 20.f ? v[i] : lg2(1.f + ex2(v[i] * kL2E)) * kLn2;
            break;
        case ZK_ACT_SIGMOID:
#pragma unroll
            for (int i = 0; i < N; ++i) v[i] = rcp(1.f + ex2(-v[i] * kL2E));
            break;
        default: act_apply_n<N>(v, act); break;
    }
}
#endif

// d act(v) / dv at the PRE-activation v
ZK_ACT_HD float act_deriv(float v, int act) {
    switch (act) {
        case 1: return v > 0.f ? 1.f : 0.f;
        case ZK_ACT_ELU: return v > 0.f ? 1.f : expf(v);
        case ZK_ACT_TANH: { const float t = tanhf(v); return 1.f - t * t; }
        case ZK_ACT_SILU: { const float s = 1.f / (1.f + expf(-v)); return s * (1.f + v * (1.f - s)); }
        case ZK_ACT_GELU:
            return 0.5f * (1.f + erff(v * 0.70710678118654752f)) + v * expf(-0.5f * v * v) * 0.39894228040143268f;
        case ZK_ACT_LEAKY_RELU: return v > 0.f ? 1.f : 0.01f;
        case ZK_ACT_SOFTPLUS: return v > 20.f ? 1.f : 1.f / (1.f + expf(-v));
        case ZK_ACT_SIGMOID: { const float s = 1.f / (1.f + expf(-v)); return s * (1.f - s); }
        default: return 1.f;
    }
}

// d^2 act(v) / dv^2 at the PRE-activation v, with torch's double-backward conventions at the kinks (ELU's is 0
// at v = 0, Softplus is linear above its threshold)
ZK_ACT_HD float act_deriv2(float v, int act) {
    switch (act) {
        case ZK_ACT_ELU: return v >= 0.f ? 0.f : expf(v);
        case ZK_ACT_TANH: { const float t = tanhf(v); return -2.f * t * (1.f - t * t); }
        case ZK_ACT_SILU: { const float s = 1.f / (1.f + expf(-v)); return s * (1.f - s) * (2.f + v * (1.f - 2.f * s)); }
        case ZK_ACT_GELU: return expf(-0.5f * v * v) * 0.39894228040143268f * (2.f - v * v);
        case ZK_ACT_SOFTPLUS: { if (v > 20.f) return 0.f; const float s = 1.f / (1.f + expf(-v)); return s * (1.f - s); }
        case ZK_ACT_SIGMOID: { const float s = 1.f / (1.f + expf(-v)); return s * (1.f - s) * (1.f - 2.f * s); }
        default: return 0.f;  // ReLU, LeakyReLU, identity
    }
}

}  // namespace zk
