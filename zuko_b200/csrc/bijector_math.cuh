// zuko_b200 — device math of the univariate bijectors (shared by the stand-alone fused
// bijector kernel in bijectors.cu and the fully fused layer kernel in fused_layer.cu).
#pragma once

#include "common.cuh"
#include "bernstein_math.cuh"
#include "sosp_math.cuh"

namespace zk {
namespace bij {

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kHalfLog2Pi = 0.9189385332046727f;

// ---------------------------------------------------------------------------
// scalar math, FAST = MUFU approximations (rcp / ex2 / lg2), else IEEE
// ---------------------------------------------------------------------------
// The MUFU approximations are issued in their .ftz form through inline PTX: the plain
// `__fdividef` / `exp2f` / `__log2f` intrinsics compile (without -ftz=true) to the MUFU plus a
// predicated rescaling sequence for denormal operands — FSETP + 2-3 FMUL around every one of the
// ~43 MUFUs of a spline evaluation, a quarter of its instructions.  None of the operands here can
// be denormal: soft-clip denominators are >= 1, softmax sums >= K * slope^(1/2), bin widths and
// the rational's denominator are bounded below through the min-slope 1e-3, exponents lie in
// [-10, 10].
__device__ __forceinline__ float rcp_ftz(float v) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}
__device__ __forceinline__ float ex2_ftz(float v) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}
__device__ __forceinline__ float lg2_ftz(float v) {
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}
template <bool FAST>
__device__ __forceinline__ float zrcp(float b) {
    if constexpr (FAST) return rcp_ftz(b);
    return 1.0f / b;
}
template <bool FAST>
__device__ __forceinline__ float zdiv(float a, float b) {
    if constexpr (FAST) return a * rcp_ftz(b);
    return a / b;
}
template <bool FAST>
__device__ __forceinline__ float zexp(float v) {
    if constexpr (FAST) return ex2_ftz(v * kLog2e);
    return expf(v);
}
template <bool FAST>
__device__ __forceinline__ float zlog(float v) {
    if constexpr (FAST) return lg2_ftz(v) * kLn2;
    return logf(v);
}
// v / (1 + |v| * a)   — the soft clip of transforms.py:480-482 with a = 2/|ln slope| (w, h)
// or 1/|ln slope| (derivatives, affine log-scale)
template <bool FAST>
__device__ __forceinline__ float softclip(float v, float a) {
    return zdiv<FAST>(v, fmaf(fabsf(v), a, 1.0f));
}

// CircularShiftTransform: remainder(x, 2B) - B with torch.remainder's sign convention
// (transforms.py:344-348; result of the remainder in [0, 2B))
__device__ __forceinline__ float circ_shift(float x, float bound) {
    const float m = 2.f * bound;
    float r = fmodf(x, m);
    if (r != 0.f && r < 0.f) r += m;
    return r - bound;
}

// ---------------------------------------------------------------------------
// RQS: select the bin and its six knot values in one sweep over the K bins.
// p points at this pair's P = 3K-1 raw parameters in shared memory:
//   p[0..K) widths, p[K..2K) heights, p[2K..3K-1) derivatives
// (flows/autoregressive.py:149,212-213; flows/spline.py:57).
// SEARCH_Y = false searches the horizontal knots (forward, transforms.py:555),
// true the vertical ones (inverse, transforms.py:535).
// ---------------------------------------------------------------------------
struct Bin {
    float x0, y0;  // left knot of the selected bin
    float dx, dy;  // bin width / height, formed directly from the softmax numerators:
                   // bound * 2 * softmax_k, i.e. WITHOUT the cancellation of knot_{k+1} - knot_k
                   // (transforms.py:505-509 subtracts two rounded knots; for a sharp spline
                   // that costs up to ulp(5)/width in the slope s — here it costs ~1 ulp)
    float d0, d1;
    bool inside;
};

template <int KT, bool FAST, bool SEARCH_Y>
__device__ __forceinline__ Bin rqs_select(const float* __restrict__ p, int Krt, float v, float bound,
                                          float aw, float ad) {
    const int K = KT > 0 ? KT : Krt;
    constexpr int KA = KT > 0 ? KT : 1;
    float ew[KA], eh[KA];
    float sw = 0.f, sh = 0.f;
    // softmax numerators.  The soft-clipped logits lie in (-|ln slope|/2, |ln slope|/2) =
    // (-3.46, 3.46), so exp cannot overflow and the max-subtraction of torch's softmax
    // (transforms.py:484-485) is mathematically a no-op that we skip.
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float e0 = zexp<FAST>(softclip<FAST>(p[k], aw));
        float e1 = zexp<FAST>(softclip<FAST>(p[K + k], aw));
        if constexpr (KT > 0) {
            ew[k] = e0;
            eh[k] = e1;
        }
        sw += e0;
        sh += e1;
    }
    // knots = bound * (2 * cumsum(softmax) - 1)  (transforms.py:488-489), evaluated as
    // fma(cum_raw, 2*bound/sum, -bound)
    const float gx = zdiv<FAST>(2.f * bound, sw);
    const float gy = zdiv<FAST>(2.f * bound, sh);
    float cw = 0.f, ch = 0.f;
    float xl = -bound, yl = -bound, rl = 0.f;  // left knot of the current bin, raw derivative
    Bin b;
    b.x0 = xl; b.y0 = yl; b.dx = 0.f; b.dy = 0.f;
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        float e0, e1;
        if constexpr (KT > 0) {
            e0 = ew[j];
            e1 = eh[j];
        } else {
            e0 = zexp<FAST>(softclip<FAST>(p[j], aw));
            e1 = zexp<FAST>(softclip<FAST>(p[K + j], aw));
        }
        cw += e0;
        ch += e1;
        const float xr = fmaf(cw, gx, -bound);
        const float yr = fmaf(ch, gy, -bound);
        const float rr = (j < K - 1) ? p[2 * K + j] : 0.f;  // pad (1,1) with 0, transforms.py:486
        // knots are non-decreasing, so "last bin whose left knot is < v" equals
        // sum_j [knot_j < v] - 1 of transforms.py:521-523 (strict <)
        const bool take = (j == 0) || ((SEARCH_Y ? yl : xl) < v);
        b.x0 = take ? xl : b.x0;
        b.y0 = take ? yl : b.y0;
        b.dx = take ? e0 : b.dx;
        b.dy = take ? e1 : b.dy;
        r0 = take ? rl : r0;
        r1 = take ? rr : r1;
        xl = xr;
        yl = yr;
        rl = rr;
    }
    // mask = 0 <= k < K (transforms.py:500): first knot (-bound) < v and NOT last knot < v
    b.inside = (-bound < v) && !((SEARCH_Y ? yl : xl) < v);
    b.dx *= gx;
    b.dy *= gy;
    b.d0 = zexp<FAST>(softclip<FAST>(r0, ad));  // transforms.py:482,490 (exp(0) = 1 at the ends)
    b.d1 = zexp<FAST>(softclip<FAST>(r1, ad));
    return b;
}

// forward spline + log-derivative, transforms.py:554-567
template <bool FAST>
__device__ __forceinline__ void rqs_forward_eval(const Bin& b, float x, float& y, float& ladj) {
    const float dx = b.dx, dy = b.dy;
    float s, z;
    if constexpr (FAST) {  // one reciprocal of the bin width serves the slope and the position
        const float rdx = rcp_ftz(dx);
        s = dy * rdx;
        z = (x - b.x0) * rdx;
    } else {
        s = dy / dx;
        z = (x - b.x0) / dx;
    }
    const float omz = 1.f - z;
    const float z1 = z * omz;
    const float den = fmaf(b.d0 + b.d1 - 2.f * s, z1, s);
    const float num = fmaf(s * z, z, b.d0 * z1);
    const float jn = s * s * (2.f * s * z1 + b.d0 * omz * omz + b.d1 * z * z);
    float yy, lj;
    if constexpr (FAST) {  // and one reciprocal of the denominator serves y and the Jacobian
        const float rden = rcp_ftz(den);
        yy = fmaf(dy, num * rden, b.y0);
        lj = lg2_ftz(jn * rden * rden) * kLn2;
    } else {
        yy = fmaf(dy, num / den, b.y0);
        lj = logf(jn / (den * den));
    }
    y = b.inside ? yy : x;
    // outside the domain the reference yields mask * log(jac) = 0 for finite x and NaN for
    // non-finite x (0 * inf); (x - x) reproduces exactly that.
    ladj = b.inside ? lj : (x - x);
}

// inverse spline, transforms.py:534-548
template <bool FAST>
__device__ __forceinline__ float rqs_inverse_eval(const Bin& b, float y) {
    const float dx = b.dx, dy = b.dy;
    const float s = zdiv<FAST>(dy, dx);
    const float y_ = y - b.y0;
    const float t = b.d0 + b.d1 - 2.f * s;
    const float qa = fmaf(dy, s - b.d0, y_ * t);
    const float qb = fmaf(dy, b.d0, -y_ * t);
    const float qc = -s * y_;
    const float disc = fmaf(qb, qb, -4.f * qa * qc);
    const float z = zdiv<FAST>(2.f * qc, -qb - sqrtf(disc));
    const float x = fmaf(z, dx, b.x0);
    return b.inside ? x : y;
}

// ---------------------------------------------------------------------------
// Gaussianization: f(x) = sqrt2 erfinv(c/K sum_k erf(u_k / sqrt2)), u_k = exp(a_k) x + b_k,
// c = 1 - 1e-6 (GaussianizationTransform.f, transforms.py:867-873).  p points at the pair's
// P = 2K raw parameters: p[0..K) shifts b, p[K..2K) unconstrained log-scales a.
//
// The mixture CDF is carried as its two tails, never as erf sums near +-1:
//   tp = 1 - c/K sum erf(v_k) = 1e-6 + c/K sum erfc(v_k)     (upper tail, = P[Y > y])
//   tn = 1 + c/K sum erf(v_k) = 1e-6 + c/K sum erfc(-v_k)    (lower tail), tp + tn = 2
// One erfcf(|v_k|) per component gives both sums without cancellation: the small term goes
// to the tail it belongs to, 2 - it to the other.  erf / erfc have no MUFU form: FAST only
// changes the exp / log around them.
// ---------------------------------------------------------------------------
constexpr float kRsqrt2 = 0.7071067811865476f;
constexpr float kSqrt2 = 1.4142135623730951f;
constexpr float kGaussFloor = 1e-6f;  // 1 - c

// tail sums of the K components at x; sp / sn = sum erfc(v_k) / sum erfc(-v_k)
template <int KT, bool FAST>
__device__ __forceinline__ void gauss_tails(const float* __restrict__ p, int Krt, const float* sreg,
                                            float x, float& sp, float& sn) {
    const int K = KT > 0 ? KT : Krt;
    sp = 0.f;
    sn = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float s = KT > 0 ? sreg[k] : zexp<FAST>(p[K + k]);
        const float v = fmaf(s, x, p[k]) * kRsqrt2;
        const float e = erfcf(fabsf(v));
        const bool pos = v >= 0.f;
        sp += pos ? e : 2.f - e;
        sn += pos ? 2.f - e : e;
    }
}

// y = f(x) from the two tail sums (cK = c / K)
__device__ __forceinline__ float gauss_from_tails(float sp, float sn, float cK) {
    return sp <= sn ? kSqrt2 * erfcinvf(fmaf(cK, sp, kGaussFloor))
                    : -kSqrt2 * erfcinvf(fmaf(cK, sn, kGaussFloor));
}

// forward value and closed-form log-derivative
//   ladj = y^2/2 + log(c/K) + logsumexp_k(a_k - u_k^2/2)
template <int KT, bool FAST>
__device__ __forceinline__ void gauss_forward_eval(const float* __restrict__ p, int Krt, float x,
                                                   float& y, float& ladj) {
    const int K = KT > 0 ? KT : Krt;
    const float cK = (1.f - kGaussFloor) / (float)K;
    float sp = 0.f, sn = 0.f;
    float mx = -INFINITY, se = 0.f;  // online logsumexp
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float a = p[K + k];
        const float u = fmaf(zexp<FAST>(a), x, p[k]);
        const float v = u * kRsqrt2;
        const float e = erfcf(fabsf(v));
        const bool pos = v >= 0.f;
        sp += pos ? e : 2.f - e;
        sn += pos ? 2.f - e : e;
        const float t = fmaf(-0.5f * u, u, a);
        if (t > mx) {
            se = fmaf(se, zexp<FAST>(mx - t), 1.f);
            mx = t;
        } else {
            se += zexp<FAST>(t - mx);
        }
    }
    y = gauss_from_tails(sp, sn, cK);
    ladj = fmaf(0.5f * y, y, zlog<FAST>(cK) + mx + zlog<FAST>(se));
}

// inverse: the reference's bisection (utils.py:159-183) on [-bound, bound], `iters` halvings,
// x = midpoint of the final interval.  "f(m) < y" is decided on the tail of y's sign:
// y >= 0: tp(m) > erfc(y / sqrt2);  y < 0: tn(m) < erfc(-y / sqrt2).
template <int KT, bool FAST>
__device__ __forceinline__ float gauss_inverse_eval(const float* __restrict__ p, int Krt, float y,
                                                    float bound, int iters) {
    const int K = KT > 0 ? KT : Krt;
    constexpr int KA = KT > 0 ? KT : 1;
    float sreg[KA];
    if constexpr (KT > 0) {
#pragma unroll
        for (int k = 0; k < KT; ++k) sreg[k] = zexp<FAST>(p[K + k]);
    }
    const float cK = (1.f - kGaussFloor) / (float)K;
    const bool upper = y >= 0.f;
    const float target = erfcf(fabsf(y) * kRsqrt2);
    return bisect(bound, iters, [&](float m) {
        float sp, sn;
        gauss_tails<KT, FAST>(p, K, sreg, m, sp, sn);
        return upper ? (fmaf(cK, sp, kGaussFloor) > target) : (fmaf(cK, sn, kGaussFloor) < target);
    });
}


}  // namespace bij
}  // namespace zk
