// zuko_b200 — one description per univariate bijector family, read by the stand-alone kernel (bijectors.cu), the
// backward kernel (backward.cu), the dimension-sequential inverse (ar_inverse.cu) and the C entry points.
//
// A family is a specialisation UniFamily<ZK_UNI_*> (circular RQS is RQS with UniSpec::circular).  It states:
//   P(K, degree); fixed_P(kt) for the compile-time shapes of the sequential inverse
//   key(s): the spec's candidate compile-time shape; Shapes: the shapes compiled per UniRole (0 = the runtime-shape
//     fallback; the sequential inverse has none and falls back to the sweeps)
//   kFastBackward, kTwoPerThread (sequential inverse), kCircular, kLayers (bits 1 << ZK_LAYER_*)
//   check_shape(s), check_scalars(s, inverse); Tables<Base> and tables(s, p): its device constants
//   forward, inverse, inverse_ladj (sequential inverse), backward: per-pair device functions over the math headers
// UniFamilyBase supplies kKind, K as the key, fixed_P(kt) = P(kt, 0), no checks and no tables.  A new family also
// needs its ZK_UNI_* define, an entry in UniKinds and, with device tables, a member in UniParams and InvParams.
#pragma once

#include <tuple>
#include <type_traits>

#include "bijector_grad.cuh"
#include "bijector_math.cuh"

namespace zk {

enum UniRole { kStandalone = 0, kBackward = 1, kSequential = 2 };  // uni_kernel, uni_bwd_kernel, ar_inverse_kernel

template <int... V>
struct KTs {};  // compile-time shapes (KT template arguments) of one role

constexpr int kAnyUniLayer = (1 << ZK_LAYER_AUTOREGRESSIVE) | (1 << ZK_LAYER_COUPLING) | (1 << ZK_LAYER_ELEMENTWISE);

template <int UNI>
struct UniFamily;

template <int UNI>
struct UniFamilyBase {
    static constexpr int kKind = UNI;
    static int key(const UniSpec& s) { return s.K; }
    // parameters per pair of the compile-time shape kt (sequential inverse): P(kt, 0) where the key is K
    __host__ __device__ static constexpr int fixed_P(int kt) { return UniFamily<UNI>::P(kt, 0); }
    static zk_status check_shape(const UniSpec&) { return ZK_OK; }
    static zk_status check_scalars(const UniSpec&, bool) { return ZK_OK; }
    template <class Base>
    using Tables = Base;  // a kernel's parameter type with the family's device constants appended
    template <class Prm>
    static void tables(const UniSpec&, Prm&) {}
};

inline zk_status k_in_range(const char* what, const UniSpec& s) {
    ZK_REQUIRE(s.K >= 1 && s.K <= 1024, "%s must be in [1, 1024], got %d", what, s.K);
    return ZK_OK;
}
inline zk_status bisection_scalars(const char* name, const UniSpec& s, bool inverse) {
    ZK_REQUIRE(s.bound > 0.f, "%s: bound must be positive, got %g", name, (double)s.bound);
    if (inverse) ZK_REQUIRE(s.iters >= 1 && s.iters <= 64, "%s: bisection steps must be in [1, 64], got %d", name, s.iters);
    return ZK_OK;
}

// a per-pair device function: KT the compile-time shape (0 = runtime), FAST the math mode, Prm the kernel's parameters
#define ZK_PAIR template <int KT, bool FAST, class Prm> static __device__ __forceinline__

// MonotonicAffineTransform, transforms.py:435-446: phi = (shift, unconstrained log-scale)
template <>
struct UniFamily<ZK_UNI_AFFINE> : UniFamilyBase<ZK_UNI_AFFINE> {
    __host__ __device__ static constexpr int P(int, int) { return 2; }
    static int key(const UniSpec&) { return 0; }
    using Shapes = std::tuple<KTs<0>, KTs<0>, KTs<0>>;
    static constexpr bool kFastBackward = false, kTwoPerThread = true, kCircular = false;  // one expf: no fast variant
    static constexpr int kLayers = kAnyUniLayer;

    ZK_PAIR float forward(const float* pp, const Prm& a, float x, float& lj) {
        const float shift = pp[0];
        const float ls = bij::softclip<FAST>(pp[1], a.ad);
        lj = ls;
        return fmaf(x, bij::zexp<FAST>(ls), shift);
    }
    ZK_PAIR float inverse(const float* pp, const Prm& a, float y) {
        const float shift = pp[0];
        const float ls = bij::softclip<FAST>(pp[1], a.ad);
        return bij::zdiv<FAST>(y - shift, bij::zexp<FAST>(ls));
    }
    ZK_PAIR float inverse_ladj(const float* u, const Prm& p, float y, float& lj) {
        lj = bij::softclip<FAST>(u[1], p.ad);
        return inverse<KT, FAST>(u, p, y);
    }
    ZK_PAIR void backward(const float* pp, const Prm& a, float x, float gy, float gl, float& gx, float* out) {
        bijgrad::affine_backward_pair(pp, x, gy, gl, a.ad, gx, out);
    }
};

// MonotonicRQSTransform, transforms.py:469-567; circular: CircularShiftTransform(bound) in front (flows/spline.py:65-72)
template <>
struct UniFamily<ZK_UNI_RQS> : UniFamilyBase<ZK_UNI_RQS> {
    __host__ __device__ static constexpr int P(int K, int) { return 3 * K - 1; }
    using Shapes = std::tuple<KTs<4, 8, 16, 0>, KTs<8, 16, 0>, KTs<8, 16>>;
    static constexpr bool kFastBackward = true, kTwoPerThread = true, kCircular = true;
    static constexpr int kLayers = kAnyUniLayer;
    static zk_status check_shape(const UniSpec& s) { return k_in_range("rqs: bins", s); }

    ZK_PAIR float forward(const float* pp, const Prm& a, float x, float& lj) {
        if (a.circ) x = bij::circ_shift(x, a.bound);
        bij::Bin b = bij::rqs_select<KT, FAST, false>(pp, a.K, x, a.bound, a.aw, a.ad);
        float y;
        bij::rqs_forward_eval<FAST>(b, x, y, lj);
        return y;
    }
    ZK_PAIR float inverse(const float* pp, const Prm& a, float y) { return solve<KT, FAST>(pp, a.K, a, y, nullptr); }
    ZK_PAIR float inverse_ladj(const float* u, const Prm& p, float y, float& lj) { return solve<KT, FAST>(u, KT, p, y, &lj); }
    // the inverse with K bins; with lj, also the ladj of the forward map at the solution
    ZK_PAIR float solve(const float* pp, int K, const Prm& a, float y, float* lj) {
        bij::Bin b = bij::rqs_select<KT, FAST, true>(pp, K, y, a.bound, a.aw, a.ad);
        float x = bij::rqs_inverse_eval<FAST>(b, y);
        float y2;
        if (lj) bij::rqs_forward_eval<FAST>(b, x, y2, *lj);
        if (a.circ) x = bij::circ_shift(x, a.bound);
        return x;
    }
    ZK_PAIR void backward(const float* pp, const Prm& a, float x, float gy, float gl, float& gx, float* out) {
        bijgrad::rqs_backward_pair<KT, FAST>(pp, a.K, x, gy, gl, a.bound, a.aw, a.ad, gx, out);
    }
};

// GaussianizationTransform, transforms.py:834-875: K erfc terms, bisection inverse (transforms.py:609-617)
template <>
struct UniFamily<ZK_UNI_GAUSS> : UniFamilyBase<ZK_UNI_GAUSS> {
    __host__ __device__ static constexpr int P(int K, int) { return 2 * K; }
    using Shapes = std::tuple<KTs<8, 16, 0>, KTs<8, 16, 0>, KTs<>>;
    static constexpr bool kFastBackward = true, kTwoPerThread = false, kCircular = false;
    static constexpr int kLayers = 1 << ZK_LAYER_ELEMENTWISE;  // the bisection inverse is element-wise only
    static zk_status check_shape(const UniSpec& s) { return k_in_range("gaussianization: components", s); }
    static zk_status check_scalars(const UniSpec& s, bool inverse) { return bisection_scalars("gaussianization", s, inverse); }

    ZK_PAIR float forward(const float* pp, const Prm& a, float x, float& lj) {
        float y;
        bij::gauss_forward_eval<KT, FAST>(pp, a.K, x, y, lj);
        return y;
    }
    ZK_PAIR float inverse(const float* pp, const Prm& a, float y) {
        return bij::gauss_inverse_eval<KT, FAST>(pp, a.K, y, a.bound, a.iters);
    }
    ZK_PAIR void backward(const float* pp, const Prm& a, float x, float gy, float gl, float& gx, float* out) {
        float y, lj;
        bij::gauss_forward_eval<KT, FAST>(pp, a.K, x, y, lj);
        bijgrad::gauss_backward_pair<FAST>(pp, KT > 0 ? KT : a.K, x, y, gy, gl, gx, out);
    }
};

// sum-of-squares polynomial bijector of SOSPF (flows/polynomial.py:23-28, sosp_math.cuh)
template <>
struct UniFamily<ZK_UNI_SOSP> : UniFamilyBase<ZK_UNI_SOSP> {
    __host__ __device__ static constexpr int P(int K, int degree) { return K * (degree + 1) + 1; }
    __host__ __device__ static constexpr int fixed_P(int) { return sosp::kDefP; }
    static int key(const UniSpec& s) { return (s.K == sosp::kDefK && s.degree == sosp::kDefL) ? sosp::kDefK : 0; }
    using Shapes = std::tuple<KTs<sosp::kDefK, 0>, KTs<sosp::kDefK, 0>, KTs<sosp::kDefK>>;
    // no transcendental in the reverse mode; two register bisections per thread would spill
    static constexpr bool kFastBackward = false, kTwoPerThread = false, kCircular = false;
    static constexpr int kLayers = 1 << ZK_LAYER_AUTOREGRESSIVE;  // the bisection runs in autoregressive layers only
    static zk_status check_shape(const UniSpec& s) {  // degree <= 15 (16 quadrature nodes), P <= 1024
        ZK_REQUIRE(s.K >= 1 && s.K <= 1023 && s.degree >= 0 && s.degree <= 15 && s.K * (s.degree + 1) + 1 <= 1024,
                   "sosp: polynomials %d / degree %d out of range (degree <= 15, K (degree + 1) + 1 <= 1024)", s.K, s.degree);
        return ZK_OK;
    }
    static zk_status check_scalars(const UniSpec& s, bool inverse) { return bisection_scalars("sosp", s, inverse); }
    template <class Base>
    struct Tables : Base {
        sosp::Const sosp;
    };
    template <class Prm>
    static void tables(const UniSpec& s, Prm& p) { p.sosp = sosp::make_const(s.K, s.degree, s.bound, s.slope, s.iters); }

    // the default shape works on a register copy of its 16 parameters (four 16-byte loads: P = 16 puts every pair on
    // the same banks, a 4-way rather than a 16-way conflict)
    template <int KT>
    static __device__ __forceinline__ const float* in_regs(const float* pp, float (&ar)[sosp::kDefP]) {
        if constexpr (KT > 0) {
#pragma unroll
            for (int q = 0; q < sosp::kDefP / 4; ++q) {
                const float4 v = reinterpret_cast<const float4*>(pp)[q];
                ar[4 * q] = v.x; ar[4 * q + 1] = v.y; ar[4 * q + 2] = v.z; ar[4 * q + 3] = v.w;
            }
            return ar;
        }
        return pp;
    }
    ZK_PAIR float forward(const float* pp, const Prm& a, float x, float& lj) {
        float ar[sosp::kDefP], gx;
        const float y = sosp::forward<KT>(in_regs<KT>(pp, ar), a.sosp, x, gx);
        lj = bij::zlog<FAST>(gx);
        return y;
    }
    ZK_PAIR float inverse(const float* pp, const Prm& a, float y) {
        float ar[sosp::kDefP];
        return sosp::inverse<KT>(in_regs<KT>(pp, ar), a.sosp, y);
    }
    ZK_PAIR float inverse_ladj(const float* u, const Prm& p, float y, float& lj) {
        const float x = sosp::inverse<KT>(u, p.sosp, y);
        lj = bij::zlog<FAST>(sosp::g<KT>(u, p.sosp, x));  // ladj of the forward map at the solution
        return x;
    }
    ZK_PAIR void backward(const float* pp, const Prm& a, float x, float gy, float gl, float& gx, float* out) {
        float ar[KT > 0 ? sosp::kDefP : 1];  // the default shape's parameters in registers: out may alias pp
        if constexpr (KT > 0) {
#pragma unroll
            for (int q = 0; q < sosp::kDefP; ++q) ar[q] = pp[q];
        }
        sosp::backward_pair<KT>(KT > 0 ? ar : pp, a.sosp, x, gy, gl, gx, out);
    }
};

// bounded Bernstein bijector of BPF (transforms.py:640-831, bernstein_math.cuh)
template <>
struct UniFamily<ZK_UNI_BERNSTEIN> : UniFamilyBase<ZK_UNI_BERNSTEIN> {
    __host__ __device__ static constexpr int P(int, int degree) { return degree + 1; }
    __host__ __device__ static constexpr int fixed_P(int) { return bern::kDefP; }
    static int key(const UniSpec& s) { return s.degree + 1; }
    using Shapes = std::tuple<KTs<bern::kDefP, 0>, KTs<bern::kDefP, 0>, KTs<bern::kDefP>>;
    // no approximated transcendental in the reverse mode; two register bisections per thread would spill
    static constexpr bool kFastBackward = false, kTwoPerThread = false, kCircular = false;
    static constexpr int kLayers = 1 << ZK_LAYER_AUTOREGRESSIVE;  // BPF is a MAF (flows/polynomial.py:79-117)
    static zk_status check_shape(const UniSpec& s) {  // order M = degree + 5 <= 64
        ZK_REQUIRE(s.degree >= 0 && s.degree <= bern::kMaxDegree, "bernstein: degree must be in [0, %d], got %d",
                   bern::kMaxDegree, s.degree);
        return ZK_OK;
    }
    static zk_status check_scalars(const UniSpec& s, bool inverse) {
        ZK_REQUIRE(s.eps > 0.f && s.eps < 0.5f, "bernstein: eps must be in (0, 1/2), got %g", (double)s.eps);
        return bisection_scalars("bernstein", s, inverse);
    }
    template <class Base>
    struct Tables : Base {
        bern::Const bern;
    };
    template <class Prm>
    static void tables(const UniSpec& s, Prm& p) { p.bern = bern::make_const(s.degree, s.bound, s.eps, s.iters); }

    // run(dl) with dl(j) the softmax differences: the default degree takes its 17 parameters to registers and keeps
    // the scaled softmax there; other degrees form each softmax entry from shared memory when the sums need it
    template <int KT, class Run>
    static __device__ __forceinline__ float with_softmax(const float* pp, const bern::Const& c, Run run) {
        constexpr int PT = KT > 0 ? bern::kDefP : 0;
        float u[PT > 0 ? PT : 1], w[PT > 0 ? PT : 1];
        if constexpr (PT > 0) {
#pragma unroll
            for (int q = 0; q < PT; ++q) u[q] = pp[q];
        }
        const float* up = PT > 0 ? u : pp;
        float mx, rs;
        bern::softmax<PT>(up, c, w, mx, rs);
        return run([&](int j) { return bern::delta<PT>(up, w, c, mx, rs, j); });
    }
    ZK_PAIR float forward(const float* pp, const Prm& a, float x, float& lj) {
        return with_softmax<KT>(pp, a.bern, [&](auto dl) {
            float fp;
            const float y = bern::forward<(KT > 0 ? bern::kDefM : 0)>(a.bern, x, dl, &fp);
            lj = bij::zlog<FAST>(fp);
            return y;
        });
    }
    ZK_PAIR float inverse(const float* pp, const Prm& a, float y) {
        return with_softmax<KT>(pp, a.bern, [&](auto dl) { return bern::inverse<(KT > 0 ? bern::kDefM : 0)>(a.bern, y, dl); });
    }
    ZK_PAIR float inverse_ladj(const float* u, const Prm& p, float y, float& lj) {
        return with_softmax<KT>(u, p.bern, [&](auto dl) {
            const float x = bern::inverse<bern::kDefM>(p.bern, y, dl);
            float fp;
            bern::forward<bern::kDefM>(p.bern, x, dl, &fp);
            lj = bij::zlog<FAST>(fp);  // ladj of the forward map at the solution
            return x;
        });
    }
    ZK_PAIR void backward(const float* pp, const Prm& a, float x, float gy, float gl, float& gx, float* out) {
        float ur[KT > 0 ? bern::kDefP : 1];  // the default degree's parameters in registers: out may alias pp
        if constexpr (KT > 0) {
#pragma unroll
            for (int q = 0; q < bern::kDefP; ++q) ur[q] = pp[q];
        }
        bern::backward_pair<KT>(KT > 0 ? ur : pp, a.bern, x, gy, gl, gx, out);
    }
};

#undef ZK_PAIR

// ---------------------------------------------------------------------------
// host side: runtime kind -> family
// ---------------------------------------------------------------------------
template <int... V>
constexpr bool kt_listed(KTs<V...>, int kt) {
    return ((kt == V) || ...);
}

// every family, once: with_family dispatches over this list and uni_known tests membership of it
using UniKinds = KTs<ZK_UNI_AFFINE, ZK_UNI_RQS, ZK_UNI_GAUSS, ZK_UNI_SOSP, ZK_UNI_BERNSTEIN>;
inline bool uni_known(int kind) { return kt_listed(UniKinds{}, kind); }

// f(UniFamily<kind>{}); an unknown kind gets a value-initialised result (callers refuse it first: uni_known)
template <class F, int... U>
auto with_family_in(KTs<U...>, int kind, F&& f) {
    decltype(f(UniFamily<ZK_UNI_RQS>{})) r{};
    ((kind == U && (r = f(UniFamily<U>{}), true)) || ...);
    return r;
}
template <class F>
auto with_family(int kind, F&& f) {
    return with_family_in(UniKinds{}, kind, f);
}

inline int uni_P(const UniSpec& s) {
    return with_family(s.kind, [&](auto fam) { return decltype(fam)::P(s.K, s.degree); });
}
inline zk_status uni_check_shape(const UniSpec& s) {
    ZK_REQUIRE(uni_known(s.kind), "univariate: unknown kind %d", s.kind);
    return with_family(s.kind, [&](auto fam) { return decltype(fam)::check_shape(s); });
}
// the family's bound / eps / bisection steps (the steps only when the call inverts) and the slope every family takes
inline zk_status uni_check_scalars(const UniSpec& s, bool inverse) {
    ZK_TRY(with_family(s.kind, [&](auto fam) { return decltype(fam)::check_scalars(s, inverse); }));
    ZK_REQUIRE(s.slope > 0.f && s.slope < 1.f, "univariate: slope must be in (0, 1), got %g", (double)s.slope);
    return ZK_OK;
}

// the compile-time shape that serves `s` in ROLE: its key when compiled, else 0 when the role has a runtime-shape
// fallback, else -1
template <UniRole ROLE>
int uni_kt(const UniSpec& s) {
    return with_family(s.kind, [&](auto fam) {
        using Fam = decltype(fam);
        const std::tuple_element_t<ROLE, typename Fam::Shapes> list;
        return kt_listed(list, Fam::key(s)) ? Fam::key(s) : (kt_listed(list, 0) ? 0 : -1);
    });
}

// bound, aw / ad (from the slope), circ and the family's tables in a kernel's parameters
template <class Fam, class Prm>
void set_uni_consts(const UniSpec& s, Prm& p) {
    p.bound = s.bound;
    const float absL = fabsf(logf(s.slope));
    p.aw = 2.f / absL;
    p.ad = 1.f / absL;
    p.circ = (Fam::kCircular && s.circular) ? 1 : 0;
    Fam::tables(s, p);
}

template <int... V, class F>
zk_status with_kt(KTs<V...>, int kt, F&& f) {
    zk_status st = ZK_OK;
    const bool hit = ((kt == V && (st = f(std::integral_constant<int, V>{}), true)) || ...);
    return hit ? st : fail(ZK_EINVAL, "univariate: no compiled shape %d", kt);
}

// The instantiation of ROLE that serves (kind, kt, fast): launch(fam, KT, FAST) with fam a UniFamily and KT / FAST
// std::integral_constants, over the shapes the family lists for the role.  FAST is false for a backward without a
// fast-math variant.
template <UniRole ROLE, class F>
zk_status uni_dispatch(int kind, int kt, bool fast, F&& launch) {
    ZK_REQUIRE(uni_known(kind), "univariate: unknown kind %d", kind);
    return with_family(kind, [&](auto fam) {
        using Fam = decltype(fam);
        return with_kt(std::tuple_element_t<ROLE, typename Fam::Shapes>{}, kt, [&](auto k) {
            if constexpr (ROLE != kBackward || Fam::kFastBackward) {
                if (fast) return launch(fam, k, std::true_type{});
            }
            return launch(fam, k, std::false_type{});
        });
    });
}

}  // namespace zk
