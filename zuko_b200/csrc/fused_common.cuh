// zuko_b200 — helpers of the fully fused layer kernel (fused_layer.cu).
#pragma once

#include <type_traits>
#include <utility>
#include <vector>

#include "bijector_math.cuh"
#include "fused_layer.cuh"
#include "tc_common.cuh"

namespace zk {

// compile-time loop: f(integral_constant<int, Start>), ..., f(integral_constant<int, Start + N - 1>)
template <int Start, class F, int... I>
__device__ __forceinline__ void for_range_impl(F& f, std::integer_sequence<int, I...>) {
    (f(std::integral_constant<int, Start + I>{}), ...);
}
template <int Start, int N, class F>
__device__ __forceinline__ void for_range(F& f) {
    for_range_impl<Start>(f, std::make_integer_sequence<int, N>{});
}

// per-(UNI, K) chunking of the last layer: DPC dims (P parameters each) per 64-column chunk, of which the first
// NL = DPC * P rounded up to the wgmma N granularity of 8 are loaded and multiplied
template <int UNI, int KT>
struct LastCfg;
template <>
struct LastCfg<ZK_UNI_RQS, 8> { static constexpr int P = 23, DPC = 2, NL = 48; };
template <>
struct LastCfg<ZK_UNI_RQS, 16> { static constexpr int P = 47, DPC = 1, NL = 48; };
template <>
struct LastCfg<ZK_UNI_AFFINE, 0> { static constexpr int P = 2, DPC = 32, NL = 64; };

inline int fused_dpc(int univariate, int bins) { return (univariate == ZK_UNI_RQS) ? (bins == 8 ? 2 : 1) : 32; }
inline int fused_p(int univariate, int bins) { return (univariate == ZK_UNI_RQS) ? 3 * bins - 1 : 2; }
inline int fused_nl(int univariate, int bins) { return (fused_dpc(univariate, bins) * fused_p(univariate, bins) + 7) / 8 * 8; }

// hidden units of every hidden layer sorted by dependency degree: perm[l][new] = old index
void fused_degree_perm(const int* dims, int L, const std::vector<std::vector<uint8_t>>& Mk,
                       std::vector<std::vector<int>>& perm);

}  // namespace zk
