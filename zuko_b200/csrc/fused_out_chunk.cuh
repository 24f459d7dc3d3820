// zuko_b200 — column order of the fused layer kernel's output chunks, and the quad exchange that gives each consumer
// thread the parameter vector of one (row, slot) straight from the wgmma accumulators.  Host/device code without
// CUDA headers: nvcc compiles it into fused_layer_kernel and fused_layer_prepare, g++ into the CPU harness
// tests/native/fused_out_chunk_host.cpp.
//
// An output chunk holds NP = DPC * P parameters of DPC whole dims per sample row, in "staging order": value k is
// parameter k % P of the chunk's dim k / P.  The chunk is split into two halves of VH = ceil(NP / 2) values; a
// slot (the share of the chunk one thread evaluates) reads NV consecutive values from value NV * slot on:
//   RQS, 8 bins:  P = 23, DPC = 2   halves = slots = dims (VH = NV = 23)
//   RQS, 16 bins: P = 47, DPC = 1   one dim in two halves (VH = 24, NV = 47: slot 0 gathers both, slot 1 idles)
//   affine:       P = 2, DPC = 32   halves = slots of 16 (shift, log-scale) pairs (VH = NV = 32)
// Value i of half h sits in packed column 8 (i / 4) + 4 h + i % 4.  In the m64nN accumulator fragment
// (d[4 j + 2 hh + e] = D[16 w + l / 4 + 8 hh][8 j + 2 (l % 4) + e], tc_common.cuh) quad lanes 2h and 2h + 1 then
// hold half h of both rows of their quad, two values per 8-column group each.  One xor-1 exchange of the other row's
// pair per group leaves lane 2h + b with half h of row b; with DPC = 1 an xor-2 exchange hands half 1 to lanes 0, 1.
#pragma once

#if defined(__CUDACC__)
#define ZK_OUT_HD __host__ __device__ __forceinline__
#else
#define ZK_OUT_HD inline
#endif

namespace zk {
namespace outchunk {

template <int P, int DPC>
struct Shape {
    static_assert(DPC == 1 || DPC % 2 == 0, "a chunk splits into two halves of whole slots");
    static constexpr int NP = DPC * P;           // staged values of a chunk
    static constexpr int VH = (NP + 1) / 2;      // values of a half
    static constexpr int NG = (VH + 3) / 4;      // 8-column groups that hold a half
    static constexpr int NV = DPC == 1 ? P : NP / 2;  // values one slot evaluates
    static constexpr int NCOL = 8 * NG;          // packed columns the chunk's MMAs must cover
};

// packed column of staging-order value k of a chunk of np values
ZK_OUT_HD int col(int k, int np) {
    const int vh = (np + 1) / 2, h = k / vh, i = k - h * vh;
    return 8 * (i >> 2) + 4 * h + (i & 3);
}

// the (row of the warp's 16, slot) that lane `lane` of a consumer warp evaluates
ZK_OUT_HD int row(int lane) { return (lane >> 2) + 8 * (lane & 1); }
ZK_OUT_HD int slot(int lane) { return (lane >> 1) & 1; }

// Output-layer row map of the pack: packed row ch * 64 + c <- row last_rows[...] of the unpacked output layer
// (parameter j of dim d is row d * P + j), -1 for padding.  A chunk's rows stay in the chunk.
inline void last_rows(int D, int P, int DPC, int n_last, int* out) {
    for (int i = 0; i < n_last * 64; ++i) out[i] = -1;
    for (int ch = 0; ch < n_last; ++ch)
        for (int k = 0; k < DPC * P; ++k) {
            const int d = ch * DPC + k / P;
            if (d < D) out[ch * 64 + col(k, DPC * P)] = d * P + k % P;
        }
}

// Assembles v[j] = staging-order value NV * slot(lane) + j of row row(lane) from the thread's accumulator fragment a.
// All four lanes of a quad call it together.  xch(mine, mask) returns the `mine` of lane lane ^ mask
// (__shfl_xor_sync on the device); every lane passes its own send value, whether or not it uses what it receives.
template <int P, int DPC, int NA, class Xch>
ZK_OUT_HD void assemble(const float (&a)[NA], int lane, Xch&& xch, float (&v)[Shape<P, DPC>::NV]) {
    using S = Shape<P, DPC>;
    static_assert(S::NCOL <= 2 * NA, "the fragment must hold every packed column");
    const bool b = lane & 1;  // the row half this lane keeps: it sends the other one
    float h[4 * S::NG];
#pragma unroll
    for (int g = 0; g < S::NG; ++g)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float r0 = a[4 * g + e], r1 = a[4 * g + 2 + e];
            const float got = xch(b ? r0 : r1, 1);
            h[4 * g + e] = b ? got : r0;
            h[4 * g + 2 + e] = b ? r1 : got;
        }
    if constexpr (DPC == 1) {  // half 1 from the lane pair above; its own copy is unused there
#pragma unroll
        for (int j = 0; j < S::VH; ++j) v[j] = h[j];
#pragma unroll
        for (int j = S::VH; j < S::NV; ++j) v[j] = xch(h[j - S::VH], 2);
    } else {
#pragma unroll
        for (int j = 0; j < S::NV; ++j) v[j] = h[j];
    }
}

}  // namespace outchunk
}  // namespace zk

#undef ZK_OUT_HD
