// zuko_b200 — wgmma / TMA PTX wrappers (sm_90a) and the packed-weight structures shared by the
// per-layer GEMM kernel (mlp_tcgen05.cu) and the fused layer kernel (fused_layer.cu).
#pragma once

#include <cuda.h>  // CUtensorMap types only; the encoder is fetched through the runtime
#include <cuda_bf16.h>

#include <vector>

#include "mlp.cuh"

namespace zk {

// ---------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// wgmma shared-memory descriptor, K-major, SWIZZLE_128B (operand rows of 128 bytes, 8-row groups
// 1024 B apart, 1024-byte aligned base):
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (unused for swizzled K-major, 1) |
//   [32,46) SBO >> 4 = 1024 B | [62,64) layout 1 = 128B swizzle
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// descriptor of the k-th 16-element K step inside a 64-wide swizzled K block: +32 bytes = +2 units
__device__ __forceinline__ uint64_t gmma_desc_advance(uint64_t desc, int k) { return desc + (uint64_t)(2 * k); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// all but the most recently committed group are complete
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// per-thread register limit of the executing warpgroup (all its warps execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int NA>
__device__ __forceinline__ void acc_fence(float (&d)[NA]) {
#pragma unroll
    for (int i = 0; i < NA; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] += A[64 x 16] * B[64 x 16]^T (one warpgroup; bf16 inputs, fp32 accumulators in registers).
// Accumulator layout (thread t of the warpgroup, w = t / 32, l = t % 32):
//   d[4 i + 2 h + e] = D[16 w + l / 4 + 8 h][8 i + 2 (l % 4) + e]
__device__ __forceinline__ void wgmma_m64n64k16_bf16(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b));
}

// D[64 x 48] += A[64 x 16] * B[48 x 16]^T: the first 48 rows (six 8-row groups) of a 64-row B tile, same descriptor.
// Accumulator layout as above with i < 6.
__device__ __forceinline__ void wgmma_m64n48k16_bf16(float (&d)[24], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23}, "
        "%24, %25, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(desc_a), "l"(desc_b));
}
// one k16 step on an accumulator of N / 2 registers per thread, N = 64 or 48
__device__ __forceinline__ void wgmma_k16(float (&d)[32], uint64_t a, uint64_t b) { wgmma_m64n64k16_bf16(d, a, b); }
__device__ __forceinline__ void wgmma_k16(float (&d)[24], uint64_t a, uint64_t b) { wgmma_m64n48k16_bf16(d, a, b); }

// The first KS 16-wide k steps of one 64-wide K block of the split-bf16 product on 64 x N tiles (N = 2 NA): hi*hi
// (+ hi*lo + lo*hi when n_terms == 3).  KS < 4 when the columns past 16 KS of the A operand are padding.
// a_hi / a_lo / b_hi / b_lo: shared-memory addresses of 128B-swizzled K-major 64-row operand tiles.
template <int KS = 4, int NA>
__device__ __forceinline__ void wgmma_kblock(float (&d)[NA], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                             int n_terms) {
    static_assert(KS >= 1 && KS <= 4, "a K block is four k16 steps");
    const uint64_t dah = gmma_desc_sw128(a_hi), dal = gmma_desc_sw128(a_lo);
    const uint64_t dbh = gmma_desc_sw128(b_hi), dbl = gmma_desc_sw128(b_lo);
    if (n_terms == 3) {  // one branch outside the MMA sequence: no register hand-off between the MMAs
#pragma unroll
        for (int k = 0; k < KS; ++k) {
            wgmma_k16(d, gmma_desc_advance(dah, k), gmma_desc_advance(dbh, k));
            wgmma_k16(d, gmma_desc_advance(dah, k), gmma_desc_advance(dbl, k));
            wgmma_k16(d, gmma_desc_advance(dal, k), gmma_desc_advance(dbh, k));
        }
    } else {
#pragma unroll
        for (int k = 0; k < KS; ++k) wgmma_k16(d, gmma_desc_advance(dah, k), gmma_desc_advance(dbh, k));
    }
}

// two consecutive fp32 at a shared-memory address (shared window)
__device__ __forceinline__ float2 lds_f32x2(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}

// four 8 x 8 b16 matrices to shared memory: lane l gives the address of row l % 8 of matrix l / 8 (16 bytes), and
// r[m] is the pair of matrix m at row l / 4, columns 2 (l % 4), 2 (l % 4) + 1 — an 8 x 8 block of the wgmma
// accumulator fragment after packing to bf16x2
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};"
                 ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3) : "memory");
}

// byte offset of K element k (< 64) of row r inside a 128B-swizzled tile of 128-byte rows
__device__ __forceinline__ uint32_t sw128_offset(int r, int k) {
    return (uint32_t)r * 128u + ((((uint32_t)k >> 3) ^ ((uint32_t)r & 7u)) << 4) + (((uint32_t)k & 7u) << 1);
}

struct TcLayer {
    int N = 0, K = 0, Kp = 0;
    __nv_bfloat16* w = nullptr;  // [2][N][Kp] (owned)
    CUtensorMap mapW;            // box (64 x 128 x 1): per-layer GEMM kernel
};
// weights as the fused layer kernel streams them: hidden units sorted by dependency degree (so
// that the masked matrices are block lower-triangular), the output layer's rows regrouped so that
// every 64-row chunk holds whole dims, and the all-zero (chunk, K block) tiles of every layer
// recorded so that their loads and MMAs are skipped
struct FusedPack {
    bool ready = false;
    int uni = 0, bins = 0, D = 0, C = 0;
    std::vector<__nv_bfloat16*> w;  // per layer [2][N][Kp], permuted (owned); output layer [2][n_last * 64][Kp]
    std::vector<float*> bias;       // per layer, permuted, padded (owned)
    std::vector<int*> dperm;        // per hidden layer: device copy of the degree permutation (owned; weight refresh)
    int* last_rows = nullptr;       // device: output-layer row of every padded output row, -1 = zero row (owned)
    int n_last = 0;                 // 64-row chunks of the output layer
    std::vector<CUtensorMap> maps;  // box (64 x 64 x 1); output layer (64 x NL x 1): a chunk's parameter rows
    uint8_t kbmask[8][128];         // [layer][chunk]: bit kb = K block kb has non-zero weights
    double issued_macs_per_row = 0;  // MACs the kernel issues per sample row (all split terms), bench bookkeeping
    int n_items = 0;                 // non-zero 64 x 64 weight tiles streamed per row tile
    size_t stream_bytes = 0;         // weight bytes those tiles bring into shared memory per row tile (all planes)
};
struct TcPack {
    std::vector<TcLayer> layers;
    std::vector<TcLayer> bwd;  // transposed weights (dgrad): N = in features, K = out features; built on first backward
    int n_terms = 3;
    int max_np = 0;  // widest padded hidden activation
    FusedPack fused;
};

inline int pad64(int v) { return (v + 63) / 64 * 64; }


// tensor map over bf16 planes [2][rows][Kp]; box = (64 x box_rows x 1), 128B swizzle
zk_status make_plane_map(CUtensorMap* map, const void* base, int64_t rows, int Kp, int box_rows);

// bf16 hi / lo split of two fp32 values, packed as (low 16 bits = first, high 16 = second).
// hi = rn_bf16(v) (one cvt.rn.bf16x2.f32 for the pair), lo = rn_bf16(v - hi): 6 instructions / pair.
__device__ __forceinline__ uint32_t pack_bf16x2_rn(float lo_half, float hi_half) {
    uint32_t d;  // cvt.rn.bf16x2.f32 d, a, b : a -> upper 16 bits, b -> lower 16 bits
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi_half), "f"(lo_half));
    return d;
}
__device__ __forceinline__ void split2_bf16(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    hi = pack_bf16x2_rn(v0, v1);  // registers only (taking the address of a __nv_bfloat162 went through local memory)
    const float h0 = __uint_as_float(hi << 16), h1 = __uint_as_float(hi & 0xffff0000u);
    lo = pack_bf16x2_rn(v0 - h0, v1 - h1);
}

}  // namespace zk
