// zuko_b200 — ONE kernel per flow layer: conditioner (all linear layers) + bijector + ladj.
//
//   x, c  --(bf16 hi/lo split, in-kernel)-->  A operand in SHARED MEMORY (64 or 128 rows x up to 512 columns)
//   for every linear layer:  wgmma  D[registers] += A[smem] * W[smem]^T
//        W is streamed from L2 by TMA as 64 x 64 tiles (hi + lo planes) through a ring of mbarrier
//        slots; the all-zero tiles of the degree-sorted masked matrices are never loaded or multiplied,
//        nor are the k16 steps of layer 0 past D + C or the padding rows of an output chunk past NL;
//        hidden layers : at most four 64 x 64 fp32 accumulators per consumer warpgroup; once every
//                        reader of an A operand is done with it, it is overwritten in place with the
//                        layer's output (bias, activation, bf16 hi/lo split): activations never
//                        leave shared memory;
//        last layer    : its rows are regrouped so that a 64-row chunk holds whole dims, in a column
//                        order (fused_out_chunk.cuh) that lets each thread gather one (sample row, dim)'s
//                        parameters from its quad's accumulators with register shuffles; it evaluates
//                        the spline / affine bijector, the log-derivative and the per-sample sum — phi
//                        never touches HBM.
//   HBM traffic per sample per layer: 4 (D + C) read + 4 (D + 1) written.
//
// Restates for one MaskedAutoregressiveTransform layer:  flows/autoregressive.py:207-215 (meta),
// nn.py:217-218 (masked linears, mask folded into W at pack time), transforms.py:469-490,
// 554-567 (RQS) or 426-446 (affine), transforms.py:210-214 (sum over D), and on the last
// layer of a flow distributions.py:115-119 + torch normal.py:87-102 (DiagNormal log-prob).
//
// Warp roles (384 threads, 1 CTA / SM, persistent over row tiles).  The row tile is 64 or 128 rows,
// chosen by the launcher from the shape (fused_plan):
//   warpgroup 0     W producer (one thread: TMA loads in a fixed tile order)
//   warpgroups 1-2  consumers: input staging, MMAs, epilogues
// 64-row tiles: the consumers split the layers' 64-column chunks (chunk ch belongs to warpgroup ch % 2); each
//   tile goes into the ring of the warpgroup that multiplies it — a ring has ONE consumer that takes every
//   slot in order, so its mbarrier phases can never be lapped.
// 128-row tiles: warpgroup 1 owns rows 0-63 of the tile and warpgroup 2 rows 64-127, each with its own A
//   operand; both multiply EVERY weight tile (one ring, two arrivals per slot, neither consumer skips a
//   slot), so a tile brought in by TMA feeds 128 rows.  MMAs are asynchronous (one group per tile, the next tile
//   issued before waiting, a slot released one tile late).  The output chunks go in pairs: a pair's tiles are one
//   such stream that completes before the two chunks' bijectors run side by side.  The warpgroups only meet at the
//   W ring.
//   The producer runs on 40 registers and the consumers on 232 (setmaxnreg).

#include <string.h>

#include <algorithm>
#include <type_traits>
#include <utility>
#include <vector>

#include "activations.cuh"
#include "fused_common.cuh"
#include "fused_out_chunk.cuh"

namespace zk {

namespace {

using namespace bij;

constexpr int FM = 64;              // rows per wgmma M (and per consumer warpgroup)
constexpr int FK = 64;              // bf16 per K block (128-byte swizzle row) = columns per chunk
constexpr int F_MAXKB = 8;          // A operand: up to 8 K blocks = 512 columns
constexpr int F_MAX_STAGES = 8;     // the W ring is as deep as shared memory allows (see fused_plan)
constexpr int F_WIDE_MAXKB = 4;     // 128-row tiles: four accumulators per consumer hold every hidden chunk
constexpr int F_THREADS = 384;
constexpr uint32_t F_TILE = FM * FK * 2;  // 8 KB: one plane of a 64 x 64 tile
constexpr uint32_t F_STAGE = 2 * F_TILE;  // hi + lo
constexpr uint32_t F_SMEM_MAX = 232448;   // 227 KB per block on sm_90

// floats per row of the former output-layer staging region: the chunk's DPC * P parameters, made odd.  The region
// still sizes the plan; output chunks are assembled in registers, and the region holds the hidden layers' biases
__host__ __device__ constexpr int f_srow(int dpc_p) { return dpc_p | 1; }

struct FusedParams {
    CUtensorMap mapW[ZK_FUSED_MAX_LINEAR];
    const float* bias[ZK_FUSED_MAX_LINEAR];
    uint8_t kbmask[ZK_FUSED_MAX_LINEAR][128];  // [layer][chunk]: K blocks with non-zero weights
    int n_linear;
    int K0, KB0;        // real input width (D + C) and its number of 64-wide K blocks
    int ks0;            // k16 steps of layer 0's last K block that hold inputs: ceil((K0 - 64 (KB0 - 1)) / 16)
    int vec_in;         // x and c rows can be read as float4 (D, C, ldx, ldc multiples of 4, 16-byte aligned bases)
    int g_shift;        // vec_in: log2 of the staging items per row (float4 groups of the staged columns, rounded up)
    int H;              // hidden width (multiple of 64, <= 512)
    int KBA;            // K blocks of the A buffer: max(KB0, H / 64)
    int D, C;
    int n_last;         // 64-row chunks of the output layer
    int n_terms;        // 3 (split bf16) or 1
    int act;            // hidden activation: 1 ReLU, else ZK_ACT_* (GACT instantiation)
    int M;
    int n_stages;       // slots of the W ring(s), 16 KB each (64-row tiles: half per consumer warpgroup)
    const float* x; int64_t ldx;
    const float* c; int64_t ldc;
    float* y; int64_t ldy;
    float* ladj; int accumulate;
    float* log_prob; const float* base_loc; const float* base_scale;
    float bound, aw, ad;
};

// f(integral_constant<int, ks>), ks in 1..4: the k16 steps of an MMA chain are a compile-time constant, chosen by
// one branch outside the chain
template <class F>
__device__ __forceinline__ void with_ksteps(int ks, F&& f) {
    if (ks == 4) f(std::integral_constant<int, 4>{});
    else if (ks == 3) f(std::integral_constant<int, 3>{});
    else if (ks == 2) f(std::integral_constant<int, 2>{});
    else f(std::integral_constant<int, 1>{});
}

// one synchronous 64 x N tile: the first KS k16 steps of an A K block times the W tile in ring slot `w_tile`
template <int KS = 4, int NA>
__device__ __forceinline__ void tile_mma(float (&acc)[NA], uint32_t a_hi, uint32_t a_plane, uint32_t w_tile, int n_terms) {
    wgmma_fence();
    wgmma_kblock<KS>(acc, a_hi, a_hi + a_plane, w_tile, w_tile + F_TILE, n_terms);
    wgmma_commit();
    wgmma_wait0();
    acc_fence(acc);
}
// the same into accumulator q of a hidden layer (compile-time index: the accumulators must stay in registers)
template <int KS>
__device__ __forceinline__ void tile_mma(float (&acc)[4][32], int q, uint32_t a_hi, uint32_t a_plane, uint32_t w_tile,
                                         int n_terms) {
    if (q == 0) tile_mma<KS>(acc[0], a_hi, a_plane, w_tile, n_terms);
    else if (q == 1) tile_mma<KS>(acc[1], a_hi, a_plane, w_tile, n_terms);
    else if (q == 2) tile_mma<KS>(acc[2], a_hi, a_plane, w_tile, n_terms);
    else tile_mma<KS>(acc[3], a_hi, a_plane, w_tile, n_terms);
#pragma unroll
    for (int i = 0; i < 4; ++i) acc_fence(acc[i]);
}

// NT: split-bf16 terms as a compile-time constant (128-row tiles: no branch between the asynchronous MMAs of an
// accumulator), or 0 to read p.n_terms
template <int UNI, int KT, bool FAST, bool GACT, int ROWS, int NT>
__global__ void __launch_bounds__(F_THREADS, 1)
fused_layer_kernel(const __grid_constant__ FusedParams p) {
    using Cfg = LastCfg<UNI, KT>;
    constexpr int P = Cfg::P, DPC = Cfg::DPC, NL = Cfg::NL;
    constexpr int NP = DPC * P, SROW = f_srow(NP);  // parameters of an output chunk, row stride of the bias region
    constexpr bool WIDE = (ROWS == 128);
    using Out = outchunk::Shape<P, DPC>;
    static_assert(NP <= NL && NL <= FK && NL % 8 == 0 && Out::NCOL <= NL, "a last-layer chunk must fit its MMA width");
    static_assert(ROWS == 64 || ROWS == 128, "row tile: one or two wgmma M");
    const int n_terms = NT ? NT : p.n_terms;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    // [W ring: n_stages x 16 KB][A: ROWS / 64 x 2 planes x KBA x 8 KB][hidden biases: region of 2 x 64 x SROW fp32]
    // [ladj partials 4 x ROWS][barriers]
    const int NS = p.n_stages;
    uint8_t* sW = smem;
    uint8_t* sA = smem + (size_t)NS * F_STAGE;
    const uint32_t a_plane = (uint32_t)p.KBA * F_TILE;
    float* s_bias = (float*)(sA + (ROWS / FM) * 2 * (size_t)a_plane);  // [L - 1][H]
    static_assert(2 * FM * SROW >= (ZK_FUSED_MAX_LINEAR - 1) * F_MAXKB * FK, "the hidden biases fit the region");
    float* s_part = s_bias + 2 * FM * SROW;
    uint64_t* full = (uint64_t*)(s_part + 4 * ROWS);         // [F_MAX_STAGES] TMA -> consumer
    uint64_t* empty = full + F_MAX_STAGES;                   // [F_MAX_STAGES] consumer -> TMA
    const int NR = WIDE ? NS : NS / 2;                       // slots per ring (64 rows: ring g = [g NR, g NR + NR))

    const int L = p.n_linear;
    const int m_tiles = (p.M + ROWS - 1) / ROWS;
    const int nch = p.H / FK;  // hidden chunks = K blocks of every layer after the first

    if (threadIdx.x == 0) {
        for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], WIDE ? 2 : 1); }
        fence_mbar_init();
    }
    __syncthreads();

    const int wg = threadIdx.x >> 7;
    if (wg == 0) {
        // ======================= W producer =======================
        // tile order (the consumers walk the same one): hidden layers K block by K block, each over
        // its chunks; the output layer chunk by chunk, each over its K blocks
        if constexpr (WIDE) setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {
            int rs[2] = {0, 0};
            uint32_t rph[2] = {0u, 0u};
            // 64 rows: chunk ch is multiplied by consumer warpgroup ch % 2.  plane: bytes of the layer's box
            auto load = [&](int l, int ch, int kb, uint32_t plane) {
                const int o = WIDE ? 0 : (ch & 1), s = o * NR + rs[o];
                mbar_wait(&empty[s], rph[o] ^ 1);
                uint8_t* dst = sW + (size_t)s * F_STAGE;
                mbar_arrive_expect_tx(&full[s], (n_terms == 3) ? 2 * plane : plane);
                tma_load_3d(dst, &p.mapW[l], &full[s], kb * FK, ch * FK, 0);
                if (n_terms == 3) tma_load_3d(dst + F_TILE, &p.mapW[l], &full[s], kb * FK, ch * FK, 1);
                if (++rs[o] == NR) { rs[o] = 0; rph[o] ^= 1; }
            };
            for (int t = blockIdx.x; t < m_tiles; t += gridDim.x) {
                for (int l = 0; l < L - 1; ++l) {
                    const int KB = (l == 0) ? p.KB0 : nch;
                    for (int kb = 0; kb < KB; ++kb)
                        for (int ch = 0; ch < nch; ++ch)
                            if ((p.kbmask[l][ch] >> kb) & 1u) load(l, ch, kb, F_TILE);
                }
                for (int ch = 0; ch < p.n_last; ++ch)
                    for (int kb = 0; kb < nch; ++kb)
                        if ((p.kbmask[L - 1][ch] >> kb) & 1u) load(L - 1, ch, kb, NL * FK * 2);
            }
        }
        return;
    }

    // ======================= consumers =======================
    if constexpr (WIDE) setmaxnreg_inc<232>();
    const int cw = wg - 1;  // 64 rows: the chunk parity this warpgroup owns; 128 rows: its half of the tile
    const int tid = threadIdx.x & 127, ctid = threadIdx.x - 128;
    const int w = tid >> 5, lane = tid & 31;
    uint8_t* myA = sA + (WIDE ? (size_t)cw * 2 * a_plane : 0);
    const uint32_t a_base = smem_u32(myA), w_base = smem_u32(sW);
    float* part = s_part + (WIDE ? cw * 4 * FM : 0);  // [4][64]: partial (chunk parity, slot) of each row
    const int s0 = WIDE ? 0 : cw * NR;                // this warpgroup's ring
    int s = s0;
    uint32_t ph = 0;
    auto advance = [&]() { if (++s == s0 + NR) { s = s0; ph ^= 1; } };
    auto release = [&](int slot) { if (tid == 0) mbar_arrive(&empty[slot]); };
    // the threads that read and write this warpgroup's A operand
    auto sync_a = [&]() { if constexpr (WIDE) named_bar_sync(2 + cw, 128); else named_bar_sync(1, 256); };

    // the hidden layers' biases, once per CTA: the epilogues read them from shared memory rather than waiting on a
    // global load per chunk
    for (int i = ctid; i < (L - 1) * p.H; i += 256) s_bias[i] = __ldg(p.bias[i / p.H] + i % p.H);
    named_bar_sync(1, 256);

    for (int t = blockIdx.x; t < m_tiles; t += gridDim.x) {
        const int64_t rb = (int64_t)t * ROWS + (WIDE ? cw * FM : 0);  // first row of this warpgroup's A
        if constexpr (!WIDE) named_bar_sync(1, 256);  // the previous tile's MMAs on A and reads of s_part are done
        // ---- stage the layer-0 operand: cat(x, c) -> bf16 hi / lo pairs, 128B-swizzled K blocks ----
        // Only the columns layer 0 multiplies are written (zeros from K0 on); what lies beyond in the last K block
        // is the previous tile's activations, which layer 0 does not read and the first epilogue overwrites.
        const int KW = (p.KB0 - 1) * FK + 16 * p.ks0;
        const int n_thr = WIDE ? 128 : 256;
        if (p.vec_in) {
            // item i = (row i >> g_shift, float4 group i & mask); four loads in flight per thread before the first split
            const int n_it = FM << p.g_shift, gmask = (1 << p.g_shift) - 1;
            for (int i0 = WIDE ? tid : ctid; i0 < n_it; i0 += 4 * n_thr) {
                float4 v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = i0 + j * n_thr, k = (i & gmask) << 2;
                    const int64_t row = rb + (i >> p.g_shift);
                    v[j] = make_float4(0.f, 0.f, 0.f, 0.f);  // masked rows and padded columns stage zeros
                    const float* src = (k < p.D) ? p.x + row * p.ldx + k : p.c + row * p.ldc + (k - p.D);
                    if (i < n_it && row < p.M && k < p.K0) v[j] = __ldg(reinterpret_cast<const float4*>(src));
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = i0 + j * n_thr, k = (i & gmask) << 2;
                    if (i >= n_it || k >= KW) continue;
                    uint2 hi, lo;
                    split2_bf16(v[j].x, v[j].y, hi.x, lo.x);
                    split2_bf16(v[j].z, v[j].w, hi.y, lo.y);
                    const uint32_t off = (uint32_t)(k >> 6) * F_TILE + sw128_offset(i >> p.g_shift, k & 63);
                    *reinterpret_cast<uint2*>(myA + off) = hi;
                    *reinterpret_cast<uint2*>(myA + a_plane + off) = lo;
                }
            }
        } else {
            const int kw = KW / 2;  // bf16 pairs per row
            for (int i = WIDE ? tid : ctid; i < FM * kw; i += n_thr) {
                const int r = i / kw, k = 2 * (i - r * kw);
                const int64_t row = rb + r;
                float v0 = 0.f, v1 = 0.f;  // masked rows and padded columns stage zeros
                if (row < p.M) {
                    if (k < p.D) v0 = __ldg(p.x + row * p.ldx + k);
                    else if (k < p.K0) v0 = __ldg(p.c + row * p.ldc + (k - p.D));
                    if (k + 1 < p.D) v1 = __ldg(p.x + row * p.ldx + k + 1);
                    else if (k + 1 < p.K0) v1 = __ldg(p.c + row * p.ldc + (k + 1 - p.D));
                }
                uint32_t hi, lo;
                split2_bf16(v0, v1, hi, lo);
                const uint32_t off = (uint32_t)(k >> 6) * F_TILE + sw128_offset(r, k & 63);
                *reinterpret_cast<uint32_t*>(myA + off) = hi;
                *reinterpret_cast<uint32_t*>(myA + a_plane + off) = lo;
            }
        }
        fence_proxy_async();  // generic-proxy writes -> visible to the MMAs (async proxy)
        sync_a();

        // ---- hidden layers: D -> bias, activation -> hi/lo -> A (in place) ----
        for (int l = 0; l < L - 1; ++l) {
            const int KB = (l == 0) ? p.KB0 : nch;
            float acc[4][32];
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;
            if constexpr (WIDE) {
                // accumulator q = chunk q; one group per tile, its slot released once the next tile is issued
                int held = -1;
                for (int kb = 0; kb < KB; ++kb) {
                    const int ks = (l == 0 && kb == KB - 1) ? p.ks0 : 4;
#pragma unroll
                    for (int q = 0; q < F_WIDE_MAXKB; ++q) {
                        if (q >= nch || !((p.kbmask[l][q] >> kb) & 1u)) continue;
                        mbar_wait(&full[s], ph);
                        const uint32_t a_hi = a_base + (uint32_t)kb * F_TILE, w_tile = w_base + (uint32_t)s * F_STAGE;
                        with_ksteps(ks, [&](auto KS) {
                            wgmma_fence();
                            wgmma_kblock<decltype(KS)::value>(acc[q], a_hi, a_hi + a_plane, w_tile, w_tile + F_TILE, n_terms);
                            wgmma_commit();
                        });
                        wgmma_wait1();
                        if (held >= 0) release(held);
                        held = s;
                        advance();
                    }
                }
                wgmma_wait0();
                if (held >= 0) release(held);
#pragma unroll
                for (int q = 0; q < 4; ++q) acc_fence(acc[q]);
            } else {
                for (int kb = 0; kb < KB; ++kb) {
                    const int ks = (l == 0 && kb == KB - 1) ? p.ks0 : 4;
                    for (int ch = 0; ch < nch; ++ch) {
                        if (!((p.kbmask[l][ch] >> kb) & 1u)) continue;
                        if ((ch & 1) == cw) {
                            mbar_wait(&full[s], ph);
                            with_ksteps(ks, [&](auto KS) {
                                tile_mma<decltype(KS)::value>(acc, ch >> 1, a_base + (uint32_t)kb * F_TILE, a_plane,
                                                              w_base + (uint32_t)s * F_STAGE, n_terms);
                            });
                            release(s);
                            advance();
                        }
                    }
                }
            }
            sync_a();  // every reader of this A operand is done with it: overwrite it
            const uint32_t bias = smem_u32(s_bias + l * p.H);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int ch = WIDE ? q : 2 * q + cw;
                if (ch >= nch) continue;
                // a warp's 16 x 16 blocks, one stmatrix.x4 per plane: matrix m holds rows 16 w + 8 (m & 1) ... and
                // columns 8 (i0 + m / 2) ...; lane t addresses row t % 8 of matrix t / 8
#pragma unroll
                for (int i0 = 0; i0 < 8; i0 += 2) {
                    uint32_t hi[4], lo[4];
#pragma unroll
                    for (int di = 0; di < 2; ++di) {
                        const int i = i0 + di;
                        const float2 bb = lds_f32x2(bias + 4u * (uint32_t)(ch * FK + 8 * i + 2 * (lane & 3)));
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            float v[2] = {acc[q][4 * i + 2 * hh] + bb.x, acc[q][4 * i + 2 * hh + 1] + bb.y};
                            if constexpr (GACT) {  // any ZK_ACT_* (nn.py:264-265)
                                if constexpr (FAST) act_apply_n_fast<2>(v, p.act); else act_apply_n<2>(v, p.act);
                            } else {
                                v[0] = fmaxf(v[0], 0.f);
                                v[1] = fmaxf(v[1], 0.f);
                            }
                            split2_bf16(v[0], v[1], hi[2 * di + hh], lo[2 * di + hh]);
                        }
                    }
                    const uint32_t off = a_base + (uint32_t)ch * F_TILE +
                                         sw128_offset(w * 16 + 8 * ((lane >> 3) & 1) + (lane & 7), 8 * (i0 + (lane >> 4)));
                    stmatrix_x4(off, hi[0], hi[1], hi[2], hi[3]);
                    stmatrix_x4(off + a_plane, lo[0], lo[1], lo[2], lo[3]);
                }
            }
            fence_proxy_async();
            sync_a();
        }

        // ---- last layer: chunk = whole dims -> parameters gathered from the quad's accumulators -> bijector + ladj ----
        // evaluation: thread = (sample row, share of the chunk's dims), both within its quad's rows
        const int r = w * 16 + outchunk::row(lane), slot = outchunk::slot(lane);
        const int64_t row = rb + r;
        const bool row_ok = row < p.M;
        const float* bias = p.bias[L - 1];
        // the bias pairs of output chunk ch that this thread adds to its accumulators
        auto load_bias = [&](float2 (&bb)[NL / 8], int ch) {
#pragma unroll
            for (int i = 0; i < NL / 8; ++i)
                bb[i] = __ldg(reinterpret_cast<const float2*>(bias + ch * FK + 8 * i + 2 * (lane & 3)));
        };
        // RQS: the input x of this thread's dim of output chunk ch (0 where the thread evaluates nothing)
        auto load_x = [&](int ch) -> float {
            if constexpr (UNI == ZK_UNI_RQS) {
                const int d = ch * DPC + slot;
                if (slot < DPC && d < p.D && row_ok) return __ldg(p.x + row * p.ldx + d);
            }
            return 0.f;
        };
        // this thread's dims of output chunk ch: NE of them (RQS: one, affine: 16), dim j is d_of(ch, j); only those
        // with keep(d) exist
        constexpr int NE = (UNI == ZK_UNI_RQS) ? 1 : 16;
        static_assert(UNI == ZK_UNI_RQS || DPC == 32, "affine chunk layout: 32 (shift, log-scale) pairs");
        auto d_of = [&](int ch, int j) { return (UNI == ZK_UNI_RQS) ? ch * DPC + slot : ch * DPC + slot * 16 + j; };
        auto keep = [&](int d) { return slot < DPC && d < p.D && row_ok; };
        // value part: the bijector and log-derivative of this thread's dims of output chunk ch, from the chunk's
        // accumulators a and bias pairs bb (RQS: xv = load_x(ch)).  Every thread of the warpgroup calls it, and it has
        // no branch: a thread computes on whatever it holds, and store_chunk drops the dims that do not exist.  So the
        // compiler can interleave two calls' dependent MUFU chains.
        auto chunk_values = [&](int ch, float xv, float (&a)[NL / 2], const float2 (&bb)[NL / 8], float (&yv)[NE],
                                float (&lj)[NE]) {
#pragma unroll
            for (int i = 0; i < NL / 8; ++i)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    a[4 * i + 2 * hh] += bb[i].x;
                    a[4 * i + 2 * hh + 1] += bb[i].y;
                }
            float pr[Out::NV];  // staging-order values NV * slot ... of row r
            outchunk::assemble<P, DPC>(a, lane, [](float mine, int mask) { return __shfl_xor_sync(0xffffffffu, mine, mask); }, pr);
            if constexpr (UNI == ZK_UNI_RQS) {
                Bin b = rqs_select<KT, FAST, false>(pr, KT, xv, p.bound, p.aw, p.ad);
                rqs_forward_eval<FAST>(b, xv, yv[0], lj[0]);
            } else {
#pragma unroll
                for (int j = 0; j < NE; ++j) {
                    const int d = d_of(ch, j);
                    const float x = keep(d) ? __ldg(p.x + row * p.ldx + d) : 0.f;
                    lj[j] = softclip<FAST>(pr[2 * j + 1], p.ad);
                    yv[j] = fmaf(x, zexp<FAST>(lj[j]), pr[2 * j]);
                }
            }
        };
        // store part: y of the dims that exist, and their log-derivatives (plus the base log-density on a flow's last
        // layer) summed into ls.  The sum takes a select rather than a zero term, so that -0 partials keep their bits.
        auto store_chunk = [&](int ch, float& ls, const float (&yv)[NE], const float (&lj)[NE]) {
#pragma unroll
            for (int j = 0; j < NE; ++j) {
                const int d = d_of(ch, j);
                const bool ok = keep(d);
                if (ok && p.y) p.y[row * p.ldy + d] = yv[j];
                float l = lj[j];
                if (p.log_prob) {
                    const float mu = (ok && p.base_loc) ? p.base_loc[d] : 0.f;
                    const float sg = (ok && p.base_scale) ? p.base_scale[d] : 1.f;
                    const float u = (yv[j] - mu) / sg;
                    l += -0.5f * u * u - logf(sg) - kHalfLog2Pi;
                }
                ls = ok ? ls + l : ls;
            }
        };
        if constexpr (WIDE) {
            // the next tile's inputs are fetched into L2 while this tile's output layer runs
            {
                const int64_t nrow = rb + (int64_t)gridDim.x * ROWS + r;
                if (nrow < p.M) {
                    const float* src = slot ? p.c + nrow * p.ldc : p.x + nrow * p.ldx;
                    const int len = slot ? p.C : p.D;
                    for (int k = 0; k < len; k += 32) prefetch_l2(src + k);
                }
            }
            // The output chunks go in pairs (A, B) = (ch, ch + 1); with n_last odd the last pair's B is empty (no
            // tiles, no dims).  A pair's tiles, A's then B's, are one stream of asynchronous MMAs with the hidden
            // layers' discipline (one group per tile, a slot released once the next tile is issued), so B's tiles
            // load and multiply behind A's and the pair ends in one full wait.  The bijector runs with no MMAs in
            // flight: its code inside a wgmma pipeline stage makes ptxas serialize every wgmma of the kernel (C7515).
            // Both chunks' bias and this thread's x are loaded before the pair's MMAs, so that their latency runs
            // under the MMAs, and the two chunks' bijectors are evaluated side by side.
            float accA[NL / 2], accB[NL / 2];
            float ls0 = 0.f, ls1 = 0.f;  // partials of the even and of the odd chunks
            for (int ch = 0; ch < p.n_last; ch += 2) {
                const bool has_b = ch + 1 < p.n_last;
#pragma unroll
                for (int i = 0; i < NL / 2; ++i) {
                    accA[i] = 0.f;
                    accB[i] = 0.f;
                }
                // B's zeros are set before A's MMAs: set inside that pipeline stage, they would serialize it (C7515)
                acc_fence(accA);
                acc_fence(accB);
                float2 bbA[NL / 8], bbB[NL / 8];
                load_bias(bbA, ch);
                load_bias(bbB, ch + has_b);  // an empty B reads A's: its results are dropped
                const float xA = load_x(ch), xB = load_x(ch + 1);
                int held = -1;
                auto issue = [&](float (&acc)[NL / 2], uint32_t kbmask) {
                    for (int kb = 0; kb < nch; ++kb) {
                        if (!((kbmask >> kb) & 1u)) continue;
                        mbar_wait(&full[s], ph);
                        const uint32_t a_hi = a_base + (uint32_t)kb * F_TILE, w_tile = w_base + (uint32_t)s * F_STAGE;
                        wgmma_fence();
                        wgmma_kblock(acc, a_hi, a_hi + a_plane, w_tile, w_tile + F_TILE, n_terms);
                        wgmma_commit();
                        wgmma_wait1();
                        if (held >= 0) release(held);
                        held = s;
                        advance();
                    }
                };
                issue(accA, p.kbmask[L - 1][ch]);
                issue(accB, has_b ? p.kbmask[L - 1][ch + 1] : 0u);
                wgmma_wait0();
                if (held >= 0) release(held);
                acc_fence(accA);
                acc_fence(accB);
                float yA[NE], ljA[NE], yB[NE], ljB[NE];
                chunk_values(ch, xA, accA, bbA, yA, ljA);
                chunk_values(ch + 1, xB, accB, bbB, yB, ljB);
                store_chunk(ch, ls0, yA, ljA);
                store_chunk(ch + 1, ls1, yB, ljB);
            }
            part[slot * FM + r] = ls0;
            part[(2 + slot) * FM + r] = ls1;
        } else {
            float lsum = 0.f;
            for (int ch = 0; ch < p.n_last; ++ch) {
                const bool mine = (ch & 1) == cw;
                float acc[NL / 2];
#pragma unroll
                for (int i = 0; i < NL / 2; ++i) acc[i] = 0.f;
                for (int kb = 0; kb < nch; ++kb) {
                    if (!((p.kbmask[L - 1][ch] >> kb) & 1u)) continue;
                    if (mine) {
                        mbar_wait(&full[s], ph);
                        tile_mma(acc, a_base + (uint32_t)kb * F_TILE, a_plane, w_base + (uint32_t)s * F_STAGE, n_terms);
                        release(s);
                        advance();
                    }
                }
                if (!mine) continue;
                float2 bb[NL / 8];
                load_bias(bb, ch);
                float yv[NE], lj[NE];
                chunk_values(ch, load_x(ch), acc, bb, yv, lj);
                store_chunk(ch, lsum, yv, lj);
            }
            part[(2 * cw + slot) * FM + r] = lsum;
        }
        // ---- per-sample sum over the four (chunk parity, share) partials, fixed order ----
        sync_a();
        const int sr = WIDE ? tid : ctid;
        if (sr < FM) {
            const int64_t rr = rb + sr;
            if (rr < p.M) {
                const float tot = part[sr] + part[FM + sr] + part[2 * FM + sr] + part[3 * FM + sr] +
                                  (p.accumulate ? p.ladj[rr] : 0.f);
                if (p.log_prob) p.log_prob[rr] = tot;
                else if (p.ladj) p.ladj[rr] = tot;
            }
        }
    }
}

template <int UNI, int KT, int ROWS, int NT>
zk_status launch_fused_t(const FusedParams& p, bool fast, int grid, size_t smem, cudaStream_t st) {
    auto go = [&](auto kern) -> zk_status {
        ZK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F_SMEM_MAX));
        kern<<<grid, F_THREADS, smem, st>>>(p);
        return check_launch("fused_layer_kernel");
    };
    if (p.act > 1)
        return fast ? go(fused_layer_kernel<UNI, KT, true, true, ROWS, NT>) : go(fused_layer_kernel<UNI, KT, false, true, ROWS, NT>);
    return fast ? go(fused_layer_kernel<UNI, KT, true, false, ROWS, NT>) : go(fused_layer_kernel<UNI, KT, false, false, ROWS, NT>);
}

template <int UNI, int KT>
zk_status launch_fused_rows(const FusedParams& p, int rows, bool fast, int grid, size_t smem, cudaStream_t st) {
    if (rows == 64) return launch_fused_t<UNI, KT, 64, 0>(p, fast, grid, smem, st);
    return p.n_terms == 3 ? launch_fused_t<UNI, KT, 128, 3>(p, fast, grid, smem, st) : launch_fused_t<UNI, KT, 128, 1>(p, fast, grid, smem, st);
}

// Row tile and W ring depth of a shape: 128-row tiles when the four accumulators of a consumer hold every
// hidden chunk (KBA <= 4) and a ring of at least four slots fits beside the two A operands; 64-row tiles
// otherwise.  The ring gets every byte of shared memory the A operand(s), staging buffers, partials and
// barriers leave.
struct FusedPlan {
    int rows = 0, n_stages = 0;
    size_t smem = 0;
};
FusedPlan fused_plan(int KBA, int univariate, int bins) {
    const uint32_t srow = (uint32_t)f_srow(fused_dpc(univariate, bins) * fused_p(univariate, bins));
    for (int rows : {128, 64}) {
        const uint32_t fixed = 1024u /*alignment slack*/ + (uint32_t)(rows / FM) * 2u * (uint32_t)KBA * F_TILE +
                               2u * FM * srow * 4u + 4u * (uint32_t)rows * 4u + 2u * F_MAX_STAGES * 8u;
        if (fixed >= F_SMEM_MAX) continue;
        int ns = (int)std::min<uint32_t>(F_MAX_STAGES, (F_SMEM_MAX - fixed) / F_STAGE);
        if (rows == 128 && (KBA > F_WIDE_MAXKB || ns < 4)) continue;
        if (rows == 64) ns &= ~1;  // two rings of equal depth
        return {rows, ns, (size_t)ns * F_STAGE + fixed};
    }
    return {};
}

}  // namespace

static bool fused_shape(const zk_mlp* m, int univariate, int bins, int D, int C) {
    const TcPack* pk = (const TcPack*)m->tc;
    if (!pk || m->gemm_mode == ZK_GEMM_FP32) return false;
    if (m->act < 1 || !m->plain) return false;  // plain MLPs only (residual blocks need the input of two layers back)
    if (m->n_linear < 2 || m->n_linear > ZK_FUSED_MAX_LINEAR) return false;
    const int H = m->dims[1];
    if (H % 64 != 0 || H < 64 || H > 64 * F_MAXKB) return false;
    for (int i = 1; i < m->n_linear; ++i)
        if (m->dims[i] != H) return false;
    if (D + C > 64 * F_MAXKB || m->dims[0] != D + C) return false;
    if (univariate == ZK_UNI_RQS) {
        if (bins != 8 && bins != 16) return false;
    } else if (univariate != ZK_UNI_AFFINE) {
        return false;
    }
    const int dpc = fused_dpc(univariate, bins);
    return (D + dpc - 1) / dpc <= 128;
}

bool fused_layer_supported(const zk_mlp* m, int univariate, int bins, int D, int C) {
    if (!fused_shape(m, univariate, bins, D, C)) return false;
    const FusedPack& f = ((const TcPack*)m->tc)->fused;
    return f.ready && f.uni == univariate && f.bins == bins && f.D == D && f.C == C;
}

int fused_layer_kind(const zk_mlp* m, int univariate, int bins, int D, int C) {
    return fused_layer_supported(m, univariate, bins, D, C) ? 1 : 0;
}

// K blocks of the fused kernel's A operand: the wider of the input and the hidden width
// k16 steps of layer 0's last K block that hold inputs
static int fused_ks0(int K0, int KB0) { return (K0 - FK * (KB0 - 1) + 15) / 16; }

static int fused_kba(const zk_mlp* m) {
    return std::max(((const TcPack*)m->tc)->layers[0].Kp / FK, m->dims[1] / FK);
}

int fused_layer_plan(const zk_mlp* m, int univariate, int bins, int D, int C, int* ring_slots, size_t* smem) {
    if (!fused_layer_supported(m, univariate, bins, D, C)) return 0;
    const FusedPlan plan = fused_plan(fused_kba(m), univariate, bins);
    if (ring_slots) *ring_slots = plan.n_stages;
    if (smem) *smem = plan.smem;
    return plan.rows;
}

int fused_tile_rows(const zk_mlp* m, int univariate, int bins, int D, int C) {
    return fused_layer_plan(m, univariate, bins, D, C, nullptr, nullptr);
}

namespace {
// planes [2][N][Kp] of W (N, K) with rows / columns gathered: row n <- W row row_map[n] (-1: zero row)
__global__ void split_permuted_kernel(const float* W, int N, int K, int Kp, const int* row_map, const int* col_perm,
                                      __nv_bfloat16* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * Kp) return;
    const int n = (int)(i / Kp), k = (int)(i - (int64_t)n * Kp);
    const int sn = row_map ? row_map[n] : n;
    const float v = (k < K && sn >= 0) ? W[(int64_t)sn * K + (col_perm ? col_perm[k] : k)] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    out[i] = h;
    out[(int64_t)N * Kp + i] = __float2bfloat16_rn(v - __bfloat162float(h));
}
__global__ void permute_bias_kernel(const float* b, int N, const int* row_map, float* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) out[i] = row_map ? (row_map[i] >= 0 ? b[row_map[i]] : 0.f) : b[i];
}
}  // namespace

// Dependency degree of every hidden unit = number of network inputs it can see
// (flows/autoregressive.py:121-124 + nn.py:270-293: units of a lower order class see fewer inputs);
// sorting by degree makes the hidden -> hidden masks block lower-triangular.  Pure host code.
void fused_degree_perm(const int* dims, int L, const std::vector<std::vector<uint8_t>>& Mk,
                       std::vector<std::vector<int>>& perm) {
    const int K0 = dims[0];
    perm.assign(L - 1, {});  // perm[l][new] = old index of hidden layer l+1's units
    // dependency sets as bit rows: dep[unit] = OR of the dep rows of the inputs it is connected to
    const int W64 = (K0 + 63) / 64;
    std::vector<uint64_t> prev, cur;
    for (int l = 0; l < L - 1; ++l) {
        const int K = dims[l], N = dims[l + 1];
        cur.assign((size_t)N * W64, 0);
        for (int n = 0; n < N; ++n) {
            uint64_t* dn = &cur[(size_t)n * W64];
            const uint8_t* mrow = &Mk[l][(size_t)n * K];
            for (int k = 0; k < K; ++k) {
                if (!mrow[k]) continue;
                if (l == 0) dn[k >> 6] |= (uint64_t)1 << (k & 63);
                else {
                    const uint64_t* dk = &prev[(size_t)k * W64];
                    for (int w = 0; w < W64; ++w) dn[w] |= dk[w];
                }
            }
        }
        std::vector<int> deg(N, 0);
        for (int n = 0; n < N; ++n)
            for (int w = 0; w < W64; ++w) deg[n] += __builtin_popcountll(cur[(size_t)n * W64 + w]);
        perm[l].resize(N);
        for (int n = 0; n < N; ++n) perm[l][n] = n;
        std::stable_sort(perm[l].begin(), perm[l].end(), [&](int a, int b) { return deg[a] < deg[b]; });
        prev.swap(cur);
    }
}

// rows of the fused pack's layer l (hidden layers: all units; output layer: n_last 64-row chunks)
static int fused_rows(const zk_mlp* m, const FusedPack& f, int l) {
    return (l == m->n_linear - 1) ? f.n_last * FK : m->dims[l + 1];
}

// split kernels of the fused pack (stream-ordered): permuted / regrouped bf16 planes and biases
static zk_status fused_split(zk_mlp* m, FusedPack& f, cudaStream_t st) {
    const TcPack* pk = (const TcPack*)m->tc;
    const int L = m->n_linear;
    for (int l = 0; l < L; ++l) {
        const int K = m->dims[l], N = fused_rows(m, f, l), Kp = pk->layers[l].Kp;
        const int* rp = (l < L - 1) ? f.dperm[l] : f.last_rows;  // output units of hidden layers are permuted
        const int* cp = (l > 0) ? f.dperm[l - 1] : nullptr;      // and so are the inputs of the layer after
        split_permuted_kernel<<<(unsigned)ceil_div((int64_t)N * Kp, 256), 256, 0, st>>>(m->w[l], N, K, Kp, rp, cp, f.w[l]);
        ZK_TRY(check_launch("split_permuted_kernel"));
        permute_bias_kernel<<<(unsigned)ceil_div(N, 256), 256, 0, st>>>(m->b[l], N, rp, f.bias[l]);
        ZK_TRY(check_launch("permute_bias_kernel"));
    }
    return ZK_OK;
}

// The weights of `m` changed in place (same shapes, same masks): rebuild the fused kernel's permuted
// planes and biases with the permutations of the last fused_layer_prepare.  Stream-ordered, no
// allocation, no host synchronisation; tensor maps and zero-tile masks depend on the masks only and stay.
zk_status fused_refresh(zk_mlp* m, cudaStream_t st) {
    TcPack* pk = (TcPack*)m->tc;
    if (!pk || !pk->fused.ready) return ZK_OK;  // no fused pack was built
    return fused_split(m, pk->fused, st);
}

// Masks to the host, hidden units sorted by dependency degree, output rows regrouped into 64-row
// chunks of whole dims, permuted bf16 hi / lo planes and biases on the device, tensor maps and the
// map of all-zero (chunk, K block) tiles.
zk_status fused_layer_prepare(zk_mlp* m, const uint8_t* const* mask_dev, int univariate, int bins, int D, int C) {
    if (!fused_shape(m, univariate, bins, D, C)) return ZK_OK;
    TcPack* pk = (TcPack*)m->tc;
    FusedPack& f = pk->fused;
    f.ready = false;
    const int L = m->n_linear;
    const int H = m->dims[1];
    const int P = fused_p(univariate, bins);
    const int DPC = fused_dpc(univariate, bins);
    // ---- host copies of the masks (dense layers: all ones) ----
    std::vector<std::vector<uint8_t>> Mk(L);
    for (int l = 0; l < L; ++l) {
        const size_t n = (size_t)m->dims[l + 1] * m->dims[l];
        Mk[l].assign(n, 1);
        if (mask_dev && mask_dev[l]) ZK_CUDA(cudaMemcpy(Mk[l].data(), mask_dev[l], n, cudaMemcpyDeviceToHost));
    }
    std::vector<std::vector<int>> perm;
    fused_degree_perm(m->dims.data(), L, Mk, perm);
    // output layer: the 64 padded rows of chunk ch hold the P parameters of dims ch * DPC ... ch * DPC + DPC - 1 (or
    // zeros), in the column order of fused_out_chunk.cuh
    f.n_last = (D + DPC - 1) / DPC;
    std::vector<int> last_rows((size_t)f.n_last * FK);
    outchunk::last_rows(D, P, DPC, f.n_last, last_rows.data());
    // ---- device buffers ----
    for (auto* q : f.w) cudaFree(q);
    for (auto* q : f.bias) cudaFree(q);
    for (auto* q : f.dperm) cudaFree(q);
    cudaFree(f.last_rows);
    f.w.assign(L, nullptr);
    f.bias.assign(L, nullptr);
    f.dperm.assign(L - 1, nullptr);
    f.last_rows = nullptr;
    auto upload = [](int** dst, const std::vector<int>& v) -> bool {
        return cudaMalloc((void**)dst, v.size() * 4) == cudaSuccess &&
               cudaMemcpy(*dst, v.data(), v.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess;
    };
    for (int l = 0; l < L - 1; ++l)
        if (!upload(&f.dperm[l], perm[l])) return fail(ZK_ENOMEM, "fused_layer_prepare: cudaMalloc failed");
    if (!upload(&f.last_rows, last_rows)) return fail(ZK_ENOMEM, "fused_layer_prepare: cudaMalloc failed");
    for (int l = 0; l < L; ++l) {
        const int N = fused_rows(m, f, l), Kp = pk->layers[l].Kp;
        if (cudaMalloc((void**)&f.w[l], (size_t)2 * N * Kp * 2) != cudaSuccess ||
            cudaMalloc((void**)&f.bias[l], ((size_t)N + 4) * 4) != cudaSuccess)
            return fail(ZK_ENOMEM, "fused_layer_prepare: cudaMalloc failed");
        ZK_CUDA(cudaMemset(f.bias[l], 0, ((size_t)N + 4) * 4));
    }
    ZK_TRY(fused_split(m, f, 0));
    ZK_CUDA(cudaStreamSynchronize(0));
    // the output layer's box covers the NL rows of a 64-row chunk that hold parameters
    const int NL = fused_nl(univariate, bins);
    f.maps.assign(L, CUtensorMap{});
    for (int l = 0; l < L; ++l)
        ZK_TRY(make_plane_map(&f.maps[l], f.w[l], fused_rows(m, f, l), pk->layers[l].Kp, l == L - 1 ? NL : FK));
    // ---- which (chunk, K block) tiles of the permuted masked matrices are non-zero ----
    memset(f.kbmask, 0, sizeof(f.kbmask));
    f.n_items = 0;
    f.issued_macs_per_row = 0;
    f.stream_bytes = 0;
    const int KB0 = pk->layers[0].Kp / FK, planes = (pk->n_terms == 3) ? 2 : 1;
    for (int l = 0; l < L; ++l) {
        const bool last = (l == L - 1);
        const int K = m->dims[l];
        const int nch = last ? f.n_last : H / FK;
        for (int ch = 0; ch < nch; ++ch) {
            uint8_t bits = 0;
            for (int j = 0; j < FK; ++j) {
                const int sn = last ? last_rows[(size_t)ch * FK + j] : perm[l][ch * FK + j];
                if (sn < 0) continue;
                for (int k = 0; k < K; ++k) {
                    const int sk = (l > 0) ? perm[l - 1][k] : k;
                    if (Mk[l][(size_t)sn * K + sk]) bits |= (uint8_t)(1u << (k / 64));
                }
            }
            f.kbmask[l][ch] = bits;
            f.n_items += __builtin_popcount(bits);
            // what the kernel issues and streams for these tiles: N = NL in the output layer, fused_ks0 k16 steps in
            // layer 0's last K block (whose box is still 64 columns wide)
            const int n = last ? NL : FK;
            for (int kb = 0; kb < 8; ++kb) {
                if (!((bits >> kb) & 1)) continue;
                const int k = (l == 0 && kb == KB0 - 1) ? 16 * fused_ks0(m->dims[0], KB0) : FK;
                f.issued_macs_per_row += (double)n * k * pk->n_terms;
                f.stream_bytes += (size_t)n * FK * 2 * planes;
            }
        }
    }
    f.uni = univariate; f.bins = bins; f.D = D; f.C = C;
    f.ready = true;
    return ZK_OK;
}

zk_status launch_fused_layer(const zk_mlp* m, const FusedLayerArgs& a, cudaStream_t st) {
    ZK_REQUIRE(fused_layer_supported(m, a.univariate, a.bins, a.D, a.C), "fused layer: the conditioner was not prepared for this bijector");
    ZK_REQUIRE(a.B < ((int64_t)1 << 31) - 2 * FM, "fused layer: batch too large for one launch");
    if (a.B == 0) return ZK_OK;
    const TcPack* pk = (const TcPack*)m->tc;
    const FusedPack& f = pk->fused;
    FusedParams p;
    memset(&p, 0, sizeof(p));
    memcpy(p.kbmask, f.kbmask, sizeof(p.kbmask));
    for (int i = 0; i < m->n_linear; ++i) {
        p.mapW[i] = f.maps[i];
        p.bias[i] = f.bias[i];
    }
    p.n_linear = m->n_linear;
    p.K0 = a.D + a.C;
    p.KB0 = pk->layers[0].Kp / FK;
    p.ks0 = fused_ks0(p.K0, p.KB0);
    const auto vec4 = [](const float* q, int n, int64_t ld) { return n % 4 == 0 && ld % 4 == 0 && ((uintptr_t)q & 15) == 0; };
    p.vec_in = vec4(a.x, a.D, a.ldx) && (a.C == 0 || vec4(a.c, a.C, a.ldc));
    while ((4 << p.g_shift) < (p.KB0 - 1) * FK + 16 * p.ks0) ++p.g_shift;
    p.H = m->dims[1];
    p.KBA = fused_kba(m);
    p.D = a.D; p.C = a.C;
    p.n_last = f.n_last;
    p.n_terms = pk->n_terms;
    p.act = m->act;
    p.M = (int)a.B;
    p.x = a.x; p.ldx = a.ldx; p.c = a.c; p.ldc = a.ldc;
    p.y = a.y; p.ldy = a.ldy; p.ladj = a.ladj; p.accumulate = a.accumulate;
    p.log_prob = a.log_prob; p.base_loc = a.base_loc; p.base_scale = a.base_scale;
    p.bound = a.bound;
    const float absL = fabsf(logf(a.slope));
    p.aw = 2.f / absL;
    p.ad = 1.f / absL;
    const FusedPlan plan = fused_plan(p.KBA, a.univariate, a.bins);
    ZK_REQUIRE(plan.n_stages >= 4, "fused layer: not enough shared memory for the weight rings");
    p.n_stages = plan.n_stages;
    const int grid = (int)std::min<int64_t>(ceil_div(a.B, plan.rows), sm_count());
    if (a.univariate == ZK_UNI_RQS && a.bins == 8)
        return launch_fused_rows<ZK_UNI_RQS, 8>(p, plan.rows, a.fast_math, grid, plan.smem, st);
    if (a.univariate == ZK_UNI_RQS) return launch_fused_rows<ZK_UNI_RQS, 16>(p, plan.rows, a.fast_math, grid, plan.smem, st);
    return launch_fused_rows<ZK_UNI_AFFINE, 0>(p, plan.rows, a.fast_math, grid, plan.smem, st);
}

}  // namespace zk
