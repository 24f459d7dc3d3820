// zuko_b200 — conditioner GEMMs on the Hopper tensor cores (wgmma, sm_90a).
//
// One linear layer  C[M, N] = act(A[M, K] W[N, K]^T + b)  of MaskedMLP / MLP
// (zuko/nn.py:217-218 with the mask folded into W at pack time) as a persistent,
// warp-specialised kernel over 128 x 128 output tiles:
//
//   warpgroup 0   TMA producer : one thread issues cp.async.bulk.tensor (128B-swizzled boxes) of the
//                                A and W tiles into a shared-memory ring, completion on mbarriers
//   warpgroups 1-2 consumers   : warpgroup g owns rows [64 (g - 1), 64 g) of the tile; it issues
//                                wgmma.mma_async m64n64k16 (both operands in shared memory, fp32
//                                accumulators in registers), releases the ring slot, and runs the
//                                epilogue (bias, activation -> fp32 phi or bf16 hi/lo planes for the
//                                next layer) straight from the accumulator registers
//
// Precision: fp32 inputs are carried as TWO bf16 planes (hi = rn(v), lo = rn(v - hi)) and the
// product is formed as  A_hi W_hi + A_hi W_lo + A_lo W_hi  with fp32 accumulation
// (ZK_GEMM_BF16X3).  A single bf16 MMA misses the 1e-5 parity bar of BASELINE.json (1.4e-4 on
// config 2, SURVEY §7.4-1); the 3-MMA split meets it.  ZK_GEMM_BF16X1 keeps only the first term
// (fast, inexact, opt-in).
//
// Operand layout in HBM: activations act[plane][M][Kp] and weights w[plane][N][Kp], bf16,
// K contiguous ("K-major"), Kp = K rounded up to 64 with zero padding.  A TMA box of
// (64 x rows) bf16 lands in shared memory as rows of 128 bytes with the 128B swizzle, which is
// the K-major SWIZZLE_128B wgmma operand layout (8-row groups 1024 B apart).

#include "activations.cuh"
#include "mlp_tcgen05.cuh"
#include "tc_common.cuh"

namespace zk {

namespace {

constexpr int BM = 128;        // rows per tile (two warpgroups of 64)
constexpr int BN = 128;        // output columns per tile (two 64-wide MMA column blocks)
constexpr int BK = 64;         // bf16 per K block = one 128-byte swizzle row
constexpr int STAGES = 3;      // shared-memory ring depth
constexpr int kThreads = 384;  // producer warpgroup + two consumer warpgroups

constexpr uint32_t A_TILE_BYTES = BM * BK * 2;  // 16 KB per plane
constexpr uint32_t W_TILE_BYTES = BN * BK * 2;  // 16 KB per plane
constexpr uint32_t STAGE_BYTES = 2 * A_TILE_BYTES + 2 * W_TILE_BYTES;  // 64 KB
constexpr size_t SMEM_BYTES = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;

struct TcParams {
    int M, N, Kp;        // rows, real output columns, padded K (multiple of 64)
    int n_chunks;        // ceil(N / BN)
    int n_terms;         // 3 = split-bf16 (hi*hi + hi*lo + lo*hi), 1 = hi*hi only
    int relu;
    const float* bias;   // (N) fp32
    // output: either fp32 (out_f32 != nullptr) or bf16 planes for the next layer
    float* out_f32;
    int64_t ldo;
    __nv_bfloat16* out_planes;  // [2][M][Np]
    int Np;                     // padded width of the next layer's K
    // backward pass (tc_gemm): ReLU gate and batch-sliced weight operand
    const __nv_bfloat16* gate;  // [M][Np] hi plane of a ReLU output: out = gate > 0 ? out : 0 (planes output only)
    // second layer of a residual block (zuko/nn.py:195-199; GENERAL_ACT instantiation, planes output only):
    // hi + lo of these planes [2][M][Np] is added to the output.  May alias out_planes: every element is read
    // by the thread that then overwrites it.
    const __nv_bfloat16* res;
    int slice_m;                // > 0: rows [s * slice_m, (s + 1) * slice_m) of A pair with W rows s * w_slice_rows + n
    int w_slice_rows;
};

// relu(bf16 v) > 0 test on the raw bits: positive and not zero
__device__ __forceinline__ bool bf16_positive(uint32_t b) { return (b & 0x7fffu) != 0u && (b & 0x8000u) == 0u; }

// ---------------------------------------------------------------------------
// the GEMM kernel
// ---------------------------------------------------------------------------
// GENERAL_ACT = false: epilogue activation none / ReLU only (the hot instantiation — every BASELINE config);
// true: any ZK_ACT_* through act_apply() and the residual input.  Two instantiations keep the general
// switch out of the hot epilogue.
template <bool GENERAL_ACT>
__global__ void __launch_bounds__(kThreads, 1)
linear_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW,
                 const TcParams p) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment: SWIZZLE_128B atoms are 8 rows x 128 B
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = (uint64_t*)(smem + (size_t)STAGES * STAGE_BYTES);
    uint64_t* full_bar = bars;            // [STAGES]   TMA -> consumers
    uint64_t* empty_bar = bars + STAGES;  // [STAGES]   consumers -> TMA (one arrival per consumer warpgroup)

    const int wg = threadIdx.x >> 7;
    const int m_tiles = (p.M + BM - 1) / BM;
    const int total_tiles = m_tiles * p.n_chunks;
    const int k_blocks = p.Kp / BK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ================= TMA producer =================
        if (threadIdx.x == 0) {
            const uint32_t bytes = (p.n_terms == 3) ? STAGE_BYTES : (A_TILE_BYTES + W_TILE_BYTES);
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                const int m0 = (t / p.n_chunks) * BM;
                const int n0 = (t % p.n_chunks) * BN;
                // split-K wgrad: the batch slice this M tile belongs to selects the W rows
                const int wr = n0 + (p.slice_m > 0 ? (m0 / p.slice_m) * p.w_slice_rows : 0);
                for (int kb = 0; kb < k_blocks; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* st = smem + (size_t)stage * STAGE_BYTES;
                    mbar_arrive_expect_tx(&full_bar[stage], bytes);
                    tma_load_3d(st, &mapA, &full_bar[stage], kb * BK, m0, 0);                      // A hi
                    tma_load_3d(st + 2 * A_TILE_BYTES, &mapW, &full_bar[stage], kb * BK, wr, 0);   // W hi
                    if (p.n_terms == 3) {
                        tma_load_3d(st + A_TILE_BYTES, &mapA, &full_bar[stage], kb * BK, m0, 1);   // A lo
                        tma_load_3d(st + 2 * A_TILE_BYTES + W_TILE_BYTES, &mapW, &full_bar[stage], kb * BK, wr, 1);  // W lo
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ================= consumers: MMA + epilogue =================
    const int h = wg - 1;                 // row half of the tile
    const int tid = threadIdx.x & 127;
    const int w = tid >> 5, lane = tid & 31;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int m0 = (t / p.n_chunks) * BM;
        const int n0 = (t % p.n_chunks) * BN;
        const int n_sz = min(BN, p.N - n0);  // real columns of this tile (> 0)
        float acc[2][32];
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
        for (int kb = 0; kb < k_blocks; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sbase = smem_u32(smem) + (uint32_t)stage * STAGE_BYTES;
            const uint32_t a_hi = sbase + (uint32_t)h * (A_TILE_BYTES / 2), a_lo = a_hi + A_TILE_BYTES;
            const uint32_t w_hi = sbase + 2 * A_TILE_BYTES, w_lo = w_hi + W_TILE_BYTES;
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < 2; ++c)
                if (c * 64 < n_sz)
                    wgmma_kblock(acc[c], a_hi, a_lo, w_hi + (uint32_t)c * (W_TILE_BYTES / 2), w_lo + (uint32_t)c * (W_TILE_BYTES / 2),
                                 p.n_terms);
            wgmma_commit();
            wgmma_wait0();
            acc_fence(acc[0]);
            acc_fence(acc[1]);
            if (tid == 0) mbar_arrive(&empty_bar[stage]);  // slot free: this warpgroup's MMAs have read it
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        // ---- epilogue straight from the accumulator registers ----
        const int r_base = m0 + h * 64 + w * 16 + (lane >> 2);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int n = n0 + c * 64 + 8 * i + 2 * (lane & 3);  // first of the thread's two columns
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int row = r_base + 8 * hh;
                    if (row >= p.M) continue;
                    float v[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float f = acc[c][4 * i + 2 * hh + e] + ((p.bias != nullptr && n + e < p.N) ? __ldg(p.bias + n + e) : 0.f);
                        if constexpr (GENERAL_ACT) {
                            if (p.relu == 1) f = fmaxf(f, 0.f);
                            else if (p.relu > 1) f = act_apply(f, p.relu);
                        } else {
                            if (p.relu) f = fmaxf(f, 0.f);
                        }
                        v[e] = (n + e < p.N) ? f : 0.f;  // padded columns feed the next layer as exact zeros
                    }
                    if (p.out_f32 != nullptr) {
                        float* dst = p.out_f32 + (int64_t)row * p.ldo + n;
                        if (n < p.N) dst[0] = v[0];
                        if (n + 1 < p.N) dst[1] = v[1];
                        continue;
                    }
                    if (n >= p.Np) continue;  // Np is even: the pair is in range together
                    const int64_t off = (int64_t)row * p.Np + n;
                    if (p.gate != nullptr) {  // d relu: zero where the forward activation was not positive
                        const uint32_t gv = __ldg(reinterpret_cast<const unsigned int*>(p.gate + off));
                        if (!bf16_positive(gv & 0xffffu)) v[0] = 0.f;
                        if (!bf16_positive(gv >> 16)) v[1] = 0.f;
                    }
                    if constexpr (GENERAL_ACT) {
                        if (p.res != nullptr) {  // plain loads: the planes may be the ones written below
                            const uint32_t a = *reinterpret_cast<const uint32_t*>(p.res + off);
                            const uint32_t b = *reinterpret_cast<const uint32_t*>(p.res + (int64_t)p.M * p.Np + off);
                            v[0] += __uint_as_float(a << 16) + __uint_as_float(b << 16);
                            v[1] += __uint_as_float(a & 0xffff0000u) + __uint_as_float(b & 0xffff0000u);
                        }
                    }
                    // split into bf16 hi / lo planes (K-major operand of the next layer)
                    uint32_t ph, pl;
                    split2_bf16(v[0], v[1], ph, pl);
                    *reinterpret_cast<uint32_t*>(p.out_planes + off) = ph;
                    *reinterpret_cast<uint32_t*>(p.out_planes + (int64_t)p.M * p.Np + off) = pl;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------
// helper kernels: fp32 -> bf16 hi/lo planes
// ---------------------------------------------------------------------------
// weights: W (N, K) fp32 (already masked) -> planes [2][N][Kp], zero padded along K
__global__ void split_weight_kernel(const float* W, int N, int K, int Kp, __nv_bfloat16* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * Kp) return;
    const int n = (int)(i / Kp), k = (int)(i - (int64_t)n * Kp);
    const float v = (k < K) ? W[(int64_t)n * K + k] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    out[i] = h;
    out[(int64_t)N * Kp + i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// first-layer input: cat(x, c) (flows/autoregressive.py:209) -> planes [2][M][Kp]; 8 columns per thread
__global__ void split_input_kernel(const float* x, int64_t ldx, int dx, const float* c, int64_t ldc, int dc,
                                   int64_t M, int Kp, __nv_bfloat16* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int per_row = Kp / 8;
    if (i >= M * per_row) return;
    const int64_t r = i / per_row;
    const int k0 = (int)(i - r * per_row) * 8;
    uint32_t ph[4], pl[4];
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
        float v[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int k = k0 + j + u;
            v[u] = (k < dx) ? x[r * ldx + k] : ((k < dx + dc) ? c[r * ldc + (k - dx)] : 0.f);
        }
        const __nv_bfloat16 h0 = __float2bfloat16_rn(v[0]), h1 = __float2bfloat16_rn(v[1]);
        const __nv_bfloat16 l0 = __float2bfloat16_rn(v[0] - __bfloat162float(h0));
        const __nv_bfloat16 l1 = __float2bfloat16_rn(v[1] - __bfloat162float(h1));
        ph[j >> 1] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        pl[j >> 1] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    __nv_bfloat16* hi = out + r * Kp + k0;
    __nv_bfloat16* lo = hi + M * Kp;
    *reinterpret_cast<uint4*>(hi) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
    *reinterpret_cast<uint4*>(lo) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

}  // namespace

zk_status make_plane_map(CUtensorMap* map, const void* base, int64_t rows, int Kp, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return fail(ZK_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[3] = {(cuuint64_t)Kp, (cuuint64_t)rows, 2};
    cuuint64_t strides[2] = {(cuuint64_t)Kp * 2, (cuuint64_t)rows * Kp * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(ZK_ECUDA, "cuTensorMapEncodeTiled failed (%d) rows=%lld Kp=%d", (int)r, (long long)rows, Kp);
    return ZK_OK;
}

namespace {

}  // namespace

void tc_destroy(zk_mlp* m) {
    TcPack* pk = (TcPack*)m->tc;
    if (!pk) return;
    for (auto& l : pk->layers) cudaFree(l.w);
    for (auto& l : pk->bwd) cudaFree(l.w);
    for (auto* q : pk->fused.w) cudaFree(q);
    for (auto* q : pk->fused.bias) cudaFree(q);
    for (auto* q : pk->fused.dperm) cudaFree(q);
    cudaFree(pk->fused.last_rows);
    delete pk;
    m->tc = nullptr;
}

zk_status tc_pack(zk_mlp* m, int requested_mode) {
    m->gemm_mode = ZK_GEMM_FP32;
    if (requested_mode == ZK_GEMM_FP32) return ZK_OK;
    // AUTO: the tensor-core path pays off once the layers are at least one tile wide
    bool eligible = true;
    int max_dim = 0;
    for (int d : m->dims) max_dim = d > max_dim ? d : max_dim;
    if (max_dim < 64) eligible = false;
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess)
        return fail(ZK_ECUDA, "tc_pack: no CUDA device");
    if (major != 9) eligible = false;  // the wgmma kernels are built for sm_90a only
    if (!encode_fn()) eligible = false;
    if (!eligible) {
        if (requested_mode == ZK_GEMM_AUTO) return ZK_OK;
        return fail(ZK_EUNSUPPORTED, "tensor-core GEMM path unavailable (needs sm_90 and layer widths >= 64; widest is %d)", max_dim);
    }
    TcPack* pk = new TcPack();
    pk->n_terms = (requested_mode == ZK_GEMM_BF16X1) ? 1 : 3;
    m->tc = pk;
    for (int i = 0; i < m->n_linear; ++i) {
        TcLayer L;
        L.K = m->dims[i];
        L.N = m->dims[i + 1];
        L.Kp = pad64(L.K);
        const size_t elems = (size_t)2 * L.N * L.Kp;
        if (cudaMalloc((void**)&L.w, elems * 2) != cudaSuccess) {
            pk->layers.push_back(L);
            return fail(ZK_ENOMEM, "tc_pack: cudaMalloc failed");
        }
        pk->layers.push_back(L);
        split_weight_kernel<<<(unsigned)ceil_div((int64_t)L.N * L.Kp, 256), 256, 0, 0>>>(m->w[i], L.N, L.K, L.Kp, L.w);
        ZK_TRY(check_launch("split_weight_kernel"));
        ZK_TRY(make_plane_map(&pk->layers.back().mapW, L.w, L.N, L.Kp, BN));
        if (i < m->n_linear - 1) pk->max_np = std::max(pk->max_np, pad64(L.N));
    }
    ZK_CUDA(cudaFuncSetAttribute(linear_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    ZK_CUDA(cudaFuncSetAttribute(linear_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    m->gemm_mode = (pk->n_terms == 3) ? ZK_GEMM_BF16X3 : ZK_GEMM_BF16X1;
    return ZK_OK;
}

zk_status tc_refresh(zk_mlp* m, cudaStream_t st) {
    TcPack* pk = (TcPack*)m->tc;
    if (!pk) return ZK_OK;
    for (int i = 0; i < m->n_linear; ++i) {
        const TcLayer& L = pk->layers[i];
        split_weight_kernel<<<(unsigned)ceil_div((int64_t)L.N * L.Kp, 256), 256, 0, st>>>(m->w[i], L.N, L.K, L.Kp, L.w);
        ZK_TRY(check_launch("split_weight_kernel"));
    }
    return ZK_OK;
}

size_t tc_workspace_bytes(const zk_mlp* m, int64_t B) {
    const TcPack* pk = (const TcPack*)m->tc;
    if (!pk || B <= 0) return 0;
    size_t in_planes = align_up((size_t)2 * B * pk->layers[0].Kp * 2, 256);
    size_t hid = (m->n_linear > 1) ? 2 * align_up((size_t)2 * B * pk->max_np * 2, 256) : 0;
    return in_planes + hid;
}

zk_status tc_forward(const zk_mlp* m, const float* x, int64_t ldx, int dx, const float* c, int64_t ldc,
                     int dc, int64_t B, float* out, int64_t ldo, void* ws, size_t ws_bytes,
                     cudaStream_t st) {
    const TcPack* pk = (const TcPack*)m->tc;
    ZK_REQUIRE(pk, "tc_forward: handle was not packed for the tensor-core path");
    ZK_REQUIRE(B < ((int64_t)1 << 31) - BM, "tc_forward: batch too large for one launch");
    ZK_REQUIRE(ws_bytes >= tc_workspace_bytes(m, B), "tc_forward: workspace too small");
    char* base = (char*)ws;
    __nv_bfloat16* in_planes = (__nv_bfloat16*)base;
    base += align_up((size_t)2 * B * pk->layers[0].Kp * 2, 256);
    __nv_bfloat16* hid[2] = {nullptr, nullptr};
    if (m->n_linear > 1) {
        hid[0] = (__nv_bfloat16*)base;
        hid[1] = (__nv_bfloat16*)(base + align_up((size_t)2 * B * pk->max_np * 2, 256));
    }
    // cat(x, c) -> bf16 hi/lo planes of the first layer
    {
        const int Kp = pk->layers[0].Kp;
        const int64_t n = B * (Kp / 8);
        split_input_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(x, ldx, dx, c, ldc, dc, B, Kp, in_planes);
        ZK_TRY(check_launch("split_input_kernel"));
    }
    const int sms = sm_count();
    const __nv_bfloat16* a = in_planes;
    for (int i = 0; i < m->n_linear; ++i) {
        const TcLayer& L = pk->layers[i];
        const bool last = (i == m->n_linear - 1);
        CUtensorMap mapA;
        ZK_TRY(make_plane_map(&mapA, a, B, L.Kp, BM));
        TcParams p;
        p.M = (int)B; p.N = L.N; p.Kp = L.Kp;
        p.n_chunks = (L.N + BN - 1) / BN;
        p.n_terms = pk->n_terms;
        p.relu = m->lact[i];  // per layer: the plain pattern is act ... act 0, residual blocks are act 0 pairs
        p.bias = m->b[i];
        p.out_f32 = last ? out : nullptr;
        p.ldo = ldo;
        p.out_planes = last ? nullptr : hid[i & 1];
        p.Np = last ? 0 : pk->layers[i + 1].Kp;
        p.gate = nullptr; p.slice_m = 0; p.w_slice_rows = 0;
        // residual block: the input of layer i-1 is what layer i-2 left in the ping-pong buffer this layer writes
        p.res = (!last && m->lres[i]) ? hid[i & 1] : nullptr;
        if (!last) {
            // the next layer reads columns [0, Np): they are all written when the chunks cover Np
            ZK_REQUIRE(p.n_chunks * BN >= p.Np, "tc_forward: internal padding error");
        }
        const int64_t tiles = ceil_div(B, BM) * p.n_chunks;
        const int grid = (int)std::min<int64_t>(tiles, sms);
        if (p.relu > 1 || p.res != nullptr) linear_tc_kernel<true><<<grid, kThreads, SMEM_BYTES, st>>>(mapA, L.mapW, p);
        else linear_tc_kernel<false><<<grid, kThreads, SMEM_BYTES, st>>>(mapA, L.mapW, p);
        ZK_TRY(check_launch("linear_tc_kernel"));
        a = p.out_planes;
    }
    return ZK_OK;
}

// ===========================================================================
// backward pass on the tensor cores: the same GEMM kernel drives
//   forward-with-saved-activations, dgrad (A = g planes, W = transposed weights, ReLU gate in the
//   epilogue) and wgrad (A = g^T, W = act^T, both batch-major; the batch is cut into S slices that
//   become extra M tiles, each pairing with its own rows of the W operand; fp32 partials are
//   reduced in a fixed order by wgrad_reduce_sliced_kernel).
// ===========================================================================
namespace {

// bf16 planes [2][M][Kp]  ->  [2][S][Rp][Bs]: out[pl][s][r][j] = in[pl][s*Bs + j][r] (0 beyond M / Kp).
// 64 x 64 tiles, 32-bit (bf16 pair) accesses on both sides: every warp reads and writes 128
// contiguous bytes per row.  Bs is a multiple of 64, so a tile never straddles two batch slices.
__global__ void __launch_bounds__(256)
transpose_planes_kernel(const __nv_bfloat16* in, int64_t M, int Kp, int S, int Rp, int Bs, __nv_bfloat16* out) {
    __shared__ uint16_t tile[64][66];
    const int pl = blockIdx.z;
    const int64_t b0 = (int64_t)blockIdx.x * 64;  // position along S*Bs (slices are contiguous in b)
    const int r0 = blockIdx.y * 64;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const uint16_t* src = reinterpret_cast<const uint16_t*>(in) + (int64_t)pl * M * Kp;
    uint16_t* dst = reinterpret_cast<uint16_t*>(out) + (int64_t)pl * S * Rp * Bs;
#pragma unroll
    for (int j = ty; j < 64; j += 8) {
        const int64_t b = b0 + j;
        const int r = r0 + 2 * tx;  // Kp is even (multiple of 64): a pair is in range together
        uint32_t w = 0u;
        if (b < M && r < Kp) w = *reinterpret_cast<const uint32_t*>(src + b * Kp + r);
        tile[j][2 * tx] = (uint16_t)(w & 0xffffu);
        tile[j][2 * tx + 1] = (uint16_t)(w >> 16);
    }
    __syncthreads();
    const int64_t s = b0 / Bs, jj0 = b0 - s * Bs;
    if (s >= S) return;
#pragma unroll
    for (int j = ty; j < 64; j += 8) {
        const int r = r0 + j;
        if (r < Rp) {
            const uint32_t w = (uint32_t)tile[2 * tx][j] | ((uint32_t)tile[2 * tx + 1][j] << 16);
            *reinterpret_cast<uint32_t*>(dst + (s * Rp + r) * Bs + jj0 + 2 * tx) = w;
        }
    }
}

// fp32 (M, N) row-major (stride ld)  ->  bf16 hi/lo planes [2][S][Rp][Bs], transposed (same tiling)
__global__ void __launch_bounds__(256)
transpose_split_f32_kernel(const float* in, int64_t ld, int64_t M, int N, int S, int Rp, int Bs, __nv_bfloat16* out) {
    __shared__ float tile[64][65];
    const int64_t b0 = (int64_t)blockIdx.x * 64;
    const int r0 = blockIdx.y * 64;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int j = ty; j < 64; j += 8) {
        const int64_t b = b0 + j;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = r0 + tx + 32 * h;
            tile[j][tx + 32 * h] = (b < M && r < N) ? in[b * ld + r] : 0.f;
        }
    }
    __syncthreads();
    const int64_t s = b0 / Bs, jj0 = b0 - s * Bs;
    if (s >= S) return;
    const int64_t plane = (int64_t)S * Rp * Bs;
    uint16_t* dst = reinterpret_cast<uint16_t*>(out);
#pragma unroll
    for (int j = ty; j < 64; j += 8) {
        const int r = r0 + j;
        if (r < Rp) {
            uint32_t hi, lo;
            split2_bf16(tile[2 * tx][j], tile[2 * tx + 1][j], hi, lo);
            const int64_t o = (s * Rp + r) * Bs + jj0 + 2 * tx;
            *reinterpret_cast<uint32_t*>(dst + o) = hi;
            *reinterpret_cast<uint32_t*>(dst + plane + o) = lo;
        }
    }
}

// gw (N, K) += mask ? sum_s partial[(s * slice_m + n) * K + k] : 0
__global__ void wgrad_reduce_sliced_kernel(const float* partial, int S, int slice_m, int N, int K,
                                           const uint8_t* mask, float* gw) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * K) return;
    if (mask && !mask[i]) return;
    const int n = (int)(i / K), k = (int)(i - (int64_t)n * K);
    float t = 0.f;
    for (int s = 0; s < S; ++s) t += partial[((int64_t)s * slice_m + n) * K + k];
    gw[i] += t;
}

// column sums of (hi + lo) planes [2][M][Np] over a row slice (stage 1 of the fixed-order reduction);
// a thread owns two adjacent columns (one 32-bit load per plane), a warp reads 128 contiguous bytes
__global__ void __launch_bounds__(256)
colsum_planes_stage1(const __nv_bfloat16* planes, int64_t M, int Np, int N, int64_t rows_per_slice, float* partial) {
    __shared__ float sm[8][66];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int col = blockIdx.x * 64 + 2 * tx;  // Np is even: col + 1 < Np whenever col < Np
    const int64_t lo_r = (int64_t)blockIdx.y * rows_per_slice;
    const int64_t hi_r = min(M, lo_r + rows_per_slice);
    const uint16_t* hi = reinterpret_cast<const uint16_t*>(planes);
    const uint16_t* lo = hi + M * (int64_t)Np;
    float a0 = 0.f, a1 = 0.f;
    if (col < Np) {
        // eight rows (16 independent 32-bit loads) in flight per thread: the kernel is bound by load latency, and
        // the running sums keep the row order of the one-row-at-a-time loop (bit-identical results)
        constexpr int U = 8;
        int64_t r = lo_r + ty;
        for (; r + 8 * (U - 1) < hi_r; r += 8 * U) {
            uint32_t h[U], l[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                h[u] = *reinterpret_cast<const uint32_t*>(hi + (r + 8 * u) * Np + col);
                l[u] = *reinterpret_cast<const uint32_t*>(lo + (r + 8 * u) * Np + col);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                a0 += __uint_as_float(h[u] << 16) + __uint_as_float(l[u] << 16);
                a1 += __uint_as_float(h[u] & 0xffff0000u) + __uint_as_float(l[u] & 0xffff0000u);
            }
        }
        for (; r < hi_r; r += 8) {
            const uint32_t h = *reinterpret_cast<const uint32_t*>(hi + r * Np + col);
            const uint32_t l = *reinterpret_cast<const uint32_t*>(lo + r * Np + col);
            a0 += __uint_as_float(h << 16) + __uint_as_float(l << 16);
            a1 += __uint_as_float(h & 0xffff0000u) + __uint_as_float(l & 0xffff0000u);
        }
    }
    sm[ty][2 * tx] = a0;
    sm[ty][2 * tx + 1] = a1;
    __syncthreads();
    if (ty < 2) {
        const int c = blockIdx.x * 64 + 2 * tx + ty;
        if (c < N) {
            float t = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) t += sm[k][2 * tx + ty];
            partial[(int64_t)blockIdx.y * N + c] = t;
        }
    }
}
__global__ void colsum_planes_stage2(const float* partial, int S, int N, float* out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float t = 0.f;
    for (int z = 0; z < S; ++z) t += partial[(int64_t)z * N + n];
    out[n] += t;
}

}  // namespace

zk_status launch_split_planes(const float* x, int64_t ldx, int dx, const float* c, int64_t ldc, int dc,
                              int64_t M, int Kp, __nv_bfloat16* out, cudaStream_t st) {
    if (M == 0) return ZK_OK;
    const int64_t n = M * (Kp / 8);
    split_input_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(x, ldx, dx, c, ldc, dc, M, Kp, out);
    return check_launch("split_input_kernel");
}

zk_status launch_transpose_planes(const __nv_bfloat16* in, int64_t M, int Kp, int S, int Rp, int Bs,
                                  __nv_bfloat16* out, cudaStream_t st) {
    dim3 grid((unsigned)ceil_div((int64_t)S * Bs, 64), (unsigned)ceil_div(Rp, 64), 2);
    transpose_planes_kernel<<<grid, 256, 0, st>>>(in, M, Kp, S, Rp, Bs, out);
    return check_launch("transpose_planes_kernel");
}

zk_status launch_transpose_split_f32(const float* in, int64_t ld, int64_t M, int N, int S, int Rp, int Bs,
                                     __nv_bfloat16* out, cudaStream_t st) {
    dim3 grid((unsigned)ceil_div((int64_t)S * Bs, 64), (unsigned)ceil_div(Rp, 64), 1);
    transpose_split_f32_kernel<<<grid, 256, 0, st>>>(in, ld, M, N, S, Rp, Bs, out);
    return check_launch("transpose_split_f32_kernel");
}

zk_status launch_wgrad_reduce_sliced(const float* partial, int S, int slice_m, int N, int K, const uint8_t* mask,
                                     float* gw, cudaStream_t st) {
    wgrad_reduce_sliced_kernel<<<(unsigned)ceil_div((int64_t)N * K, 256), 256, 0, st>>>(partial, S, slice_m, N, K, mask, gw);
    return check_launch("wgrad_reduce_sliced_kernel");
}

size_t colsum_planes_scratch_bytes(int N) { return (size_t)256 * N * 4; }
zk_status launch_colsum_planes_add(const __nv_bfloat16* planes, int64_t M, int Np, int N, float* out, void* scratch,
                                   cudaStream_t st) {
    if (M == 0) return ZK_OK;
    int64_t S = std::min<int64_t>(256, ceil_div(M, 256));
    const int64_t rows = ceil_div(M, S);
    S = ceil_div(M, rows);
    dim3 grid((unsigned)ceil_div(N, 64), (unsigned)S);
    colsum_planes_stage1<<<grid, 256, 0, st>>>(planes, M, Np, N, rows, (float*)scratch);
    ZK_TRY(check_launch("colsum_planes_stage1"));
    colsum_planes_stage2<<<(unsigned)ceil_div(N, 256), 256, 0, st>>>((const float*)scratch, (int)S, N, out);
    return check_launch("colsum_planes_stage2");
}

zk_status tc_gemm(const TcGemmArgs& a, cudaStream_t st) {
    ZK_REQUIRE(a.a_planes && a.mapW && a.M > 0 && a.N > 0 && a.Kp > 0 && a.Kp % BK == 0, "tc_gemm: bad arguments");
    ZK_REQUIRE((a.out_f32 != nullptr) != (a.out_planes != nullptr), "tc_gemm: exactly one output kind");
    ZK_REQUIRE(a.M < ((int64_t)1 << 31) - BM, "tc_gemm: too many rows for one launch");
    CUtensorMap mapA;
    ZK_TRY(make_plane_map(&mapA, a.a_planes, a.M, a.Kp, BM));
    TcParams p;
    p.M = (int)a.M; p.N = a.N; p.Kp = a.Kp;
    p.n_chunks = (a.N + BN - 1) / BN;
    p.n_terms = a.n_terms;
    p.relu = a.relu;
    p.bias = a.bias;
    p.out_f32 = a.out_f32; p.ldo = a.ldo;
    p.out_planes = a.out_planes; p.Np = a.Np;
    p.gate = a.gate; p.slice_m = a.slice_m; p.w_slice_rows = a.w_slice_rows;
    p.res = nullptr;
    if (a.out_planes) ZK_REQUIRE(p.n_chunks * BN >= p.Np && a.Np % 64 == 0, "tc_gemm: internal padding error");
    if (a.slice_m) ZK_REQUIRE(a.slice_m % BM == 0, "tc_gemm: slice_m must be a multiple of %d", BM);
    const int64_t tiles = ceil_div(a.M, BM) * p.n_chunks;
    const int grid = (int)std::min<int64_t>(tiles, sm_count());
    if (p.relu > 1) linear_tc_kernel<true><<<grid, kThreads, SMEM_BYTES, st>>>(mapA, *a.mapW, p);
    else linear_tc_kernel<false><<<grid, kThreads, SMEM_BYTES, st>>>(mapA, *a.mapW, p);
    return check_launch("linear_tc_kernel");
}

// transposed weights as bf16 planes for dgrad: wt[i] is (K_i, N_i) fp32 row-major
zk_status tc_pack_backward(zk_mlp* m, cudaStream_t st) {
    TcPack* pk = (TcPack*)m->tc;
    ZK_REQUIRE(pk, "tc_pack_backward: handle has no tensor-core pack");
    ZK_REQUIRE((int)m->wt.size() == m->n_linear, "tc_pack_backward: transposed weights missing");
    if ((int)pk->bwd.size() == m->n_linear) {
        if (!m->bwd_dirty) return ZK_OK;
        for (int i = 0; i < m->n_linear; ++i) {  // same planes, new values
            const TcLayer& L = pk->bwd[i];
            split_weight_kernel<<<(unsigned)ceil_div((int64_t)L.N * L.Kp, 256), 256, 0, st>>>(m->wt[i], L.N, L.K, L.Kp, L.w);
            ZK_TRY(check_launch("split_weight_kernel"));
        }
        return ZK_OK;
    }
    for (auto& l : pk->bwd) cudaFree(l.w);
    pk->bwd.clear();
    for (int i = 0; i < m->n_linear; ++i) {
        TcLayer L;
        L.K = m->dims[i + 1];  // contraction over the layer's outputs
        L.N = m->dims[i];
        L.Kp = pad64(L.K);
        if (cudaMalloc((void**)&L.w, (size_t)2 * L.N * L.Kp * 2) != cudaSuccess) return fail(ZK_ENOMEM, "tc_pack_backward: cudaMalloc failed");
        pk->bwd.push_back(L);
        split_weight_kernel<<<(unsigned)ceil_div((int64_t)L.N * L.Kp, 256), 256, 0, st>>>(m->wt[i], L.N, L.K, L.Kp, L.w);
        ZK_TRY(check_launch("split_weight_kernel"));
        ZK_TRY(make_plane_map(&pk->bwd.back().mapW, L.w, L.N, L.Kp, BN));
    }
    return ZK_OK;
}

const TcPack* tc_pack_of(const zk_mlp* m) { return (const TcPack*)m->tc; }

}  // namespace zk
