// zuko_b200 — fp32 CUDA-core linear layer (exact-arithmetic path of the conditioner).
//
// relu?(A W^T + b) with fp32 FMA accumulation, any shape.  This is the reference-order
// path (ZK_GEMM_FP32): it serves shapes too small for a tensor-core tile (BASELINE cfg1:
// 4 -> 32 -> 32 -> 8) and validates the tensor-core split-bf16 path (mlp_tcgen05.cu), which is
// the production path for the large conditioners.  Restates zuko/nn.py:217-218 with the
// mask multiplication hoisted to pack time.

#include "activations.cuh"
#include "mlp.cuh"

namespace zk {

namespace {

constexpr int BM = 64, BN = 64, BK = 16;
constexpr int TM = 4, TN = 4;
constexpr int kThreads = (BM / TM) * (BN / TN);  // 256

__global__ void __launch_bounds__(kThreads)
linear_fp32_kernel(const float* __restrict__ a0, int64_t lda0, int k0, const float* __restrict__ a1,
                   int64_t lda1, int K, const float* __restrict__ W, const float* __restrict__ bias,
                   int64_t M, int N, int relu, float* C, int64_t ldc, const float* res, int64_t ldres) {
    __shared__ __align__(16) float As[BK][BM];
    __shared__ __align__(16) float Ws[BK][BN];

    const int tid = threadIdx.x;
    const int tx = tid % (BN / TN), ty = tid / (BN / TN);
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    // loader mapping: 64 rows x 16 k, 4 consecutive k per thread
    const int lr = tid / 4, lk = (tid % 4) * 4;
    const int64_t arow = m0 + lr;
    const int wrow = n0 + lr;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    for (int kb = 0; kb < K; kb += BK) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int k = kb + lk + q;
            float av = 0.f, wv = 0.f;
            if (k < K) {
                if (arow < M) av = (k < k0) ? a0[arow * lda0 + k] : a1[arow * lda1 + (k - k0)];
                if (wrow < N) wv = W[(int64_t)wrow * K + k];
            }
            As[lk + q][lr] = av;
            Ws[lk + q][lr] = wv;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * TM]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Ws[k][tx * TN]);
            const float av[4] = {a4.x, a4.y, a4.z, a4.w};
            const float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t m = m0 + ty * TM + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + tx * TN + j;
            if (n >= N) continue;
            float v = acc[i][j] + (bias ? bias[n] : 0.f);
            if (relu) v = act_apply(v, relu);  // 1 = ReLU, >= 2 = ZK_ACT_*
            if (res) v += res[m * ldres + n];  // residual add; res may be C itself (element read before written)
            C[m * ldc + n] = v;
        }
    }
}

__global__ void apply_mask_kernel(const float* W, const uint8_t* mask, int64_t n, float* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (mask == nullptr || mask[i]) ? W[i] : 0.f;
}

}  // namespace

zk_status launch_linear_fp32(const float* a0, int64_t lda0, int k0, const float* a1, int64_t lda1,
                             int K, const float* W, const float* bias, int64_t M, int N, int act,
                             float* C, int64_t ldc, cudaStream_t stream, const float* res, int64_t ldres) {
    ZK_REQUIRE(M >= 0 && N > 0 && K > 0 && k0 >= 0 && k0 <= K, "linear: bad shape");
    ZK_REQUIRE(a0 != nullptr || k0 == 0, "linear: null A");
    ZK_REQUIRE(a1 != nullptr || k0 == K, "linear: null context");
    if (M == 0) return ZK_OK;
    const int64_t gx = ceil_div(M, BM);
    ZK_REQUIRE(gx <= 0x7fffffff, "linear: batch too large");
    dim3 grid((unsigned)gx, (unsigned)ceil_div(N, BN));
    linear_fp32_kernel<<<grid, kThreads, 0, stream>>>(a0, lda0, k0, a1, lda1, K, W, bias, M, N,
                                                       act, C, ldc, res, ldres);
    return check_launch("linear_fp32_kernel");
}

zk_status launch_apply_mask(const float* W, const uint8_t* mask, int64_t n, float* W_out,
                            cudaStream_t stream) {
    if (n == 0) return ZK_OK;
    apply_mask_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(W, mask, n, W_out);
    return check_launch("apply_mask_kernel");
}

}  // namespace zk
