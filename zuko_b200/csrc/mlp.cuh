// zuko_b200 — conditioner (MaskedMLP / MLP) handle and GEMM launch interface.
#pragma once

#include <vector>

#include "common.cuh"

struct zk_mlp {
    int n_linear = 0;
    std::vector<int> dims;       // n_linear + 1
    std::vector<float*> w;       // device, pre-masked fp32 (dims[i+1], dims[i]) row-major (owned)
    std::vector<float*> b;       // device fp32 (dims[i+1]) (owned; zeros when the layer has no bias)
    std::vector<uint8_t*> mask;  // device bool bytes (dims[i+1], dims[i]) or nullptr = dense (owned): d(mask*W)/dW
    std::vector<float*> wt;      // device, w[i] transposed (dims[i], dims[i+1]) for dgrad; built on first backward (owned)
    int act = 1;                 // activation between layers: 1 = ReLU, >= 2 = ZK_ACT_* (activations.cuh)
    bool plain = true;           // activation after every layer but the last, no residual adds
    std::vector<int> lact;       // per layer: activation applied to its output (0 none, 1 ReLU, ZK_ACT_*)
    std::vector<int> lres;       // per layer: add the input of layer i-1 to the output (residual block)
    bool bwd_dirty = false;        // weights refreshed since wt / the backward planes were built
    int gemm_mode = ZK_GEMM_FP32;  // resolved path
    int max_hidden = 0;
    // tensor-core path: packed bf16 hi/lo weights (owned), see mlp_tcgen05.cu
    void* tc = nullptr;
};

namespace zk {

// C[M, N] = act(A[M, K] * W[N, K]^T + bias), fp32 FMA on CUDA cores.
// A is read from up to two row-major sources: columns [0, k0) from a0 (row stride lda0) and
// [k0, K) from a1 (row stride lda1, 0 = broadcast one row) — the torch.cat((x, c)) of
// flows/autoregressive.py:209 folded into the loader.
zk_status launch_linear_fp32(const float* a0, int64_t lda0, int k0, const float* a1, int64_t lda1,
                             int K, const float* W, const float* bias, int64_t M, int N, int act,
                             float* C, int64_t ldc, cudaStream_t stream, const float* res = nullptr,
                             int64_t ldres = 0);  // act: 0 none, 1 ReLU, ZK_ACT_*; C = act(..) + res (res may be C)

// W_out = mask ? W : 0  (mask may be null = copy) — zuko/nn.py:218 `self.mask * self.weight`, done once
zk_status launch_apply_mask(const float* W, const uint8_t* mask, int64_t n, float* W_out,
                            cudaStream_t stream);

}  // namespace zk
