// zuko_b200 — internals shared by the C-ABI translation units (api.cu, api_backward.cu, gmm.cu).
#pragma once

#include <algorithm>
#include <vector>

#include "ar_inverse.cuh"
#include "bijectors.cuh"
#include "fused_layer.cuh"
#include "mlp.cuh"
#include "mlp_tcgen05.cuh"
#include "uni_family.cuh"

namespace zk {

// bump allocator over the caller's workspace (256-byte granules)
struct Arena {
    char* base;
    size_t size, off = 0;
    bool ok = true;
    Arena(void* p, size_t n) : base((char*)p), size(n) {}
    template <typename T>
    T* take(size_t count) {
        size_t bytes = align_up(count * sizeof(T), 256);
        if (off + bytes > size) {
            ok = false;
            return nullptr;
        }
        T* r = (T*)(base + off);
        off += bytes;
        return r;
    }
};
inline size_t a256(size_t bytes) { return align_up(bytes, 256); }

template <typename T>
inline zk_status dev_copy_from_host(const T* host, size_t n, T** out) {
    *out = nullptr;
    if (n == 0) return ZK_OK;
    ZK_CUDA(cudaMalloc((void**)out, n * sizeof(T)));
    ZK_CUDA(cudaMemcpy(*out, host, n * sizeof(T), cudaMemcpyHostToDevice));
    return ZK_OK;
}


}  // namespace zk

// ===========================================================================
// layer handle
// ===========================================================================
struct zk_layer {
    int kind = 0, D = 0, C = 0, P = 0, passes = 0;
    zk::UniSpec spec;              // the bijector (ZK_UNI_CRQS: RQS + circular); spec.bound is also the softclip bound
    zk_mlp* hyper = nullptr;       // owned
    float* phi_shared = nullptr;   // device (D, P), owned
    float* rotation = nullptr;     // device (D, D), owned
    int64_t* perm = nullptr;       // device (D), owned
    int64_t* perm_inv = nullptr;   // device (D), owned
    int* idx_a = nullptr;          // device: constant-split columns (coupling), owned
    int* idx_b = nullptr;          // device: transformed columns (coupling), owned
    int n_a = 0, n_b = 0;
    zk::ArInvPack* inv = nullptr;  // step-ordered weights for the dimension-sequential inverse (owned)
    bool inv_dirty = false;        // weights refreshed in place since `inv` was built: rebuilt on the next inverse call
    std::vector<int64_t> order;    // host copy of the order classes (autoregressive), for that rebuild
};


namespace zkapi {

// forward of one layer (api.cu); with log_prob != nullptr the DiagNormal term is fused
zk_status layer_forward_impl(const zk_layer* l, const float* x, int64_t ldx, const float* c,
                             int64_t ldc, int64_t B, float* y, int64_t ldy, float* ladj,
                             int accumulate, float* log_prob, const float* loc, const float* scale,
                             void* ws, size_t ws_bytes, cudaStream_t st);
zk_status flow_check(const zk_flow_desc* f);
zk_status copy_rows(const float* x, int64_t ldx, int64_t B, int D, float* y, int64_t ldy, cudaStream_t st);
// refreshes a conditioner's weights in place (api.cu): masks re-applied, tensor-core / fused packs re-split
zk_status mlp_update_weights(zk_mlp* m, const float* const* weight, const float* const* bias, cudaStream_t st);

// ---------------------------------------------------------------------------
// conditioner backward with saved activations (api_backward.cu), shared by every caller that differentiates
// through a zk_mlp: fp32 CUDA-core path (mlp_*) and tensor-core path (tc_*, handles packed for wgmma)
// ---------------------------------------------------------------------------
struct MlpBwdBufs {
    std::vector<float*> acts;  // acts[i]: input of linear layer i, (B, dims[i])
    std::vector<float*> pre;   // pre[i]: pre-activation of hidden layer i + 1 (non-ReLU activations only)
    float* out = nullptr;      // (B, dims[n]): conditioner output, later its gradient
    float* gbuf[2] = {nullptr, nullptr};
    float* gin = nullptr;      // (B, dims[0])
    void* scratch = nullptr;
};

struct TcBwdPlan {
    int n = 0;
    std::vector<int> Kp;       // pad64(dims[i]), i = 0..n
    std::vector<int> S, Bs, slice_m;  // per linear layer: batch slices of the wgrad GEMM
    int max_hidden_kp = 0;
    size_t gT = 0, aT = 0, partial = 0, scratch = 0;
};

struct TcBwdBufs {
    float* a0 = nullptr;
    float* gin = nullptr;
    std::vector<__nv_bfloat16*> P;  // saved activation planes, [2][B][Kp[i]]
    float* out = nullptr;           // phi, then gphi
    __nv_bfloat16* G = nullptr;     // planes of gphi
    __nv_bfloat16* gbuf[2] = {nullptr, nullptr};
    __nv_bfloat16* gT = nullptr;
    __nv_bfloat16* aT = nullptr;
    float* partial = nullptr;
    void* scratch = nullptr;
};

bool tc_backward_on();  // zk_set_tc_backward
// transposed pre-masked weights for dgrad, built on first use
zk_status mlp_ensure_backward(const zk_mlp* cm, cudaStream_t st);
size_t mlp_bwd_scratch(const zk_mlp* m);
size_t mlp_bwd_ws(const zk_mlp* m, int64_t B);
bool mlp_bwd_carve(const zk_mlp* m, int64_t B, zk::Arena& ar, MlpBwdBufs& b);
// forward with every activation kept (fp32 CUDA-core path); acts[0] must be filled
zk_status mlp_forward_save(const zk_mlp* m, const MlpBwdBufs& b, int64_t B, cudaStream_t st);
// b.out holds dL/d(out) on entry; on exit b.gin = dL/d(input) when want_gin
zk_status mlp_backward(const zk_mlp* m, const MlpBwdBufs& b, int64_t B, bool want_gin,
                       const zk_layer_grads* grads, cudaStream_t st);
TcBwdPlan tc_plan(const zk_mlp* m, int64_t B);
bool mlp_uses_tc(const zk_mlp* m);
size_t tc_bwd_ws(const zk_mlp* m, int64_t B);
bool tc_bwd_carve(const zk_mlp* m, const TcBwdPlan& p, int64_t B, zk::Arena& ar, TcBwdBufs& b);
// b.a0 = the conditioner input must be filled; leaves the output in b.out and every layer input in b.P
zk_status tc_forward_save(const zk_mlp* m, const TcBwdPlan& p, const TcBwdBufs& b, int64_t B, cudaStream_t st);
// b.out holds dL/d(out) (fp32); on exit b.gin = dL/d(input) when want_gin
zk_status tc_mlp_backward(const zk_mlp* m, const TcBwdPlan& p, const TcBwdBufs& b, int64_t B, bool want_gin,
                          const zk_layer_grads* grads, cudaStream_t st);

}  // namespace zkapi
