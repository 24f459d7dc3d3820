// zuko_b200 — internals shared by the C-ABI translation units (api.cu, api_backward.cu).
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

}  // namespace zkapi
