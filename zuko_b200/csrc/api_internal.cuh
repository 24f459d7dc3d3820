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

// Largest row count n <= B whose workspace need(n) fits in ws_bytes; 0 when one row does not fit (or B <= 0).
// need is monotone in n up to small bumps: with granule > 1, a count of at least two granules is rounded down
// to a whole number of granules (aligned tiles) when the rounded count still fits.
template <class Need>
int64_t largest_fitting_rows(int64_t B, size_t ws_bytes, Need need, int64_t granule) {
    if (B <= 0) return 0;
    if (need(B) <= ws_bytes) return B;
    if (need(1) > ws_bytes) return 0;
    int64_t lo = 1, hi = B;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo + 1) / 2;
        if (need(mid) <= ws_bytes) lo = mid; else hi = mid - 1;
    }
    if (granule > 1 && lo >= 2 * granule && need(lo / granule * granule) <= ws_bytes) lo = lo / granule * granule;
    return lo;
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

// One conditioner backward over `rows` input rows.  recompute() carves its buffers from `ar`, writes the input
// cat(x[:, cols] (x[:, :nx] when cols is null), c) and reruns the conditioner keeping every activation: its output
// is `phi`.  The caller turns phi into dL/dphi (in place or in its own buffer), then backward() accumulates the
// weight / bias gradients into `grads` and, with want_gin, leaves dL/d(input) (B, nx + nc) in `gin`; `scratch`
// (>= colsum_scratch_bytes(nx + nc)) is free for the caller's scatter of gin.  The tensor cores run it when the
// handle is packed for them, allow_tc is set and zk_set_tc_backward is on; otherwise the fp32 kernels do.
struct ConditionerBackward {
    float* phi = nullptr;
    const float* gin = nullptr;
    void* scratch = nullptr;

    zk_status recompute(const zk_mlp* mlp, bool allow_tc, const float* x, int64_t ldx, const int* cols, int nx,
                        const float* c, int64_t ldc, int nc, int64_t rows, zk::Arena& ar, const char* what,
                        cudaStream_t st);
    zk_status backward(float* gphi, bool want_gin, const zk_layer_grads* grads, cudaStream_t st);
    // workspace of recompute() + backward() over `rows` rows, on the path they would take now
    static size_t bytes(const zk_mlp* mlp, int64_t rows, bool allow_tc);

    // kept by recompute() for backward()
    const zk_mlp* m = nullptr;
    int64_t B = 0;
    bool tc = false;
    TcBwdPlan plan;
    TcBwdBufs tb;
    MlpBwdBufs mb;
};

}  // namespace zkapi
