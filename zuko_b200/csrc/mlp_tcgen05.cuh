// zuko_b200 — tensor-core (wgmma) conditioner path: interface.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>

#include "mlp.cuh"

namespace zk {

// Resolves m->gemm_mode from the requested mode and packs bf16 hi/lo weights when the
// tensor-core path is selected.  Runs on stream 0.
zk_status tc_pack(zk_mlp* m, int requested_mode);
void tc_destroy(zk_mlp* m);
// re-splits m->w into the existing bf16 planes (weights changed, shapes / masks did not); stream-ordered
zk_status tc_refresh(zk_mlp* m, cudaStream_t stream);
size_t tc_workspace_bytes(const zk_mlp* m, int64_t B);
zk_status tc_forward(const zk_mlp* m, const float* x, int64_t ldx, int dx, const float* c,
                     int64_t ldc, int dc, int64_t B, float* out, int64_t ldo, void* ws,
                     size_t ws_bytes, cudaStream_t stream);

// ---- building blocks of the tensor-core backward pass (api_backward.cu) ----
struct TcGemmArgs {
    const __nv_bfloat16* a_planes = nullptr;  // [2][M][Kp] bf16 hi / lo
    int64_t M = 0;
    int Kp = 0;
    const CUtensorMap* mapW = nullptr;  // planes [2][rows][Kp], box (64 x 128 x 1)
    int N = 0;                          // real output columns
    const float* bias = nullptr;
    int relu = 0;
    float* out_f32 = nullptr; int64_t ldo = 0;        // fp32 output, or
    __nv_bfloat16* out_planes = nullptr; int Np = 0;  // bf16 hi / lo planes [2][M][Np]
    const __nv_bfloat16* gate = nullptr;              // [M][Np]: zero the output where gate <= 0
    int slice_m = 0, w_slice_rows = 0;                // split-K wgrad (see linear_tc_kernel)
    int n_terms = 3;
};
zk_status tc_gemm(const TcGemmArgs& a, cudaStream_t stream);
zk_status tc_pack_backward(zk_mlp* m, cudaStream_t stream);  // needs m->wt
struct TcPack;
const TcPack* tc_pack_of(const zk_mlp* m);
// cat(x, c) fp32 -> planes [2][M][Kp]
zk_status launch_split_planes(const float* x, int64_t ldx, int dx, const float* c, int64_t ldc, int dc,
                              int64_t M, int Kp, __nv_bfloat16* out, cudaStream_t stream);
// planes [2][M][Kp] -> batch-major planes [2][S][Rp][Bs] (zero padded)
zk_status launch_transpose_planes(const __nv_bfloat16* in, int64_t M, int Kp, int S, int Rp, int Bs,
                                  __nv_bfloat16* out, cudaStream_t stream);
zk_status launch_transpose_split_f32(const float* in, int64_t ld, int64_t M, int N, int S, int Rp, int Bs,
                                     __nv_bfloat16* out, cudaStream_t stream);
zk_status launch_wgrad_reduce_sliced(const float* partial, int S, int slice_m, int N, int K, const uint8_t* mask,
                                     float* gw, cudaStream_t stream);
size_t colsum_planes_scratch_bytes(int N);
zk_status launch_colsum_planes_add(const __nv_bfloat16* planes, int64_t M, int Np, int N, float* out, void* scratch,
                                   cudaStream_t stream);

}  // namespace zk
