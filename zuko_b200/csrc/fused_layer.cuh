// zuko_b200 — fully fused flow-layer kernel (conditioner + bijector + ladj): interface.
#pragma once

#include <atomic>

#include "mlp.cuh"

#define ZK_FUSED_MAX_LINEAR 6

namespace zk {

struct FusedLayerArgs {
    int univariate = ZK_UNI_RQS;
    int bins = 8;
    int D = 0, C = 0;
    float bound = 5.f, slope = 1e-3f;
    const float* x = nullptr; int64_t ldx = 0;
    const float* c = nullptr; int64_t ldc = 0;
    int64_t B = 0;
    float* y = nullptr; int64_t ldy = 0;  // may be null (log_prob only)
    float* ladj = nullptr; int accumulate = 0;
    float* log_prob = nullptr; const float* base_loc = nullptr; const float* base_scale = nullptr;
    bool fast_math = true;
};

// true when the autoregressive layer (conditioner `m`, univariate, D, C) can run as ONE kernel
bool fused_layer_supported(const zk_mlp* m, int univariate, int bins, int D, int C);
// which kernel: 0 none, 1 the fused layer kernel (fused_layer.cu)
int fused_layer_kind(const zk_mlp* m, int univariate, int bins, int D, int C);
// rows per tile of the fused layer kernel for this layer (64 or 128, from the shape); 0 when it does not run fused
int fused_tile_rows(const zk_mlp* m, int univariate, int bins, int D, int C);
// the same, with the plan launch_fused_layer uses: W ring slots (64-row tiles: both rings together) and dynamic
// shared memory bytes (outputs may be null; untouched when the layer does not run fused)
int fused_layer_plan(const zk_mlp* m, int univariate, int bins, int D, int C, int* ring_slots, size_t* smem);
// Builds the fused kernel's weight pack for this conditioner (degree-sorted hidden units, zero-tile
// map); `mask_dev` are the DEVICE mask pointers of zk_mlp_desc (may be null = dense).  No-op when
// the shape is not supported by the fused kernel.
zk_status fused_layer_prepare(zk_mlp* m, const uint8_t* const* mask_dev, int univariate, int bins, int D, int C);
zk_status fused_refresh(zk_mlp* m, cudaStream_t stream);  // weights changed in place: re-split into the fused packs
zk_status launch_fused_layer(const zk_mlp* m, const FusedLayerArgs& a, cudaStream_t stream);

}  // namespace zk
