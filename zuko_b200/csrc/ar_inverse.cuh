// zuko_b200 — dimension-sequential inverse of a masked autoregressive layer: interface.
#pragma once

#include "mlp.cuh"

namespace zk {

struct ArInvPack;  // step-ordered weight stream of one layer (ar_inverse.cu)

// Builds the pack when the layer has a pure order-class structure (an `order` vector) and its bijector has a
// compiled sequential-inverse shape (uni_kt<kSequential>); leaves *out null (and returns ZK_OK) when
// the layer must use the generic sweep-based inverse instead.  `mask_dev` are the DEVICE mask pointers
// of zk_mlp_desc (may be null).
zk_status ar_inverse_pack(const zk_mlp* m, const uint8_t* const* mask_dev, const int64_t* order, int D, int C,
                          const UniSpec& spec, int passes, ArInvPack** out);
void ar_inverse_free(ArInvPack* pk);
bool ar_inverse_threads(const ArInvPack* pk, int* threads, size_t* smem);
// the launch geometry launch_ar_inverse uses (ZK_INV_GEOM honoured): threads per CTA, samples per
// thread, dynamic shared memory; false when the state does not fit
bool ar_inverse_geometry(const ArInvPack* pk, int* threads, int* per_thread, size_t* smem);

struct ArInvArgs {
    const float* y = nullptr; int64_t ldy = 0;  // the layer's output (input of the inverse)
    const float* c = nullptr; int64_t ldc = 0;
    int64_t B = 0;
    float* x = nullptr; int64_t ldx = 0;
    UniSpec spec;  // the one the pack was built for
    bool fast = true;
    // optional: per-sample sum over D of the FORWARD log-derivative at the solution x (what
    // rsample_and_log_prob needs, distributions.py:129-138), accumulated into `ladj` when
    // `accumulate`; with `base` the DiagNormal(loc, scale) log-density of y is added as well
    float* ladj = nullptr; int accumulate = 0;
    bool base = false; const float* base_loc = nullptr; const float* base_scale = nullptr;
    // the layer as an INVERTED member of a flow (LazyInverse): the member's own ladj is minus the forward
    // ladj at the solution, and the base density (if fused here) is evaluated on the OUTPUT x
    bool as_inverse_member = false;
};
zk_status launch_ar_inverse(const ArInvPack* pk, const ArInvArgs& a, cudaStream_t stream);

}  // namespace zk
