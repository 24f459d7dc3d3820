// zuko_b200 — launch interface of the element-wise bijector kernels (bijectors.cu).
#pragma once

#include "common.cuh"

namespace zk {

// One fused pass of a univariate bijector over a (B, D) batch with (B, D, P)
// per-sample parameters (or one shared (D, P) table when phi_ld == 0).
struct UniArgs {
    UniSpec spec;
    bool inverse = false;
    const float* x = nullptr;  // input (B, *) ; forward: x, inverse: y
    int64_t ldx = 0;
    const float* phi = nullptr;
    int64_t phi_ld = 0;  // row stride of phi in elements, >= D*P (padded rows allowed); 0 = one shared table
    float* y = nullptr;  // output (B, *), may be null (forward + log_prob only)
    int64_t ldy = 0;
    float* ladj = nullptr;  // (B) summed over dims; forward only; may be null
    int accumulate = 0;     // ladj[b] += ... (also seeds log_prob when set)
    float* log_prob = nullptr;  // (B): ladj total + DiagNormal(loc, scale).log_prob(y); forward only
    const float* base_loc = nullptr;    // (D) or null = 0
    const float* base_scale = nullptr;  // (D) or null = 1
    const int* dim_map = nullptr;  // (D) device: pair d lives in column dim_map[d] of x / y (coupling)
    int64_t B = 0;
    int D = 0;      // number of transformed dims (pairs per sample)
    bool fast_math = true;  // MUFU rcp/ex2/lg2 fast path (default) vs IEEE div + expf/logf
};

// Tile plan of uni_kernel (launch_univariate and zk_univariate_plan both take it from uni_plan).
struct UniPlan {
    int rows_per_tile = 0;   // R: >= ceil(256 / D) rows and ~24 KB of phi, shrunk to <= 96 KB, capped by B
    int grid = 0;            // ceil(B / R) CTAs
    size_t smem = 0;         // dynamic shared memory: phi (R rows, or one shared table) + R*D reduction floats
    bool smem_attr = false;  // smem + the static barrier exceed the 48 KB default: raise the attribute
    bool bulk = false;       // cp.async.bulk for full tiles: dense rows, 16-byte aligned phi and tile
    bool shuffle = false;    // D <= 32 and a power of two: warp-shuffle ladj sum, else the fixed-order sum
    int kt = 0;              // compile-time shape of the instantiation (uni_kt<kStandalone>); 0 = runtime
};
// Validates the shape arguments as launch_univariate does and fills `out`; B = 0 leaves it zero.  Host only.
zk_status uni_plan(const UniSpec& s, int64_t B, int D, int64_t phi_ld, const float* phi, UniPlan& out);
zk_status launch_univariate(const UniArgs& a, cudaStream_t stream);

zk_status launch_softclip(const float* x, int64_t ldx, int64_t B, int D, float bound, bool inverse,
                          float* y, int64_t ldy, float* ladj, int accumulate, cudaStream_t stream);
zk_status launch_permute(const float* x, int64_t ldx, const int64_t* order, int64_t B, int D,
                         float* y, int64_t ldy, cudaStream_t stream);
zk_status launch_rotate(const float* x, int64_t ldx, const float* R, int transpose, int64_t B, int D,
                        float* y, int64_t ldy, cudaStream_t stream);
zk_status launch_circular_shift(const float* x, int64_t ldx, int64_t B, int D, float bound, float* y,
                                int64_t ldy, cudaStream_t stream);
zk_status launch_box_uniform(const float* z, int64_t ldz, const float* lower, const float* upper,
                             const float* ladj, int64_t B, int D, float* out, cudaStream_t stream);
zk_status launch_diag_normal(const float* z, int64_t ldz, const float* loc, const float* scale,
                             const float* ladj, int64_t B, int D, float* out, cudaStream_t stream);
// out[0] = sum_b v[b] in double, fixed-order two-stage reduction; scratch >= reduce_scratch_bytes()
size_t reduce_scratch_bytes();
zk_status launch_sum_f32_to_f64(const float* v, int64_t B, double* out, void* scratch,
                                cudaStream_t stream);
// copy selected columns: y[:, cols[j]] = x[:, cols[j]] for j < n (coupling passthrough)
zk_status launch_copy_columns(const float* x, int64_t ldx, const int* cols, int n, int64_t B,
                              float* y, int64_t ldy, cudaStream_t stream);
zk_status launch_fill(float* p, int64_t n, float v, cudaStream_t stream);

}  // namespace zk
