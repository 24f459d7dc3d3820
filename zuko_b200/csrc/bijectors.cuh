// zuko_b200 — launch interface of the element-wise bijector kernels (bijectors.cu).
#pragma once

#include "common.cuh"

namespace zk {

// One fused pass of a univariate bijector over a (B, D) batch with (B, D, P)
// per-sample parameters (or one shared (D, P) table when phi_ld == 0).
struct UniArgs {
    int univariate = ZK_UNI_RQS;  // ZK_UNI_*
    bool inverse = false;
    const float* x = nullptr;  // input (B, *) ; forward: x, inverse: y
    int64_t ldx = 0;
    const float* phi = nullptr;
    int64_t phi_ld = 0;  // elements per sample row of phi (0 = shared table)
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
    int K = 0;      // bins (RQS) / mixture components (Gaussianization) / polynomials (SOSP)
    int degree = 0; // SOSP: polynomial degree L; Bernstein: BPF degree (P = degree + 1)
    float bound = 5.f;
    int iters = 0;  // Gaussianization / SOSP / Bernstein inverse: bisection steps on [-bound, bound]
    float eps = kBernsteinEps;  // Bernstein: branch threshold on t = (x + bound) / 2 bound
    float slope = 1e-3f;
    bool circular = false;  // RQS only: CircularShiftTransform(bound) in front (forward) / behind (inverse)
    bool fast_math = true;  // MUFU rcp/ex2/lg2 fast path (default) vs IEEE div + expf/logf
};

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
