// zuko_b200 — backward pass (reverse mode) of the flow hot path: launch interface.
//
// What torch.autograd does for the reference when a training loop calls
// `(-flow(c).log_prob(x).mean()).backward()` (README.md:43-49, tests/test_flows.py:22-29),
// re-derived per kernel:
//   * univariate bijectors (zuko/transforms.py:469-567, 426-446, 299-316, 834-875, 878-963, 640-831): uni_bwd_kernel
//   * (masked) MLP conditioner (zuko/nn.py:217-218): dgrad = linear_fp32_kernel on the
//     transposed pre-masked weights, wgrad = wgrad_fp32_kernel (split over the batch,
//     fixed-order reduction, mask applied to the result), bias = column sums
//   * DiagNormal base (torch/distributions/normal.py:87-102): base_grad_kernel
#pragma once

#include "common.cuh"
#include "mlp.cuh"

namespace zk {

// d(loss)/d(x, phi) of one univariate bijector pass.  gy (B, *) and gl (B) are the upstream
// gradients of y and of the per-sample summed ladj (either may be null = 0).  gphi receives the
// per-sample parameter gradients (B, D*P) (may be phi itself when phi_ld == D*P); gx the direct
// input gradient (column dim_map[d] like the forward pass).
struct UniBwdArgs {
    UniSpec spec;
    const float* x = nullptr; int64_t ldx = 0;
    const float* phi = nullptr; int64_t phi_ld = 0;  // 0 = shared (D, P) table
    const float* gy = nullptr; int64_t ldgy = 0;
    const float* gl = nullptr;
    float* gx = nullptr; int64_t ldgx = 0;
    float* gphi = nullptr;  // (B, D*P) contiguous
    const int* dim_map = nullptr;
    int64_t B = 0;
    int D = 0;
    bool fast_math = false; // MUFU reciprocal / ex2 where the family has a fast-math backward (zk_set_fast_math)
};

// Tile plan of uni_bwd_kernel (launch_univariate_backward and zk_univariate_backward_plan both take it from
// uni_bwd_plan).  A tile stages R parameter rows (or the shared table) and rewrites them with the gradients.
struct UniBwdPlan {
    int rows_per_tile = 0;        // R: ~24 KB of phi and >= ceil(256 / D) rows, shrunk to <= 96 KB with the table, capped by B
    int grid = 0;                 // ceil(B / R) CTAs
    size_t smem = 0;              // dynamic shared memory: R rows, plus the shared table unless it is rewritten in place
    bool smem_attr = false;       // smem > 40 KB: the launch raises the dynamic shared memory attribute
    bool table_in_place = false;  // shared table and R = 1: the kernel writes the gradients over the staged table
    int kt = 0;                   // compile-time shape (uni_kt<kBackward>); 0 = runtime
};
// Validates the shape arguments as launch_univariate_backward does and fills `out`; B = 0 leaves it zero.  Host only.
zk_status uni_bwd_plan(const UniSpec& s, int64_t B, int D, int64_t phi_ld, UniBwdPlan& out);
zk_status launch_univariate_backward(const UniBwdArgs& a, cudaStream_t stream);

// gx = gy / (1 + t)^2 - 2 gl sign(x) / (bound (1 + t)), t = |x| / bound  (transforms.py:309-316)
zk_status launch_softclip_backward(const float* x, int64_t ldx, const float* gy, int64_t ldgy,
                                   const float* gl, int64_t B, int D, float bound, float* gx,
                                   int64_t ldgx, cudaStream_t stream);

// gz (B, D) = [gz_in] + g_lp * (-(z - loc) / scale^2);  gl (B) = [gl_in] + g_lp
// (distributions.py:115-119, torch normal.py:87-102); inputs may be null.
zk_status launch_base_grad(const float* z, int64_t ldz, const float* loc, const float* scale,
                           const float* g_lp, const float* gz_in, int64_t ldgz_in,
                           const float* gl_in, int64_t B, int D, float* gz, float* gl,
                           cudaStream_t stream);  // loc == scale == nullptr with g_lp: standard normal; see `flat_base`
// same seed for a base whose density is constant on its support (BoxUniform): d log p / dz = 0
zk_status launch_base_grad_flat(const float* g_lp, const float* gz_in, int64_t ldgz_in, const float* gl_in,
                                int64_t B, int D, float* gz, float* gl, cudaStream_t stream);

// out (B, nx + nc) = cat(x[:, cols] (or x[:, :nx] when cols == null), c)  (autoregressive.py:209)
zk_status launch_concat(const float* x, int64_t ldx, const int* cols, int nx, const float* c,
                        int64_t ldc, int nc, int64_t B, float* out, cudaStream_t stream);

// Distributes the conditioner's input gradient gin (B, nx + nc):
//   gx[:, col_j] (+)= gin[:, j]  for j < nx  (col_j = cols[j] or j; `add_x` = accumulate,
//                                             otherwise gx[:, col_j] = base[:, col_j] + gin[:, j])
//   gc[:, j] += gin[:, nx + j]   (gc may be null)
zk_status launch_input_grad(const float* gin, int nx, int nc, const int* cols, int64_t B, float* gx,
                            int64_t ldgx, const float* base, int64_t ldbase, float* gc,
                            int64_t ldgc, cudaStream_t stream);

// g[i] = a[i] > 0 ? g[i] : 0   (ReLU gate, n elements)
zk_status launch_relu_gate(float* g, const float* a, int64_t n, cudaStream_t stream);

// general activation (activations.cuh): y[i] = act(pre[i]);  g[i] *= act'(pre[i])
zk_status launch_act_apply(const float* pre, float* y, int64_t n, int act, cudaStream_t stream);
zk_status launch_act_gate(float* g, const float* pre, int64_t n, int act, cudaStream_t stream);

// out[n] += sum_b v[b, n]  (fixed-order two-stage); scratch >= colsum_scratch_bytes(N)
size_t colsum_scratch_bytes(int N);
zk_status launch_colsum_add(const float* v, int64_t ldv, int64_t B, int N, float* out, void* scratch,
                            cudaStream_t stream);

// gw (N, K) += mask ? sum_b g[b, n] * a[b, k] : 0   (mask (N, K) bytes or null = dense);
// scratch >= wgrad_scratch_bytes(N, K)
size_t wgrad_scratch_bytes(int N, int K);
zk_status launch_wgrad_fp32(const float* g, int64_t ldg, const float* a, int64_t lda, int64_t B,
                            int N, int K, const uint8_t* mask, float* gw, void* scratch,
                            cudaStream_t stream);

// out (K, N) = in (N, K)^T
zk_status launch_transpose(const float* in, int N, int K, float* out, cudaStream_t stream);

// y[i] += x[i]
zk_status launch_add(float* y, const float* x, int64_t n, cudaStream_t stream);
// out[i] = alpha * in[i]
zk_status launch_scale(float* out, const float* in, float alpha, int64_t n, cudaStream_t stream);
// out[i] = g[i] / s[i];   v[i] += (g[i] - jtv[i]) / s[i]   (Richardson sweep of the triangular solve J^T v = g)
zk_status launch_div(float* out, const float* g, const float* s, int64_t n, cudaStream_t stream);
zk_status launch_richardson(float* v, const float* g, const float* jtv, const float* s, int64_t n, cudaStream_t stream);

}  // namespace zk
