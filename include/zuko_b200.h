/*
 * zuko_b200 — C ABI of the H100-native (sm_90a) engine for Zuko's flow hot path.
 *
 * The reference (probabilists/zuko @ 1063ae4) has NO FFI, plugin registry or
 * native code: its seams are Python protocols.  The entry points below are the
 * boundary a native replacement of the hot path binds at; each cites the
 * reference interface (file:line in /root/reference) it replaces.  The Python
 * host side in zuko_b200/ mirrors the reference's LazyTransform /
 * LazyDistribution / Flow API on top of these calls (see INTEGRATION.md for the
 * ctypes stub a reference maintainer would add).
 *
 * Conventions
 *   - every function returns a zk_status (0 = OK) and never throws;
 *     zk_last_error() gives a thread-local message for the last failure;
 *   - all tensor pointers are DEVICE pointers to fp32 row-major data unless the
 *     parameter comment says "host"; `ld*` are row strides in ELEMENTS;
 *     ldc == 0 broadcasts a single context row (zuko/utils.py:236-244,
 *     zuko/flows/autoregressive.py:209);
 *   - calls are asynchronous on the given CUDA stream (cudaStream_t passed as
 *     void*); the caller owns every input / output / workspace buffer;
 *   - handles (zk_mlp, zk_layer) own only packed copies of the weights and are
 *     immutable after creation => re-entrant across streams when each call has
 *     its own workspace;
 *   - there is no CPU fallback: without a CUDA device every compute entry point
 *     returns ZK_ECUDA.
 */
#ifndef ZUKO_B200_H
#define ZUKO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    ZK_OK = 0,
    ZK_EINVAL = 1,       /* bad shape / pointer / alignment / workspace too small */
    ZK_EUNSUPPORTED = 2, /* option the engine does not implement */
    ZK_ECUDA = 3,        /* CUDA runtime error (message in zk_last_error) */
    ZK_ENOMEM = 4
} zk_status;

typedef void* zk_stream; /* cudaStream_t */

/* univariate bijector applied per (sample, dim) */
#define ZK_UNI_AFFINE 1 /* MonotonicAffineTransform, zuko/transforms.py:412-446; phi = (shift, scale) */
#define ZK_UNI_RQS 2    /* MonotonicRQSTransform,    zuko/transforms.py:449-567; phi = (w[K], h[K], d[K-1]) */
#define ZK_UNI_CRQS 3   /* CircularRQSTransform = CircularShiftTransform(bound) then RQS(bound), zuko/flows/spline.py:65-72
                           (layers only: NCSF; `bound` of the layer is pi) */
#define ZK_UNI_GAUSS 4  /* GaussianizationTransform, zuko/transforms.py:834-875; phi = (shift[K], scale[K]), inverse by
                           bisection on [-bound, bound] (transforms.py:609-617); element-wise layers only */
#define ZK_UNI_SOSP 5   /* ShiftedSOSPTransform = SOSPolynomialTransform(a, slope) then AdditiveTransform(constant),
                           zuko/flows/polynomial.py:23-28, transforms.py:878-963; phi = (a[K][L+1] row-major, constant),
                           P = K (L + 1) + 1 (K = `bins`, L = `degree`); inverse by bisection on [-bound, bound];
                           autoregressive layers only */
#define ZK_UNI_BERNSTEIN 6 /* BoundedBernsteinTransform, zuko/transforms.py:640-831 (BPF, flows/polynomial.py:79-117);
                              phi = u[degree + 1] (unconstrained, softmax-constrained coefficient differences),
                              order M = degree + 5 <= 64; bound B = `bound`, eps = 1e-6; inverse by the two linear
                              branches beyond [-B, B] and bisection on [-B, B] inside; autoregressive layers only */
/* base distribution of a flow */
#define ZK_BASE_DIAG_NORMAL 0 /* DiagNormal(loc, scale)    zuko/distributions.py:337-363 */
#define ZK_BASE_BOX_UNIFORM 1 /* BoxUniform(lower, upper)  zuko/distributions.py:366-396; base_loc = lower, base_scale = upper */

/* layer kinds (elements of a ComposedTransform, zuko/transforms.py:59-160) */
#define ZK_LAYER_AUTOREGRESSIVE 1 /* flows/autoregressive.py:24-218 + transforms.py:966-1007 */
#define ZK_LAYER_COUPLING 2       /* flows/coupling.py:25-139 + transforms.py:1010-1073 */
#define ZK_LAYER_ELEMENTWISE 3    /* flows/gaussianization.py:28-94 */
#define ZK_LAYER_SOFTCLIP 4       /* transforms.py:286-316 */
#define ZK_LAYER_PERMUTATION 5    /* transforms.py:1182-1214 */
#define ZK_LAYER_ROTATION 6       /* transforms.py:1217-1244 */

/* arithmetic of the conditioner GEMMs (zuko/nn.py:217-218) */
#define ZK_GEMM_AUTO 0    /* tensor-core split-bf16 when the shape allows it, else fp32 SIMT */
#define ZK_GEMM_FP32 1    /* fp32 FMA on CUDA cores (exact-order reference path, any shape) */
#define ZK_GEMM_BF16X3 2  /* wgmma bf16, hi/lo split (3 MMAs), fp32 accumulate in registers */
#define ZK_GEMM_BF16X1 3  /* single bf16 MMA: fast, does NOT meet the 1e-5 parity bar */

/* activation between the linear layers of a conditioner (zuko/nn.py:264-265: `activation()` modules);
 * torch defaults of each: ELU(alpha=1), GELU(approximate='none'), LeakyReLU(0.01), Softplus(beta=1,
 * threshold=20).  0 keeps the reference's default (ReLU). */
#define ZK_ACT_RELU 0
#define ZK_ACT_ELU 2
#define ZK_ACT_TANH 3
#define ZK_ACT_SILU 4
#define ZK_ACT_GELU 5
#define ZK_ACT_LEAKY_RELU 6
#define ZK_ACT_SOFTPLUS 7
#define ZK_ACT_SIGMOID 8

int zk_version(void);
const char* zk_last_error(void);
/* sm count / compute capability of the current device; ZK_ECUDA if none. */
zk_status zk_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------- *
 * Stand-alone bijector kernels (one fused pass each: z and summed ladj).
 * `ladj` is per SAMPLE: sum over D of log|dy/dx| — i.e. what
 * DependentTransform.call_and_ladj returns (transforms.py:210-214); with
 * accumulate != 0 it is added to the buffer (transforms.py:147).
 * `phi_ld` is the row stride of phi in elements: D*P for dense per-sample
 * parameters as produced by MaskedAutoregressiveTransform.meta (flows/
 * autoregressive.py:207-215), any larger value for padded rows (the pads are
 * never read), or 0 for one shared (D, P) table (flows/gaussianization.py:74-77).
 * y may alias x; y or ladj may be NULL when not needed.
 * ------------------------------------------------------------------------- */

/* Tile plan of the stand-alone bijector kernel for these arguments, as the next launch would choose it (univariate is
 * ZK_UNI_AFFINE, _RQS, _GAUSS, _SOSP or _BERNSTEIN; K = bins / components / polynomials; degree of SOSP / Bernstein;
 * phi only for its alignment).  Returns ZK_OK and fills the non-NULL outputs, or the status the launch would return for
 * these arguments.  rows_per_tile: sample rows per CTA; smem: dynamic shared memory bytes; bulk_staging: 1 when full
 * tiles stage phi with one bulk copy; shuffle_sum: 1 when the ladj sum over D is the warp-shuffle reduction (D <= 32, a
 * power of two), 0 for the fixed-order one; bins_instantiated: the compile-time shape the launch picks (RQS 4, 8 or 16,
 * Gaussianization 8 or 16, SOSP 3 for (K, degree) = (3, 4), Bernstein 17 for degree 16; 0 for the runtime-shape
 * kernel).  B = 0 reports 0 everywhere.  Read-only, no device work. */
zk_status zk_univariate_plan(int univariate, int64_t B, int D, int K, int degree, int64_t phi_ld, const float* phi,
                             int* rows_per_tile, size_t* smem, int* bulk_staging, int* shuffle_sum, int* bins_instantiated);

/* MonotonicRQSTransform(*phi).call_and_ladj(x)   — transforms.py:469-490,554-567 */
zk_status zk_rqs_forward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                         int D, int K, float bound, float slope, float* y, int64_t ldy,
                         float* ladj, int accumulate, zk_stream stream);
/* MonotonicRQSTransform(*phi)._inverse(y)        — transforms.py:534-548 */
zk_status zk_rqs_inverse(const float* y, int64_t ldy, const float* phi, int64_t phi_ld, int64_t B,
                         int D, int K, float bound, float slope, float* x, int64_t ldx,
                         zk_stream stream);
/* MonotonicAffineTransform(shift, scale)         — transforms.py:426-446 */
zk_status zk_affine_forward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld,
                            int64_t B, int D, float slope, float* y, int64_t ldy, float* ladj,
                            int accumulate, zk_stream stream);
zk_status zk_affine_inverse(const float* y, int64_t ldy, const float* phi, int64_t phi_ld,
                            int64_t B, int D, float slope, float* x, int64_t ldx,
                            zk_stream stream);
/* GaussianizationTransform(shift, scale, bound, eps) — transforms.py:834-875; phi = (shift[K], scale[K]) per pair.
 * Forward: y and the closed-form ladj.  Inverse: `iterations` bisection steps on [-bound, bound] (utils.py:159-183);
 * a y beyond the range of f returns +-(bound - half the final interval), as the reference does. */
zk_status zk_gaussianization_forward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                                     int D, int K, float* y, int64_t ldy, float* ladj, int accumulate,
                                     zk_stream stream);
zk_status zk_gaussianization_inverse(const float* y, int64_t ldy, const float* phi, int64_t phi_ld, int64_t B,
                                     int D, int K, float bound, int iterations, float* x, int64_t ldx,
                                     zk_stream stream);
/* ShiftedSOSPTransform(a, constant, slope) with SOSPolynomialTransform's bound — flows/polynomial.py:23-28,
 * transforms.py:878-963; phi = (a[K][degree+1] row-major, constant) per pair, 1 <= K, 0 <= degree <= 15,
 * K (degree + 1) + 1 <= 1024.  Forward: y = x sum_i w_i g(t_i x) + constant (degree + 1 Gauss-Legendre nodes)
 * and ladj = log g(x).  Inverse: `iterations` bisection steps on [-bound, bound] of y - constant; a y beyond
 * the range of f returns +-(bound - half the final interval), as the reference does. */
zk_status zk_sosp_forward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B, int D,
                          int K, int degree, float bound, float slope, float* y, int64_t ldy, float* ladj,
                          int accumulate, zk_stream stream);
zk_status zk_sosp_inverse(const float* y, int64_t ldy, const float* phi, int64_t phi_ld, int64_t B, int D,
                          int K, int degree, float bound, float slope, int iterations, float* x, int64_t ldx,
                          zk_stream stream);
/* BoundedBernsteinTransform(u, bound, eps) — transforms.py:640-831; phi = u[degree + 1] per pair, 0 <= degree <= 59,
 * bound > 0, 0 < eps < 1/2.  Forward: t = (x + B) / 2B; y = sum_i theta_i b_{i,M}(t) for eps < t < 1 - eps, else
 * the linear branches 2B (t - eps) - B and 2B (t - 1 + eps) + B (so x -+ 2B eps outside [-B, B]), and ladj =
 * log f'(x) (0 in the linear branches).  Inverse: the linear branches exactly for y <= -B and y >= B, else
 * ceil(log2(2 B / eps)) bisection steps on [-B, B] (utils.py:159-183). */
zk_status zk_bernstein_forward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B, int D,
                               int degree, float bound, float eps, float* y, int64_t ldy, float* ladj,
                               int accumulate, zk_stream stream);
zk_status zk_bernstein_inverse(const float* y, int64_t ldy, const float* phi, int64_t phi_ld, int64_t B, int D,
                               int degree, float bound, float eps, float* x, int64_t ldx, zk_stream stream);
/* SoftclipTransform(bound)                       — transforms.py:299-316 */
zk_status zk_softclip_forward(const float* x, int64_t ldx, int64_t B, int D, float bound, float* y,
                              int64_t ldy, float* ladj, int accumulate, zk_stream stream);
zk_status zk_softclip_inverse(const float* y, int64_t ldy, int64_t B, int D, float bound, float* x,
                              int64_t ldx, zk_stream stream);
/* PermutationTransform: y[:, j] = x[:, order[j]] (bit-exact) — transforms.py:1207-1211.
 * `order` is a DEVICE int64 vector of length D.  x and y must not alias. */
zk_status zk_permute(const float* x, int64_t ldx, const int64_t* order, int64_t B, int D, float* y,
                     int64_t ldy, zk_stream stream);
/* RotationTransform: y = R x (transpose = 0) or R^T x (1); R is DEVICE (D, D)
 * row-major, = matrix_exp(A - A^T) built by the caller — transforms.py:1235-1241. */
zk_status zk_rotate(const float* x, int64_t ldx, const float* R, int transpose, int64_t B, int D,
                    float* y, int64_t ldy, zk_stream stream);
/* CircularShiftTransform(bound): y = remainder(x, 2 bound) - bound (torch.remainder semantics), its own
 * inverse, ladj 0 — transforms.py:319-351. */
zk_status zk_circular_shift(const float* x, int64_t ldx, int64_t B, int D, float bound, float* y,
                            int64_t ldy, zk_stream stream);
/* BoxUniform(lower, upper).log_prob(z) + ladj — distributions.py:366-396, torch/distributions/uniform.py:
 * -sum_d log(upper_d - lower_d) when lower <= z < upper in every dim, -inf otherwise; ladj may be NULL. */
zk_status zk_box_uniform_log_prob(const float* z, int64_t ldz, const float* lower, const float* upper,
                                  const float* ladj, int64_t B, int D, float* out, zk_stream stream);
/* DiagNormal(loc, scale).log_prob(z) + ladj — distributions.py:115-119,337-363;
 * loc/scale DEVICE (D) or both NULL for the standard normal; ladj may be NULL. */
zk_status zk_diag_normal_log_prob(const float* z, int64_t ldz, const float* loc, const float* scale,
                                  const float* ladj, int64_t B, int D, float* out,
                                  zk_stream stream);

/* ------------------------------------------------------------------------- *
 * Conditioner: MaskedMLP (zuko/nn.py:221-318) or MLP (zuko/nn.py:122-192) with
 * an element-wise activation (ReLU by default, ZK_ACT_*) between layers and none after the last.  Creation applies `mask * W`
 * ONCE (the reference redoes it on every call, nn.py:217-218) and packs the
 * weights for the selected GEMM path.
 * ------------------------------------------------------------------------- */
typedef struct zk_mlp zk_mlp;

typedef struct {
    int n_linear;                /* number of linear layers (>= 1) */
    const int* dims;             /* host, n_linear + 1 widths: in, hidden..., out */
    const float* const* weight;  /* host array of DEVICE ptrs, (dims[i+1], dims[i]) row-major */
    const float* const* bias;    /* host array of DEVICE ptrs, (dims[i+1]); entries may be NULL */
    const uint8_t* const* mask;  /* host array of DEVICE ptrs (bool bytes), or NULL / NULL entries = dense */
    int gemm_mode;               /* ZK_GEMM_* */
    int activation;              /* ZK_ACT_* between the linear layers (0 = ReLU) */
    /* residual conditioners (MaskedMLP(residual=True), zuko/nn.py:195-199, 297-309): per linear layer, host
     * arrays of n_linear ints or NULL for the plain pattern (activation after every layer but the last):
     * layer_act[i] = 0 none / 1 ReLU / ZK_ACT_* applied to the output of layer i; layer_res[i] != 0 adds the
     * INPUT of layer i-1 to the output of layer i (second layer of a residual block; needs i >= 2 and equal
     * widths).  Such handles run the per-layer GEMM kernels (tensor cores or fp32 by gemm_mode), never the
     * fused layer kernels; their backward pass runs the fp32 kernels. */
    const int* layer_act;
    const int* layer_res;
} zk_mlp_desc;

zk_status zk_mlp_create(const zk_mlp_desc* desc, zk_mlp** out);
zk_status zk_mlp_destroy(zk_mlp* mlp);
size_t zk_mlp_workspace_bytes(const zk_mlp* mlp, int64_t B);
/* out = mlp(cat(x, c)): x (B, dx), c (B, dc) or one row (ldc = 0) or NULL (dc = 0);
 * dx + dc must equal dims[0]; out is (B, dims[n_linear]) with row stride ldo.  The workspace must be 256-byte
 * aligned on a tensor-core handle (ZK_GEMM_BF16X3 / BF16X1; cudaMalloc and torch allocations are) and 4-byte
 * aligned on an fp32 one (ZK_EINVAL otherwise). */
zk_status zk_mlp_forward(const zk_mlp* mlp, const float* x, int64_t ldx, int dx, const float* c,
                         int64_t ldc, int dc, int64_t B, float* out, int64_t ldo, void* workspace,
                         size_t workspace_bytes, zk_stream stream);
/* which GEMM path the handle resolved to (ZK_GEMM_FP32 / BF16X3 / BF16X1) */
int zk_mlp_gemm_mode(const zk_mlp* mlp);

/* ------------------------------------------------------------------------- *
 * Layers: one lazy transformation of the reference, packed.
 * ------------------------------------------------------------------------- */
typedef struct zk_layer zk_layer;

typedef struct {
    int kind;       /* ZK_LAYER_* */
    int features;   /* D */
    int context;    /* C (0 = unconditional) */
    int univariate; /* ZK_UNI_* (autoregressive / coupling / elementwise) */
    int bins;       /* K for ZK_UNI_RQS, mixture components K for ZK_UNI_GAUSS, polynomials K for ZK_UNI_SOSP */
    float bound;    /* spline bound B (5.0), softclip bound, the bisection bound of ZK_UNI_GAUSS / ZK_UNI_SOSP (10.0)
                       or the Bernstein bound B of ZK_UNI_BERNSTEIN (5.0) */
    float slope;    /* minimum slope (1e-3) */
    int passes;     /* autoregressive: number of inverse sweeps (transforms.py:994-1000) */
    const int64_t* order;         /* host (D): autoregressive order classes (MaskedAutoregressiveTransform.order,
                                     flows/autoregressive.py:121-124; may be NULL) or the permutation order */
    const uint8_t* coupling_mask; /* host (D) bool: 1 = constant split x_a (transforms.py:1037-1041) */
    const zk_mlp_desc* hyper;     /* conditioner; NULL for parameter-free / shared-table layers */
    const float* phi;             /* DEVICE (D, P) shared table: elementwise without context */
    const float* rotation;        /* DEVICE (D, D) R for ZK_LAYER_ROTATION */
    int iterations;               /* ZK_UNI_GAUSS / ZK_UNI_SOSP / ZK_UNI_BERNSTEIN: bisection steps of the inverse,
                                     ceil(log2(2 bound / eps)) (>= 1; eps = 1e-6) */
    int degree;                   /* ZK_UNI_SOSP: polynomial degree L (0 .. 15); ZK_UNI_BERNSTEIN: BPF degree (0 .. 59) */
} zk_layer_desc;

zk_status zk_layer_create(const zk_layer_desc* desc, zk_layer** out);
zk_status zk_layer_destroy(zk_layer* layer);
/* The conditioner's weights / biases changed (optimizer step, nn.py:217-218 reads them on every
 * call) but shapes, masks and options did not: refreshes every packed copy IN PLACE — `mask * W`, the
 * bf16 hi / lo planes of the GEMM and fused kernels — with kernels on `stream`: no allocation, no
 * host synchronisation, no mask download.  The transposed weights of the backward pass and the
 * step-ordered stream of the sequential inverse are rebuilt by the next call that needs them.
 * weight / bias: host arrays of n_linear DEVICE pointers as in zk_mlp_desc.  Unlike zk_mlp_desc, a NULL
 * bias array or a NULL bias entry KEEPS that layer's current bias (it does not mean a zero bias).
 * Every weight pointer is checked before any work is queued: a refusal (ZK_EINVAL) changes nothing.
 * Calls already queued on `stream` see the old weights, later ones the new. */
zk_status zk_layer_update_weights(zk_layer* layer, const float* const* weight, const float* const* bias,
                                  zk_stream stream);
/* Names the stream the caller's tensors are produced on (thread-local; NULL = none): zk_mlp_create /
 * zk_layer_create synchronise it before their pack kernels (legacy default stream) read the weights. */
void zk_set_pack_stream(zk_stream stream);
size_t zk_layer_workspace_bytes(const zk_layer* layer, int64_t B);
/* Bench bookkeeping: which kernel runs an autoregressive layer's forward (flows/autoregressive.py:
 * 207-215) and how much tensor-core work it issues.  Returns 0 = per-layer GEMM kernels,
 * 1 = fused layer kernel; out[0] = the same,
 * out[1] = non-zero 64 x 64 weight tiles per row tile, out[2] = MACs ISSUED per sample row (non-zero tiles only, all
 * split-bf16 terms; an output-layer tile is multiplied at the width of its parameter rows, 48 for RQS, and layer 0's
 * last K block over the 16-wide steps that hold inputs), out[3] = dense MACs per sample row (what nn.py:218
 * executes). */
int zk_layer_fused_info(const zk_layer* layer, double* out);
/* Weight bytes the fused layer kernel brings into shared memory per row tile (the tiles of out[1], all bf16 planes
 * of the GEMM mode: 64 x 64 boxes, 48 x 64 for the output layer of RQS); 0 when the layer does not run fused. */
size_t zk_layer_fused_stream_bytes(const zk_layer* layer);
/* Rows per tile of the fused layer kernel for this layer, chosen from its shape: 128 (two consumer warpgroups
 * share every streamed weight tile), 64, or 0 when the layer does not run as the fused kernel.  Read-only. */
int zk_layer_fused_tile_rows(const zk_layer* layer);
/* The fused layer kernel's plan for this layer, as its next launch would choose it: returns the rows per tile (the
 * value of zk_layer_fused_tile_rows) and, when it is not 0, fills the non-NULL outputs with the number of 16 KB
 * weight-ring slots (64-row tiles: both consumer warpgroups' rings together) and the dynamic shared memory bytes.
 * Read-only. */
int zk_layer_fused_plan(const zk_layer* layer, int* ring_slots, size_t* smem);
/* Launch geometry of the layer's dimension-sequential inverse kernel, as its next launch would choose it
 * (the ZK_INV_GEOM=TxR override included): threads per CTA, samples per thread and dynamic shared memory
 * bytes.  Returns 1 and fills the non-NULL outputs when the layer's inverse runs as that kernel (with the
 * fused kernels enabled, zk_set_fused_layers), 0 when it runs the `passes` sweeps.  Read-only. */
int zk_layer_inverse_geometry(const zk_layer* layer, int* threads, int* samples_per_thread, size_t* smem);
/* 1 when the layer's inverse runs as the dimension-sequential kernel (one launch, emits the ladj): the
 * precondition for using it as an inverted member of a zk_flow_desc. */
int zk_layer_sequential_inverse(const zk_layer* layer);
/* t(c).call_and_ladj(x): y (B, D), ladj (B) summed over the event dim; y must not alias x. */
zk_status zk_layer_forward(const zk_layer* layer, const float* x, int64_t ldx, const float* c,
                           int64_t ldc, int64_t B, float* y, int64_t ldy, float* ladj,
                           int accumulate, void* workspace, size_t workspace_bytes,
                           zk_stream stream);
/* t(c).inv(y); x must not alias y. */
zk_status zk_layer_inverse(const zk_layer* layer, const float* y, int64_t ldy, const float* c,
                           int64_t ldc, int64_t B, float* x, int64_t ldx, void* workspace,
                           size_t workspace_bytes, zk_stream stream);

/* ------------------------------------------------------------------------- *
 * Flow: NormalizingFlow(ComposedTransform(layers...), DiagNormal(loc, scale))
 * — zuko/lazy.py:156-172, zuko/distributions.py:39-138.
 * ------------------------------------------------------------------------- */
typedef struct {
    int n_layers;
    const zk_layer* const* layers; /* host array of handles, applied first to last in the forward direction */
    int features;
    int context;
    const float* base_loc;   /* DEVICE (D) or NULL (0)   — BoxUniform: lower bounds (required) */
    const float* base_scale; /* DEVICE (D) or NULL (1)   — BoxUniform: upper bounds (required) */
    int base_kind;           /* ZK_BASE_* */
    const int* inverted;     /* host (n_layers) or NULL: != 0 = this member is the INVERSE of its layer — LazyInverse
                                (zuko/lazy.py:81-98: IAF-style flows, cheap sampling / sequential density).  Supported for
                                autoregressive layers with a dimension-sequential inverse (zk_layer_sequential_inverse);
                                zk_flow_forward / zk_flow_log_prob / zk_flow_inverse (without log_prob) honour it, the
                                backward entry points refuse such flows (ZK_EUNSUPPORTED). */
} zk_flow_desc;

/* bytes of workspace that let a batch of B rows run in a single chunk; any
 * workspace >= zk_flow_min_workspace_bytes() is accepted (the batch is then
 * processed in row chunks). */
size_t zk_flow_workspace_bytes(const zk_flow_desc* flow, int64_t B);
/* Workspace that lets zk_flow_log_prob_host run its preferred chunk plan for a batch of B rows (first chunk one
   wave of the persistent kernels, later chunks growing; two staging slots of the largest chunk + the flow's own
   scratch).  A smaller workspace still works: the plan is capped to what fits. */
size_t zk_flow_host_workspace_bytes(const zk_flow_desc* flow, int64_t B);
/* Test hook: the row chunks zk_flow_log_prob_host would use for B rows with the given wave size (rows one wave
   of the persistent kernels covers) and chunk cap; returns their number. */
int64_t zk_debug_host_chunk_plan(int64_t B, int64_t wave, int64_t max_chunk, int64_t* out, int64_t cap);
size_t zk_flow_min_workspace_bytes(const zk_flow_desc* flow);

/* transform.call_and_ladj(x) — transforms.py:141-150: z (B, D), ladj (B). */
zk_status zk_flow_forward(const zk_flow_desc* flow, const float* x, int64_t ldx, const float* c,
                          int64_t ldc, int64_t B, float* z, int64_t ldz, float* ladj,
                          void* workspace, size_t workspace_bytes, zk_stream stream);
/* NormalizingFlow.log_prob(x) — distributions.py:115-119: log_prob (B).
 * sum_log_prob: optional DEVICE double[1] receiving sum_b log_prob[b] by a
 * fixed-order two-stage reduction (the per-device term of the mean NLL). */
zk_status zk_flow_log_prob(const zk_flow_desc* flow, const float* x, int64_t ldx, const float* c,
                           int64_t ldc, int64_t B, float* log_prob, double* sum_log_prob,
                           void* workspace, size_t workspace_bytes, zk_stream stream);
/* transform.inv(z) — distributions.py:121-127 (z supplied by the caller);
 * with log_prob != NULL also NormalizingFlow.rsample_and_log_prob's second
 * output for that z — distributions.py:129-138. */
zk_status zk_flow_inverse(const zk_flow_desc* flow, const float* z, int64_t ldz, const float* c,
                          int64_t ldc, int64_t B, float* x, int64_t ldx, float* log_prob,
                          void* workspace, size_t workspace_bytes, zk_stream stream);

/* Host-buffer entry point (end-to-end path): x_host (B, D), c_host (B, C) or
 * one row (ldc = 0) or NULL, log_prob_host (B) are HOST pointers (pinned for
 * overlap); rows are streamed through the device in chunks with the copies
 * overlapped with compute.  `workspace` is a DEVICE buffer. */
zk_status zk_flow_log_prob_host(const zk_flow_desc* flow, const float* x_host, int64_t ldx,
                                const float* c_host, int64_t ldc, int64_t B, float* log_prob_host,
                                double* sum_log_prob_host, void* workspace, size_t workspace_bytes,
                                zk_stream stream);

/* ------------------------------------------------------------------------- *
 * Backward pass (reverse mode) — what torch.autograd computes for the reference
 * when a training loop calls (-flow(c).log_prob(x).mean()).backward()
 * (README.md:43-49, tests/test_flows.py:22-29), SURVEY section 8(f) rank 1.
 * The forward activations are recomputed inside the call (nothing is saved by the
 * forward entry points).  Parameter gradients are ACCUMULATED (+=) into caller
 * buffers with the shapes of the reference's parameters, so a batch processed in
 * several calls / row chunks sums up like autograd's .grad does; grad_x is
 * overwritten.  Gradients w.r.t. a masked weight are w.r.t. the RAW weight
 * (already multiplied by the mask, nn.py:218).  Reductions over the batch run in a
 * fixed order (bit-reproducible run to run).
 * ------------------------------------------------------------------------- */
typedef struct {
    float* const* grad_weight; /* host array [n_linear] of DEVICE (dims[i+1], dims[i]) buffers; NULL array / entries = not wanted */
    float* const* grad_bias;   /* host array [n_linear] of DEVICE (dims[i+1]) buffers; NULL array / entries = not wanted */
    float* grad_phi;           /* DEVICE (D, P): element-wise layer with a shared table (gaussianization.py:74-77) */
    float* grad_rotation;      /* DEVICE (D, D): dL/dR of a rotation layer (the caller chains through matrix_exp) */
} zk_layer_grads;

/* d/d(x, phi) of MonotonicRQSTransform(*phi).call_and_ladj(x) (transforms.py:469-567) for upstream
 * gradients grad_y (B, D) and grad_ladj (B, of the per-sample summed ladj); either may be NULL (= 0).
 * grad_phi: (B, D*P) per-sample gradients when phi_ld != 0, or the (D, P) table gradient, ACCUMULATED,
 * when phi_ld == 0.  grad_phi must not overlap phi, except grad_phi == phi with phi_ld == D*P (the
 * gradients overwrite the parameters); any other overlap, a shared table included, returns ZK_EINVAL
 * before anything runs.  grad_x / grad_phi may be NULL.
 * workspace >= zk_univariate_backward_workspace_bytes(B, D, P, phi_ld). */
size_t zk_univariate_backward_workspace_bytes(int64_t B, int D, int P, int64_t phi_ld);
/* Tile plan of the bijector backward kernel for these arguments (as zk_univariate_plan for the forward): returns ZK_OK
 * and fills the non-NULL outputs, or the status the launch would return for this shape.  rows_per_tile: sample rows
 * per CTA; smem: dynamic shared memory bytes (R parameter rows, plus a shared table beside them when R > 1; at R = 1
 * the table is rewritten in place, so one row of up to 200 KB fits either way); instantiated: the compile-time shape
 * (RQS 8 or 16, Gaussianization 8 or 16, SOSP 3 for (K, degree) = (3, 4), Bernstein 17 for degree 16; 0 for the
 * runtime-shape and affine kernels).  B = 0 reports 0 everywhere.  Read-only, no device work. */
zk_status zk_univariate_backward_plan(int univariate, int64_t B, int D, int K, int degree, int64_t phi_ld,
                                      int* rows_per_tile, size_t* smem, int* instantiated);
zk_status zk_rqs_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                          int D, int K, float bound, float slope, const float* grad_y, int64_t ldgy,
                          const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi,
                          void* workspace, size_t workspace_bytes, zk_stream stream);
/* same for MonotonicAffineTransform (transforms.py:426-446), P = 2 */
zk_status zk_affine_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                             int D, float slope, const float* grad_y, int64_t ldgy,
                             const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi,
                             void* workspace, size_t workspace_bytes, zk_stream stream);
/* same for GaussianizationTransform (transforms.py:834-875), P = 2K */
zk_status zk_gaussianization_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                                      int D, int K, const float* grad_y, int64_t ldgy, const float* grad_ladj,
                                      float* grad_x, int64_t ldgx, float* grad_phi, void* workspace,
                                      size_t workspace_bytes, zk_stream stream);
/* same for ShiftedSOSPTransform (flows/polynomial.py:23-28, transforms.py:878-963), P = K (degree + 1) + 1 */
zk_status zk_sosp_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B, int D,
                           int K, int degree, float bound, float slope, const float* grad_y, int64_t ldgy,
                           const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi, void* workspace,
                           size_t workspace_bytes, zk_stream stream);
/* same for BoundedBernsteinTransform (transforms.py:640-831), P = degree + 1 */
zk_status zk_bernstein_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B, int D,
                                int degree, float bound, float eps, const float* grad_y, int64_t ldgy,
                                const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi, void* workspace,
                                size_t workspace_bytes, zk_stream stream);
/* SoftclipTransform (transforms.py:299-316) */
zk_status zk_softclip_backward(const float* x, int64_t ldx, int64_t B, int D, float bound,
                               const float* grad_y, int64_t ldgy, const float* grad_ladj,
                               float* grad_x, int64_t ldgx, zk_stream stream);

/* Reverse mode of zk_layer_forward: given x, c and the upstream gradients grad_y (B, D) and
 * grad_ladj (B, may be NULL), writes grad_x (B, D) and accumulates the parameter gradients
 * selected in `grads` (may be NULL) and, when grad_c != NULL, the context gradient: += into
 * (B, C) rows (ldgc >= C), or into ONE row (C) holding the sum over the batch when ldc == 0. */
size_t zk_layer_backward_workspace_bytes(const zk_layer* layer, int64_t B);
zk_status zk_layer_backward(const zk_layer* layer, const float* x, int64_t ldx, const float* c,
                            int64_t ldc, int64_t B, const float* grad_y, int64_t ldgy,
                            const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_c,
                            int64_t ldgc, const zk_layer_grads* grads, void* workspace,
                            size_t workspace_bytes, zk_stream stream);

/* Reverse mode of zk_flow_forward and / or zk_flow_log_prob in one call:
 *   L = <grad_z, z> + <grad_ladj, ladj> + <grad_log_prob, log_prob>      (each may be NULL)
 * writes grad_x (B, D) (may be NULL), OVERWRITES grad_c ((B, C) rows, or one summed row when
 * ldc == 0; may be NULL) and accumulates parameter gradients: grads[i] belongs to layers[i]
 * (array or entries may be NULL).  Any workspace >= zk_flow_backward_min_workspace_bytes() is
 * accepted: the batch is processed in row chunks that fit. */
size_t zk_flow_backward_workspace_bytes(const zk_flow_desc* flow, int64_t B);
size_t zk_flow_backward_min_workspace_bytes(const zk_flow_desc* flow);
zk_status zk_flow_backward(const zk_flow_desc* flow, const float* x, int64_t ldx, const float* c,
                           int64_t ldc, int64_t B, const float* grad_z, int64_t ldgz,
                           const float* grad_ladj, const float* grad_log_prob, float* grad_x,
                           int64_t ldgx, float* grad_c, int64_t ldgc,
                           const zk_layer_grads* const* grads, void* workspace,
                           size_t workspace_bytes, zk_stream stream);

/* Reverse mode of zk_flow_inverse (SURVEY section 8f rank 2: reparameterised sampling, reverse-KL training):
 *   x = transform.inv(z)                      L = <grad_x, x> [+ <grad_log_prob, log_prob>]
 * where log_prob is the second output of zk_flow_inverse / NormalizingFlow.rsample_and_log_prob
 * (distributions.py:129-138).  `x` is the SAMPLE the forward call returned (the engine walks the
 * forward chain from it); `z` is only read for the base term of grad_log_prob.  Writes grad_z (B, D),
 * OVERWRITES grad_c and accumulates parameter gradients exactly like zk_flow_backward.  Implicit
 * differentiation: per layer `passes` sweeps of J^T v = g, each one call of the forward direction's
 * backward — torch.autograd reaches the same numbers by back-propagating through the inverse sweeps
 * of transforms.py:994-1000. */
size_t zk_flow_inverse_backward_workspace_bytes(const zk_flow_desc* flow, int64_t B);
size_t zk_flow_inverse_backward_min_workspace_bytes(const zk_flow_desc* flow);
zk_status zk_flow_inverse_backward(const zk_flow_desc* flow, const float* x, int64_t ldx, const float* c,
                                   int64_t ldc, int64_t B, const float* grad_x, int64_t ldgx,
                                   const float* grad_log_prob, const float* z, int64_t ldz, float* grad_z,
                                   int64_t ldgz, float* grad_c, int64_t ldgc,
                                   const zk_layer_grads* const* grads, void* workspace,
                                   size_t workspace_bytes, zk_stream stream);

/* ------------------------------------------------------------------------- *
 * Multi-GPU: the path shards by rows with no data-path collective (every op is row-wise: nn.py:217-218,
 * transforms.py:554-567, distributions.py:115-119); the ONLY exchange is the all-reduce(sum) of the
 * per-device {sum log p, count} doubles for the scalar mean NLL (SURVEY §8e).  Single-process form over
 * NCCL (resolved with dlopen at run time); the Python mirror uses torch.distributed with one process per
 * GPU (zuko_b200/dist.py).
 * ------------------------------------------------------------------------- */
typedef struct zk_comm zk_comm;
/* one communicator over devices 0 .. ndev-1 of this process (ncclCommInitAll) */
zk_status zk_comm_init_all(int ndev, zk_comm** out);
zk_status zk_comm_destroy(zk_comm* comm);
int zk_comm_size(const zk_comm* comm);
/* buf[0..n) (DEVICE doubles on device `dev`) <- element-wise sum over all devices, asynchronously on `stream`
 * (a stream of device `dev`).  One thread driving several devices brackets its calls — one per device — with
 * zk_comm_group_begin / zk_comm_group_end (ncclGroupStart / ncclGroupEnd). */
zk_status zk_comm_group_begin(zk_comm* comm);
zk_status zk_allreduce_sum(zk_comm* comm, int dev, double* buf, int n, zk_stream stream);
zk_status zk_comm_group_end(zk_comm* comm);

/* ------------------------------------------------------------------------- *
 * Continuous normalizing flow: FreeFormJacobianTransform (zuko/transforms.py:1095-1179) with the vector field
 * of FFJTransform.f (flows/continuous.py:88-97): f(t, x, c) = ode(cat(cos(freqs t), sin(freqs t), x, c)),
 * integrated by adaptive Dormand-Prince (utils.py:443-554).  The step size is shared by the whole batch: the
 * error of a trial is the maximum over every row and column, so a row's result depends on the rest of the
 * batch through the step sequence, and one call integrates its whole batch (it never chunks it).
 * Gradients through the integration: zk_cnf_backward (the adaptive checkpoint adjoint, utils.py:556-593).
 * ------------------------------------------------------------------------- */
#define ZK_CNF_TRACE_NONE 0       /* integrate x alone (_call / _inverse, transforms.py:1130-1144) */
#define ZK_CNF_TRACE_EXACT 1      /* call_and_ladj with the exact trace of df/dx (transforms.py:1150-1174) */
#define ZK_CNF_TRACE_HUTCHINSON 2 /* call_and_ladj with eps^T (df/dx) eps, eps supplied by the caller */

typedef struct zk_cnf zk_cnf;

/* ode: plain dense fp32 MLP (no masks, no residual blocks, any ZK_ACT_*) with dims[0] = features + context +
 * 2 freqs and dims[n_linear] = features; freq_values: DEVICE float[freqs] (the module's `freqs` buffer).  The
 * handle keeps a packed copy of the weights.  An MLP whose weights and per-row buffers do not fit one CTA's
 * shared memory is refused with ZK_EUNSUPPORTED by zk_cnf_plan / zk_cnf_integrate. */
zk_status zk_cnf_create(const zk_mlp_desc* ode, int features, int context, int freqs, const float* freq_values,
                        zk_cnf** out);
zk_status zk_cnf_destroy(zk_cnf* cnf);
/* workspace of zk_cnf_integrate for B rows (a smaller one is ZK_EINVAL; it must be 256-byte aligned) */
size_t zk_cnf_workspace_bytes(const zk_cnf* cnf, int64_t B, int trace);
/* launch plan of zk_cnf_integrate: cooperative CTAs (co-resident CTAs per SM x SMs), threads per CTA (one row
 * per thread and pass), passes over the rows per thread, dynamic shared memory; or the refusal status.  Outputs
 * may be NULL.  No device work. */
zk_status zk_cnf_plan(const zk_cnf* cnf, int64_t B, int trace, int* ctas, int* threads, int* passes, size_t* smem);
/* Integrates x (B, D) with context c (B, C) (ldc = 0: one broadcast row; NULL when C = 0) from times[0] to
 * times[1] (`times`: DEVICE float[2]; the inverse is the same call with the times swapped) with atol / rtol
 * (utils.py:532-552).  trace: ZK_CNF_TRACE_*; eps (B, D), row stride ldeps, for ZK_CNF_TRACE_HUTCHINSON only.
 * Writes y (B, D) (y may alias x) and, with a trace, ladj (B) = the integrated trace (NULL iff trace = NONE).
 * counts: DEVICE int32[2] (trials, accepted steps) or NULL; step_log: DEVICE float[max_trials][4] (t, dt, error,
 * accepted) per trial or NULL.  After max_trials trials without reaching times[1], or when t + dt == t in fp32
 * (where the reference would loop forever), every output is NaN and counts[1] = -1 - accepted.  One cooperative launch, no host synchronisation. */
zk_status zk_cnf_integrate(const zk_cnf* cnf, const float* x, int64_t ldx, const float* c, int64_t ldc, int64_t B,
                           const float* times, float atol, float rtol, int trace, const float* eps, int64_t ldeps,
                           int max_trials, float* y, int64_t ldy, float* ladj, int* counts, float* step_log,
                           void* workspace, size_t ws_bytes, zk_stream stream);

/* Reverse mode of one zk_cnf_integrate call (AdaptiveCheckpointAdjoint.backward, utils.py:556-593, on the packed
 * state (x, L) of call_and_ladj): for L = <grad_y, y> + <grad_ladj, ladj>.  x, c, ldc, B, trace and eps are the
 * call's own; x is its INPUT.  step_log / trials / accepted are its device log and counts (trials, accepted).
 * Each row is replayed from x along the logged accepted steps, bit for bit the call's states, then walked back
 * one 6-stage Dormand-Prince step of -dt per step, second-order terms of the trace included.  The call's rows
 * are independent once the steps are fixed, so the batch is processed in row chunks that fit the workspace.
 * grad_y (may be NULL = 0); grad_ladj (B) non-NULL iff trace != NONE; eps non-NULL iff trace = HUTCHINSON.
 * Writes grad_x (B, D) (may be NULL) and OVERWRITES grad_c ((B, C) rows, or one summed row when ldc == 0; may
 * be NULL).  Weight and bias gradients are ACCUMULATED into grads (module (out, in) layout; NULL entries are not
 * computed); reductions over rows run in a fixed order that does not depend on the chunking, so results are
 * bit-identical run to run and for any workspace size.
 * With no accepted step (t0 == t1) grad_x = grad_y and the rest is 0.  Ordinary launches, no host sync. */
size_t zk_cnf_backward_workspace_bytes(const zk_cnf* cnf, int64_t B, int trace, int accepted); /* one chunk */
/* chunks of one CTA's rows (threads per CTA) */
size_t zk_cnf_backward_min_workspace_bytes(const zk_cnf* cnf, int trace, int accepted);
/* threads per CTA (cnf_geometry's rule on the backward's per-row state), CTAs (co-resident x SMs), rows per chunk
 * for this workspace, dynamic shared memory of the adjoint kernel; ZK_EUNSUPPORTED when the backward state does
 * not fit; ZK_EINVAL when ws_bytes is below the minimum.  Outputs may be NULL.  No device work. */
zk_status zk_cnf_backward_plan(const zk_cnf* cnf, int64_t B, int trace, int accepted, size_t ws_bytes, int* ctas,
                               int* threads, int64_t* chunk_rows, size_t* smem);
zk_status zk_cnf_backward(const zk_cnf* cnf, const float* x, int64_t ldx, const float* c, int64_t ldc, int64_t B,
                          const float* step_log, int trials, int accepted, int trace, const float* eps, int64_t ldeps,
                          const float* grad_y, int64_t ldgy, const float* grad_ladj, float* grad_x, int64_t ldgx,
                          float* grad_c, int64_t ldgc, const zk_layer_grads* grads, void* workspace, size_t ws_bytes,
                          zk_stream stream);

/* ------------------------------------------------------------------------- *
 * Gaussian mixture model: GMM (zuko/mixtures.py:25-99) with Mixture.log_prob / sample
 * (zuko/distributions.py:216-290).  A row's parameters phi come in the reference's unpack order
 *     logits (K) | loc (K, D) | diag (L, Dd) | tril (L, D (D - 1) / 2)      L = tied ? 1 : K
 * (Dd = 1 spherical, D otherwise; tril for ZK_COV_FULL only), zk_gmm_params_per_row() floats.  They are
 * the conditioner's output rows hyper(c) when context > 0, else one caller-owned unconditional table `phi`
 * read by every row.  Scale matrices: L_ii = exp(diag_i) + epsilon, tril below the diagonal in
 * torch.tril_indices(D, D, -1) order; the per-row math is zuko_b200/csrc/gmm_math.cuh.
 * Covered shapes: 1 <= features <= 64, 1 <= components <= 32; others are ZK_EUNSUPPORTED.
 * Every call processes its batch in row chunks that fit the workspace (any workspace of at least
 * zk_gmm_min_workspace_bytes() is accepted).
 * ------------------------------------------------------------------------- */
#define ZK_COV_FULL 0
#define ZK_COV_DIAGONAL 1
#define ZK_COV_SPHERICAL 2

typedef struct {
    int features, context, components, covariance, tied;
    float epsilon;
    const zk_mlp_desc* hyper; /* MLP(context -> params per row); NULL when context == 0 */
} zk_gmm_desc;
typedef struct zk_gmm zk_gmm;

zk_status zk_gmm_create(const zk_gmm_desc* desc, zk_gmm** out);
zk_status zk_gmm_destroy(zk_gmm* gmm);
/* new conditioner weights / biases in place, as zk_layer_update_weights (NULL bias entries keep the current
 * bias; a refusal changes nothing) */
zk_status zk_gmm_update_weights(zk_gmm* gmm, const float* const* weight, const float* const* bias, zk_stream stream);
int64_t zk_gmm_params_per_row(int features, int components, int covariance, int tied);
/* Launch plan of the mixture kernels (one thread per row, `threads` rows per CTA, per-row vectors in
 * shared memory): threads, rows per CTA, dynamic shared memory of the log-density and of the backward
 * kernel, and the instantiation (covariance * 2 + tied).  ZK_EUNSUPPORTED outside the covered shapes,
 * ZK_EINVAL for an unknown covariance.  Outputs may be NULL.  No device work. */
zk_status zk_gmm_plan(int features, int components, int covariance, int tied, int* threads, int* rows_per_cta,
                      size_t* smem_log_prob, size_t* smem_backward, int* instantiated);
/* workspace of log_prob / sample (resp. backward) processing B rows in one chunk; the minimum of any call */
size_t zk_gmm_workspace_bytes(const zk_gmm* gmm, int64_t B);
size_t zk_gmm_backward_workspace_bytes(const zk_gmm* gmm, int64_t B);
size_t zk_gmm_min_workspace_bytes(const zk_gmm* gmm);
/* rows of one chunk for this workspace (0 when it is below the minimum); backward != 0 for zk_gmm_backward */
int64_t zk_gmm_chunk_rows(const zk_gmm* gmm, int64_t B, int backward, size_t ws_bytes);
/* log_prob (B) of x (B, D); c (B, C) rows, or one broadcast row when ldc == 0 (NULL when C == 0);
 * phi: the (params per row) table when C == 0, else NULL */
zk_status zk_gmm_log_prob(const zk_gmm* gmm, const float* x, int64_t ldx, const float* c, int64_t ldc,
                          const float* phi, int64_t B, float* log_prob, void* workspace, size_t ws_bytes,
                          zk_stream stream);
/* x (B, D) drawn from uniforms u (B) in [0, 1) (component) and standard normals z (B, D) */
zk_status zk_gmm_sample(const zk_gmm* gmm, const float* c, int64_t ldc, const float* phi, const float* u,
                        const float* z, int64_t ldz, int64_t B, float* x, int64_t ldx, void* workspace,
                        size_t ws_bytes, zk_stream stream);
/* Reverse mode of zk_gmm_log_prob for L = <grad_log_prob, log_prob>: writes grad_x (B, D) (may be NULL),
 * ACCUMULATES grad_c ((B, C) rows, or one summed row when ldc == 0; may be NULL) and the parameter
 * gradients: grads->grad_weight / grad_bias of the conditioner, or grads->grad_phi (params per row) of the
 * unconditional table.  Sums over rows run in a fixed order: bit-identical run to run for one workspace. */
zk_status zk_gmm_backward(const zk_gmm* gmm, const float* x, int64_t ldx, const float* c, int64_t ldc,
                          const float* phi, int64_t B, const float* grad_log_prob, float* grad_x, int64_t ldgx,
                          float* grad_c, int64_t ldgc, const zk_layer_grads* grads, void* workspace,
                          size_t ws_bytes, zk_stream stream);

/* 1 (default): the conditioner GEMMs of the backward pass (forward recompute, dgrad, wgrad) of a
 * handle packed for the tensor cores run on them (split-bf16, fp32 accumulate); 0: fp32 FMA on
 * CUDA cores (exact-order arbitration path).  Returns the previous value. */
int zk_set_tc_backward(int on);

/* Transcendental arithmetic of the bijector kernels: 1 (default) = MUFU rcp / ex2 / lg2
 * approximations, 0 = IEEE division + expf / logf (erf / erfc / erfcinv of the Gaussianization
 * bijector are IEEE-library calls in both settings; the sum-of-squares polynomial bijector uses the
 * approximation only for the log of its ladj, the bounded Bernstein bijector only for the log of its
 * ladj).  Process-wide; returns the previous
 * value.  Both settings meet the 1e-5 parity bar on the BASELINE configs (tests/). */
int zk_set_fast_math(int on);
/* 1 (default): an autoregressive layer whose conditioner fits the fused kernel (hidden widths
 * equal, a multiple of 64 and <= 512; D + C <= 512; RQS with
 * 8 / 16 bins or affine; tensor-core GEMM mode; any supported activation, no residual blocks) runs as ONE kernel —
 * conditioner + bijector + ladj, activations and phi stay on chip (nn.py:217-218,
 * flows/autoregressive.py:207-215, transforms.py:554-567 in one launch).
 * 0: always one GEMM kernel per linear layer + the stand-alone bijector kernel.  Returns the
 * previous value. */
int zk_set_fused_layers(int on);
/* number of kernel launches issued by this library since load (bench evidence) */
int64_t zk_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* ZUKO_B200_H */
