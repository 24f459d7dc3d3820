// zuko_b200 — fused element-wise bijector kernels for sm_90a.
//
// uni_kernel: one pass per flow layer over (B, D) with per-sample parameters
//   phi (B, D, P):  x, phi  ->  y, sum_d log|dy/dx|  (+ optional DiagNormal log-prob)
// for every univariate bijector family of uni_family.cuh (affine, RQS, Gaussianization, SOSP, Bernstein),
// replacing the eager per-pair ops of the reference's transforms and DependentTransform's ladj sum
// (zuko/transforms.py:210-214); the family's forward / inverse pair functions run in registers.
//
// Data movement: a CTA owns a tile of R consecutive sample rows.  With dense rows
// (phi_ld = D*P) their phi block is one contiguous range of R*D*P floats in HBM; it is
// staged into shared memory with a single 1-D TMA bulk copy (cp.async.bulk, mbarrier
// complete_tx) — or with coalesced loads when the 16-byte alignment rules of the bulk copy
// do not hold.  Padded rows (phi_ld > D*P) are gathered row by row with coalesced loads
// into the same dense layout.  The tile plan is uni_plan's (zk_univariate_plan).  Thread t then
// owns pair (row = t / D, dim = t % D): its P parameters sit at smem word t*P (P = 3K-1
// is odd for even K => conflict-free), x / y are accessed coalesced, and the per-sample
// sum over D is a warp-shuffle reduction (D a power of two <= 32) or a fixed-order
// shared-memory reduction (any D).
//
// Algorithmic HBM bytes per sample per layer: 4 * (D + D*P + D + 1)   (SURVEY §8d).

#include <math_constants.h>

#include "bijectors.cuh"
#include "uni_family.cuh"

namespace zk {

namespace {

constexpr int kUniThreads = 256;
using namespace bij;

// ---------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------
struct UniParams {
    const float* x; int64_t ldx;
    const float* phi; int64_t phi_ld;
    float* y; int64_t ldy;
    float* ladj; int accumulate;
    float* log_prob;
    const float* base_loc; const float* base_scale;
    const int* dim_map;
    int64_t B; int D; int K; int P;
    float bound, aw, ad;
    int rows_per_tile;
    int circ;      // RQS: circular shift by `bound` before the spline (forward) / after it (inverse)
    int use_bulk;  // host-side verdict: alignment rules for cp.async.bulk hold for full tiles
    int iters;     // Gaussianization inverse: bisection steps
    sosp::Const sosp;  // SOSP: shape, bisection and pre-scaled quadrature
    bern::Const bern;  // Bernstein: order, bound, eps and bisection
};

// UNI: the family (uni_family.cuh); KT: compile-time shape (0 = runtime shape); INVERSE; FAST math
template <int UNI, int KT, bool INVERSE, bool FAST>
__global__ void __launch_bounds__(kUniThreads) uni_kernel(const UniParams a) {
    using Fam = UniFamily<UNI>;
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t bar;

    const int tid = threadIdx.x;
    const int64_t r0 = (int64_t)blockIdx.x * a.rows_per_tile;
    const int nrows = (int)min((int64_t)a.rows_per_tile, a.B - r0);
    const int D = a.D, P = a.P;
    const int npairs = nrows * D;
    const bool shared_tbl = (a.phi_ld == 0);
    float* s_phi = smem;
    const int n_phi = shared_tbl ? D * P : nrows * D * P;
    float* s_red = smem + (shared_tbl ? D * P : a.rows_per_tile * D * P);  // [rows_per_tile * D]

    // ---- stage phi ----
    const float* g_phi = shared_tbl ? a.phi : a.phi + r0 * a.phi_ld;
    const uint32_t bytes = (uint32_t)n_phi * 4u;
    const bool bulk = a.use_bulk && !shared_tbl && (bytes % 16u == 0);
    if (bulk) {
        if (tid == 0) {
            mbar_init(&bar, 1);
            fence_mbar_init();
            mbar_arrive_expect_tx(&bar, bytes);
            bulk_g2s(s_phi, g_phi, bytes, &bar);
        }
    } else if (shared_tbl || a.phi_ld == (int64_t)D * P) {
        for (int i = tid; i < n_phi; i += kUniThreads) s_phi[i] = g_phi[i];
    } else {  // padded rows: row r of the tile starts at g_phi + r * phi_ld and lands dense at s_phi + r * D * P
        const int row_len = D * P;
#pragma unroll 1
        for (int i = tid; i < n_phi; i += kUniThreads) {
            const int r = i / row_len;
            s_phi[i] = g_phi[r * a.phi_ld + (i - r * row_len)];
        }
    }
    __syncthreads();
    if (bulk) mbar_wait(&bar, 0);

    // ---- per-pair work ----
    const bool want_sum = (!INVERSE) && (a.ladj != nullptr || a.log_prob != nullptr);
    const bool shfl = want_sum && (D <= 32) && ((D & (D - 1)) == 0);
    const int iters = (npairs + kUniThreads - 1) / kUniThreads;
    for (int it = 0; it < iters; ++it) {
        const int p = it * kUniThreads + tid;
        const bool valid = p < npairs;
        float lj = 0.f;
        int row = 0, d = 0;
        if (valid) {
            row = p / D;
            d = p - row * D;
            const int col = a.dim_map ? a.dim_map[d] : d;
            float xv = a.x[(r0 + row) * a.ldx + col];
            const float* pp = s_phi + (shared_tbl ? d * P : p * P);
            float yv;
            if constexpr (!INVERSE)
                yv = Fam::template forward<KT, FAST>(pp, a, xv, lj);
            else
                yv = Fam::template inverse<KT, FAST>(pp, a, xv);
            if (a.y) a.y[(r0 + row) * a.ldy + col] = yv;
            if (!INVERSE && a.log_prob) {
                // DiagNormal.log_prob term of this dim (torch/distributions/normal.py:87-102)
                const float mu = a.base_loc ? a.base_loc[col] : 0.f;
                const float sg = a.base_scale ? a.base_scale[col] : 1.f;
                const float u = (yv - mu) / sg;
                lj += -0.5f * u * u - logf(sg) - kHalfLog2Pi;
            }
        }
        if (want_sum) {
            if (shfl) {
                for (int o = D >> 1; o > 0; o >>= 1) lj += __shfl_xor_sync(0xffffffffu, lj, o);
                if (valid && d == 0) s_red[row] = lj;
            } else if (valid) {
                s_red[p] = lj;
            }
        }
    }
    if (!want_sum) return;
    __syncthreads();
    for (int row = tid; row < nrows; row += kUniThreads) {
        float s;
        if (shfl) {
            s = s_red[row];
        } else {
            s = 0.f;
            for (int d = 0; d < D; ++d) s += s_red[row * D + d];
        }
        const int64_t r = r0 + row;
        const float prev = a.accumulate ? a.ladj[r] : 0.f;
        if (a.log_prob)
            a.log_prob[r] = prev + s;
        else
            a.ladj[r] = prev + s;
    }
}

}  // namespace

zk_status uni_plan(const UniSpec& s, int64_t B, int D, int64_t phi_ld, const float* phi, UniPlan& out) {
    ZK_REQUIRE(B >= 0 && D > 0, "univariate: bad shape B=%lld D=%d", (long long)B, D);
    out = UniPlan{};
    if (B == 0) return ZK_OK;
    ZK_TRY(uni_check_shape(s));
    out.kt = uni_kt<kStandalone>(s);
    const int P = uni_P(s);
    ZK_REQUIRE(phi_ld == 0 || phi_ld >= (int64_t)D * P, "univariate: phi_ld too small");

    // tile = R rows: aim at >= 256 pairs and ~24 KB of phi per CTA, bounded by shared memory
    const size_t row_bytes = (size_t)D * P * 4;
    const size_t kMaxSmem = 200 * 1024;
    ZK_REQUIRE(row_bytes + D * 4 <= kMaxSmem, "univariate: D*P too large for one tile (%zu B)", row_bytes);
    int64_t R = (int64_t)(24 * 1024 / row_bytes);
    const int64_t r_pairs = ceil_div(kUniThreads, D);
    if (R < r_pairs) R = r_pairs;
    while (R > 1 && R * (row_bytes + (size_t)D * 4) > 96 * 1024) --R;
    if (R < 1) R = 1;
    if (R > B) R = B;
    const int64_t grid = ceil_div(B, R);
    ZK_REQUIRE(grid <= 0x7fffffff, "univariate: batch too large for one launch");
    out.rows_per_tile = (int)R;
    out.grid = (int)grid;
    const bool contiguous = (phi_ld == (int64_t)D * P);
    out.bulk = contiguous && (((uintptr_t)phi) % 16 == 0) && ((R * row_bytes) % 16 == 0);
    out.smem = (phi_ld == 0 ? row_bytes : R * row_bytes) + (size_t)R * D * 4;
    out.smem_attr = out.smem + 2048 > 48 * 1024;  // static smem (barrier) counts against the 48 KB default
    out.shuffle = D <= 32 && (D & (D - 1)) == 0;
    return ZK_OK;
}

zk_status launch_univariate(const UniArgs& a, cudaStream_t stream) {
    ZK_REQUIRE(a.B >= 0 && a.D > 0, "univariate: bad shape B=%lld D=%d", (long long)a.B, a.D);
    if (a.B == 0) return ZK_OK;
    ZK_REQUIRE(a.x && a.phi, "univariate: null input");
    UniPlan plan;
    ZK_TRY(uni_plan(a.spec, a.B, a.D, a.phi_ld, a.phi, plan));
    ZK_TRY(uni_check_scalars(a.spec, a.inverse));
    if (a.inverse) ZK_REQUIRE(a.y != nullptr, "univariate inverse: null output");
    if (a.accumulate) ZK_REQUIRE(a.ladj != nullptr, "univariate: accumulate needs ladj");

    UniParams p;
    p.x = a.x; p.ldx = a.ldx; p.phi = a.phi; p.phi_ld = a.phi_ld;
    p.y = a.y; p.ldy = a.ldy; p.ladj = a.ladj; p.accumulate = a.accumulate;
    p.log_prob = a.log_prob; p.base_loc = a.base_loc; p.base_scale = a.base_scale;
    p.dim_map = a.dim_map; p.B = a.B; p.D = a.D; p.K = a.spec.K; p.P = uni_P(a.spec);
    p.iters = a.spec.iters;
    p.rows_per_tile = plan.rows_per_tile;
    p.use_bulk = plan.bulk ? 1 : 0;
    return uni_dispatch<kStandalone>(a.spec.kind, plan.kt, a.fast_math, [&](auto fam, auto kt, auto fast) {
        using Fam = decltype(fam);
        set_uni_consts<Fam>(a.spec, p);
        auto kern = a.inverse ? uni_kernel<Fam::kKind, decltype(kt)::value, true, decltype(fast)::value>
                              : uni_kernel<Fam::kKind, decltype(kt)::value, false, decltype(fast)::value>;
        if (plan.smem_attr)
            ZK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem));
        kern<<<plan.grid, kUniThreads, plan.smem, stream>>>(p);
        return check_launch("uni_kernel");
    });
}

// ---------------------------------------------------------------------------
// small element-wise kernels
// ---------------------------------------------------------------------------
namespace {

// SoftclipTransform, transforms.py:309-316; one thread per sample row (D is small)
__global__ void softclip_kernel(const float* x, int64_t ldx, int64_t B, int D, float bound,
                                int inverse, float* y, int64_t ldy, float* ladj, int accumulate) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) {
        const float v = x[r * ldx + d];
        if (!inverse) {
            const float t = fabsf(v / bound);
            if (y) y[r * ldy + d] = v / (1.f + t);
            acc += -2.f * log1pf(t);
        } else {
            y[r * ldy + d] = v / (1.f - fabsf(v / bound));
        }
    }
    if (!inverse && ladj) ladj[r] = (accumulate ? ladj[r] : 0.f) + acc;
}

// PermutationTransform._call, transforms.py:1207-1208: bit-exact gather on the last dim
__global__ void permute_kernel(const float* x, int64_t ldx, const int64_t* order, int64_t B, int D,
                               float* y, int64_t ldy) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * D) return;
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    y[r * ldy + d] = x[r * ldx + order[d]];
}

// RotationTransform, transforms.py:1237-1241: y_i = sum_j R_ij x_j (or R_ji)
__global__ void rotate_kernel(const float* x, int64_t ldx, const float* R, int transpose, int64_t B,
                              int D, float* y, int64_t ldy) {
    extern __shared__ float sR[];
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) sR[i] = R[i];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * D) return;
    const int64_t r = i / D;
    const int o = (int)(i - r * D);
    float acc = 0.f;
    for (int j = 0; j < D; ++j)
        acc = fmaf(transpose ? sR[j * D + o] : sR[o * D + j], x[r * ldx + j], acc);
    y[r * ldy + o] = acc;
}

// CircularShiftTransform, transforms.py:344-348
__global__ void circular_shift_kernel(const float* x, int64_t ldx, int64_t B, int D, float bound, float* y, int64_t ldy) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * D) return;
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    y[r * ldy + d] = circ_shift(x[r * ldx + d], bound);
}

// BoxUniform.log_prob (+ ladj): Independent(Uniform(lower, upper), 1) — torch/distributions/uniform.py:
// log(lower <= z) + log(z < upper) - log(upper - lower), summed over the event dim
__global__ void box_uniform_kernel(const float* z, int64_t ldz, const float* lower, const float* upper,
                                   const float* ladj, int64_t B, int D, float* out) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    float acc = 0.f;
    bool inside = true;
    for (int d = 0; d < D; ++d) {
        const float v = z[r * ldz + d];
        inside = inside && (lower[d] <= v) && (v < upper[d]);
        acc -= logf(upper[d] - lower[d]);
    }
    out[r] = inside ? acc + (ladj ? ladj[r] : 0.f) : -CUDART_INF_F;
}

// DiagNormal.log_prob (+ ladj), one thread per sample row
__global__ void diag_normal_kernel(const float* z, int64_t ldz, const float* loc,
                                   const float* scale, const float* ladj, int64_t B, int D,
                                   float* out) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) {
        const float mu = loc ? loc[d] : 0.f;
        const float sg = scale ? scale[d] : 1.f;
        const float u = (z[r * ldz + d] - mu) / sg;
        acc += -0.5f * u * u - logf(sg) - kHalfLog2Pi;
    }
    out[r] = acc + (ladj ? ladj[r] : 0.f);
}

constexpr int kRedBlocks = 256;
constexpr int kRedThreads = 256;

// stage 1: block b sums a fixed contiguous slice in double (fixed order => deterministic)
__global__ void sum_stage1(const float* v, int64_t B, double* partial) {
    __shared__ double s[kRedThreads];
    const int64_t per = (B + kRedBlocks - 1) / kRedBlocks;
    const int64_t lo = (int64_t)blockIdx.x * per;
    const int64_t hi = min(B, lo + per);
    double acc = 0.0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += kRedThreads) acc += (double)v[i];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int o = kRedThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = s[0];
}
__global__ void sum_stage2(const double* partial, double* out) {
    __shared__ double s[kRedBlocks];
    s[threadIdx.x] = partial[threadIdx.x];
    __syncthreads();
    for (int o = kRedBlocks / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = s[0];
}

__global__ void copy_columns_kernel(const float* x, int64_t ldx, const int* cols, int n, int64_t B,
                                    float* y, int64_t ldy) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * n) return;
    const int64_t r = i / n;
    const int c = cols[(int)(i - r * n)];
    y[r * ldy + c] = x[r * ldx + c];
}

__global__ void fill_kernel(float* p, int64_t n, float v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

}  // namespace

zk_status launch_softclip(const float* x, int64_t ldx, int64_t B, int D, float bound, bool inverse,
                          float* y, int64_t ldy, float* ladj, int accumulate, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && x, "softclip: bad arguments");
    ZK_REQUIRE(bound > 0.f, "softclip: bound must be positive");
    if (inverse) ZK_REQUIRE(y != nullptr, "softclip inverse: null output");
    if (B == 0) return ZK_OK;
    softclip_kernel<<<(unsigned)ceil_div(B, 256), 256, 0, st>>>(x, ldx, B, D, bound, inverse ? 1 : 0,
                                                                y, ldy, ladj, accumulate);
    return check_launch("softclip_kernel");
}

zk_status launch_permute(const float* x, int64_t ldx, const int64_t* order, int64_t B, int D,
                         float* y, int64_t ldy, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && x && y && order, "permute: bad arguments");
    ZK_REQUIRE(x != y, "permute: x and y must not alias");
    if (B == 0) return ZK_OK;
    permute_kernel<<<(unsigned)ceil_div(B * D, 256), 256, 0, st>>>(x, ldx, order, B, D, y, ldy);
    return check_launch("permute_kernel");
}

zk_status launch_rotate(const float* x, int64_t ldx, const float* R, int transpose, int64_t B, int D,
                        float* y, int64_t ldy, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && x && y && R, "rotate: bad arguments");
    ZK_REQUIRE(x != y, "rotate: x and y must not alias");
    ZK_REQUIRE((size_t)D * D * 4 <= 48 * 1024, "rotate: D=%d too large (R must fit 48 KB)", D);
    if (B == 0) return ZK_OK;
    rotate_kernel<<<(unsigned)ceil_div(B * D, 256), 256, (size_t)D * D * 4, st>>>(x, ldx, R, transpose,
                                                                                 B, D, y, ldy);
    return check_launch("rotate_kernel");
}

zk_status launch_diag_normal(const float* z, int64_t ldz, const float* loc, const float* scale,
                             const float* ladj, int64_t B, int D, float* out, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && z && out, "diag_normal: bad arguments");
    ZK_REQUIRE((loc == nullptr) == (scale == nullptr), "diag_normal: loc/scale must both be set or null");
    if (B == 0) return ZK_OK;
    diag_normal_kernel<<<(unsigned)ceil_div(B, 256), 256, 0, st>>>(z, ldz, loc, scale, ladj, B, D, out);
    return check_launch("diag_normal_kernel");
}

zk_status launch_circular_shift(const float* x, int64_t ldx, int64_t B, int D, float bound, float* y,
                                int64_t ldy, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && x && y && bound > 0.f, "circular shift: bad arguments");
    if (B == 0) return ZK_OK;
    circular_shift_kernel<<<(unsigned)ceil_div(B * D, 256), 256, 0, st>>>(x, ldx, B, D, bound, y, ldy);
    return check_launch("circular_shift_kernel");
}

zk_status launch_box_uniform(const float* z, int64_t ldz, const float* lower, const float* upper,
                             const float* ladj, int64_t B, int D, float* out, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && z && out && lower && upper, "box_uniform: bad arguments");
    if (B == 0) return ZK_OK;
    box_uniform_kernel<<<(unsigned)ceil_div(B, 256), 256, 0, st>>>(z, ldz, lower, upper, ladj, B, D, out);
    return check_launch("box_uniform_kernel");
}

size_t reduce_scratch_bytes() { return kRedBlocks * sizeof(double); }

zk_status launch_sum_f32_to_f64(const float* v, int64_t B, double* out, void* scratch,
                                cudaStream_t st) {
    ZK_REQUIRE(v && out && scratch && B >= 0, "sum: bad arguments");
    sum_stage1<<<kRedBlocks, kRedThreads, 0, st>>>(v, B, (double*)scratch);
    ZK_TRY(check_launch("sum_stage1"));
    sum_stage2<<<1, kRedBlocks, 0, st>>>((const double*)scratch, out);
    return check_launch("sum_stage2");
}

zk_status launch_copy_columns(const float* x, int64_t ldx, const int* cols, int n, int64_t B,
                              float* y, int64_t ldy, cudaStream_t st) {
    if (B == 0 || n == 0) return ZK_OK;
    copy_columns_kernel<<<(unsigned)ceil_div(B * n, 256), 256, 0, st>>>(x, ldx, cols, n, B, y, ldy);
    return check_launch("copy_columns_kernel");
}

zk_status launch_fill(float* p, int64_t n, float v, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    fill_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(p, n, v);
    return check_launch("fill_kernel");
}

}  // namespace zk
