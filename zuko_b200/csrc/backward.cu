// zuko_b200 — backward-pass kernels of the flow hot path (interface + citations: backward.cuh).
//
// First correct version of SURVEY §8(f) rank 1: plain fp32 CUDA-core kernels with fixed-order
// (deterministic) reductions.  The three GEMM-shaped pieces — forward recompute, dgrad, wgrad —
// run on fp32 FMA here; moving them to tensor-core split-bf16 like the forward path is the next step.

#include <algorithm>

#include "activations.cuh"
#include "backward.cuh"
#include "uni_family.cuh"

namespace zk {

// outside the anonymous namespace: a family's Tables<UniBwdParams> derives from it
struct UniBwdParams {
    const float* x; int64_t ldx;
    const float* phi; int64_t phi_ld;
    const float* gy; int64_t ldgy;
    const float* gl;
    float* gx; int64_t ldgx;
    float* gphi;
    const int* dim_map;
    int64_t B; int D; int K; int P;
    float bound, aw, ad;
    int rows_per_tile;
    int circ;
};

namespace {

constexpr int kBwdThreads = 256;

// A family with device tables gets them in a parameter type of its own (UniFamily::Tables): appending the tables
// to UniBwdParams changes the register allocation of the instantiations that do not read them.
template <class Fam>
using BwdParams = typename Fam::template Tables<UniBwdParams>;

// thread = (sample row, dim) pair; the tile's parameter block is staged in shared memory, every
// pair rewrites its P slots with the parameter gradients, and the tile is written back with
// coalesced stores (per-sample gradients (B, D*P); a shared table is reduced by the caller).
// A shared table is rewritten in place too when the tile holds one row (uni_bwd_plan): pair d then
// reads and writes only slots d*P.., and every CTA stages its own copy of the table.
template <int UNI, int KT, bool FAST>
__global__ void __launch_bounds__(kBwdThreads) uni_bwd_kernel(const BwdParams<UniFamily<UNI>> a) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const int64_t r0 = (int64_t)blockIdx.x * a.rows_per_tile;
    const int nrows = (int)min((int64_t)a.rows_per_tile, a.B - r0);
    const int D = a.D, P = a.P;
    const int npairs = nrows * D;
    const bool shared_tbl = (a.phi_ld == 0);
    float* s_phi = smem;
    float* s_out = (shared_tbl && a.rows_per_tile > 1) ? smem + D * P : smem;
    const int n_phi = shared_tbl ? D * P : npairs * P;
    if (shared_tbl) {
        for (int i = tid; i < n_phi; i += kBwdThreads) s_phi[i] = a.phi[i];
    } else {
        for (int row = 0; row < nrows; ++row) {
            const float* src = a.phi + (r0 + row) * a.phi_ld;
            for (int i = tid; i < D * P; i += kBwdThreads) s_phi[row * D * P + i] = src[i];
        }
    }
    __syncthreads();
    for (int p = tid; p < npairs; p += kBwdThreads) {
        const int row = p / D;
        const int d = p - row * D;
        const int col = a.dim_map ? a.dim_map[d] : d;
        float xv = a.x[(r0 + row) * a.ldx + col];
        if (UniFamily<UNI>::kCircular && a.circ) xv = bij::circ_shift(xv, a.bound);
        const float gyv = a.gy ? a.gy[(r0 + row) * a.ldgy + col] : 0.f;
        const float glv = a.gl ? a.gl[r0 + row] : 0.f;
        const float* pp = s_phi + (shared_tbl ? d * P : p * P);
        float* out = s_out + p * P;
        float gxv;
        UniFamily<UNI>::template backward<KT, FAST>(pp, a, xv, gyv, glv, gxv, out);
        if (a.gx) a.gx[(r0 + row) * a.ldgx + col] = gxv;
    }
    __syncthreads();
    if (a.gphi) {
        float* dst = a.gphi + r0 * (int64_t)D * P;
        for (int i = tid; i < npairs * P; i += kBwdThreads) dst[i] = s_out[i];
    }
}

__global__ void softclip_bwd_kernel(const float* x, int64_t ldx, const float* gy, int64_t ldgy,
                                    const float* gl, int64_t B, int D, float bound, float* gx,
                                    int64_t ldgx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * D) return;
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    const float v = x[r * ldx + d];
    const float t1 = 1.f + fabsf(v / bound);
    const float g_y = gy ? gy[r * ldgy + d] : 0.f;
    const float g_l = gl ? gl[r] : 0.f;
    const float sgn = (v > 0.f) ? 1.f : (v < 0.f ? -1.f : 0.f);
    gx[r * ldgx + d] = g_y / (t1 * t1) - 2.f * g_l * sgn / (bound * t1);
}

__global__ void base_grad_kernel(const float* z, int64_t ldz, const float* loc, const float* scale,
                                 const float* g_lp, const float* gz_in, int64_t ldgz_in,
                                 const float* gl_in, int64_t B, int D, float* gz, float* gl) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * D) return;
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    float g = gz_in ? gz_in[r * ldgz_in + d] : 0.f;
    const float w = g_lp ? g_lp[r] : 0.f;
    if (g_lp) {
        const float mu = loc ? loc[d] : 0.f;
        const float sg = scale ? scale[d] : 1.f;
        g -= w * (z[r * ldz + d] - mu) / (sg * sg);
    }
    gz[r * D + d] = g;
    if (d == 0) gl[r] = (gl_in ? gl_in[r] : 0.f) + w;
}

__global__ void concat_kernel(const float* x, int64_t ldx, const int* cols, int nx, const float* c,
                              int64_t ldc, int nc, int64_t B, float* out) {
    const int W = nx + nc;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * W) return;
    const int64_t r = i / W;
    const int k = (int)(i - r * W);
    out[i] = (k < nx) ? x[r * ldx + (cols ? cols[k] : k)] : c[r * ldc + (k - nx)];
}

__global__ void input_grad_kernel(const float* gin, int nx, int nc, const int* cols, int64_t B,
                                  float* gx, int64_t ldgx, const float* base, int64_t ldbase,
                                  float* gc, int64_t ldgc) {
    const int W = nx + nc;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * W) return;
    const int64_t r = i / W;
    const int k = (int)(i - r * W);
    const float v = gin[i];
    if (k < nx) {
        if (gx) {
            const int col = cols ? cols[k] : k;
            float* dst = gx + r * ldgx + col;
            *dst = (base ? base[r * ldbase + col] : *dst) + v;
        }
    } else if (gc) {
        gc[r * ldgc + (k - nx)] += v;
    }
}

__global__ void relu_gate_kernel(float* g, const float* a, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && !(a[i] > 0.f)) g[i] = 0.f;
}

__global__ void act_apply_kernel(const float* pre, float* y, int64_t n, int act) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = act_apply(pre[i], act);
}
__global__ void act_gate_kernel(float* g, const float* pre, int64_t n, int act) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) g[i] *= act_deriv(pre[i], act);
}

__global__ void scale_kernel(float* out, const float* in, float alpha, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = alpha * in[i];
}
__global__ void div_kernel(float* out, const float* g, const float* s, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = g[i] / s[i];
}
__global__ void richardson_kernel(float* v, const float* g, const float* jtv, const float* s, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] += (g[i] - jtv[i]) / s[i];
}

__global__ void add_kernel(float* y, const float* x, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] += x[i];
}

// ---- column sums: stage 1 = 32 columns x 8 row lanes per block over one row slice ----
constexpr int kColSlices = 64;
__global__ void colsum_stage1(const float* v, int64_t ldv, int64_t B, int N, int64_t rows_per_slice,
                              float* partial) {
    __shared__ float s[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int col = blockIdx.x * 32 + tx;
    const int64_t lo = (int64_t)blockIdx.y * rows_per_slice;
    const int64_t hi = min(B, lo + rows_per_slice);
    float acc = 0.f;
    if (col < N)
        for (int64_t r = lo + ty; r < hi; r += 8) acc += v[r * ldv + col];
    s[ty][tx] = acc;
    __syncthreads();
    if (ty == 0 && col < N) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += s[k][tx];
        partial[(int64_t)blockIdx.y * N + col] = t;
    }
}
__global__ void colsum_stage2(const float* partial, int S, int N, float* out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float t = 0.f;
    for (int z = 0; z < S; ++z) t += partial[(int64_t)z * N + n];
    out[n] += t;
}

// ---- wgrad: partial[z][n][k] = sum_{rows of slice z} g[r, n] * a[r, k] ----
constexpr int WO = 64, WI = 64, WR = 16;
__global__ void __launch_bounds__(256)
wgrad_fp32_kernel(const float* __restrict__ g, int64_t ldg, const float* __restrict__ a, int64_t lda,
                  int64_t B, int N, int K, int64_t rows_per_slice, float* __restrict__ partial) {
    __shared__ __align__(16) float sG[WR][WO];
    __shared__ __align__(16) float sA[WR][WI];
    const int tid = threadIdx.x;
    const int ty = tid / 16, tx = tid % 16;  // 4x4 micro tile: rows ty*4.. of N, cols tx*4.. of K
    const int n0 = blockIdx.x * WO, k0 = blockIdx.y * WI;
    const int64_t rbeg = (int64_t)blockIdx.z * rows_per_slice;
    const int64_t rend = min(B, rbeg + rows_per_slice);
    const int lr = tid / 16, lc = (tid % 16) * 4;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int64_t r = rbeg; r < rend; r += WR) {
        const int64_t row = r + lr;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int cn = n0 + lc + q, ck = k0 + lc + q;
            sG[lr][lc + q] = (row < rend && cn < N) ? g[row * ldg + cn] : 0.f;
            sA[lr][lc + q] = (row < rend && ck < K) ? a[row * lda + ck] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < WR; ++k) {
            const float4 g4 = *reinterpret_cast<const float4*>(&sG[k][ty * 4]);
            const float4 a4 = *reinterpret_cast<const float4*>(&sA[k][tx * 4]);
            const float gv[4] = {g4.x, g4.y, g4.z, g4.w};
            const float av[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(gv[i], av[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* dst = partial + (int64_t)blockIdx.z * N * K;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + ty * 4 + i;
        if (n >= N) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + tx * 4 + j;
            if (k < K) dst[(int64_t)n * K + k] = acc[i][j];
        }
    }
}
__global__ void wgrad_reduce_kernel(const float* partial, int S, int64_t NK, const uint8_t* mask,
                                    float* gw) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NK) return;
    if (mask && !mask[i]) return;  // d(mask * W)/dW = mask (nn.py:218)
    float t = 0.f;
    for (int z = 0; z < S; ++z) t += partial[(int64_t)z * NK + i];
    gw[i] += t;
}

__global__ void transpose_kernel(const float* in, int N, int K, float* out) {
    __shared__ float tile[32][33];
    const int n0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int n = n0 + j, k = k0 + threadIdx.x;
        tile[j][threadIdx.x] = (n < N && k < K) ? in[(int64_t)n * K + k] : 0.f;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int k = k0 + j, n = n0 + threadIdx.x;
        if (k < K && n < N) out[(int64_t)k * N + n] = tile[threadIdx.x][j];
    }
}

int wgrad_slices_max(int N, int K) {
    const int64_t tiles = ceil_div(N, WO) * ceil_div(K, WI);
    int64_t S = ceil_div(8 * sm_count(), tiles);
    if (S > 64) S = 64;
    if (S < 1) S = 1;
    while (S > 1 && S * (int64_t)N * K * 4 > ((int64_t)256 << 20)) S /= 2;
    return (int)S;
}

}  // namespace

zk_status uni_bwd_plan(const UniSpec& s, int64_t B, int D, int64_t phi_ld, UniBwdPlan& out) {
    ZK_REQUIRE(B >= 0 && D > 0, "univariate backward: bad shape B=%lld D=%d", (long long)B, D);
    out = UniBwdPlan{};
    if (B == 0) return ZK_OK;
    ZK_TRY(uni_check_shape(s));
    out.kt = uni_kt<kBackward>(s);
    const int P = uni_P(s);
    ZK_REQUIRE(phi_ld == 0 || phi_ld >= (int64_t)D * P, "univariate backward: phi_ld too small");

    // tile = R rows: aim at >= 256 pairs and ~24 KB of phi per CTA, at most 96 KB with a shared table staged
    // beside the rows; one row up to 200 KB (a shared table is then rewritten in place)
    const size_t row_bytes = (size_t)D * P * 4;
    const size_t table = (phi_ld == 0) ? row_bytes : 0;
    ZK_REQUIRE(row_bytes <= 200 * 1024, "univariate backward: D*P too large for one tile (%zu B)", row_bytes);
    int64_t R = (int64_t)(24 * 1024 / row_bytes);
    const int64_t r_pairs = ceil_div(kBwdThreads, D);
    if (R < r_pairs) R = r_pairs;
    while (R > 1 && R * row_bytes + table > 96 * 1024) --R;
    if (R < 1) R = 1;
    if (R > B) R = B;
    const int64_t grid = ceil_div(B, R);
    ZK_REQUIRE(grid <= 0x7fffffff, "univariate backward: batch too large for one launch");
    out.rows_per_tile = (int)R;
    out.grid = (int)grid;
    out.table_in_place = (phi_ld == 0 && R == 1);
    out.smem = (size_t)R * row_bytes + (out.table_in_place ? 0 : table);
    out.smem_attr = out.smem > 40 * 1024;
    return ZK_OK;
}

zk_status launch_univariate_backward(const UniBwdArgs& a, cudaStream_t stream) {
    ZK_REQUIRE(a.B >= 0 && a.D > 0, "univariate backward: bad shape B=%lld D=%d", (long long)a.B, a.D);
    if (a.B == 0) return ZK_OK;
    ZK_REQUIRE(a.x && a.phi, "univariate backward: null input");
    UniBwdPlan plan;
    ZK_TRY(uni_bwd_plan(a.spec, a.B, a.D, a.phi_ld, plan));
    ZK_TRY(uni_check_scalars(a.spec, false));
    ZK_REQUIRE(!(a.phi_ld == 0 && a.gphi == a.phi), "univariate backward: gphi cannot alias a shared table");
    return uni_dispatch<kBackward>(a.spec.kind, plan.kt, a.fast_math, [&](auto fam, auto kt, auto fast) {
        using Fam = decltype(fam);
        BwdParams<Fam> p;
        p.x = a.x; p.ldx = a.ldx; p.phi = a.phi; p.phi_ld = a.phi_ld; p.gy = a.gy; p.ldgy = a.ldgy;
        p.gl = a.gl; p.gx = a.gx; p.ldgx = a.ldgx; p.gphi = a.gphi; p.dim_map = a.dim_map; p.B = a.B;
        p.D = a.D; p.K = a.spec.K; p.P = uni_P(a.spec);
        p.rows_per_tile = plan.rows_per_tile;
        set_uni_consts<Fam>(a.spec, p);
        auto kern = uni_bwd_kernel<Fam::kKind, decltype(kt)::value, decltype(fast)::value>;
        if (plan.smem_attr)
            ZK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem));
        kern<<<plan.grid, kBwdThreads, plan.smem, stream>>>(p);
        return check_launch("uni_bwd_kernel");
    });
}

zk_status launch_softclip_backward(const float* x, int64_t ldx, const float* gy, int64_t ldgy,
                                   const float* gl, int64_t B, int D, float bound, float* gx,
                                   int64_t ldgx, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && x && gx && bound > 0.f, "softclip backward: bad arguments");
    if (B == 0) return ZK_OK;
    softclip_bwd_kernel<<<(unsigned)ceil_div(B * D, 256), 256, 0, st>>>(x, ldx, gy, ldgy, gl, B, D, bound, gx, ldgx);
    return check_launch("softclip_bwd_kernel");
}

zk_status launch_base_grad(const float* z, int64_t ldz, const float* loc, const float* scale,
                           const float* g_lp, const float* gz_in, int64_t ldgz_in,
                           const float* gl_in, int64_t B, int D, float* gz, float* gl,
                           cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && gz && gl && (z || !g_lp), "base grad: bad arguments");
    if (B == 0) return ZK_OK;
    base_grad_kernel<<<(unsigned)ceil_div(B * D, 256), 256, 0, st>>>(z, ldz, loc, scale, g_lp, gz_in, ldgz_in, gl_in, B, D, gz, gl);
    return check_launch("base_grad_kernel");
}

zk_status launch_base_grad_flat(const float* g_lp, const float* gz_in, int64_t ldgz_in, const float* gl_in,
                                int64_t B, int D, float* gz, float* gl, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && D > 0 && gz && gl, "base grad: bad arguments");
    if (B == 0) return ZK_OK;
    base_grad_kernel<<<(unsigned)ceil_div(B * D, 256), 256, 0, st>>>(nullptr, 0, nullptr, nullptr, nullptr, gz_in, ldgz_in, gl_in, B, D, gz, gl);
    ZK_TRY(check_launch("base_grad_kernel"));
    if (g_lp) return launch_add(gl, g_lp, B, st);
    return ZK_OK;
}

zk_status launch_concat(const float* x, int64_t ldx, const int* cols, int nx, const float* c,
                        int64_t ldc, int nc, int64_t B, float* out, cudaStream_t st) {
    ZK_REQUIRE(B >= 0 && nx >= 0 && nc >= 0 && nx + nc > 0 && out, "concat: bad arguments");
    ZK_REQUIRE((nx == 0 || x) && (nc == 0 || c), "concat: null source");
    if (B == 0) return ZK_OK;
    concat_kernel<<<(unsigned)ceil_div(B * (nx + nc), 256), 256, 0, st>>>(x, ldx, cols, nx, c, ldc, nc, B, out);
    return check_launch("concat_kernel");
}

zk_status launch_input_grad(const float* gin, int nx, int nc, const int* cols, int64_t B, float* gx,
                            int64_t ldgx, const float* base, int64_t ldbase, float* gc,
                            int64_t ldgc, cudaStream_t st) {
    ZK_REQUIRE(gin && nx + nc > 0, "input grad: bad arguments");
    if (B == 0) return ZK_OK;
    input_grad_kernel<<<(unsigned)ceil_div(B * (nx + nc), 256), 256, 0, st>>>(gin, nx, nc, cols, B, gx, ldgx, base, ldbase, gc, ldgc);
    return check_launch("input_grad_kernel");
}

zk_status launch_relu_gate(float* g, const float* a, int64_t n, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    relu_gate_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(g, a, n);
    return check_launch("relu_gate_kernel");
}

zk_status launch_act_apply(const float* pre, float* y, int64_t n, int act, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    act_apply_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(pre, y, n, act);
    return check_launch("act_apply_kernel");
}
zk_status launch_act_gate(float* g, const float* pre, int64_t n, int act, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    act_gate_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(g, pre, n, act);
    return check_launch("act_gate_kernel");
}

zk_status launch_scale(float* out, const float* in, float alpha, int64_t n, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    scale_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(out, in, alpha, n);
    return check_launch("scale_kernel");
}
zk_status launch_div(float* out, const float* g, const float* s, int64_t n, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    div_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(out, g, s, n);
    return check_launch("div_kernel");
}
zk_status launch_richardson(float* v, const float* g, const float* jtv, const float* s, int64_t n, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    richardson_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(v, g, jtv, s, n);
    return check_launch("richardson_kernel");
}

zk_status launch_add(float* y, const float* x, int64_t n, cudaStream_t st) {
    if (n == 0) return ZK_OK;
    add_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(y, x, n);
    return check_launch("add_kernel");
}

size_t colsum_scratch_bytes(int N) { return (size_t)kColSlices * N * 4; }

zk_status launch_colsum_add(const float* v, int64_t ldv, int64_t B, int N, float* out, void* scratch,
                            cudaStream_t st) {
    ZK_REQUIRE(v && out && scratch && N > 0 && B >= 0, "colsum: bad arguments");
    if (B == 0) return ZK_OK;
    int64_t S = std::min<int64_t>(kColSlices, ceil_div(B, 256));
    const int64_t rows = ceil_div(B, S);
    S = ceil_div(B, rows);
    dim3 grid((unsigned)ceil_div(N, 32), (unsigned)S);
    colsum_stage1<<<grid, 256, 0, st>>>(v, ldv, B, N, rows, (float*)scratch);
    ZK_TRY(check_launch("colsum_stage1"));
    colsum_stage2<<<(unsigned)ceil_div(N, 256), 256, 0, st>>>((const float*)scratch, (int)S, N, out);
    return check_launch("colsum_stage2");
}

size_t wgrad_scratch_bytes(int N, int K) { return (size_t)wgrad_slices_max(N, K) * N * K * 4; }

zk_status launch_wgrad_fp32(const float* g, int64_t ldg, const float* a, int64_t lda, int64_t B,
                            int N, int K, const uint8_t* mask, float* gw, void* scratch,
                            cudaStream_t st) {
    ZK_REQUIRE(g && a && gw && scratch && N > 0 && K > 0 && B >= 0, "wgrad: bad arguments");
    if (B == 0) return ZK_OK;
    int64_t S = std::min<int64_t>(wgrad_slices_max(N, K), ceil_div(B, 64));
    int64_t rows = ceil_div(B, S);
    rows = ceil_div(rows, WR) * WR;
    S = ceil_div(B, rows);
    dim3 grid((unsigned)ceil_div(N, WO), (unsigned)ceil_div(K, WI), (unsigned)S);
    wgrad_fp32_kernel<<<grid, 256, 0, st>>>(g, ldg, a, lda, B, N, K, rows, (float*)scratch);
    ZK_TRY(check_launch("wgrad_fp32_kernel"));
    const int64_t NK = (int64_t)N * K;
    wgrad_reduce_kernel<<<(unsigned)ceil_div(NK, 256), 256, 0, st>>>((const float*)scratch, (int)S, NK, mask, gw);
    return check_launch("wgrad_reduce_kernel");
}

zk_status launch_transpose(const float* in, int N, int K, float* out, cudaStream_t st) {
    ZK_REQUIRE(in && out && N > 0 && K > 0, "transpose: bad arguments");
    dim3 grid((unsigned)ceil_div(K, 32), (unsigned)ceil_div(N, 32));
    transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(in, N, K, out);
    return check_launch("transpose_kernel");
}

}  // namespace zk
