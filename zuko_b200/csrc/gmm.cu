// zuko_b200 — Gaussian mixture model (zuko/mixtures.py:25-99, Mixture: zuko/distributions.py:216-290):
// log-density, backward and sampling kernels and their C ABI (include/zuko_b200.h).
//
// Each kernel runs one thread per row and loops over the components; the per-row math is gmm_math.cuh.
// A thread keeps its row's vectors v, w (D each) and t (K) in shared memory, one column per thread
// ([i][thread] layout: conflict-free), and reads its parameter row from global memory.  The three
// families are templated on the covariance type and on `tied`.
//
// The conditioner runs on the existing MLP paths: zk_mlp_forward for log_prob / sample, and the saved-
// activation backward of api_backward.cu (tensor cores when the handle is packed for them) for the
// gradients.  Its output rows are phi; the backward kernel writes one gradient row per sample into a
// separate buffer that then seeds the conditioner's backward.  A broadcast context (ldc == 0) or the
// unconditional table is one phi row read by every sample (ld 0); its gradient is the fixed-order column
// sum of the per-sample rows.

#include "api_internal.cuh"
#include "backward.cuh"
#include "gmm_math.cuh"

using namespace zk;
using namespace zkapi;
using zk::gmm::Layout;

struct zk_gmm {
    int D = 0, C = 0, K = 0, cov = 0, tied = 0;
    float eps = 1e-6f;
    Layout lay;
    zk_mlp* hyper = nullptr;  // owned; nullptr when C == 0
};

namespace {

constexpr size_t kSmemCap = 48 * 1024;  // default dynamic shared memory limit: no opt-in needed

struct GmmArgs {
    Layout l;
    float eps;
    int64_t B;
    const float* x; int64_t ldx;
    const float* phi; int64_t ldphi;  // ldphi = 0: one row shared by every sample
    float* out;                       // log_prob (B)
    const float* glp; float* gx; int64_t ldgx; float* gphi;  // backward: gphi (B, l.total)
    const float* u; const float* z; int64_t ldz;              // sample; x is then the output
    float* xs; int64_t ldxs;
};

bool shape_ok(int D, int K) { return D >= 1 && D <= gmm::kMaxD && K >= 1 && K <= gmm::kMaxK; }

int plan_threads(int D, int K) {
    int T = 128;
    while (T > 32 && (size_t)T * (2 * D + K) * 4 > kSmemCap) T /= 2;
    return T;
}

template <int COV, int TIED>
__device__ __forceinline__ Layout fixed_layout(const Layout& in) {
    Layout l = in;
    l.cov = COV;
    l.tied = TIED;
    return l;
}

template <int COV, int TIED>
__global__ void __launch_bounds__(128) gmm_log_prob_kernel(GmmArgs a) {
    extern __shared__ float sm[];
    const int T = blockDim.x;
    const int64_t row = (int64_t)blockIdx.x * T + threadIdx.x;
    if (row >= a.B) return;
    const Layout l = fixed_layout<COV, TIED>(a.l);
    float* v = sm + threadIdx.x;
    float* t = sm + (size_t)l.D * T + threadIdx.x;
    a.out[row] = gmm::row_log_prob(a.x + row * a.ldx, a.phi + row * a.ldphi, l, a.eps, v, T, t, T);
}

template <int COV, int TIED>
__global__ void __launch_bounds__(128) gmm_backward_kernel(GmmArgs a) {
    extern __shared__ float sm[];
    const int T = blockDim.x;
    const int64_t row = (int64_t)blockIdx.x * T + threadIdx.x;
    if (row >= a.B) return;
    const Layout l = fixed_layout<COV, TIED>(a.l);
    float* v = sm + threadIdx.x;
    float* w = sm + (size_t)l.D * T + threadIdx.x;
    float* t = sm + (size_t)2 * l.D * T + threadIdx.x;
    gmm::row_backward(a.x + row * a.ldx, a.phi + row * a.ldphi, l, a.eps, a.glp[row],
                      a.gx ? a.gx + row * a.ldgx : nullptr, a.gphi + row * l.total, v, T, w, T, t, T);
}

template <int COV, int TIED>
__global__ void __launch_bounds__(128) gmm_sample_kernel(GmmArgs a) {
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= a.B) return;
    const Layout l = fixed_layout<COV, TIED>(a.l);
    gmm::row_sample(a.phi + row * a.ldphi, l, a.eps, a.u[row], a.z + row * a.ldz, a.xs + row * a.ldxs);
}

enum Family { kGmmLogProb, kGmmBackward, kGmmSample };

template <int COV, int TIED>
zk_status launch_one(Family f, const GmmArgs& a, cudaStream_t st) {
    const int T = plan_threads(a.l.D, a.l.K);
    const unsigned grid = (unsigned)ceil_div(a.B, T);
    switch (f) {
        case kGmmLogProb:
            gmm_log_prob_kernel<COV, TIED><<<grid, T, (size_t)T * (a.l.D + a.l.K) * 4, st>>>(a);
            return check_launch("gmm_log_prob_kernel");
        case kGmmBackward:
            gmm_backward_kernel<COV, TIED><<<grid, T, (size_t)T * (2 * a.l.D + a.l.K) * 4, st>>>(a);
            return check_launch("gmm_backward_kernel");
        default:
            gmm_sample_kernel<COV, TIED><<<grid, T, 0, st>>>(a);
            return check_launch("gmm_sample_kernel");
    }
}

zk_status launch_gmm(Family f, const GmmArgs& a, cudaStream_t st) {
    if (a.B == 0) return ZK_OK;
    switch (a.l.cov * 2 + a.l.tied) {
        case 0: return launch_one<gmm::kFull, 0>(f, a, st);
        case 1: return launch_one<gmm::kFull, 1>(f, a, st);
        case 2: return launch_one<gmm::kDiagonal, 0>(f, a, st);
        case 3: return launch_one<gmm::kDiagonal, 1>(f, a, st);
        case 4: return launch_one<gmm::kSpherical, 0>(f, a, st);
        default: return launch_one<gmm::kSpherical, 1>(f, a, st);
    }
}

GmmArgs base_args(const zk_gmm* g) {
    GmmArgs a{};
    a.l = g->lay;
    a.eps = g->eps;
    return a;
}

size_t row_bytes(const zk_gmm* g, int64_t n) { return a256((size_t)n * g->lay.total * 4); }

// workspace of one call over n rows: `bcast` = one phi row for every sample (broadcast context or the
// unconditional table), whose chunks share the fixed part
size_t ws_for(const zk_gmm* g, int64_t n, bool bwd, bool bcast) {
    const zk_mlp* m = g->hyper;
    const size_t colsum = a256(colsum_scratch_bytes(g->lay.total));
    if (!m) return bwd ? row_bytes(g, n) + colsum : 0;
    if (bcast)
        return bwd ? ConditionerBackward::bytes(m, 1, false) + row_bytes(g, 1) + colsum + row_bytes(g, n)
                   : a256(zk_mlp_workspace_bytes(m, 1)) + row_bytes(g, 1);
    if (!bwd) return a256(zk_mlp_workspace_bytes(m, n)) + row_bytes(g, n);
    return ConditionerBackward::bytes(m, n, true) + row_bytes(g, n);
}

// chunks are not rounded to aligned row counts: that would reorder the sums of the weight gradients
int64_t chunk_rows(const zk_gmm* g, int64_t B, bool bwd, bool bcast, size_t bytes) {
    return largest_fitting_rows(B, bytes, [&](int64_t n) { return ws_for(g, n, bwd, bcast); }, 1);
}

zk_status check_call(const zk_gmm* g, const float* c, const float* phi, int64_t B, const char* what) {
    ZK_REQUIRE(g, "%s: null handle", what);
    ZK_REQUIRE(B >= 0, "%s: negative batch", what);
    if (g->C > 0) ZK_REQUIRE(c != nullptr && phi == nullptr, "%s: a conditional GMM takes c and no phi table", what);
    else ZK_REQUIRE(phi != nullptr, "%s: an unconditional GMM takes its phi table", what);
    return ZK_OK;
}

// the conditioner's output rows phi (n, params per row) for n context rows
zk_status conditioner_rows(const zk_gmm* g, const float* c, int64_t ldc, int64_t n, float* rows, void* ws,
                           size_t ws_bytes, cudaStream_t st) {
    return zk_mlp_forward(g->hyper, c, ldc, g->C, nullptr, 0, 0, n, rows, g->lay.total, ws, ws_bytes, st);
}

// shared forward plumbing of log_prob and sample: `run(phi, ldphi, r0, n)` per chunk
template <class Run>
zk_status forward_chunks(const zk_gmm* g, const float* c, int64_t ldc, const float* phi, int64_t B, void* ws,
                         size_t ws_bytes, cudaStream_t st, const char* what, Run run) {
    if (B == 0) return ZK_OK;
    if (!g->hyper) return run(phi, 0, 0, B);
    const bool bcast = (ldc == 0);
    const int64_t rows = chunk_rows(g, B, false, bcast, ws_bytes);
    ZK_REQUIRE(rows > 0, "%s: workspace too small (%zu < %zu)", what, ws_bytes, ws_for(g, 1, false, bcast));
    Arena ar(ws, ws_bytes);
    if (bcast) {
        float* row = ar.take<float>(g->lay.total);
        const size_t mb = a256(zk_mlp_workspace_bytes(g->hyper, 1));
        void* mws = mb ? ar.take<char>(mb) : nullptr;
        ZK_TRY(conditioner_rows(g, c, 0, 1, row, mws, mb, st));
        return run(row, 0, 0, B);
    }
    float* buf = ar.take<float>((size_t)rows * g->lay.total);
    const size_t mb = a256(zk_mlp_workspace_bytes(g->hyper, rows));
    void* mws = mb ? ar.take<char>(mb) : nullptr;
    for (int64_t r0 = 0; r0 < B; r0 += rows) {
        const int64_t n = std::min(rows, B - r0);
        ZK_TRY(conditioner_rows(g, c + r0 * ldc, ldc, n, buf, mws, mb, st));
        ZK_TRY(run(buf, g->lay.total, r0, n));
    }
    return ZK_OK;
}

// per-row context: conditioner recompute with saved activations, mixture backward, conditioner backward
zk_status backward_rows(const zk_gmm* g, const float* x, int64_t ldx, const float* c, int64_t ldc, int64_t n,
                        const float* glp, float* gx, int64_t ldgx, float* gc, int64_t ldgc,
                        const zk_layer_grads* grads, void* ws, size_t ws_bytes, cudaStream_t st) {
    Arena ar(ws, ws_bytes);
    ConditionerBackward cb;
    ZK_TRY(cb.recompute(g->hyper, true, nullptr, 0, nullptr, 0, c, ldc, g->C, n, ar, "gmm_backward", st));
    GmmArgs a = base_args(g);
    a.B = n; a.x = x; a.ldx = ldx; a.phi = cb.phi; a.ldphi = g->lay.total; a.glp = glp; a.gx = gx; a.ldgx = ldgx;
    a.gphi = ar.take<float>((size_t)n * g->lay.total);
    ZK_REQUIRE(ar.ok, "gmm_backward: workspace too small");
    ZK_TRY(launch_gmm(kGmmBackward, a, st));
    ZK_TRY(cb.backward(a.gphi, gc != nullptr, grads, st));
    if (gc) ZK_TRY(launch_input_grad(cb.gin, 0, g->C, nullptr, n, nullptr, 0, nullptr, 0, gc, ldgc, st));
    return ZK_OK;
}

}  // namespace

extern "C" {

int64_t zk_gmm_params_per_row(int features, int components, int covariance, int tied) {
    if (features < 1 || components < 1 || covariance < ZK_COV_FULL || covariance > ZK_COV_SPHERICAL) return 0;
    return gmm::make_layout(features, components, covariance, tied ? 1 : 0).total;
}

zk_status zk_gmm_plan(int features, int components, int covariance, int tied, int* threads, int* rows_per_cta,
                      size_t* smem_log_prob, size_t* smem_backward, int* instantiated) {
    ZK_REQUIRE(covariance >= ZK_COV_FULL && covariance <= ZK_COV_SPHERICAL, "gmm_plan: unknown covariance %d", covariance);
    if (!shape_ok(features, components))
        return fail(ZK_EUNSUPPORTED, "gmm: features %d, components %d outside the covered 1..%d, 1..%d", features,
                    components, gmm::kMaxD, gmm::kMaxK);
    const int T = plan_threads(features, components);
    if (threads) *threads = T;
    if (rows_per_cta) *rows_per_cta = T;
    if (smem_log_prob) *smem_log_prob = (size_t)T * (features + components) * 4;
    if (smem_backward) *smem_backward = (size_t)T * (2 * features + components) * 4;
    if (instantiated) *instantiated = covariance * 2 + (tied ? 1 : 0);
    return ZK_OK;
}

zk_status zk_gmm_destroy(zk_gmm* g) {
    if (!g) return ZK_OK;
    zk_mlp_destroy(g->hyper);
    delete g;
    return ZK_OK;
}

zk_status zk_gmm_create(const zk_gmm_desc* d, zk_gmm** out) {
    ZK_REQUIRE(d && out, "gmm_create: null argument");
    *out = nullptr;
    ZK_TRY(zk_gmm_plan(d->features, d->components, d->covariance, d->tied, nullptr, nullptr, nullptr, nullptr, nullptr));
    ZK_REQUIRE(d->context >= 0, "gmm_create: negative context");
    ZK_REQUIRE((d->context > 0) == (d->hyper != nullptr), "gmm_create: a conditioner iff context > 0");
    zk_gmm* g = new zk_gmm;
    g->D = d->features; g->C = d->context; g->K = d->components; g->cov = d->covariance; g->tied = d->tied ? 1 : 0;
    g->eps = d->epsilon;
    g->lay = gmm::make_layout(g->D, g->K, g->cov, g->tied);
    if (d->hyper) {
        zk_status s = zk_mlp_create(d->hyper, &g->hyper);
        if (s == ZK_OK && (g->hyper->dims[0] != g->C || g->hyper->dims[g->hyper->n_linear] != g->lay.total))
            s = fail(ZK_EINVAL, "gmm_create: conditioner (%d -> %d) != (context %d -> %d parameters)", g->hyper->dims[0],
                     g->hyper->dims[g->hyper->n_linear], g->C, g->lay.total);
        if (s != ZK_OK) {
            const std::string keep = g_last_error;
            zk_gmm_destroy(g);
            g_last_error = keep;
            return s;
        }
    }
    *out = g;
    return ZK_OK;
}

zk_status zk_gmm_update_weights(zk_gmm* g, const float* const* weight, const float* const* bias, zk_stream stream) {
    ZK_REQUIRE(g && weight, "gmm_update_weights: null argument");
    ZK_REQUIRE(g->hyper, "gmm_update_weights: the model has no conditioner");
    return mlp_update_weights(g->hyper, weight, bias, (cudaStream_t)stream);
}

size_t zk_gmm_workspace_bytes(const zk_gmm* g, int64_t B) {
    if (!g || B <= 0) return 0;
    return std::max(ws_for(g, B, false, false), ws_for(g, B, false, true));
}

size_t zk_gmm_backward_workspace_bytes(const zk_gmm* g, int64_t B) {
    if (!g || B <= 0) return 0;
    return std::max(ws_for(g, B, true, false), ws_for(g, B, true, true));
}

size_t zk_gmm_min_workspace_bytes(const zk_gmm* g) {
    return std::max(zk_gmm_workspace_bytes(g, 1), zk_gmm_backward_workspace_bytes(g, 1));
}

int64_t zk_gmm_chunk_rows(const zk_gmm* g, int64_t B, int backward, size_t ws_bytes) {
    if (!g) return 0;
    return std::min(chunk_rows(g, B, backward != 0, false, ws_bytes), chunk_rows(g, B, backward != 0, true, ws_bytes));
}

zk_status zk_gmm_log_prob(const zk_gmm* g, const float* x, int64_t ldx, const float* c, int64_t ldc, const float* phi,
                          int64_t B, float* log_prob, void* ws, size_t ws_bytes, zk_stream stream) {
    ZK_TRY(check_call(g, c, phi, B, "gmm_log_prob"));
    ZK_REQUIRE(B == 0 || (x && log_prob), "gmm_log_prob: null x / log_prob");
    cudaStream_t st = (cudaStream_t)stream;
    return forward_chunks(g, c, ldc, phi, B, ws, ws_bytes, st, "gmm_log_prob",
                          [&](const float* p, int64_t ldp, int64_t r0, int64_t n) {
                              GmmArgs a = base_args(g);
                              a.B = n; a.x = x + r0 * ldx; a.ldx = ldx; a.phi = p; a.ldphi = ldp; a.out = log_prob + r0;
                              return launch_gmm(kGmmLogProb, a, st);
                          });
}

zk_status zk_gmm_sample(const zk_gmm* g, const float* c, int64_t ldc, const float* phi, const float* u, const float* z,
                        int64_t ldz, int64_t B, float* x, int64_t ldx, void* ws, size_t ws_bytes, zk_stream stream) {
    ZK_TRY(check_call(g, c, phi, B, "gmm_sample"));
    ZK_REQUIRE(B == 0 || (u && z && x), "gmm_sample: null u / z / x");
    cudaStream_t st = (cudaStream_t)stream;
    return forward_chunks(g, c, ldc, phi, B, ws, ws_bytes, st, "gmm_sample",
                          [&](const float* p, int64_t ldp, int64_t r0, int64_t n) {
                              GmmArgs a = base_args(g);
                              a.B = n; a.phi = p; a.ldphi = ldp; a.u = u + r0; a.z = z + r0 * ldz; a.ldz = ldz;
                              a.xs = x + r0 * ldx; a.ldxs = ldx;
                              return launch_gmm(kGmmSample, a, st);
                          });
}

zk_status zk_gmm_backward(const zk_gmm* g, const float* x, int64_t ldx, const float* c, int64_t ldc, const float* phi,
                          int64_t B, const float* glp, float* gx, int64_t ldgx, float* gc, int64_t ldgc,
                          const zk_layer_grads* grads, void* ws, size_t ws_bytes, zk_stream stream) {
    ZK_TRY(check_call(g, c, phi, B, "gmm_backward"));
    if (B == 0) return ZK_OK;
    ZK_REQUIRE(x && glp, "gmm_backward: null x / grad_log_prob");
    cudaStream_t st = (cudaStream_t)stream;
    const int P = g->lay.total;
    const bool bcast = (g->hyper == nullptr || ldc == 0);
    const int64_t rows = chunk_rows(g, B, true, bcast, ws_bytes);
    ZK_REQUIRE(rows > 0, "gmm_backward: workspace too small (%zu < %zu)", ws_bytes, ws_for(g, 1, true, bcast));
    if (!bcast) {
        for (int64_t r0 = 0; r0 < B; r0 += rows) {
            const int64_t n = std::min(rows, B - r0);
            ZK_TRY(backward_rows(g, x + r0 * ldx, ldx, c + r0 * ldc, ldc, n, glp + r0, gx ? gx + r0 * ldgx : nullptr,
                                 ldgx, gc ? gc + r0 * ldgc : nullptr, ldgc, grads, ws, ws_bytes, st));
        }
        return ZK_OK;
    }
    // one phi row for every sample: per-sample gradient rows, summed over the batch in a fixed order
    Arena ar(ws, ws_bytes);
    ConditionerBackward cb;
    const float* row = phi;
    float* gsum = grads ? grads->grad_phi : nullptr;
    if (g->hyper) {  // fp32 conditioner over its one row
        ZK_TRY(cb.recompute(g->hyper, false, nullptr, 0, nullptr, 0, c, 0, g->C, 1, ar, "gmm_backward", st));
        row = cb.phi;
        gsum = ar.take<float>(P);
        ZK_REQUIRE(ar.ok, "gmm_backward: workspace too small");
        ZK_CUDA(cudaMemsetAsync(gsum, 0, (size_t)P * 4, st));
    }
    void* scr = ar.take<char>(colsum_scratch_bytes(P));
    float* grows = ar.take<float>((size_t)rows * P);
    ZK_REQUIRE(ar.ok, "gmm_backward: workspace too small");
    for (int64_t r0 = 0; r0 < B; r0 += rows) {
        GmmArgs a = base_args(g);
        a.B = std::min(rows, B - r0);
        a.x = x + r0 * ldx; a.ldx = ldx; a.phi = row; a.ldphi = 0; a.glp = glp + r0;
        a.gx = gx ? gx + r0 * ldgx : nullptr; a.ldgx = ldgx; a.gphi = grows;
        ZK_TRY(launch_gmm(kGmmBackward, a, st));
        if (gsum) ZK_TRY(launch_colsum_add(grows, P, a.B, P, gsum, scr, st));
    }
    if (g->hyper) {
        ZK_TRY(cb.backward(gsum, gc != nullptr, grads, st));
        if (gc) ZK_TRY(launch_add(gc, cb.gin, g->C, st));
    }
    return ZK_OK;
}

}  // extern "C"
