// zuko_b200 — C ABI of the backward pass: layer / flow orchestration of the reverse-mode kernels
// (backward.cu).  Declarations and reference citations: include/zuko_b200.h.
//
// Structure of one layer's backward (autoregressive, transforms.py:1005-1007):
//   A0 = cat(x, c)                                   concat_kernel
//   h_i = relu(h_{i-1} W_i^T + b_i), phi = last      linear_fp32_kernel, activations KEPT
//   (gx_direct, gphi) = d bijector(x; phi)           uni_bwd_kernel (gphi overwrites phi)
//   for i = last..first: gW_i += mask * g^T h_{i-1}  wgrad_fp32_kernel + fixed-order reduce
//                        gb_i += colsum(g)           colsum_stage1/2
//                        g = (g W_i) * [h_{i-1} > 0] linear_fp32_kernel on W_i^T + relu_gate_kernel
//   gx = gx_direct + g[:, :D];  gc += g[:, D:]       input_grad_kernel
// The flow-level call recomputes the forward chain z_0..z_T with the production forward kernels
// (fused layer kernel where it applies), then walks the layers in reverse.

#include <mutex>

#include "api_internal.cuh"
#include "backward.cuh"
#include "tc_common.cuh"

using namespace zk;
namespace zkapi {}
using namespace zkapi;

namespace zkapi {

namespace {

std::mutex g_bwd_mu;
std::atomic<int> g_tc_backward{1};

}  // namespace

bool tc_backward_on() { return g_tc_backward.load() != 0; }

// transposed pre-masked weights for dgrad, built on first use
zk_status mlp_ensure_backward(const zk_mlp* cm, cudaStream_t st) {
    zk_mlp* m = const_cast<zk_mlp*>(cm);
    std::lock_guard<std::mutex> lk(g_bwd_mu);
    if ((int)m->wt.size() == m->n_linear) {
        if (!m->bwd_dirty) return ZK_OK;
        // the weights were refreshed in place (zk_layer_update_weights): same buffers, new transposes
        for (int i = 0; i < m->n_linear; ++i) ZK_TRY(launch_transpose(m->w[i], m->dims[i + 1], m->dims[i], m->wt[i], st));
        if (m->gemm_mode != ZK_GEMM_FP32 && m->tc != nullptr && m->act == 1 && m->plain) ZK_TRY(tc_pack_backward(m, st));
        m->bwd_dirty = false;
        return ZK_OK;
    }
    for (float* p : m->wt) cudaFree(p);
    m->wt.clear();
    for (int i = 0; i < m->n_linear; ++i) {
        float* t = nullptr;
        ZK_CUDA(cudaMalloc((void**)&t, (size_t)m->dims[i] * m->dims[i + 1] * 4));
        m->wt.push_back(t);
        ZK_TRY(launch_transpose(m->w[i], m->dims[i + 1], m->dims[i], t, st));
    }
    if (m->gemm_mode != ZK_GEMM_FP32 && m->tc != nullptr && m->act == 1 && m->plain) ZK_TRY(tc_pack_backward(m, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    return ZK_OK;
}

size_t mlp_bwd_scratch(const zk_mlp* m) {
    size_t s = colsum_scratch_bytes(m->dims[0]);  // broadcast-context column sum of the input gradient
    for (int i = 0; i < m->n_linear; ++i)
        s = std::max(s, std::max(wgrad_scratch_bytes(m->dims[i + 1], m->dims[i]), colsum_scratch_bytes(m->dims[i + 1])));
    return a256(s);
}

size_t mlp_bwd_ws(const zk_mlp* m, int64_t B) {
    size_t s = 0;
    for (int i = 0; i <= m->n_linear; ++i) s += a256((size_t)B * m->dims[i] * 4);  // acts + out
    for (int i = 1; i < m->n_linear; ++i)
        if (m->lact[i - 1] > 1) s += a256((size_t)B * m->dims[i] * 4);  // pre-activations (non-ReLU layers)
    if (m->n_linear > 1) s += 2 * a256((size_t)B * m->max_hidden * 4);
    s += a256((size_t)B * m->dims[0] * 4);  // gin
    return s + mlp_bwd_scratch(m);
}

bool mlp_bwd_carve(const zk_mlp* m, int64_t B, Arena& ar, MlpBwdBufs& b) {
    b.acts.resize(m->n_linear);
    for (int i = 0; i < m->n_linear; ++i) b.acts[i] = ar.take<float>((size_t)B * m->dims[i]);
    b.pre.assign(m->n_linear, nullptr);
    for (int i = 1; i < m->n_linear; ++i)
        if (m->lact[i - 1] > 1) b.pre[i] = ar.take<float>((size_t)B * m->dims[i]);
    b.out = ar.take<float>((size_t)B * m->dims[m->n_linear]);
    if (m->n_linear > 1) {
        b.gbuf[0] = ar.take<float>((size_t)B * m->max_hidden);
        b.gbuf[1] = ar.take<float>((size_t)B * m->max_hidden);
    }
    b.gin = ar.take<float>((size_t)B * m->dims[0]);
    b.scratch = ar.take<char>(mlp_bwd_scratch(m));
    return ar.ok;
}

// forward with every activation kept (fp32 CUDA-core path); acts[0] must be filled
zk_status mlp_forward_save(const zk_mlp* m, const MlpBwdBufs& b, int64_t B, cudaStream_t st) {
    const int n = m->n_linear;
    for (int i = 0; i < n; ++i) {
        const bool hidden = (i < n - 1);
        const int act = m->lact[i];
        if (hidden && act > 1) {  // general activation: keep the pre-activation for act'
            ZK_TRY(launch_linear_fp32(b.acts[i], m->dims[i], m->dims[i], nullptr, 0, m->dims[i], m->w[i], m->b[i],
                                      B, m->dims[i + 1], 0, b.pre[i + 1], m->dims[i + 1], st));
            ZK_TRY(launch_act_apply(b.pre[i + 1], b.acts[i + 1], B * (int64_t)m->dims[i + 1], act, st));
            continue;
        }
        float* dst = hidden ? b.acts[i + 1] : b.out;
        // second layer of a residual block: + input of the previous layer (zuko/nn.py:195-199)
        const float* res = m->lres[i] ? b.acts[i - 1] : nullptr;
        ZK_TRY(launch_linear_fp32(b.acts[i], m->dims[i], m->dims[i], nullptr, 0, m->dims[i], m->w[i], m->b[i],
                                  B, m->dims[i + 1], act, dst, m->dims[i + 1], st, res, m->dims[i + 1]));
    }
    return ZK_OK;
}

// b.out holds dL/d(out) on entry; on exit b.gin = dL/d(input) when want_gin
zk_status mlp_backward(const zk_mlp* m, const MlpBwdBufs& b, int64_t B, bool want_gin,
                       const zk_layer_grads* grads, cudaStream_t st) {
    const int n = m->n_linear;
    const float* g = b.out;
    for (int i = n - 1; i >= 0; --i) {
        const int N = m->dims[i + 1], K = m->dims[i];
        if (grads && grads->grad_weight && grads->grad_weight[i])
            ZK_TRY(launch_wgrad_fp32(g, N, b.acts[i], K, B, N, K, m->mask[i], grads->grad_weight[i], b.scratch, st));
        if (grads && grads->grad_bias && grads->grad_bias[i])
            ZK_TRY(launch_colsum_add(g, N, B, N, grads->grad_bias[i], b.scratch, st));
        if (i > 0 || want_gin) {
            float* dst = (i == 0) ? b.gin : b.gbuf[i & 1];
            // g (B, N) x W (N, K) = "linear" with the transposed weights (K, N).  When layer i + 1 closed a
            // residual block, its output gradient also flows straight into this layer's input: it still sits
            // in the ping-pong buffer this dgrad writes, and the epilogue adds it in place
            const float* pend = (i + 1 < n && m->lres[i + 1]) ? dst : nullptr;
            ZK_TRY(launch_linear_fp32(g, N, N, nullptr, 0, N, m->wt[i], nullptr, B, K, 0, dst, K, st, pend, K));
            if (i > 0) {  // through the activation of layer i - 1 (none inside / after a residual block's sum)
                const int act = m->lact[i - 1];
                if (act == 1) ZK_TRY(launch_relu_gate(dst, b.acts[i], B * (int64_t)K, st));
                else if (act > 1) ZK_TRY(launch_act_gate(dst, b.pre[i], B * (int64_t)K, act, st));
            }
            g = dst;
        }
    }
    return ZK_OK;
}


// ---------------------------------------------------------------------------
// conditioner backward on the tensor cores (handles packed for wgmma): every GEMM-shaped piece —
// forward recompute with saved activations, dgrad, wgrad — is linear_tc_kernel (split-bf16, fp32
// accumulation); see the block comment at the end of mlp_tcgen05.cu.
// ---------------------------------------------------------------------------
TcBwdPlan tc_plan(const zk_mlp* m, int64_t B) {
    TcBwdPlan p;
    p.n = m->n_linear;
    for (int i = 0; i <= p.n; ++i) p.Kp.push_back(pad64(m->dims[i]));
    for (int i = 1; i < p.n; ++i) p.max_hidden_kp = std::max(p.max_hidden_kp, p.Kp[i]);
    p.scratch = colsum_scratch_bytes(m->dims[0]);
    for (int i = 0; i < p.n; ++i) {
        const int N = m->dims[i + 1], K = m->dims[i];
        const int sm = (N + 127) / 128 * 128;
        const int64_t tiles = (int64_t)(sm / 128) * ((K + 127) / 128);
        int64_t S = ceil_div(2 * sm_count(), tiles);
        S = std::max<int64_t>(1, std::min<int64_t>(S, B / 512));
        const int Bs = pad64((int)ceil_div(B, S));
        p.S.push_back((int)S);
        p.Bs.push_back(Bs);
        p.slice_m.push_back(sm);
        p.gT = std::max(p.gT, (size_t)4 * S * sm * Bs);
        p.aT = std::max(p.aT, (size_t)4 * S * p.Kp[i] * Bs);
        p.partial = std::max(p.partial, (size_t)4 * S * sm * K);
        p.scratch = std::max(p.scratch, std::max(colsum_scratch_bytes(N), colsum_planes_scratch_bytes(N)));
    }
    return p;
}

bool mlp_uses_tc(const zk_mlp* m) {  // the tensor-core backward gates with ReLU in the GEMM epilogue
    return m->gemm_mode != ZK_GEMM_FP32 && m->tc != nullptr && m->act == 1 && m->plain;
}

size_t tc_bwd_ws(const zk_mlp* m, int64_t B) {
    const TcBwdPlan p = tc_plan(m, B);
    size_t s = 2 * a256((size_t)B * m->dims[0] * 4);  // A0 (fp32 cat) + gin
    for (int i = 0; i < p.n; ++i) s += a256((size_t)B * p.Kp[i] * 4);  // saved activation planes
    s += a256((size_t)B * m->dims[p.n] * 4);                            // phi / gphi (fp32)
    s += a256((size_t)B * p.Kp[p.n] * 4);                               // planes of gphi
    if (p.n > 1) s += 2 * a256((size_t)B * p.max_hidden_kp * 4);        // dgrad ping-pong planes
    return s + a256(p.gT) + a256(p.aT) + a256(p.partial) + a256(p.scratch);
}

bool tc_bwd_carve(const zk_mlp* m, const TcBwdPlan& p, int64_t B, Arena& ar, TcBwdBufs& b) {
    b.a0 = ar.take<float>((size_t)B * m->dims[0]);
    b.gin = ar.take<float>((size_t)B * m->dims[0]);
    b.P.resize(p.n);
    for (int i = 0; i < p.n; ++i) b.P[i] = ar.take<__nv_bfloat16>((size_t)2 * B * p.Kp[i]);
    b.out = ar.take<float>((size_t)B * m->dims[p.n]);
    b.G = ar.take<__nv_bfloat16>((size_t)2 * B * p.Kp[p.n]);
    if (p.n > 1) {
        b.gbuf[0] = ar.take<__nv_bfloat16>((size_t)2 * B * p.max_hidden_kp);
        b.gbuf[1] = ar.take<__nv_bfloat16>((size_t)2 * B * p.max_hidden_kp);
    }
    b.gT = (__nv_bfloat16*)ar.take<char>(p.gT);
    b.aT = (__nv_bfloat16*)ar.take<char>(p.aT);
    b.partial = (float*)ar.take<char>(p.partial);
    b.scratch = ar.take<char>(p.scratch);
    return ar.ok;
}

// b.a0 = cat(x, c) must be filled; leaves phi in b.out and every layer input in b.P
zk_status tc_forward_save(const zk_mlp* m, const TcBwdPlan& p, const TcBwdBufs& b, int64_t B, cudaStream_t st) {
    const TcPack* pk = tc_pack_of(m);
    ZK_TRY(launch_split_planes(b.a0, m->dims[0], m->dims[0], nullptr, 0, 0, B, p.Kp[0], b.P[0], st));
    for (int i = 0; i < p.n; ++i) {
        const bool last = (i == p.n - 1);
        TcGemmArgs g;
        g.a_planes = b.P[i]; g.M = B; g.Kp = p.Kp[i]; g.mapW = &pk->layers[i].mapW; g.N = m->dims[i + 1];
        g.bias = m->b[i]; g.relu = last ? 0 : 1; g.n_terms = pk->n_terms;
        if (last) { g.out_f32 = b.out; g.ldo = m->dims[p.n]; }
        else { g.out_planes = b.P[i + 1]; g.Np = p.Kp[i + 1]; }
        ZK_TRY(tc_gemm(g, st));
    }
    return ZK_OK;
}

// b.out holds dL/d(out) (fp32); on exit b.gin = dL/d(input) when want_gin
zk_status tc_mlp_backward(const zk_mlp* m, const TcBwdPlan& p, const TcBwdBufs& b, int64_t B, bool want_gin,
                          const zk_layer_grads* grads, cudaStream_t st) {
    const TcPack* pk = tc_pack_of(m);
    const int n = p.n;
    ZK_TRY(launch_split_planes(b.out, m->dims[n], m->dims[n], nullptr, 0, 0, B, p.Kp[n], b.G, st));
    const __nv_bfloat16* g = b.G;  // planes [2][B][Kp[i + 1]] of dL/d(output of layer i)
    for (int i = n - 1; i >= 0; --i) {
        const int N = m->dims[i + 1], K = m->dims[i];
        if (grads && grads->grad_weight && grads->grad_weight[i]) {
            const int S = p.S[i], Bs = p.Bs[i], sm = p.slice_m[i];
            if (i == n - 1) ZK_TRY(launch_transpose_split_f32(b.out, N, B, N, S, sm, Bs, b.gT, st));
            else ZK_TRY(launch_transpose_planes(g, B, p.Kp[i + 1], S, sm, Bs, b.gT, st));
            ZK_TRY(launch_transpose_planes(b.P[i], B, p.Kp[i], S, p.Kp[i], Bs, b.aT, st));
            CUtensorMap mapAT;
            ZK_TRY(make_plane_map(&mapAT, b.aT, (int64_t)S * p.Kp[i], Bs, 128));
            TcGemmArgs w;
            w.a_planes = b.gT; w.M = (int64_t)S * sm; w.Kp = Bs; w.mapW = &mapAT; w.N = K;
            w.out_f32 = b.partial; w.ldo = K; w.slice_m = sm; w.w_slice_rows = p.Kp[i]; w.n_terms = pk->n_terms;
            ZK_TRY(tc_gemm(w, st));
            ZK_TRY(launch_wgrad_reduce_sliced(b.partial, S, sm, N, K, m->mask[i], grads->grad_weight[i], st));
        }
        if (grads && grads->grad_bias && grads->grad_bias[i]) {
            if (i == n - 1) ZK_TRY(launch_colsum_add(b.out, N, B, N, grads->grad_bias[i], b.scratch, st));
            else ZK_TRY(launch_colsum_planes_add(g, B, p.Kp[i + 1], N, grads->grad_bias[i], b.scratch, st));
        }
        if (i > 0 || want_gin) {
            TcGemmArgs d;
            d.a_planes = g; d.M = B; d.Kp = p.Kp[i + 1]; d.mapW = &pk->bwd[i].mapW; d.N = K; d.n_terms = pk->n_terms;
            if (i == 0) { d.out_f32 = b.gin; d.ldo = K; }
            else { d.out_planes = b.gbuf[i & 1]; d.Np = p.Kp[i]; d.gate = b.P[i]; }
            ZK_TRY(tc_gemm(d, st));
            g = b.gbuf[i & 1];
        }
    }
    return ZK_OK;
}

namespace {

size_t layer_bwd_ws(const zk_layer* l, int64_t B) {
    if (!l || B <= 0) return 0;
    const size_t table = a256((size_t)B * l->D * l->P * 4) + a256(colsum_scratch_bytes(std::max(1, l->D * l->P)));
    switch (l->kind) {
        case ZK_LAYER_AUTOREGRESSIVE:
        case ZK_LAYER_COUPLING:
            return (mlp_uses_tc(l->hyper) ? std::max(tc_bwd_ws(l->hyper, B), mlp_bwd_ws(l->hyper, B)) : mlp_bwd_ws(l->hyper, B)) + 1024;
        case ZK_LAYER_ELEMENTWISE:
            return (l->hyper ? mlp_bwd_ws(l->hyper, B) : 0) + table + 1024;
        case ZK_LAYER_ROTATION:
            return a256(wgrad_scratch_bytes(l->D, l->D)) + 1024;
        default:
            return 0;
    }
}

// direct_only (autoregressive / coupling): stop after the bijector's own derivative — gx receives
// gy * dy_d/dx_d on the transformed dims, nothing flows through the conditioner
zk_status layer_backward_impl(const zk_layer* l, const float* x, int64_t ldx, const float* c,
                              int64_t ldc, int64_t B, const float* gy, int64_t ldgy, const float* gl,
                              float* gx, int64_t ldgx, float* gc, int64_t ldgc,
                              const zk_layer_grads* grads, void* ws, size_t ws_bytes, cudaStream_t st,
                              bool direct_only = false) {
    if (B == 0) return ZK_OK;
    ZK_REQUIRE(l->C == 0 || c != nullptr, "layer needs a context of %d features", l->C);
    Arena ar(ws, ws_bytes);
    UniBwdArgs u;
    u.spec = l->spec; u.B = B;
    u.fast_math = g_fast_math.load() != 0;
    u.x = x; u.ldx = ldx; u.gy = gy; u.ldgy = ldgy; u.gl = gl; u.gx = gx; u.ldgx = ldgx;
    switch (l->kind) {
        case ZK_LAYER_AUTOREGRESSIVE:
        case ZK_LAYER_COUPLING: {
            const bool coupling = (l->kind == ZK_LAYER_COUPLING);
            const zk_mlp* m = l->hyper;
            const int nx = coupling ? l->n_a : l->D;
            const int nt = coupling ? l->n_b : l->D;  // transformed dims
            ZK_TRY(mlp_ensure_backward(m, st));
            u.phi_ld = (int64_t)nt * l->P; u.D = nt;
            u.dim_map = coupling ? l->idx_b : nullptr;
            const bool per_row_gc = (gc != nullptr && l->C > 0 && ldc != 0);
            if (mlp_uses_tc(m) && g_tc_backward.load()) {
                // tensor-core path: forward recompute, dgrad and wgrad on linear_tc_kernel
                const TcBwdPlan plan = tc_plan(m, B);
                TcBwdBufs tb;
                ZK_REQUIRE(tc_bwd_carve(m, plan, B, ar, tb), "layer_backward: workspace too small");
                ZK_TRY(launch_concat(x, ldx, coupling ? l->idx_a : nullptr, nx, c, ldc, l->C, B, tb.a0, st));
                ZK_TRY(tc_forward_save(m, plan, tb, B, st));
                u.phi = tb.out; u.gphi = direct_only ? nullptr : tb.out;
                ZK_TRY(launch_univariate_backward(u, st));
                if (direct_only) return ZK_OK;
                ZK_TRY(tc_mlp_backward(m, plan, tb, B, true, grads, st));
                ZK_TRY(launch_input_grad(tb.gin, nx, l->C, coupling ? l->idx_a : nullptr, B, gx, ldgx,
                                         coupling ? gy : nullptr, ldgy, per_row_gc ? gc : nullptr, ldgc, st));
                if (gc != nullptr && l->C > 0 && ldc == 0)
                    ZK_TRY(launch_colsum_add(tb.gin + nx, m->dims[0], B, l->C, gc, tb.scratch, st));
                return ZK_OK;
            }
            MlpBwdBufs b;
            ZK_REQUIRE(mlp_bwd_carve(m, B, ar, b), "layer_backward: workspace too small");
            ZK_TRY(launch_concat(x, ldx, coupling ? l->idx_a : nullptr, nx, c, ldc, l->C, B, b.acts[0], st));
            ZK_TRY(mlp_forward_save(m, b, B, st));
            u.phi = b.out; u.gphi = direct_only ? nullptr : b.out;
            ZK_TRY(launch_univariate_backward(u, st));  // gx[:, transformed] = direct term
            if (direct_only) return ZK_OK;
            ZK_TRY(mlp_backward(m, b, B, true, grads, st));
            // coupling: gx[:, idx_a] = gy[:, idx_a] + gin[:, :n_a] (y_a = x_a, transforms.py:1069)
            ZK_TRY(launch_input_grad(b.gin, nx, l->C, coupling ? l->idx_a : nullptr, B, gx, ldgx,
                                     coupling ? gy : nullptr, ldgy, per_row_gc ? gc : nullptr, ldgc, st));
            if (gc != nullptr && l->C > 0 && ldc == 0)  // broadcast context: one summed row
                ZK_TRY(launch_colsum_add(b.gin + nx, m->dims[0], B, l->C, gc, b.scratch, st));
            return ZK_OK;
        }
        case ZK_LAYER_ELEMENTWISE: {
            const int DP = l->D * l->P;
            u.D = l->D;
            if (!l->hyper) {  // shared (D, P) table (gaussianization.py:74-77)
                float* rows = ar.take<float>((size_t)B * DP);
                void* scr = ar.take<char>(colsum_scratch_bytes(DP));
                ZK_REQUIRE(ar.ok, "layer_backward: workspace too small");
                u.phi = l->phi_shared; u.phi_ld = 0;
                u.gphi = (grads && grads->grad_phi) ? rows : nullptr;
                ZK_TRY(launch_univariate_backward(u, st));
                if (grads && grads->grad_phi) ZK_TRY(launch_colsum_add(rows, DP, B, DP, grads->grad_phi, scr, st));
                return ZK_OK;
            }
            const zk_mlp* m = l->hyper;
            ZK_TRY(mlp_ensure_backward(m, st));
            const int64_t rows = (ldc == 0) ? 1 : B;  // gaussianization.py:89-92: phi = hyper(c)
            MlpBwdBufs b;
            ZK_REQUIRE(mlp_bwd_carve(m, rows, ar, b), "layer_backward: workspace too small");
            float* grows = nullptr;
            void* scr = nullptr;
            if (rows == 1) {
                grows = ar.take<float>((size_t)B * DP);
                scr = ar.take<char>(colsum_scratch_bytes(DP));
                ZK_REQUIRE(ar.ok, "layer_backward: workspace too small");
            }
            ZK_TRY(launch_concat(nullptr, 0, nullptr, 0, c, ldc, l->C, rows, b.acts[0], st));
            ZK_TRY(mlp_forward_save(m, b, rows, st));
            u.phi = b.out;
            if (rows == 1) {
                u.phi_ld = 0; u.gphi = grows;
                ZK_TRY(launch_univariate_backward(u, st));
                ZK_CUDA(cudaMemsetAsync(b.out, 0, (size_t)DP * 4, st));
                ZK_TRY(launch_colsum_add(grows, DP, B, DP, b.out, scr, st));
            } else {
                u.phi_ld = DP; u.gphi = b.out;
                ZK_TRY(launch_univariate_backward(u, st));
            }
            ZK_TRY(mlp_backward(m, b, rows, gc != nullptr, grads, st));
            if (gc) {
                if (rows == 1) ZK_TRY(launch_add(gc, b.gin, l->C, st));
                else ZK_TRY(launch_input_grad(b.gin, 0, l->C, nullptr, B, nullptr, 0, nullptr, 0, gc, ldgc, st));
            }
            return ZK_OK;
        }
        case ZK_LAYER_SOFTCLIP:
            return launch_softclip_backward(x, ldx, gy, ldgy, gl, B, l->D, l->spec.bound, gx, ldgx, st);
        case ZK_LAYER_PERMUTATION:  // y[:, j] = x[:, order[j]]  =>  gx[:, i] = gy[:, argsort(order)[i]]
            return launch_permute(gy, ldgy, l->perm_inv, B, l->D, gx, ldgx, st);
        case ZK_LAYER_ROTATION: {  // y = R x  =>  gx = R^T gy, gR += gy^T x
            ZK_TRY(launch_rotate(gy, ldgy, l->rotation, 1, B, l->D, gx, ldgx, st));
            if (grads && grads->grad_rotation) {
                void* scr = ar.take<char>(wgrad_scratch_bytes(l->D, l->D));
                ZK_REQUIRE(ar.ok, "layer_backward: workspace too small");
                ZK_TRY(launch_wgrad_fp32(gy, ldgy, x, ldx, B, l->D, l->D, nullptr, grads->grad_rotation, scr, st));
            }
            return ZK_OK;
        }
    }
    return fail(ZK_EUNSUPPORTED, "layer_backward: unknown kind %d", l->kind);
}

size_t flow_bwd_ws_for(const zk_flow_desc* f, int64_t Bc) {
    const int D = f->features;
    size_t layer_max = 0;
    for (int i = 0; i < f->n_layers; ++i)
        layer_max = std::max(layer_max, std::max(zk_layer_workspace_bytes(f->layers[i], Bc), layer_bwd_ws(f->layers[i], Bc)));
    return (size_t)(f->n_layers + 2) * a256((size_t)Bc * D * 4)  // z_1..z_T + two gradient buffers
           + 2 * a256((size_t)Bc * 4)                            // gl, ladj scratch
           + layer_max + 1024;
}

int64_t flow_bwd_chunk_rows(const zk_flow_desc* f, int64_t B, size_t ws_bytes) {
    if (flow_bwd_ws_for(f, B) <= ws_bytes) return B;
    if (flow_bwd_ws_for(f, 1) > ws_bytes) return 0;
    int64_t lo = 1, hi = B;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo + 1) / 2;
        if (flow_bwd_ws_for(f, mid) <= ws_bytes) lo = mid; else hi = mid - 1;
    }
    // keep tiles aligned when that still fits (the batch-slice plan of the tensor-core wgrad makes the
    // requirement only approximately monotone in the row count, so the rounded value is re-checked)
    if (lo >= 2048 && flow_bwd_ws_for(f, lo / 1024 * 1024) <= ws_bytes) lo = lo / 1024 * 1024;
    return lo;
}

zk_status flow_backward_chunk(const zk_flow_desc* f, const float* x, int64_t ldx, const float* c,
                              int64_t ldc, int64_t B, const float* gz_in, int64_t ldgz,
                              const float* gl_in, const float* g_lp, float* grad_x, int64_t ldgx,
                              float* grad_c, int64_t ldgc, const zk_layer_grads* const* grads,
                              void* ws, size_t ws_bytes, cudaStream_t st) {
    const int D = f->features, T = f->n_layers;
    Arena ar(ws, ws_bytes);
    std::vector<const float*> z(T + 1);
    std::vector<int64_t> ldz(T + 1, D);
    std::vector<float*> zbuf(T + 1, nullptr);
    z[0] = x;
    ldz[0] = ldx;
    for (int i = 1; i <= T; ++i) z[i] = zbuf[i] = ar.take<float>((size_t)B * D);
    float* gA = ar.take<float>((size_t)B * D);
    float* gB = ar.take<float>((size_t)B * D);
    float* gl = ar.take<float>((size_t)B);
    float* lscr = ar.take<float>((size_t)B);
    ZK_REQUIRE(ar.ok, "flow_backward: workspace too small");
    void* lws = ar.base + ar.off;
    const size_t lws_bytes = ar.size - ar.off;
    // forward chain with the production kernels, every z_i kept
    for (int i = 0; i < T; ++i) {
        const zk_layer* l = f->layers[i];
        ZK_TRY(layer_forward_impl(l, z[i], ldz[i], l->C ? c : nullptr, ldc, B, zbuf[i + 1], D, lscr, 0, nullptr,
                                  nullptr, nullptr, lws, lws_bytes, st));
    }
    // seed: dL/dz_T and dL/dladj (distributions.py:115-119)
    if (f->base_kind == ZK_BASE_BOX_UNIFORM)  // constant density on the support: no d/dz term
        ZK_TRY(launch_base_grad_flat(g_lp, gz_in, ldgz, gl_in, B, D, gA, gl, st));
    else
        ZK_TRY(launch_base_grad(z[T], ldz[T], f->base_loc, f->base_scale, g_lp, gz_in, ldgz, gl_in, B, D, gA, gl, st));
    const float* cur = gA;
    int64_t ldcur = D;
    for (int i = T - 1; i >= 0; --i) {
        const zk_layer* l = f->layers[i];
        float* dst = (i == 0 && grad_x) ? grad_x : (cur == gA ? gB : gA);
        const int64_t ldd = (i == 0 && grad_x) ? ldgx : D;
        ZK_TRY(layer_backward_impl(l, z[i], ldz[i], l->C ? c : nullptr, ldc, B, cur, ldcur, gl, dst, ldd,
                                   l->C ? grad_c : nullptr, ldgc, grads ? grads[i] : nullptr, lws, lws_bytes, st));
        cur = dst;
        ldcur = ldd;
    }
    if (T == 0 && grad_x) ZK_TRY(copy_rows(gA, D, B, D, grad_x, ldgx, st));
    return ZK_OK;
}


// ---------------------------------------------------------------------------
// inverse direction (reparameterised sampling, SURVEY section 8f rank 2): x = layer^{-1}(y; theta, c).
// By the implicit-function theorem on y = f(x; theta, c) at the solution x, with J = df/dx:
//     dL/dy = J^{-T} g,     dL/dtheta = -(df/dtheta)^T v,     dL/dc = -(df/dc)^T v,     v = dL/dy.
// J is triangular in the layer's order classes with diagonal s = dy_d/dx_d, so J^T v = g is solved
// exactly by `passes` Richardson sweeps  v <- v + (g - J^T v) / s  (I - S J^T is nilpotent), and
// J^T v is ONE call of the forward direction's backward (gy = v, no parameter gradients).
// (torch.autograd gets the same numbers by back-propagating through the sweeps of transforms.py:994-1000.)
// ---------------------------------------------------------------------------
struct InvBwdBufs { float *s, *jtv, *negv, *ones; };

zk_status layer_inverse_backward_impl(const zk_layer* l, const float* x, int64_t ldx, const float* c, int64_t ldc,
                                      int64_t B, const float* g /*(B, D)*/, float* v /*(B, D)*/, float* gc,
                                      int64_t ldgc, const zk_layer_grads* grads, const InvBwdBufs& ib, void* ws,
                                      size_t ws_bytes, cudaStream_t st) {
    const int D = l->D;
    const int64_t n = B * (int64_t)D;
    bool has_params = false;
    switch (l->kind) {
        case ZK_LAYER_PERMUTATION:  // J = P (orthogonal): J^{-T} g = P g
            return launch_permute(g, D, l->perm, B, D, v, D, st);
        case ZK_LAYER_ROTATION:     // J = R (orthogonal): J^{-T} g = R g
            ZK_TRY(launch_rotate(g, D, l->rotation, 0, B, D, v, D, st));
            has_params = true;
            break;
        default: {
            const bool cond = (l->kind == ZK_LAYER_AUTOREGRESSIVE || l->kind == ZK_LAYER_COUPLING);
            const int sweeps = (l->kind == ZK_LAYER_AUTOREGRESSIVE) ? std::max(1, l->passes) : (l->kind == ZK_LAYER_COUPLING ? 2 : 1);
            // s = diag J: the bijector's own derivative (1 on the constant split of a coupling layer)
            ZK_TRY(launch_fill(ib.s, n, 1.f, st));
            ZK_TRY(layer_backward_impl(l, x, ldx, c, ldc, B, ib.ones, D, nullptr, ib.s, D, nullptr, 0, nullptr, ws, ws_bytes, st, cond));
            ZK_TRY(launch_div(v, g, ib.s, n, st));
            for (int it = 1; it < sweeps; ++it) {
                ZK_TRY(layer_backward_impl(l, x, ldx, c, ldc, B, v, D, nullptr, ib.jtv, D, nullptr, 0, nullptr, ws, ws_bytes, st));
                ZK_TRY(launch_richardson(v, g, ib.jtv, ib.s, n, st));
            }
            has_params = (l->hyper != nullptr) || (l->phi_shared != nullptr);
        }
    }
    if (has_params && (grads != nullptr || (gc != nullptr && l->C > 0))) {
        ZK_TRY(launch_scale(ib.negv, v, -1.f, n, st));
        ZK_TRY(layer_backward_impl(l, x, ldx, c, ldc, B, ib.negv, D, nullptr, ib.jtv, D, l->C ? gc : nullptr, ldgc, grads, ws, ws_bytes, st));
    }
    return ZK_OK;
}

size_t flow_invbwd_ws_for(const zk_flow_desc* f, int64_t Bc) {
    return flow_bwd_ws_for(f, Bc) + (size_t)(f->n_layers + 9) * a256((size_t)Bc * f->features * 4) + a256((size_t)Bc * 4);
}

int64_t flow_invbwd_chunk_rows(const zk_flow_desc* f, int64_t B, size_t ws_bytes) {
    if (flow_invbwd_ws_for(f, B) <= ws_bytes) return B;
    if (flow_invbwd_ws_for(f, 1) > ws_bytes) return 0;
    int64_t lo = 1, hi = B;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo + 1) / 2;
        if (flow_invbwd_ws_for(f, mid) <= ws_bytes) lo = mid; else hi = mid - 1;
    }
    if (lo >= 2048 && flow_invbwd_ws_for(f, lo / 1024 * 1024) <= ws_bytes) lo = lo / 1024 * 1024;
    return lo;
}

zk_status flow_inverse_backward_chunk(const zk_flow_desc* f, const float* x, int64_t ldx, const float* c, int64_t ldc,
                                      int64_t B, const float* grad_x, int64_t ldgx, const float* g_lp, const float* z,
                                      int64_t ldz, float* grad_z, int64_t ldgz, float* grad_c, int64_t ldgc,
                                      const zk_layer_grads* const* grads, void* ws, size_t ws_bytes, cudaStream_t st) {
    const int D = f->features, T = f->n_layers;
    const int64_t n = B * (int64_t)D;
    Arena ar(ws, ws_bytes);
    std::vector<const float*> xs(T + 1);
    std::vector<int64_t> ldxs(T + 1, D);
    std::vector<float*> xbuf(T + 1, nullptr);
    xs[0] = x;
    ldxs[0] = ldx;
    for (int i = 1; i <= T; ++i) xs[i] = xbuf[i] = ar.take<float>((size_t)n);
    float* ga = ar.take<float>((size_t)n);
    float* gb = ar.take<float>((size_t)n);
    float* gxl = ar.take<float>((size_t)n);
    InvBwdBufs ib;
    ib.s = ar.take<float>((size_t)n); ib.jtv = ar.take<float>((size_t)n); ib.negv = ar.take<float>((size_t)n);
    ib.ones = ar.take<float>((size_t)n);
    float* out = ar.take<float>((size_t)n);
    float* lscr = ar.take<float>((size_t)B);
    ZK_REQUIRE(ar.ok, "flow_inverse_backward: workspace too small");
    void* lws = ar.base + ar.off;
    const size_t lws_bytes = ar.size - ar.off;
    ZK_TRY(launch_fill(ib.ones, n, 1.f, st));
    // forward chain from the sample: xs[l] is the input of layer l in the forward direction
    for (int i = 0; i < T; ++i) {
        const zk_layer* l = f->layers[i];
        ZK_TRY(layer_forward_impl(l, xs[i], ldxs[i], l->C ? c : nullptr, ldc, B, xbuf[i + 1], D, lscr, 0, nullptr,
                                  nullptr, nullptr, lws, lws_bytes, st));
    }
    if (grad_x) ZK_TRY(copy_rows(grad_x, ldgx, B, D, ga, D, st));
    else ZK_TRY(launch_fill(ga, n, 0.f, st));
    if (g_lp) {
        // log p = base.log_prob(z) + sum_l ladj_l(x_l; theta): explicit gradients at fixed x, d/dx joins g
        ZK_TRY(flow_backward_chunk(f, x, ldx, c, ldc, B, nullptr, 0, g_lp, nullptr, gxl, D, grad_c, ldgc, grads, lws, lws_bytes, st));
        ZK_TRY(launch_add(ga, gxl, n, st));
    }
    float* g = ga;
    float* v = gb;
    for (int i = 0; i < T; ++i) {
        const zk_layer* l = f->layers[i];
        ZK_TRY(layer_inverse_backward_impl(l, xs[i], ldxs[i], l->C ? c : nullptr, ldc, B, g, v, l->C ? grad_c : nullptr, ldgc,
                                           grads ? grads[i] : nullptr, ib, lws, lws_bytes, st));
        std::swap(g, v);
    }
    if (grad_z) {
        if (g_lp && f->base_kind == ZK_BASE_DIAG_NORMAL) {  // + g_lp * d base.log_prob(z) / dz
            ZK_REQUIRE(z != nullptr, "flow_inverse_backward: grad_log_prob needs z");
            ZK_TRY(launch_base_grad(z, ldz, f->base_loc, f->base_scale, g_lp, g, D, nullptr, B, D, out, lscr, st));
            ZK_TRY(copy_rows(out, D, B, D, grad_z, ldgz, st));
        } else {
            ZK_TRY(copy_rows(g, D, B, D, grad_z, ldgz, st));
        }
    }
    return ZK_OK;
}

zk_status uni_backward_entry(const UniSpec& spec, const float* x, int64_t ldx, const float* phi, int64_t phi_ld,
                             int64_t B, int D, const float* gy, int64_t ldgy, const float* gl, float* gx, int64_t ldgx,
                             float* gphi, void* ws, size_t ws_bytes, zk_stream stream, bool shape_first = false) {
    const cudaStream_t st = (cudaStream_t)stream;
    // the Gaussianization, SOSP and Bernstein entries refuse a bad shape even with B = 0; RQS and affine do not
    if (shape_first) ZK_TRY(uni_check_shape(spec));
    ZK_REQUIRE(x && phi && B >= 0 && D > 0, "univariate backward: bad arguments");
    const int P = uni_P(spec);
    if (gphi != nullptr && B > 0 && P > 0) {
        // grad_phi may only be phi itself with dense rows: each tile then rewrites the rows it staged.  Any
        // other overlap lets one CTA's (or one chunk's) writes reach parameters another one still reads
        const int64_t DP = (int64_t)D * P;
        const int64_t n_phi = (phi_ld == 0) ? DP : (B - 1) * phi_ld + DP;
        const int64_t n_gphi = (phi_ld == 0) ? DP : B * DP;
        const bool overlap = (uintptr_t)gphi < (uintptr_t)(phi + n_phi) && (uintptr_t)phi < (uintptr_t)(gphi + n_gphi);
        ZK_REQUIRE(!overlap || (gphi == phi && phi_ld == DP),
                   "univariate backward: grad_phi overlaps phi (only grad_phi == phi with phi_ld == D*P is allowed)");
    }
    UniBwdArgs u;
    u.spec = spec; u.D = D;
    u.fast_math = g_fast_math.load() != 0;
    u.phi = phi; u.phi_ld = phi_ld;
    if (phi_ld != 0 || gphi == nullptr) {
        u.x = x; u.ldx = ldx; u.gy = gy; u.ldgy = ldgy; u.gl = gl; u.gx = gx; u.ldgx = ldgx; u.gphi = gphi; u.B = B;
        return launch_univariate_backward(u, st);
    }
    // shared table: per-row gradients go through the workspace in row chunks, then a fixed-order column sum
    const size_t DP = (size_t)D * P;
    const size_t scr = a256(colsum_scratch_bytes((int)DP));
    ZK_REQUIRE(ws && ws_bytes >= scr + a256(DP * 4), "univariate backward: workspace too small");
    const int64_t fit = std::min<int64_t>(B, (int64_t)((ws_bytes - scr) / (DP * 4)));
    float* rows = (float*)((char*)ws + scr);
    for (int64_t i0 = 0; i0 < B; i0 += fit) {
        const int64_t n = std::min(fit, B - i0);
        u.x = x + i0 * ldx; u.ldx = ldx; u.gy = gy ? gy + i0 * ldgy : nullptr; u.ldgy = ldgy;
        u.gl = gl ? gl + i0 : nullptr; u.gx = gx ? gx + i0 * ldgx : nullptr; u.ldgx = ldgx; u.gphi = rows; u.B = n;
        ZK_TRY(launch_univariate_backward(u, st));
        ZK_TRY(launch_colsum_add(rows, (int64_t)DP, n, (int)DP, gphi, ws, st));
    }
    return ZK_OK;
}

}  // namespace
}  // namespace zkapi

extern "C" {

int zk_set_tc_backward(int on) { return g_tc_backward.exchange(on ? 1 : 0); }

zk_status zk_univariate_backward_plan(int univariate, int64_t B, int D, int K, int degree, int64_t phi_ld,
                                      int* rows_per_tile, size_t* smem, int* instantiated) {
    UniBwdPlan p;
    ZK_TRY(uni_bwd_plan(UniSpec{univariate, K, degree}, B, D, phi_ld, p));
    if (rows_per_tile) *rows_per_tile = p.rows_per_tile;
    if (smem) *smem = p.smem;
    if (instantiated) *instantiated = p.kt;
    return ZK_OK;
}

size_t zk_univariate_backward_workspace_bytes(int64_t B, int D, int P, int64_t phi_ld) {
    if (phi_ld != 0 || B <= 0 || D <= 0 || P <= 0) return 0;
    return a256(colsum_scratch_bytes(D * P)) + a256((size_t)B * D * P * 4);
}

zk_status zk_rqs_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                          int D, int K, float bound, float slope, const float* grad_y, int64_t ldgy,
                          const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi,
                          void* ws, size_t ws_bytes, zk_stream stream) {
    return uni_backward_entry({ZK_UNI_RQS, K, 0, bound, slope}, x, ldx, phi, phi_ld, B, D, grad_y, ldgy, grad_ladj,
                              grad_x, ldgx, grad_phi, ws, ws_bytes, stream);
}

zk_status zk_affine_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                             int D, float slope, const float* grad_y, int64_t ldgy,
                             const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi,
                             void* ws, size_t ws_bytes, zk_stream stream) {
    return uni_backward_entry({ZK_UNI_AFFINE, 0, 0, 5.f, slope}, x, ldx, phi, phi_ld, B, D, grad_y, ldgy, grad_ladj,
                              grad_x, ldgx, grad_phi, ws, ws_bytes, stream);
}

zk_status zk_gaussianization_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B,
                                      int D, int K, const float* grad_y, int64_t ldgy, const float* grad_ladj,
                                      float* grad_x, int64_t ldgx, float* grad_phi, void* ws, size_t ws_bytes,
                                      zk_stream stream) {
    return uni_backward_entry({ZK_UNI_GAUSS, K, 0, 10.f}, x, ldx, phi, phi_ld, B, D, grad_y, ldgy, grad_ladj, grad_x, ldgx,
                              grad_phi, ws, ws_bytes, stream, true);
}

zk_status zk_sosp_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B, int D,
                           int K, int degree, float bound, float slope, const float* grad_y, int64_t ldgy,
                           const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi, void* ws,
                           size_t ws_bytes, zk_stream stream) {
    return uni_backward_entry({ZK_UNI_SOSP, K, degree, bound, slope}, x, ldx, phi, phi_ld, B, D, grad_y, ldgy,
                              grad_ladj, grad_x, ldgx, grad_phi, ws, ws_bytes, stream, true);
}

zk_status zk_bernstein_backward(const float* x, int64_t ldx, const float* phi, int64_t phi_ld, int64_t B, int D,
                                int degree, float bound, float eps, const float* grad_y, int64_t ldgy,
                                const float* grad_ladj, float* grad_x, int64_t ldgx, float* grad_phi, void* ws,
                                size_t ws_bytes, zk_stream stream) {
    return uni_backward_entry({ZK_UNI_BERNSTEIN, 0, degree, bound, 1e-3f, eps}, x, ldx, phi, phi_ld, B, D, grad_y, ldgy,
                              grad_ladj, grad_x, ldgx, grad_phi, ws, ws_bytes, stream, true);
}

zk_status zk_softclip_backward(const float* x, int64_t ldx, int64_t B, int D, float bound,
                               const float* grad_y, int64_t ldgy, const float* grad_ladj,
                               float* grad_x, int64_t ldgx, zk_stream stream) {
    return launch_softclip_backward(x, ldx, grad_y, ldgy, grad_ladj, B, D, bound, grad_x, ldgx, (cudaStream_t)stream);
}

size_t zk_layer_backward_workspace_bytes(const zk_layer* l, int64_t B) { return layer_bwd_ws(l, B); }

zk_status zk_layer_backward(const zk_layer* l, const float* x, int64_t ldx, const float* c, int64_t ldc,
                            int64_t B, const float* grad_y, int64_t ldgy, const float* grad_ladj,
                            float* grad_x, int64_t ldgx, float* grad_c, int64_t ldgc,
                            const zk_layer_grads* grads, void* ws, size_t ws_bytes, zk_stream stream) {
    ZK_REQUIRE(l && x && grad_y && grad_x, "layer_backward: null argument");
    ZK_REQUIRE(grad_x != grad_y && grad_x != x, "layer_backward: grad_x must not alias its inputs");
    ZK_REQUIRE(B >= 0 && ldx >= l->D && ldgy >= l->D && ldgx >= l->D, "layer_backward: bad shape");
    ZK_REQUIRE(!grad_c || ldc == 0 || ldgc >= l->C, "layer_backward: bad ldgc");
    ZK_REQUIRE(ws_bytes >= layer_bwd_ws(l, B), "layer_backward: workspace too small (%zu < %zu)", ws_bytes, layer_bwd_ws(l, B));
    return layer_backward_impl(l, x, ldx, c, ldc, B, grad_y, ldgy, grad_ladj, grad_x, ldgx, l->C ? grad_c : nullptr,
                               ldgc, grads, ws, ws_bytes, (cudaStream_t)stream);
}

size_t zk_flow_backward_workspace_bytes(const zk_flow_desc* f, int64_t B) {
    if (!f || B <= 0) return 1024;
    return flow_bwd_ws_for(f, B);
}
size_t zk_flow_backward_min_workspace_bytes(const zk_flow_desc* f) { return f ? flow_bwd_ws_for(f, 1) : 1024; }

zk_status zk_flow_backward(const zk_flow_desc* f, const float* x, int64_t ldx, const float* c,
                           int64_t ldc, int64_t B, const float* grad_z, int64_t ldgz,
                           const float* grad_ladj, const float* grad_log_prob, float* grad_x,
                           int64_t ldgx, float* grad_c, int64_t ldgc,
                           const zk_layer_grads* const* grads, void* ws, size_t ws_bytes,
                           zk_stream stream) {
    ZK_TRY(flow_check(f));
    if (f->inverted)
        for (int i = 0; i < f->n_layers; ++i)
            if (f->inverted[i]) return fail(ZK_EUNSUPPORTED, "backward through inverted flow members (LazyInverse) is not implemented");
    ZK_REQUIRE(x, "flow_backward: null x");
    ZK_REQUIRE(B >= 0 && ldx >= f->features, "flow_backward: bad shape");
    ZK_REQUIRE(!grad_z || ldgz >= f->features, "flow_backward: bad ldgz");
    ZK_REQUIRE(!grad_x || ldgx >= f->features, "flow_backward: bad ldgx");
    ZK_REQUIRE(f->context == 0 || c, "flow_backward: flow needs a context");
    ZK_REQUIRE(!grad_c || f->context == 0 || ldc == 0 || ldgc >= f->context, "flow_backward: bad ldgc");
    ZK_REQUIRE(grad_x != x || !grad_x, "flow_backward: grad_x must not alias x");
    cudaStream_t st = (cudaStream_t)stream;
    const int C = f->context;
    if (C == 0) grad_c = nullptr;
    if (grad_c && ldc == 0) ZK_CUDA(cudaMemsetAsync(grad_c, 0, (size_t)C * 4, st));
    if (B == 0) return ZK_OK;
    const int64_t Bc = flow_bwd_chunk_rows(f, B, ws_bytes);
    ZK_REQUIRE(Bc > 0, "flow_backward: workspace too small (%zu < %zu)", ws_bytes, zk_flow_backward_min_workspace_bytes(f));
    for (int64_t i0 = 0; i0 < B; i0 += Bc) {
        const int64_t n = std::min(Bc, B - i0);
        float* gc = grad_c ? (ldc == 0 ? grad_c : grad_c + i0 * ldgc) : nullptr;
        if (gc && ldc != 0) ZK_CUDA(cudaMemset2DAsync(gc, (size_t)ldgc * 4, 0, (size_t)C * 4, (size_t)n, st));
        ZK_TRY(flow_backward_chunk(f, x + i0 * ldx, ldx, c ? c + i0 * ldc : nullptr, ldc, n,
                                   grad_z ? grad_z + i0 * ldgz : nullptr, ldgz, grad_ladj ? grad_ladj + i0 : nullptr,
                                   grad_log_prob ? grad_log_prob + i0 : nullptr, grad_x ? grad_x + i0 * ldgx : nullptr,
                                   ldgx, gc, ldgc, grads, ws, ws_bytes, st));
    }
    return ZK_OK;
}

size_t zk_flow_inverse_backward_workspace_bytes(const zk_flow_desc* f, int64_t B) {
    if (!f || B <= 0) return 1024;
    return flow_invbwd_ws_for(f, B);
}
size_t zk_flow_inverse_backward_min_workspace_bytes(const zk_flow_desc* f) { return f ? flow_invbwd_ws_for(f, 1) : 1024; }

zk_status zk_flow_inverse_backward(const zk_flow_desc* f, const float* x, int64_t ldx, const float* c, int64_t ldc,
                                   int64_t B, const float* grad_x, int64_t ldgx, const float* grad_log_prob,
                                   const float* z, int64_t ldz, float* grad_z, int64_t ldgz, float* grad_c,
                                   int64_t ldgc, const zk_layer_grads* const* grads, void* ws, size_t ws_bytes,
                                   zk_stream stream) {
    ZK_TRY(flow_check(f));
    if (f->inverted)
        for (int i = 0; i < f->n_layers; ++i)
            if (f->inverted[i]) return fail(ZK_EUNSUPPORTED, "backward through inverted flow members (LazyInverse) is not implemented");
    ZK_REQUIRE(x, "flow_inverse_backward: null x");
    ZK_REQUIRE(B >= 0 && ldx >= f->features, "flow_inverse_backward: bad shape");
    ZK_REQUIRE(!grad_x || ldgx >= f->features, "flow_inverse_backward: bad ldgx");
    ZK_REQUIRE(!grad_z || ldgz >= f->features, "flow_inverse_backward: bad ldgz");
    ZK_REQUIRE(!grad_log_prob || !grad_z || f->base_kind != ZK_BASE_DIAG_NORMAL || (z && ldz >= f->features),
               "flow_inverse_backward: grad_log_prob needs z");
    ZK_REQUIRE(f->context == 0 || c, "flow_inverse_backward: flow needs a context");
    ZK_REQUIRE(!grad_c || f->context == 0 || ldc == 0 || ldgc >= f->context, "flow_inverse_backward: bad ldgc");
    cudaStream_t st = (cudaStream_t)stream;
    const int C = f->context;
    if (C == 0) grad_c = nullptr;
    if (grad_c && ldc == 0) ZK_CUDA(cudaMemsetAsync(grad_c, 0, (size_t)C * 4, st));
    if (B == 0) return ZK_OK;
    const int64_t Bc = flow_invbwd_chunk_rows(f, B, ws_bytes);
    ZK_REQUIRE(Bc > 0, "flow_inverse_backward: workspace too small (%zu < %zu)", ws_bytes, zk_flow_inverse_backward_min_workspace_bytes(f));
    for (int64_t i0 = 0; i0 < B; i0 += Bc) {
        const int64_t n = std::min(Bc, B - i0);
        float* gc = grad_c ? (ldc == 0 ? grad_c : grad_c + i0 * ldgc) : nullptr;
        if (gc && ldc != 0) ZK_CUDA(cudaMemset2DAsync(gc, (size_t)ldgc * 4, 0, (size_t)C * 4, (size_t)n, st));
        ZK_TRY(flow_inverse_backward_chunk(f, x + i0 * ldx, ldx, c ? c + i0 * ldc : nullptr, ldc, n,
                                           grad_x ? grad_x + i0 * ldgx : nullptr, ldgx, grad_log_prob ? grad_log_prob + i0 : nullptr,
                                           z ? z + i0 * ldz : nullptr, ldz, grad_z ? grad_z + i0 * ldgz : nullptr, ldgz, gc,
                                           ldgc, grads, ws, ws_bytes, st));
    }
    return ZK_OK;
}

}  // extern "C"
