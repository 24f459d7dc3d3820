// zuko_b200 — dimension-sequential inverse of a masked autoregressive layer.
//
// The reference inverts  y = f(x | x_<, c)  with `passes` fixed-point sweeps, each running the
// FULL conditioner and the full bijector over all D dims (zuko/transforms.py:994-1000): for
// BASELINE config 4 that is 64 sweeps x 8 layers of a 64-64-64-3008 MLP, although sweep p only
// finalises the dims of order class p.  The masks make the dependency structure explicit
// (zuko/nn.py:270-293, flows/autoregressive.py:121-124): a hidden unit / output row depends on the
// x dims of a bounded order class only, so everything can be evaluated exactly once, in order:
//
//   step p = 0 .. passes-1:
//     every hidden unit whose inputs became final at step p is computed;
//     the P parameter rows of every dim of class p are computed from the last hidden layer;
//     the family's inverse (uni_family.cuh: inverse_ladj, in registers) yields x_d, which is stored and
//     becomes an input of the later steps.
//
// This visits every weight once instead of `passes` times and reproduces the reference's fixed
// point up to summation order (SURVEY §3.2, §7.2).  The same sweep also yields what
// `rsample_and_log_prob` needs (distributions.py:129-138): with the bin of the solved dimension in
// registers, the FORWARD log-derivative at x_d costs a few flops, so the kernel accumulates
// ladj(x) — and, on the first layer it inverts, the base log-density of its input z — instead of
// the reference's second conditioner evaluation (the extra meta(x) of transforms.py:1002-1003).
//
// Mapping: thread = R samples (R = 2 when the state fits: every weight fetched from L1 feeds two
// samples, which takes the inner loop from LDS-bound — 3 shared-memory wavefronts per 8 FMA
// instructions — to 4 per 16), state vectors (c | x, hidden activations) live in shared memory as
// [k][sample].  Every state section is stored SORTED by the step at which an entry becomes final
// (context first, x dims by order class, hidden units by readiness), so the inputs a tile may
// depend on at step p are a PREFIX of its section: the dot products run over that prefix only and
// the weight stream holds only those rows (half the FMAs and half the bytes of full-K tiles).
// The block of a step is staged into shared memory by the whole CTA (coalesced 16-byte loads) and read
// by broadcast.  (Reading it through L1 instead — no barriers, prefetch of the next block — was
// measured 33 % SLOWER on cfg4: with one warp per scheduler every L1 miss of the weight stream is
// exposed, 303 ms against 228 ms.)

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "activations.cuh"
#include "ar_inverse.cuh"
#include "uni_family.cuh"

namespace zk {

struct ArInvPack {
    int D = 0, C = 0, P = 0, uni = 0, kt = 0, passes = 0, act = 1;
    int n_linear = 0;
    std::vector<int> dims;         // n_linear + 1
    std::vector<int> sec_off;      // state section offsets (floats): IN, H1 .. H_{L-1}, end
    int state_floats = 0;
    int max_step_words = 0;
    float* stream = nullptr;       // device: all step blocks
    int* step_off = nullptr;       // device (passes + 1): word offsets of the step blocks
    std::vector<int> h_step_off;
};

namespace {

using namespace bij;

constexpr int TILE = 8;

struct InvParams {
    const float* stream;
    const int* step_off;
    int passes, n_linear, D, C, P;
    int sec_off[9];    // state sections: IN, H1 .. H_{L-1}, end
    int sec_len[8];    // entries per section
    const float* y; int64_t ldy;
    const float* c; int64_t ldc;
    float* x; int64_t ldx;
    int64_t B;
    float bound, aw, ad;
    int act;           // activation between the linear layers: 1 = ReLU, else ZK_ACT_*
    int circ;          // circular RQS (NCSF): CircularShiftTransform(bound) applied to the solved dimension
    float* ladj;       // nullable: per-sample sum of the FORWARD log-derivatives at the solution
    int accumulate;    // ladj += (else =)
    int base;          // 1: also add DiagNormal(loc, scale).log_prob of the input y (distributions.py:129-138); 2: of the output x
    float sign;        // +1: accumulate the forward ladj at the solution; -1: the layer is an inverted flow member
    const float* base_loc; const float* base_scale;
    sosp::Const sosp;  // SOSP: bisection and pre-scaled quadrature of the default shape
    bern::Const bern;  // Bernstein: order, bound, eps and bisection of the default degree
};

// two fp32 FMAs on a pair (fmaf rounding)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// acc[j][.] += sum_{k < K} state[k][sample j] * w[k][.]  over NT 8-row tiles stored k-major
// ([k][NT * 8] weights): one state load per k feeds 8 NT FMAs.  The weights are read by every lane
// from the same address (broadcast).
template <int R, int NT>
__device__ __forceinline__ void tile_dot(const float* __restrict__ w, const float* __restrict__ st, int K, int S, int T,
                                         float2 (&acc)[R][NT * 4]) {
#pragma unroll 2
    for (int k = 0; k < K; ++k) {
        float2 sv[R];
#pragma unroll
        for (int j = 0; j < R; ++j) {
            const float s = st[k * S + j * T];
            sv[j] = make_float2(s, s);
        }
#pragma unroll
        for (int q = 0; q < NT * 2; ++q) {
            const float4 wv = *reinterpret_cast<const float4*>(w + k * (NT * TILE) + 4 * q);
#pragma unroll
            for (int j = 0; j < R; ++j) {
                acc[j][2 * q] = fma2(sv[j], make_float2(wv.x, wv.y), acc[j][2 * q]);
                acc[j][2 * q + 1] = fma2(sv[j], make_float2(wv.z, wv.w), acc[j][2 * q + 1]);
            }
        }
    }
}

// step block (32-bit words, 16-byte aligned sections):
//   header  [n8_0 .. n8_{L-2}] [n_dims] [K_0 .. K_{L-1}] [n2_0 .. n2_{L-2}]      padded to 4
//           n8 / n2: 8-wide and 2-wide hidden tiles of the layer (a fully autoregressive conditioner
//           finalises ONE unit per layer and step: an 8-wide tile would spend 7/8 of its FMAs on padding)
//   dest    per layer: 8 state positions per 8-wide tile, then 2 per 2-wide tile (or -1); padded to 4
//   dims    per dim of this class: feature index d, state position of x_d   (2 words each, padded to 4)
//   tiles   hidden tiles: K_l x 8 weights (k-major over the section's ready prefix) + 8 biases each;
//           then per dim ONE block of its PT tiles: K x (PT * 8) weights k-major + PT * 8 biases
template <int UNI, int KT, bool FAST, int R, bool GACT>
__global__ void __launch_bounds__(256) ar_inverse_kernel(const InvParams p) {
    constexpr int P = UniFamily<UNI>::fixed_P(KT);
    constexpr int PT = (P + TILE - 1) / TILE;  // tiles per dim
    extern __shared__ __align__(16) float state[];  // [state_floats][S], S = R * T samples
    const int T = blockDim.x;
    const int S = R * T;
    const int tid = threadIdx.x;
    const int L = p.n_linear;
    const int64_t row0 = (int64_t)blockIdx.x * S + tid;  // sample j of this thread: row0 + j * T
    bool ok[R];
#pragma unroll
    for (int j = 0; j < R; ++j) ok[j] = row0 + (int64_t)j * T < p.B;
    float* S_in = state + (size_t)p.sec_off[0] * S + tid;
    float* wbuf = state + (size_t)p.sec_off[L] * S;  // one step block

    // sorted input section: context first (always final), then the x dims by order class;
    // x = zeros_like(y) (transforms.py:995)
#pragma unroll
    for (int j = 0; j < R; ++j) {
        const int64_t row = row0 + (int64_t)j * T;
        for (int k = 0; k < p.C; ++k) S_in[k * S + j * T] = ok[j] ? p.c[row * p.ldc + k] : 0.f;
        for (int k = p.C; k < p.C + p.D; ++k) S_in[k * S + j * T] = 0.f;
        for (int l = 1; l < L; ++l) {
            float* Sh = state + (size_t)p.sec_off[l] * S + tid + j * T;
            for (int k = 0; k < p.sec_len[l]; ++k) Sh[k * S] = 0.f;
        }
    }
    float lsum[R];
#pragma unroll
    for (int j = 0; j < R; ++j) lsum[j] = 0.f;

    for (int step = 0; step < p.passes; ++step) {
        const int off = __ldg(p.step_off + step), len = __ldg(p.step_off + step + 1) - off;
        __syncthreads();  // the previous step's weights are no longer read
        {
            const float4* src = reinterpret_cast<const float4*>(p.stream + off);
            float4* dst = reinterpret_cast<float4*>(wbuf);
            for (int i = tid; i < len / 4; i += T) dst[i] = __ldg(src + i);
        }
        __syncthreads();
        const float* blk = wbuf;
        const int* hdr = reinterpret_cast<const int*>(blk);
        const int HW = (3 * L + 3) & ~3;
        const int n_dims = hdr[L - 1];
        int dest_words = 0;
        for (int l = 0; l < L - 1; ++l) dest_words += hdr[l] * TILE + hdr[2 * L + l] * 2;
        dest_words = (dest_words + 3) & ~3;
        const int* dest = hdr + HW;
        const int* dim_ids = dest + dest_words;
        const float* wp = blk + HW + dest_words + ((2 * n_dims + 3) & ~3);
        // ---- hidden units that become final at this step ----
        for (int l = 0; l < L - 1; ++l) {
            const int K = hdr[L + l];
            const float* Sl = state + (size_t)p.sec_off[l] * S + tid;
            float* So = state + (size_t)p.sec_off[l + 1] * S + tid;
            const int n8 = hdr[l], n2 = hdr[2 * L + l];
            for (int t = 0; t < n8; ++t, dest += TILE) {
                float2 acc[R][4];
                const float4 b0 = *reinterpret_cast<const float4*>(wp + K * TILE);  // bias follows the tile
                const float4 b1 = *reinterpret_cast<const float4*>(wp + K * TILE + 4);
#pragma unroll
                for (int j = 0; j < R; ++j) {
                    acc[j][0] = make_float2(b0.x, b0.y); acc[j][1] = make_float2(b0.z, b0.w);
                    acc[j][2] = make_float2(b1.x, b1.y); acc[j][3] = make_float2(b1.z, b1.w);
                }
                tile_dot<R, 1>(wp, Sl, K, S, T, acc);
                wp += (K + 1) * TILE;
#pragma unroll
                for (int i = 0; i < TILE; ++i) {
                    const int u = dest[i];
                    if (u >= 0) {
#pragma unroll
                        for (int j = 0; j < R; ++j) {
                            const float v = (i & 1) ? acc[j][i >> 1].y : acc[j][i >> 1].x;
                            if constexpr (GACT) So[u * S + j * T] = act_apply(v, p.act);  // any ZK_ACT_* (nn.py:264-265)
                            else So[u * S + j * T] = fmaxf(v, 0.f);
                        }
                    }
                }
            }
            for (int t = 0; t < n2; ++t, dest += 2) {  // 2-wide tiles: K x 2 weights (k-major) + 2 biases, padded to 16 bytes
                float2 acc[R];
                const float2 bb = *reinterpret_cast<const float2*>(wp + K * 2);
#pragma unroll
                for (int j = 0; j < R; ++j) acc[j] = bb;
#pragma unroll 4
                for (int k = 0; k < K; ++k) {
                    const float2 wv = *reinterpret_cast<const float2*>(wp + 2 * k);
#pragma unroll
                    for (int j = 0; j < R; ++j) {
                        const float sv = Sl[k * S + j * T];
                        acc[j] = fma2(make_float2(sv, sv), wv, acc[j]);
                    }
                }
                wp += ((K + 1) * 2 + 3) & ~3;
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int u = dest[i];
                    if (u >= 0) {
#pragma unroll
                        for (int j = 0; j < R; ++j) {
                            const float v = i ? acc[j].y : acc[j].x;
                            if constexpr (GACT) So[u * S + j * T] = act_apply(v, p.act);
                            else So[u * S + j * T] = fmaxf(v, 0.f);
                        }
                    }
                }
            }
            // a later layer of this step reads what this layer just wrote — same thread, same
            // column of the state: no barrier needed
        }
        // ---- dims of this order class: parameters -> inverse bijector (+ forward log-derivative) ----
        {
            const int K = hdr[2 * L - 1];  // K_{L-1}
            const float* Sl = state + (size_t)p.sec_off[L - 1] * S + tid;
            for (int i = 0; i < n_dims; ++i) {
                const int d = dim_ids[2 * i], pos = dim_ids[2 * i + 1];
                float yv[R];
#pragma unroll
                for (int j = 0; j < R; ++j)  // issued early: overlaps the dot products
                    yv[j] = ok[j] ? __ldg(p.y + (row0 + (int64_t)j * T) * p.ldy + d) : 0.f;
                float2 acc[R][PT * 4];
                {
                    const float* bp = wp + K * (PT * TILE);  // the dim's PT * 8 biases follow its weights
#pragma unroll
                    for (int q = 0; q < PT * 2; ++q) {
                        const float4 bv = *reinterpret_cast<const float4*>(bp + 4 * q);
#pragma unroll
                        for (int j = 0; j < R; ++j) {
                            acc[j][2 * q] = make_float2(bv.x, bv.y);
                            acc[j][2 * q + 1] = make_float2(bv.z, bv.w);
                        }
                    }
                }
                tile_dot<R, PT>(wp, Sl, K, S, T, acc);
                wp += (K + 1) * (PT * TILE);
                float phi[R][PT * TILE];
#pragma unroll
                for (int j = 0; j < R; ++j)
#pragma unroll
                    for (int q = 0; q < PT * 4; ++q) {
                        phi[j][2 * q] = acc[j][q].x;
                        phi[j][2 * q + 1] = acc[j][q].y;
                    }
                float mu = 0.f, isg = 1.f, lsg = kHalfLog2Pi;
                if (p.base) {
                    const float sg = p.base_scale ? __ldg(p.base_scale + d) : 1.f;
                    mu = p.base_loc ? __ldg(p.base_loc + d) : 0.f;
                    isg = 1.f / sg;
                    lsg = logf(sg) + kHalfLog2Pi;
                }
#pragma unroll
                for (int j = 0; j < R; ++j) {
                    float lj;
                    const float xv = UniFamily<UNI>::template inverse_ladj<KT, FAST>(phi[j], p, yv[j], lj);
                    lj *= p.sign;
                    if (p.base) {
                        const float u = ((p.base == 2 ? xv : yv[j]) - mu) * isg;
                        lj += -0.5f * u * u - lsg;
                    }
                    lsum[j] += lj;
                    S_in[pos * S + j * T] = xv;
                    if (ok[j]) p.x[(row0 + (int64_t)j * T) * p.ldx + d] = xv;
                }
            }
        }
    }
    if (p.ladj != nullptr) {
#pragma unroll
        for (int j = 0; j < R; ++j) {
            const int64_t row = row0 + (int64_t)j * T;
            if (ok[j]) p.ladj[row] = lsum[j] + (p.accumulate ? p.ladj[row] : 0.f);
        }
    }
}

// threads per CTA, samples per thread and shared memory for a pack.  ZK_INV_GEOM=TxR overrides the
// choice (experiments); the default has not been re-tuned since the port to sm_90a.
bool inv_geometry(const ArInvPack* pk, int* threads, int* per_thread, size_t* smem) {
    const size_t per_sample = (size_t)pk->state_floats * 4;
    const size_t wbytes = (size_t)pk->max_step_words * 4 + 16;
    const size_t budget = 226 * 1024;
    auto fits = [&](int T, int R) { return per_sample * T * R + wbytes <= budget; };
    auto set = [&](int T, int R) { *threads = T; *per_thread = R; *smem = per_sample * T * R + wbytes; return true; };
    if (const char* e = getenv("ZK_INV_GEOM")) {
        int T = 0, R = 0;
        const bool r2 = with_family(pk->uni, [](auto fam) { return decltype(fam)::kTwoPerThread; });  // else not compiled
        if (sscanf(e, "%dx%d", &T, &R) == 2 && (R == 1 || (R == 2 && r2)) && T >= 32 && T <= 256 && T % 32 == 0 && fits(T, R)) return set(T, R);
    }
    // two CTAs of 128 samples per SM when they fit (8 warps hide the FMA / LDS latencies of the dot
    // products far better than 4), else one CTA with as many samples as shared memory holds
    if (per_sample * 128 + wbytes <= 112 * 1024) return set(128, 1);
    int T = (int)((budget - std::min(budget, wbytes)) / per_sample);
    T = std::min(256, T / 32 * 32);
    if (T < 32) return false;
    return set(T, 1);
}

}  // namespace

void ar_inverse_free(ArInvPack* pk) {
    if (!pk) return;
    cudaFree(pk->stream);
    cudaFree(pk->step_off);
    delete pk;
}

zk_status ar_inverse_pack(const zk_mlp* m, const uint8_t* const* mask_dev, const int64_t* order, int D, int C,
                          const UniSpec& spec, int passes, ArInvPack** out) {
    *out = nullptr;
    const int L = m->n_linear;
    if (!order || L < 1 || L > 7) return ZK_OK;
    if (!m->plain) return ZK_OK;  // residual blocks use the sweeps
    const int kt = uni_kt<kSequential>(spec);
    if (kt < 0) return ZK_OK;  // no compiled shape
    if (m->dims[0] != D + C) return ZK_OK;
    const int P = uni_P(spec);
    if (m->dims[L] != D * P) return ZK_OK;
    for (int d = 0; d < D; ++d)
        if (order[d] < 0 || order[d] >= passes) return ZK_OK;

    // host copies of the masked weights, biases and masks
    std::vector<std::vector<float>> W_(L), Bv(L);
    std::vector<std::vector<uint8_t>> Mk(L);
    for (int l = 0; l < L; ++l) {
        const size_t n = (size_t)m->dims[l + 1] * m->dims[l];
        W_[l].resize(n);
        Bv[l].resize(m->dims[l + 1]);
        Mk[l].assign(n, 1);
        ZK_CUDA(cudaMemcpy(W_[l].data(), m->w[l], n * 4, cudaMemcpyDeviceToHost));
        ZK_CUDA(cudaMemcpy(Bv[l].data(), m->b[l], (size_t)m->dims[l + 1] * 4, cudaMemcpyDeviceToHost));
        if (mask_dev && mask_dev[l]) ZK_CUDA(cudaMemcpy(Mk[l].data(), mask_dev[l], n, cudaMemcpyDeviceToHost));
    }
    // step at which every unit's inputs are final: 1 + max order class of the x dims it depends on
    std::vector<std::vector<int>> ready(L);
    for (int l = 0; l < L; ++l) {
        const int K = m->dims[l], N = m->dims[l + 1];
        ready[l].assign(N, 0);
        for (int n = 0; n < N; ++n) {
            int r = 0;
            for (int k = 0; k < K; ++k) {
                if (!Mk[l][(size_t)n * K + k]) continue;
                const int rk = (l == 0) ? (k < D ? (int)order[k] + 1 : 0) : ready[l - 1][k];
                r = std::max(r, rk);
            }
            ready[l][n] = r;
        }
    }
    // every parameter row of dim d must be computable at step order[d] (autoregressive property)
    for (int d = 0; d < D; ++d)
        for (int q = 0; q < P; ++q)
            if (ready[L - 1][d * P + q] > order[d]) return ZK_OK;  // not a pure order-class structure

    ArInvPack* pk = new ArInvPack();
    pk->D = D; pk->C = C; pk->P = P; pk->uni = spec.kind; pk->kt = kt; pk->passes = passes; pk->n_linear = L;
    pk->act = m->act;
    pk->dims = m->dims;
    int off = 0;
    pk->sec_off.push_back(off);
    off += D + C;
    for (int l = 1; l < L; ++l) { pk->sec_off.push_back(off); off += m->dims[l]; }
    pk->sec_off.push_back(off);  // end
    pk->state_floats = off;

    // ---- sorted state layout: entry `slot[l][k]` = original index of the k-th entry of section l,
    //      ascending in the step at which it becomes final; avail[l][p] = entries final before step p
    //      computes its tiles of layer l (a tile of step p may read exactly those) ----
    std::vector<std::vector<int>> slot(L), pos(L), fin(L);
    for (int l = 0; l < L; ++l) {
        const int n = (l == 0) ? D + C : m->dims[l];
        fin[l].resize(n);
        for (int k = 0; k < n; ++k)
            fin[l][k] = (l == 0) ? (k < D ? (int)order[k] + 1 : 0) : ready[l - 1][k];
        slot[l].resize(n);
        for (int k = 0; k < n; ++k) slot[l][k] = k;
        std::stable_sort(slot[l].begin(), slot[l].end(), [&](int a, int b) { return fin[l][a] < fin[l][b]; });
        pos[l].resize(n);
        for (int k = 0; k < n; ++k) pos[l][slot[l][k]] = k;
    }
    auto avail = [&](int l, int p) {  // inputs of layer l that are final when step p runs: fin <= p
        int cnt = 0;
        for (int v : fin[l]) cnt += (v <= p) ? 1 : 0;
        return cnt;
    };

    std::vector<float> stream;
    pk->h_step_off.assign(passes + 1, 0);
    const int PT = (P + TILE - 1) / TILE;
    auto as_float = [](int v) { float f; memcpy(&f, &v, 4); return f; };
    for (int step = 0; step < passes; ++step) {
        while (stream.size() % 4) stream.push_back(0.f);
        pk->h_step_off[step] = (int)stream.size();
        std::vector<std::vector<int>> rows(L - 1 > 0 ? L - 1 : 0);
        for (int l = 0; l < L - 1; ++l)
            for (int n = 0; n < m->dims[l + 1]; ++n)
                if (ready[l][n] == step) rows[l].push_back(n);
        std::vector<int> dims_p;
        for (int d = 0; d < D; ++d)
            if (order[d] == step) dims_p.push_back(d);
        std::vector<int> Kl(L);
        for (int l = 0; l < L; ++l) Kl[l] = avail(l, step);
        // header: 8-wide tiles for full groups of 8 units (and remainders of 5..7), 2-wide tiles for remainders of 1..4
        std::vector<int> hdr((3 * L + 3) & ~3, 0);
        std::vector<int> n8(L, 0), n2(L, 0);
        for (int l = 0; l < L - 1; ++l) {
            const int n = (int)rows[l].size(), rem = n % TILE;
            n8[l] = n / TILE + (rem > 4 ? 1 : 0);
            n2[l] = (rem >= 1 && rem <= 4) ? (rem + 1) / 2 : 0;
            hdr[l] = n8[l];
            hdr[2 * L + l] = n2[l];
        }
        hdr[L - 1] = (int)dims_p.size();
        for (int l = 0; l < L; ++l) hdr[L + l] = Kl[l];
        for (int v : hdr) stream.push_back(as_float(v));
        auto unit = [&](int l, size_t i) { return i < rows[l].size() ? rows[l][i] : -1; };
        size_t dest_words = 0;
        for (int l = 0; l < L - 1; ++l) {
            for (int t = 0; t < n8[l]; ++t)
                for (int j = 0; j < TILE; ++j, ++dest_words) {
                    const int r = unit(l, (size_t)t * TILE + j);
                    stream.push_back(as_float(r >= 0 ? pos[l + 1][r] : -1));
                }
            for (int t = 0; t < n2[l]; ++t)
                for (int j = 0; j < 2; ++j, ++dest_words) {
                    const int r = unit(l, (size_t)n8[l] * TILE + (size_t)t * 2 + j);
                    stream.push_back(as_float(r >= 0 ? pos[l + 1][r] : -1));
                }
        }
        for (; dest_words % 4; ++dest_words) stream.push_back(as_float(-1));
        for (size_t i = 0; i < dims_p.size(); ++i) {
            stream.push_back(as_float(dims_p[i]));
            stream.push_back(as_float(pos[0][dims_p[i]]));
        }
        while (stream.size() % 4) stream.push_back(as_float(-1));
        // tile data: K_l x W weights (k-major over the ready prefix of the sorted section) + W biases
        auto emit_tile = [&](int l, const int* row_ids, int W) {
            const int K = m->dims[l];
            for (int k = 0; k < Kl[l]; ++k) {
                const int src = slot[l][k];
                for (int j = 0; j < W; ++j)
                    stream.push_back(row_ids[j] >= 0 && Mk[l][(size_t)row_ids[j] * K + src] ? W_[l][(size_t)row_ids[j] * K + src] : 0.f);
            }
            for (int j = 0; j < W; ++j) stream.push_back(row_ids[j] >= 0 ? Bv[l][row_ids[j]] : 0.f);
            while (stream.size() % 4) stream.push_back(0.f);
        };
        for (int l = 0; l < L - 1; ++l) {
            for (int t = 0; t < n8[l]; ++t) {
                int ids[TILE];
                for (int j = 0; j < TILE; ++j) ids[j] = unit(l, (size_t)t * TILE + j);
                emit_tile(l, ids, TILE);
            }
            for (int t = 0; t < n2[l]; ++t) {
                int ids[2];
                for (int j = 0; j < 2; ++j) ids[j] = unit(l, (size_t)n8[l] * TILE + (size_t)t * 2 + j);
                emit_tile(l, ids, 2);
            }
        }
        for (int d : dims_p) {  // one block per dim: K x (PT * 8) weights k-major, then PT * 8 biases
            const int l = L - 1, K = m->dims[l];
            for (int k = 0; k < Kl[l]; ++k) {
                const int src = slot[l][k];
                for (int q = 0; q < PT * TILE; ++q) {
                    const int row = d * P + q;
                    stream.push_back(q < P && Mk[l][(size_t)row * K + src] ? W_[l][(size_t)row * K + src] : 0.f);
                }
            }
            for (int q = 0; q < PT * TILE; ++q) stream.push_back(q < P ? Bv[l][d * P + q] : 0.f);
        }
    }
    while (stream.size() % 4) stream.push_back(0.f);
    pk->h_step_off[passes] = (int)stream.size();
    for (int step = 0; step < passes; ++step)
        pk->max_step_words = std::max(pk->max_step_words, pk->h_step_off[step + 1] - pk->h_step_off[step]);
    // every weight outside a tile's prefix must be masked out (guaranteed by `ready`): verify
    zk_status st = ZK_OK;
    if (cudaMalloc((void**)&pk->stream, std::max<size_t>(stream.size(), 4) * 4) != cudaSuccess ||
        cudaMalloc((void**)&pk->step_off, (size_t)(passes + 1) * 4) != cudaSuccess)
        st = fail(ZK_ENOMEM, "ar_inverse_pack: cudaMalloc failed");
    if (st == ZK_OK && (cudaMemcpy(pk->stream, stream.data(), stream.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
                        cudaMemcpy(pk->step_off, pk->h_step_off.data(), (size_t)(passes + 1) * 4, cudaMemcpyHostToDevice) != cudaSuccess))
        st = fail(ZK_ECUDA, "ar_inverse_pack: upload failed");
    if (st != ZK_OK) {
        ar_inverse_free(pk);
        return st;
    }
    *out = pk;
    return ZK_OK;
}

bool ar_inverse_threads(const ArInvPack* pk, int* threads, size_t* smem) {
    int R = 0;
    return inv_geometry(pk, threads, &R, smem);
}

bool ar_inverse_geometry(const ArInvPack* pk, int* threads, int* per_thread, size_t* smem) {
    return inv_geometry(pk, threads, per_thread, smem);
}

zk_status launch_ar_inverse(const ArInvPack* pk, const ArInvArgs& a, cudaStream_t st) {
    if (a.B == 0) return ZK_OK;
    int T = 0, R = 0;
    size_t smem = 0;
    ZK_REQUIRE(inv_geometry(pk, &T, &R, &smem), "ar_inverse: state does not fit shared memory");
    InvParams p;
    p.stream = pk->stream; p.step_off = pk->step_off; p.passes = pk->passes; p.n_linear = pk->n_linear;
    p.D = pk->D; p.C = pk->C; p.P = pk->P;
    for (size_t i = 0; i < pk->sec_off.size(); ++i) p.sec_off[i] = pk->sec_off[i];
    p.sec_len[0] = pk->D + pk->C;
    for (int l = 1; l < pk->n_linear; ++l) p.sec_len[l] = pk->dims[l];
    p.y = a.y; p.ldy = a.ldy; p.c = a.c; p.ldc = a.ldc; p.x = a.x; p.ldx = a.ldx; p.B = a.B;
    p.act = pk->act;
    p.ladj = a.ladj; p.accumulate = a.accumulate; p.base = a.base ? (a.as_inverse_member ? 2 : 1) : 0;
    p.sign = a.as_inverse_member ? -1.f : 1.f;
    p.base_loc = a.base_loc; p.base_scale = a.base_scale;
    const int64_t grid = ceil_div(a.B, (int64_t)T * R);
    ZK_REQUIRE(grid <= 0x7fffffff, "ar_inverse: batch too large for one launch");
    ZK_TRY(uni_check_scalars(a.spec, true));
    return uni_dispatch<kSequential>(pk->uni, pk->kt, a.fast, [&](auto fam, auto kt, auto fast) {
        using Fam = decltype(fam);
        set_uni_consts<Fam>(a.spec, p);
        auto go = [&](auto kern) -> zk_status {
            ZK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<(int)grid, T, smem, st>>>(p);
            return check_launch("ar_inverse_kernel");
        };
        // GACT: a general activation (IEEE math in the activation) instead of ReLU
        auto tiled = [&](auto gact) {
            constexpr int K = decltype(kt)::value;
            constexpr bool F = decltype(fast)::value, G = decltype(gact)::value;
            if constexpr (Fam::kTwoPerThread)
                if (R == 2) return go(ar_inverse_kernel<Fam::kKind, K, F, 2, G>);
            return go(ar_inverse_kernel<Fam::kKind, K, F, 1, G>);
        };
        return p.act != 1 ? tiled(std::true_type{}) : tiled(std::false_type{});
    });
}

}  // namespace zk
