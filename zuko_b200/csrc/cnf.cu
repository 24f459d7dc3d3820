// zuko_b200 — continuous normalizing flow (CNF): FreeFormJacobianTransform (zuko/transforms.py:1095-1179) with the
// vector field of FFJTransform.f (zuko/flows/continuous.py:88-97), integrated by the adaptive Dormand-Prince
// method of zuko/utils.py:443-554 with the step size shared by the whole batch.
//
// One cooperative persistent launch per integration.  Every CTA stages the whole MLP in shared memory; each
// thread owns rows (statically strided over the grid) and runs all stages of a trial for them in fp32 FMA.
// Per trial the CTAs fold their rows' error ratios into one device slot (atomic max on the bit pattern of a
// non-negative float, NaN -> +inf), meet at a grid barrier, and all run the same scalar step controller on the
// same maximum, so every CTA takes the same decision without a host round trip.

#include <cooperative_groups.h>

#include <algorithm>
#include <new>
#include <vector>

#include "activations.cuh"
#include "common.cuh"

namespace cg = cooperative_groups;

namespace zk {
namespace cnf {

constexpr int kMaxLinear = 16;
constexpr int kMaxFreqs = 32;
constexpr int kStages = 7;
constexpr size_t kSmemCap = 232448;     // opt-in dynamic shared memory per CTA on sm_90
constexpr size_t kSmemPerSm = 233472;   // shared memory per SM
constexpr int kThreadChoices[] = {256, 128, 64, 32};
constexpr float kTraceScale = 1e-2f;    // transforms.py:1127 (relaxes the tolerance of the ladj column)
constexpr int kCtrlSlots = 3;

// Dormand-Prince tableau (utils.py:454-495), each coefficient the double quotient rounded to fp32 as torch
// does for a Python scalar times an fp32 tensor; subtractions are additions of the negated coefficient
__constant__ float kA[kStages][kStages - 1] = {
    {0.f, 0.f, 0.f, 0.f, 0.f, 0.f},
    {(float)(1. / 5), 0.f, 0.f, 0.f, 0.f, 0.f},
    {(float)(3. / 40), (float)(9. / 40), 0.f, 0.f, 0.f, 0.f},
    {(float)(44. / 45), -(float)(56. / 15), (float)(32. / 9), 0.f, 0.f, 0.f},
    {(float)(19372. / 6561), -(float)(25360. / 2187), (float)(64448. / 6561), -(float)(212. / 729), 0.f, 0.f},
    {(float)(9017. / 3168), -(float)(355. / 33), (float)(46732. / 5247), (float)(49. / 176), -(float)(5103. / 18656), 0.f},
    {(float)(35. / 384), 0.f, (float)(500. / 1113), (float)(125. / 192), -(float)(2187. / 6784), (float)(11. / 84)},
};
__constant__ float kE[kStages] = {(float)(5179. / 57600), 0.f, (float)(7571. / 16695), (float)(393. / 640),
                                  -(float)(92097. / 339200), (float)(187. / 2100), (float)(1. / 40)};
// stage times t + c dt (c = 1 for stages 6 and 7: t + dt)
__constant__ float kC[kStages] = {0.f, (float)(1. / 5), (float)(3. / 10), (float)(4. / 5), (float)(8. / 9), 1.f, 1.f};

struct Params {
    const float* w;  // packed: per layer W^T (in, pad) then bias (pad); then freqs
    int wfloats, nl, act, D, C, F, trace;
    int in[kMaxLinear], pad[kMaxLinear], woff[kMaxLinear], boff[kMaxLinear], dact_off[kMaxLinear];
    int S;  // per-thread slots of each activation buffer
    const float* x; int64_t ldx;
    const float* c; int64_t ldc;
    const float* eps; int64_t ldeps;
    const float* times;
    float atol, rtol;
    int max_trials;
    int64_t B;
    float* y; int64_t ldy;
    float* ladj;
    int* counts;
    float* log;
    float* X;        // (2, W, B) ping-pong state, column-major per row
    float* Fk;       // (7, W, B) stage values of f
    unsigned* ctrl;  // kCtrlSlots error slots
    int W, passes;
};

// bias[o] + sum_j W[o, j] in(j) (0 without bias) for all `pad` outputs, 8 at a time, each block of 8 handed to
// epi(o0, acc)
template <class In, class Epi>
__device__ __forceinline__ void dense_to(const float* __restrict__ WT, int pad, int n_in, const float* __restrict__ bias,
                                         In in, Epi epi) {
    for (int o0 = 0; o0 < pad; o0 += 8) {
        float acc[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) acc[r] = bias ? bias[o0 + r] : 0.f;
        for (int j = 0; j < n_in; ++j) {
            const float v = in(j);
            const float4 w0 = *reinterpret_cast<const float4*>(WT + (size_t)j * pad + o0);
            const float4 w1 = *reinterpret_cast<const float4*>(WT + (size_t)j * pad + o0 + 4);
            acc[0] = fmaf(w0.x, v, acc[0]);
            acc[1] = fmaf(w0.y, v, acc[1]);
            acc[2] = fmaf(w0.z, v, acc[2]);
            acc[3] = fmaf(w0.w, v, acc[3]);
            acc[4] = fmaf(w1.x, v, acc[4]);
            acc[5] = fmaf(w1.y, v, acc[5]);
            acc[6] = fmaf(w1.z, v, acc[6]);
            acc[7] = fmaf(w1.w, v, acc[7]);
        }
        epi(o0, acc);
    }
}

// out[o] = act(bias[o] + sum_j W[o, j] in(j)) (or, without bias, (sum_j W[o, j] in(j)) * scale[o]) for all
// `pad` outputs, 8 at a time; per-thread buffers are strided by nt
template <class In>
__device__ __forceinline__ void dense(const float* __restrict__ WT, int pad, int n_in, const float* __restrict__ bias,
                                      In in, float* out, int nt, int act, float* dact, const float* scale) {
    dense_to(WT, pad, n_in, bias, in, [&](int o0, float (&acc)[8]) {
        if (dact) {
#pragma unroll
            for (int r = 0; r < 8; ++r) dact[(o0 + r) * nt] = act_deriv(acc[r], act);
        }
        if (scale) {
#pragma unroll
            for (int r = 0; r < 8; ++r) acc[r] *= scale[(o0 + r) * nt];
        }
        if (act) act_apply_n<8>(acc, act);
#pragma unroll
        for (int r = 0; r < 8; ++r) out[(o0 + r) * nt] = acc[r];
    });
}

// column j of stage s's state x + sum_m A[s][m] (dt f_m) of one row, f_m in slot(m) of Fk ((slots, W, B)
// column-major); shared by the integration and the backward's replay, so the replayed states are bit for bit
// the integration's
template <class Slot>
__device__ __forceinline__ float stage_state(const float* X, const float* Fk, int W, int64_t B, int64_t row, int j,
                                             int s, float dt, Slot slot) {
    float v = X[(int64_t)j * B + row];
    for (int m = 0; m < s; ++m) {
        const float k = __fmul_rn(dt, Fk[((int64_t)slot(m) * W + j) * B + row]);
        if (kA[s][m] != 0.f) v = __fadd_rn(v, __fmul_rn(kA[s][m], k));
    }
    return v;
}

// time embedding (cos, sin)(freqs t_s) of the 7 stage times of a step (t, dt), by the CTA into emb (7, 2F)
__device__ __forceinline__ void stage_embedding(const float* freqs, int F, float t, float dt, float* emb) {
    for (int k = threadIdx.x; k < kStages * F; k += blockDim.x) {
        const int s = k / F, i = k % F;
        const float ts = __fadd_rn(t, __fmul_rn(kC[s], dt));
        const float a = __fmul_rn(freqs[i], s >= 5 ? __fadd_rn(t, dt) : ts);
        emb[s * 2 * F + i] = cosf(a);
        emb[s * 2 * F + F + i] = sinf(a);
    }
}

// f(t_s, x_s) of one row: x_s and c already in bufA[0 .. D + C); writes f (D) and, with a trace, its
// trace * 1e-2 to the stage slot fs (column-major, row `row`)
__device__ __forceinline__ void eval_row(const Params& p, const float* sw, const float* emb, float* bufA, float* bufB, float* dact,
                         int nt, int64_t row, float* fs) {
    const int F2 = 2 * p.F, nl = p.nl, D = p.D;
    const bool deriv = p.trace != ZK_CNF_TRACE_NONE;
    float* cur = bufA;
    float* nxt = bufB;
    for (int l = 0; l < nl; ++l) {
        const bool last = l == nl - 1;
        const int act = last ? 0 : p.act;
        float* d = (deriv && !last) ? dact + p.dact_off[l] * nt : nullptr;
        if (l == 0) {
            const float* a = cur;
            dense(sw + p.woff[0], p.pad[0], p.in[0], sw + p.boff[0],
                  [&](int j) { return j < F2 ? emb[j] : a[(j - F2) * nt]; }, nxt, nt, act, d, nullptr);
        } else {
            const float* a = cur;
            dense(sw + p.woff[l], p.pad[l], p.in[l], sw + p.boff[l], [&](int j) { return a[j * nt]; }, nxt, nt, act, d,
                  nullptr);
        }
        float* t = cur;
        cur = nxt;
        nxt = t;
    }
    for (int j = 0; j < D; ++j) fs[(int64_t)j * p.B + row] = cur[j * nt];
    if (!deriv) return;

    // forward-mode tangents: T1 = W1[:, x columns] * act'(pre1), T(l+1) = W(l+1) T(l) * act'(pre(l+1)); only the
    // diagonal of the last layer is formed (exact), or the tangent along eps dotted with eps (Hutchinson)
    const float* W0 = sw + p.woff[0];
    const int pad0 = p.pad[0];
    float tr = 0.f;
    const int L = nl - 1;
    const float* WL = sw + p.woff[L];
    const int padL = p.pad[L];
    if (p.trace == ZK_CNF_TRACE_EXACT) {
        for (int i = 0; i < D; ++i) {
            const float* col = W0 + (size_t)(F2 + i) * pad0;
            if (nl == 1) {
                tr += col[i];
                continue;
            }
            for (int o = 0; o < pad0; ++o) bufA[o * nt] = col[o] * dact[o * nt];
            float* a = bufA;
            float* b = bufB;
            for (int l = 1; l < L; ++l) {
                const float* ca = a;
                dense(sw + p.woff[l], p.pad[l], p.in[l], nullptr, [&](int j) { return ca[j * nt]; }, b, nt, 0, nullptr,
                      dact + p.dact_off[l] * nt);
                float* t = a;
                a = b;
                b = t;
            }
            float s = 0.f;
            for (int j = 0; j < p.in[L]; ++j) s = fmaf(WL[(size_t)j * padL + i], a[j * nt], s);
            tr += s;
        }
    } else {
        const float* e = p.eps + row * p.ldeps;
        float* a = bufA;
        float* b = bufB;
        dense(W0 + (size_t)F2 * pad0, pad0, D, nullptr, [&](int j) { return __ldg(e + j); }, a, nt, 0, nullptr,
              nl == 1 ? nullptr : dact);
        for (int l = 1; l < nl; ++l) {
            const float* ca = a;
            dense(sw + p.woff[l], p.pad[l], p.in[l], nullptr, [&](int j) { return ca[j * nt]; }, b, nt, 0, nullptr,
                  l == L ? nullptr : dact + p.dact_off[l] * nt);
            float* t = a;
            a = b;
            b = t;
        }
        for (int i = 0; i < D; ++i) tr = fmaf(__ldg(e + i), a[i * nt], tr);
    }
    fs[(int64_t)D * p.B + row] = tr * kTraceScale;
}

__global__ void __launch_bounds__(256, 1) cnf_dopri_kernel(Params p) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, nt = blockDim.x;
    float* sw = smem;
    float* emb = sw + p.wfloats;                     // (7, 2F) time embedding of the stage times
    float* red = emb + kStages * 2 * kMaxFreqs;      // 32 warp maxima
    float* scr = red + 32 + tid;                     // per-thread buffers, stride nt
    float* bufA = scr;
    float* bufB = scr + (size_t)p.S * nt;
    float* dact = scr + (size_t)2 * p.S * nt;
    for (int k = tid; k < p.wfloats; k += nt) sw[k] = p.w[k];
    const float* freqs = p.w + p.wfloats;

    cg::grid_group grid = cg::this_grid();
    const int64_t stride = (int64_t)gridDim.x * nt;
    const int64_t base = (int64_t)blockIdx.x * nt + tid;
    const int64_t B = p.B;
    const int D = p.D, W = p.W, F2 = 2 * p.F;

    for (int ps = 0; ps < p.passes; ++ps) {
        const int64_t row = base + ps * stride;
        if (row >= B) break;
        for (int j = 0; j < D; ++j) p.X[(int64_t)j * B + row] = p.x[row * p.ldx + j];
        if (W > D) p.X[(int64_t)D * B + row] = 0.f;
    }

    // AdaptiveCheckpointAdjoint.forward, utils.py:532-552, in fp32 (t, dt) with the factor in double
    const float t0 = p.times[0], t1 = p.times[1];
    float t = t0;
    float dt = __fsub_rn(t1, t0);
    const float sign = dt > 0.f ? 1.f : (dt < 0.f ? -1.f : 0.f);
    int par = 0, s1 = 0, s7 = kStages - 1, trials = 0, accepted = 0;
    bool clip = true, failed = false, have_f1 = false;
    while (__fmul_rn(sign, __fsub_rn(t1, t)) > 0.f) {
        if (clip) {
            dt = __fmul_rn(sign, fminf(fabsf(dt), fabsf(__fsub_rn(t1, t))));
            clip = false;
        }
        if (trials >= p.max_trials || __fadd_rn(t, dt) == t) {
            failed = true;
            break;
        }
        __syncthreads();  // the previous trial's readers of emb are done
        stage_embedding(freqs, p.F, t, dt, emb);
        __syncthreads();

        float emax = 0.f;
        const float* Xc = p.X + (size_t)par * W * B;
        float* Xn = p.X + (size_t)(par ^ 1) * W * B;
        auto slot = [&](int m) { return m == 0 ? s1 : (m == kStages - 1 ? s7 : m); };
        for (int ps = 0; ps < p.passes; ++ps) {
            const int64_t row = base + ps * stride;
            if (row >= B) break;
            const float* cr = p.c ? p.c + row * p.ldc : nullptr;
            for (int s = have_f1 ? 1 : 0; s < kStages; ++s) {
                for (int j = 0; j < D; ++j) {
                    const float v = stage_state(Xc, p.Fk, W, B, row, j, s, dt, slot);
                    bufA[j * nt] = v;
                    if (s == kStages - 1) Xn[(int64_t)j * B + row] = v;
                }
                for (int j = 0; j < p.C; ++j) bufA[(D + j) * nt] = __ldg(cr + j);
                eval_row(p, sw, emb + s * F2, bufA, bufB, dact, nt, row, p.Fk + (int64_t)slot(s) * W * B);
            }
            // error of the embedded 4th-order solution, every packed column (ladj included)
            for (int j = 0; j < W; ++j) {
                const float x0 = Xc[(int64_t)j * B + row];
                float xn = x0, xs = x0;
                for (int m = 0; m < kStages; ++m) {
                    const float k = __fmul_rn(dt, p.Fk[((int64_t)slot(m) * W + j) * B + row]);
                    if (m < kStages - 1 && kA[kStages - 1][m] != 0.f) xn = __fadd_rn(xn, __fmul_rn(kA[kStages - 1][m], k));
                    if (kE[m] != 0.f) xs = __fadd_rn(xs, __fmul_rn(kE[m], k));
                }
                if (j == D) Xn[(int64_t)j * B + row] = xn;
                const float err = fabsf(__fsub_rn(xn, xs));
                const float tol = __fadd_rn(p.atol, __fmul_rn(p.rtol, fmaxf(fabsf(x0), fabsf(xn))));
                float r = __fdiv_rn(err, tol);
                if (isnan(r) || isnan(x0) || isnan(xn)) r = INFINITY;
                emax = fmaxf(emax, r);
            }
        }
        // CTA maximum, then one atomic per CTA
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) emax = fmaxf(emax, __shfl_xor_sync(0xffffffffu, emax, o));
        if ((tid & 31) == 0) red[tid >> 5] = emax;
        __syncthreads();
        if (tid == 0) {
            float m = 0.f;
            for (int w = 0; w < (nt + 31) / 32; ++w) m = fmaxf(m, red[w]);
            if (m > 0.f) atomicMax(p.ctrl + trials % kCtrlSlots, __float_as_uint(m));
        }
        grid.sync();
        float e = __uint_as_float(__ldcg(p.ctrl + trials % kCtrlSlots));
        // slot (trials - 1) % 3 was read by every CTA before this barrier and is next used two trials on
        if (blockIdx.x == 0 && tid == 0) p.ctrl[(trials + 2) % kCtrlSlots] = 0u;
        e = fmaxf(e, 1e-9f);  // .clip(min=1e-9)
        const bool accept = e < 1.f;
        if (p.log && blockIdx.x == 0 && tid == 0) {
            float* lg = p.log + (size_t)trials * 4;
            lg[0] = t;
            lg[1] = dt;
            lg[2] = e;
            lg[3] = accept ? 1.f : 0.f;
        }
        if (accept) {
            t = __fadd_rn(t, dt);
            par ^= 1;
            const int sw7 = s1;  // first same as last: f(t + dt, x_next) is the next trial's f(t, x)
            s1 = s7;
            s7 = sw7;
            clip = true;
            ++accepted;
        }
        const double fac = fmin(10.0, fmax(0.1, 0.9 / pow((double)e, 0.2)));
        dt = __fmul_rn(dt, (float)fac);
        ++trials;
        have_f1 = true;
    }

    const float* Xc = p.X + (size_t)par * W * B;
    for (int ps = 0; ps < p.passes; ++ps) {
        const int64_t row = base + ps * stride;
        if (row >= B) break;
        for (int j = 0; j < D; ++j) p.y[row * p.ldy + j] = failed ? NAN : Xc[(int64_t)j * B + row];
        if (p.ladj) p.ladj[row] = failed ? NAN : __fmul_rn(Xc[(int64_t)D * B + row], 100.f);  // * (1 / 1e-2)
    }
    if (p.counts && blockIdx.x == 0 && tid == 0) {
        p.counts[0] = trials;
        p.counts[1] = failed ? -1 - accepted : accepted;
    }
}

// ---------------------------------------------------------------------------
// Backward: AdaptiveCheckpointAdjoint.backward (utils.py:556-593) on the packed state (x, L) of call_and_ladj.
// The accepted steps of the forward's log are known, so rows are independent: each row is replayed from x0
// (cnf_replay_kernel, the integration's own stage arithmetic), then walked back one 6-stage Dormand-Prince step
// of -dt per accepted step (cnf_adjoint_kernel) on (a, g_phi) with
//   da/dt = -(a^T df/dx + a_L 1e-2 dtau/dx),   dg_phi/dt = -(a^T df/dphi + a_L 1e-2 dtau/dphi),
// where tau = sum_k r_k^T (df/dx) s_k (exact: s_k = r_k = e_k, k < D; Hutchinson: s = r = eps) is differentiated
// in reverse mode through the forward-mode tangent program, one tangent at a time, act'' included.  Since g_phi
// never feeds the dynamics, g_phi += dt sum_s b_s VJP_phi(stage s): per stage, every thread adds the CTA's rows
// (in order) of the outer products it owns into the CTA's partial; cnf_grad_reduce_kernel sums the partials in
// CTA order.
// ---------------------------------------------------------------------------
constexpr int kAdjStages = 6;

struct BackParams {
    Params m;   // MLP shape and the chunk's x / c / eps (B = rows of the chunk); m.trace = NONE for the replay
    int trace;  // the differentiated call's trace
    int out[kMaxLinear], hoff[kMaxLinear];
    int H, ns, passes;  // passes: the replay's
    int64_t blk0;       // adjoint: global index of the chunk's first block of blockDim.x rows; block b of the whole
    int gtot;           // call belongs to CTA b % gtot, whatever the chunking (bit-identical partials)
    const float* log;
    int trials, accepted;
    const float* gy; int64_t ldgy;
    const float* gl;
    float* gx; int64_t ldgx;
    float* gc; int64_t ldgc;  // per-row context gradient (ldc != 0) or NULL
    float* Xs;    // (accepted + 1, D, R) replayed states
    float* Fk;    // (7, D, R) stage values of f
    float* Ka;    // (6, D, R) stage values of da/dt
    float* Aa;    // (D, R) adjoint of x
    float* Gc;    // (R, C) context gradient
    float* part;  // (CTAs, wfloats) parameter-gradient partials in the packed weight layout
};

__global__ void __launch_bounds__(256) cnf_replay_kernel(BackParams q) {
    extern __shared__ __align__(16) float smem[];
    const Params& p = q.m;
    const int tid = threadIdx.x, nt = blockDim.x;
    float* sw = smem;
    float* emb = sw + p.wfloats;
    float* bufA = emb + kStages * 2 * kMaxFreqs + tid;
    float* bufB = bufA + (size_t)p.S * nt;
    for (int k = tid; k < p.wfloats; k += nt) sw[k] = p.w[k];
    const float* freqs = p.w + p.wfloats;
    const int64_t R = p.B, stride = (int64_t)gridDim.x * nt, base = (int64_t)blockIdx.x * nt + tid;
    const int D = p.D, F2 = 2 * p.F;
    for (int ps = 0; ps < q.passes; ++ps) {
        const int64_t row = base + ps * stride;
        if (row >= R) break;
        for (int j = 0; j < D; ++j) q.Xs[(int64_t)j * R + row] = p.x[row * p.ldx + j];
    }
    auto same = [](int m) { return m; };
    int k = 0;
    for (int i = 0; i < q.trials && k < q.accepted; ++i) {
        if (q.log[4 * i + 3] == 0.f) continue;
        const float t = q.log[4 * i], dt = q.log[4 * i + 1];
        __syncthreads();
        stage_embedding(freqs, p.F, t, dt, emb);
        __syncthreads();
        const float* Xc = q.Xs + (int64_t)k * D * R;
        float* Xn = q.Xs + (int64_t)(k + 1) * D * R;
        for (int ps = 0; ps < q.passes; ++ps) {
            const int64_t row = base + ps * stride;
            if (row >= R) break;
            const float* cr = p.c ? p.c + row * p.ldc : nullptr;
            for (int s = 0; s < kStages; ++s) {
                for (int j = 0; j < D; ++j) {
                    const float v = stage_state(Xc, q.Fk, D, R, row, j, s, dt, same);
                    if (s == kStages - 1)
                        Xn[(int64_t)j * R + row] = v;
                    else
                        bufA[j * nt] = v;
                }
                if (s == kStages - 1) break;
                for (int j = 0; j < p.C; ++j) bufA[(D + j) * nt] = __ldg(cr + j);
                eval_row(p, sw, emb + s * F2, bufA, bufB, nullptr, nt, row, q.Fk + (int64_t)s * D * R);
            }
        }
        ++k;
    }
}

// v_j = sum_{o < n_out} W[o, j] g[o] for j < n_in (g strided by ns), each handed to epi(j, v)
template <class Epi>
__device__ __forceinline__ void dense_t(const float* WT, int pad, int n_in, int n_out, const float* g, int ns, Epi epi) {
    for (int j = 0; j < n_in; ++j) {
        const float* w = WT + (size_t)j * pad;
        float v = 0.f;
        for (int o = 0; o < n_out; ++o) v = fmaf(w[o], g[o * ns], v);
        epi(j, v);
    }
}

// part[(j0 + j) pad + o] += wgt sum_r g[o][r] in(j, r) over the CTA's live rows r in order, for j < nj, o < n_out;
// g is the CTA's buffer (row r at offset r, stride ns).  Each entry belongs to one thread: bit-reproducible.
template <class In>
__device__ __forceinline__ void reduce_outer(float* part, int pad, int j0, int nj, int n_out, const float* g, int ns,
                                             const int* alive, float wgt, In in) {
    const int nt = blockDim.x;
    for (int e = threadIdx.x; e < nj * n_out; e += nt) {
        const int j = e / n_out, o = e % n_out;
        float s = 0.f;
        for (int r = 0; r < nt; ++r)
            if (alive[r]) s = fmaf(g[o * ns + r], in(j, r), s);
        float* d = part + (size_t)(j0 + j) * pad + o;
        *d = fmaf(wgt, s, *d);
    }
}

__global__ void __launch_bounds__(256, 1) cnf_adjoint_kernel(BackParams q) {
    extern __shared__ __align__(16) float smem[];
    const Params& p = q.m;
    const int tid = threadIdx.x, nt = blockDim.x, ns = q.ns;
    const int D = p.D, C = p.C, F2 = 2 * p.F, nl = p.nl, L = nl - 1, H = q.H, S = p.S;
    const bool tr = q.trace != ZK_CNF_TRACE_NONE, exact = q.trace == ZK_CNF_TRACE_EXACT;
    float* sw = smem;
    float* emb = sw + p.wfloats;
    int* alive = reinterpret_cast<int*>(emb + kStages * 2 * kMaxFreqs);
    // per-row buffers (row r at offset r, stride ns = nt + 1: the reductions read across rows without bank conflicts)
    float* B_in = reinterpret_cast<float*>(alive + nt);  // x_s, c
    float* B_h = B_in + (size_t)(D + C) * ns;            // act(pre) of the hidden layers
    float* B_d = B_h + (size_t)H * ns;                   // act'(pre)
    float* B_g0 = B_d + (size_t)H * ns;                  // three vectors of up to S
    float* B_g1 = B_g0 + (size_t)S * ns;
    float* B_g2 = B_g1 + (size_t)S * ns;
    float* B_d2 = B_g2 + (size_t)S * ns;                 // with a trace: act''(pre)
    float* B_u = B_d2 + (size_t)H * ns;                  // tangent of the hidden pre-activations
    float* B_zb = B_u + (size_t)H * ns;                  // d tau / d pre of the hidden layers
    float* B_e = B_zb + (size_t)H * ns;                  // Hutchinson eps
    float *in = B_in + tid, *h = B_h + tid, *d = B_d + tid, *g0 = B_g0 + tid, *d2 = B_d2 + tid, *u = B_u + tid,
          *zb = B_zb + tid, *e = B_e + tid;
    for (int k = tid; k < p.wfloats; k += nt) sw[k] = p.w[k];
    const float* freqs = p.w + p.wfloats;
    float* part = q.part + (size_t)blockIdx.x * p.wfloats;
    const int64_t R = p.B;
    const float* W0 = sw + p.woff[0];
    const int pad0 = p.pad[0];
    auto same = [](int m) { return m; };

    const int64_t nblk = (R + nt - 1) / nt;
    const int64_t first = q.blk0 + ((blockIdx.x - q.blk0 % q.gtot) % q.gtot + q.gtot) % q.gtot;
    for (int64_t blk = first; blk < q.blk0 + nblk; blk += q.gtot) {  // uniform over the CTA
        const int64_t row = (blk - q.blk0) * nt + tid;
        const bool live = row < R;
        __syncthreads();
        alive[tid] = live;
        float alpha = 0.f;
        const float* cr = nullptr;
        if (live) {
            for (int j = 0; j < D; ++j) q.Aa[(int64_t)j * R + row] = q.gy ? q.gy[row * q.ldgy + j] : 0.f;
            for (int j = 0; j < C; ++j) q.Gc[row * C + j] = 0.f;
            if (tr) alpha = __fmul_rn(__fmul_rn(q.gl[row], 100.f), kTraceScale);  // a_L = gl / 1e-2, times 1e-2
            if (q.trace == ZK_CNF_TRACE_HUTCHINSON)
                for (int j = 0; j < D; ++j) e[j * ns] = p.eps[row * p.ldeps + j];
            cr = p.c ? p.c + row * p.ldc : nullptr;
        }
        int k = q.accepted;
        for (int i = q.trials - 1; i >= 0 && k > 0; --i) {
            if (q.log[4 * i + 3] == 0.f) continue;
            const float dt = q.log[4 * i + 1];
            const float tp = __fadd_rn(q.log[4 * i], dt), hs = -dt;  // from (t + dt, x_k) with step -dt
            __syncthreads();
            stage_embedding(freqs, p.F, tp, hs, emb);
            __syncthreads();
            const float* Xk = q.Xs + (int64_t)k * D * R;
            for (int s = 0; s < kAdjStages; ++s) {
                const float* es = emb + s * F2;
                const float bs = kA[kStages - 1][s];
                const bool wred = bs != 0.f;  // b_1 = 0: that stage feeds the later ones through a only
                const float wgt = __fmul_rn(dt, bs);
                if (live) {
                    for (int j = 0; j < D; ++j) {
                        in[j * ns] = stage_state(Xk, q.Fk, D, R, row, j, s, hs, same);
                        g0[j * ns] = stage_state(q.Aa, q.Ka, D, R, row, j, s, hs, same);
                    }
                    for (int j = 0; j < C; ++j) in[(D + j) * ns] = __ldg(cr + j);
                    // f at the stage, keeping act, act' (and act'') of every hidden layer
                    for (int l = 0; l < nl; ++l) {
                        const float* WT = sw + p.woff[l];
                        const int ho = l < L ? q.hoff[l] : 0;
                        auto epi = [&](int o0, float (&acc)[8]) {
#pragma unroll
                            for (int r = 0; r < 8; ++r) {
                                const int o = o0 + r;
                                if (l == L) {
                                    if (o < D) q.Fk[((int64_t)s * D + o) * R + row] = acc[r];
                                } else {
                                    h[(ho + o) * ns] = act_apply(acc[r], p.act);
                                    d[(ho + o) * ns] = act_deriv(acc[r], p.act);
                                    if (tr) d2[(ho + o) * ns] = act_deriv2(acc[r], p.act);
                                }
                            }
                        };
                        if (l == 0)
                            dense_to(WT, pad0, p.in[0], sw + p.boff[0], [&](int j) { return j < F2 ? es[j] : in[(j - F2) * ns]; }, epi);
                        else {
                            const int hi = q.hoff[l - 1];
                            dense_to(WT, p.pad[l], p.in[l], sw + p.boff[l], [&](int j) { return h[(hi + j) * ns]; }, epi);
                        }
                    }
                    if (tr)
                        for (int o = 0; o < H; ++o) zb[o * ns] = 0.f;
                }
                // the trace term, one tangent at a time: forward tangent u, then back from a_L 1e-2 r
                const int K = tr ? (exact ? D : 1) : 0;
                for (int kk = 0; kk < K; ++kk) {
                    float* ga = B_g1;
                    float* gb = B_g2;
                    if (live) {
                        if (nl > 1) {
                            if (exact)
                                for (int o = 0; o < pad0; ++o) u[o * ns] = W0[(size_t)(F2 + kk) * pad0 + o];
                            else
                                dense_to(W0 + (size_t)F2 * pad0, pad0, D, nullptr, [&](int j) { return e[j * ns]; },
                                         [&](int o0, float (&acc)[8]) {
#pragma unroll
                                             for (int r = 0; r < 8; ++r) u[(o0 + r) * ns] = acc[r];
                                         });
                            for (int l = 1; l < L; ++l) {
                                const int hi = q.hoff[l - 1], ho = q.hoff[l];
                                dense_to(sw + p.woff[l], p.pad[l], p.in[l], nullptr,
                                         [&](int j) { return d[(hi + j) * ns] * u[(hi + j) * ns]; },
                                         [&](int o0, float (&acc)[8]) {
#pragma unroll
                                             for (int r = 0; r < 8; ++r) u[(ho + o0 + r) * ns] = acc[r];
                                         });
                            }
                        }
                        for (int o = 0; o < D; ++o) ga[tid + o * ns] = exact ? (o == kk ? alpha : 0.f) : alpha * e[o * ns];
                    }
                    for (int l = L; l >= 1; --l) {
                        const int hi = q.hoff[l - 1], nin = p.in[l], nout = q.out[l];
                        if (wred) {
                            __syncthreads();
                            reduce_outer(part + p.woff[l], p.pad[l], 0, nin, nout, ga, ns, alive, wgt,
                                         [&](int j, int r) { return B_d[(hi + j) * ns + r] * B_u[(hi + j) * ns + r]; });
                            __syncthreads();
                        }
                        if (live) {
                            float* gbo = gb + tid;
                            dense_t(sw + p.woff[l], p.pad[l], nin, nout, ga + tid, ns, [&](int j, float v) {
                                const int x2 = (hi + j) * ns;
                                zb[x2] = fmaf(u[x2] * v, d2[x2], zb[x2]);
                                gbo[j * ns] = d[x2] * v;
                            });
                        }
                        float* t2 = ga;
                        ga = gb;
                        gb = t2;
                    }
                    if (wred) {
                        __syncthreads();
                        if (exact)
                            reduce_outer(part + p.woff[0], pad0, F2 + kk, 1, q.out[0], ga, ns, alive, wgt,
                                         [](int, int) { return 1.f; });
                        else
                            reduce_outer(part + p.woff[0], pad0, F2, D, q.out[0], ga, ns, alive, wgt,
                                         [&](int j, int r) { return B_e[j * ns + r]; });
                        __syncthreads();
                    }
                }
                // reverse pass of f from a_s, the trace's d/d pre added at every hidden layer
                float* ga = B_g0;
                float* gb = B_g1;
                for (int l = L; l >= 0; --l) {
                    const int nin = p.in[l], nout = q.out[l];
                    const int hi = l > 0 ? q.hoff[l - 1] : 0;
                    if (wred) {
                        __syncthreads();
                        if (l == 0)
                            reduce_outer(part + p.woff[0], pad0, 0, nin + 1, nout, ga, ns, alive, wgt, [&](int j, int r) {
                                return j == nin ? 1.f : (j < F2 ? es[j] : B_in[(j - F2) * ns + r]);
                            });
                        else
                            reduce_outer(part + p.woff[l], p.pad[l], 0, nin + 1, nout, ga, ns, alive, wgt,
                                         [&](int j, int r) { return j == nin ? 1.f : B_h[(hi + j) * ns + r]; });
                        __syncthreads();
                    }
                    if (live) {
                        float* gbo = gb + tid;
                        if (l > 0)
                            dense_t(sw + p.woff[l], p.pad[l], nin, nout, ga + tid, ns, [&](int j, float v) {
                                const int x2 = (hi + j) * ns;
                                gbo[j * ns] = tr ? fmaf(d[x2], v, zb[x2]) : d[x2] * v;
                            });
                        else
                            dense_t(W0 + (size_t)F2 * pad0, pad0, D + C, nout, ga + tid, ns, [&](int j, float v) {
                                if (j < D) {
                                    q.Ka[((int64_t)s * D + j) * R + row] = -v;
                                } else if (wred) {
                                    float* gcp = q.Gc + row * C + (j - D);
                                    *gcp = fmaf(wgt, v, *gcp);
                                }
                            });
                    }
                    float* t2 = ga;
                    ga = gb;
                    gb = t2;
                }
            }
            if (live)
                for (int j = 0; j < D; ++j)
                    q.Aa[(int64_t)j * R + row] = stage_state(q.Aa, q.Ka, D, R, row, j, kStages - 1, hs, same);
            --k;
        }
        if (live) {
            if (q.gx)
                for (int j = 0; j < D; ++j) q.gx[row * q.ldgx + j] = q.Aa[(int64_t)j * R + row];
            if (q.gc)
                for (int j = 0; j < C; ++j) q.gc[row * q.ldgc + j] = q.Gc[row * C + j];
        }
    }
}

struct GradOut {
    float* gw[kMaxLinear];
    float* gb[kMaxLinear];
    int in[kMaxLinear], out[kMaxLinear], pad[kMaxLinear], woff[kMaxLinear];
    int nl, wfloats, ctas;
    const float* part;
};

// one thread per packed entry: the CTA partials summed in CTA order, added into the (out, in) / (out) buffers
__global__ void cnf_grad_reduce_kernel(GradOut g) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.wfloats) return;
    int l = g.nl - 1;
    while (l > 0 && e < g.woff[l]) --l;
    const int rel = e - g.woff[l], j = rel / g.pad[l], o = rel % g.pad[l];
    if (o >= g.out[l]) return;
    float* dst = j < g.in[l] ? (g.gw[l] ? g.gw[l] + (size_t)o * g.in[l] + j : nullptr) : (g.gb[l] ? g.gb[l] + o : nullptr);
    if (!dst) return;
    float s = 0.f;
    for (int c = 0; c < g.ctas; ++c) s += g.part[(size_t)c * g.wfloats + e];
    *dst += s;
}

// grad_c (C) += the chunk's rows, one after the other in row order (a broadcast context): the same sequence of
// additions whatever the chunking
__global__ void cnf_context_sum_kernel(const float* Gc, int64_t R, int C, float* gc) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= C) return;
    float s = gc[j];
    for (int64_t r = 0; r < R; ++r) s += Gc[r * C + j];
    gc[j] = s;
}

}  // namespace cnf
}  // namespace zk

struct zk_cnf {
    int nl = 0, D = 0, C = 0, F = 0, act = 1;
    std::vector<int> dims, pad, woff, boff;
    int wfloats = 0, hidden_pad = 0, S = 0;
    float* w = nullptr;  // device, owned: packed weights then freqs
};

using namespace zk;

namespace {

size_t cnf_fixed_smem(const zk_cnf* h) { return ((size_t)h->wfloats + cnf::kStages * 2 * cnf::kMaxFreqs + 32) * 4; }

// per-thread floats: two activation buffers of S slots, and act'(pre) of every hidden layer with a trace
int cnf_thread_floats(const zk_cnf* h, int trace) { return 2 * h->S + (trace ? h->hidden_pad : 0); }

// threads per CTA: the choice with the most resident threads per SM by shared memory, ties to more threads
zk_status cnf_geometry(const zk_cnf* h, int trace, int* threads, size_t* smem) {
    int best = 0;
    size_t best_smem = 0;
    int64_t best_res = 0;
    for (int nt : cnf::kThreadChoices) {
        const size_t s = cnf_fixed_smem(h) + (size_t)nt * cnf_thread_floats(h, trace) * 4;
        if (s > cnf::kSmemCap) continue;
        const int64_t per_sm = std::min<int64_t>({(int64_t)(cnf::kSmemPerSm / (s + 1024)), 2048 / nt, 32});
        if (per_sm * nt > best_res) {
            best_res = per_sm * nt;
            best = nt;
            best_smem = s;
        }
    }
    if (!best)
        return fail(ZK_EUNSUPPORTED, "cnf: the MLP does not fit in shared memory (%zu bytes of weights, %d floats per row)",
                    (size_t)h->wfloats * 4, cnf_thread_floats(h, trace));
    *threads = best;
    *smem = best_smem;
    return ZK_OK;
}

zk_status cnf_ctas(int threads, size_t smem, int* ctas) {
    ZK_CUDA(cudaFuncSetAttribute(cnf::cnf_dopri_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    ZK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cnf::cnf_dopri_kernel, threads, smem));
    if (per_sm <= 0) return fail(ZK_EUNSUPPORTED, "cnf: no CTA of %d threads and %zu bytes fits an SM", threads, smem);
    *ctas = per_sm * sm_count();
    return ZK_OK;
}

size_t cnf_ws(const zk_cnf* h, int64_t B, int trace) {
    const int64_t W = h->D + (trace ? 1 : 0);
    return 256 + align_up((size_t)2 * W * B * 4, 256) + align_up((size_t)cnf::kStages * W * B * 4, 256);
}

}  // namespace

extern "C" {

zk_status zk_cnf_create(const zk_mlp_desc* ode, int features, int context, int freqs, const float* freq_values,
                        zk_cnf** out) {
    ZK_REQUIRE(ode && out, "cnf_create: null argument");
    *out = nullptr;
    ZK_REQUIRE(features >= 1 && context >= 0, "cnf_create: features=%d context=%d", features, context);
    ZK_REQUIRE(freqs >= 0 && freqs <= cnf::kMaxFreqs, "cnf_create: freqs=%d outside [0, %d]", freqs, cnf::kMaxFreqs);
    ZK_REQUIRE(freqs == 0 || freq_values, "cnf_create: null freq_values");
    ZK_REQUIRE(ode->n_linear >= 1 && ode->dims && ode->weight, "cnf_create: bad MLP descriptor");
    if (ode->n_linear > cnf::kMaxLinear)
        return fail(ZK_EUNSUPPORTED, "cnf_create: %d linear layers (at most %d)", ode->n_linear, cnf::kMaxLinear);
    ZK_REQUIRE(ode->activation >= 0 && ode->activation <= ZK_ACT_SIGMOID && ode->activation != 1,
               "cnf_create: unknown activation %d", ode->activation);
    if (ode->layer_act || ode->layer_res) return fail(ZK_EUNSUPPORTED, "cnf_create: residual blocks are not supported");
    const int nl = ode->n_linear;
    ZK_REQUIRE(ode->dims[0] == features + context + 2 * freqs && ode->dims[nl] == features,
               "cnf_create: MLP widths %d -> %d do not match features + context + 2 freqs -> features", ode->dims[0],
               ode->dims[nl]);
    for (int l = 0; l < nl; ++l) {
        ZK_REQUIRE(ode->dims[l + 1] >= 1 && ode->weight[l], "cnf_create: bad layer %d", l);
        if (ode->mask && ode->mask[l]) return fail(ZK_EUNSUPPORTED, "cnf_create: masked layers are not supported");
    }
    zk_cnf* h = new (std::nothrow) zk_cnf();
    if (!h) return fail(ZK_ENOMEM, "cnf_create: out of host memory");
    h->nl = nl;
    h->D = features;
    h->C = context;
    h->F = freqs;
    h->act = ode->activation == ZK_ACT_RELU ? 1 : ode->activation;
    h->dims.assign(ode->dims, ode->dims + nl + 1);
    int off = 0, S = features + context;
    for (int l = 0; l < nl; ++l) {
        const int pad = (int)align_up(h->dims[l + 1], 8);
        h->pad.push_back(pad);
        h->woff.push_back(off);
        off += h->dims[l] * pad;
        h->boff.push_back(off);
        off += pad;
        S = std::max(S, pad);
        if (l < nl - 1) h->hidden_pad += pad;
    }
    h->wfloats = off;
    h->S = S;
    std::vector<float> pack((size_t)off + freqs, 0.f), wl;
    // the weights may still be written by work queued on any stream: creation is not on the hot path
    cudaError_t e = cudaDeviceSynchronize();
    for (int l = 0; l < nl && e == cudaSuccess; ++l) {
        const int in = h->dims[l], o = h->dims[l + 1];
        wl.resize((size_t)in * o);
        e = cudaMemcpy(wl.data(), ode->weight[l], wl.size() * 4, cudaMemcpyDeviceToHost);
        for (int r = 0; r < o; ++r)
            for (int j = 0; j < in; ++j) pack[h->woff[l] + (size_t)j * h->pad[l] + r] = wl[(size_t)r * in + j];
        if (e == cudaSuccess && ode->bias && ode->bias[l])
            e = cudaMemcpy(pack.data() + h->boff[l], ode->bias[l], (size_t)o * 4, cudaMemcpyDeviceToHost);
    }
    if (e == cudaSuccess && freqs) e = cudaMemcpy(pack.data() + off, freq_values, (size_t)freqs * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMalloc((void**)&h->w, pack.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpy(h->w, pack.data(), pack.size() * 4, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(h->w);
        delete h;
        return fail(ZK_ECUDA, "cnf_create: %s", cudaGetErrorString(e));
    }
    *out = h;
    return ZK_OK;
}

zk_status zk_cnf_destroy(zk_cnf* h) {
    if (!h) return ZK_OK;
    cudaFree(h->w);
    delete h;
    return ZK_OK;
}

size_t zk_cnf_workspace_bytes(const zk_cnf* h, int64_t B, int trace) {
    if (!h || B < 0) return 0;
    return cnf_ws(h, B, trace != ZK_CNF_TRACE_NONE);
}

zk_status zk_cnf_plan(const zk_cnf* h, int64_t B, int trace, int* ctas, int* threads, int* passes, size_t* smem) {
    ZK_REQUIRE(h && B >= 0, "cnf_plan: bad argument");
    ZK_REQUIRE(trace >= ZK_CNF_TRACE_NONE && trace <= ZK_CNF_TRACE_HUTCHINSON, "cnf_plan: unknown trace %d", trace);
    int nt = 0, g = 0;
    size_t s = 0;
    ZK_TRY(cnf_geometry(h, trace != ZK_CNF_TRACE_NONE, &nt, &s));
    ZK_TRY(cnf_ctas(nt, s, &g));
    if (ctas) *ctas = g;
    if (threads) *threads = nt;
    if (passes) *passes = (int)ceil_div(B, (int64_t)g * nt);
    if (smem) *smem = s;
    return ZK_OK;
}

zk_status zk_cnf_integrate(const zk_cnf* h, const float* x, int64_t ldx, const float* c, int64_t ldc, int64_t B,
                           const float* times, float atol, float rtol, int trace, const float* eps, int64_t ldeps,
                           int max_trials, float* y, int64_t ldy, float* ladj, int* counts, float* step_log,
                           void* workspace, size_t ws_bytes, zk_stream stream) {
    ZK_REQUIRE(h, "cnf_integrate: null handle");
    ZK_REQUIRE(B >= 0, "cnf_integrate: B=%lld", (long long)B);
    ZK_REQUIRE(trace >= ZK_CNF_TRACE_NONE && trace <= ZK_CNF_TRACE_HUTCHINSON, "cnf_integrate: unknown trace %d", trace);
    ZK_REQUIRE((trace == ZK_CNF_TRACE_NONE) == (ladj == nullptr), "cnf_integrate: ladj must be NULL iff trace is NONE");
    ZK_REQUIRE(trace != ZK_CNF_TRACE_HUTCHINSON || (eps && ldeps >= h->D), "cnf_integrate: Hutchinson needs eps (B, D)");
    ZK_REQUIRE(max_trials >= 1, "cnf_integrate: max_trials=%d", max_trials);
    ZK_REQUIRE(times, "cnf_integrate: null times");
    if (B == 0) return ZK_OK;
    ZK_REQUIRE(x && y && ldx >= h->D && ldy >= h->D, "cnf_integrate: bad x / y");
    ZK_REQUIRE(h->C == 0 || (c && (ldc == 0 || ldc >= h->C)), "cnf_integrate: bad context");
    const size_t need = cnf_ws(h, B, trace != ZK_CNF_TRACE_NONE);
    ZK_REQUIRE(workspace && ws_bytes >= need && ((uintptr_t)workspace & 255) == 0,
               "cnf_integrate: workspace of %zu bytes (256-byte aligned) needed, %zu given", need, ws_bytes);
    int nt = 0, g = 0;
    size_t s = 0;
    ZK_TRY(cnf_geometry(h, trace != ZK_CNF_TRACE_NONE, &nt, &s));
    ZK_TRY(cnf_ctas(nt, s, &g));

    cnf::Params p{};
    p.w = h->w;
    p.wfloats = h->wfloats;
    p.nl = h->nl;
    p.act = h->act;
    p.D = h->D;
    p.C = h->C;
    p.F = h->F;
    p.trace = trace;
    int doff = 0;
    for (int l = 0; l < h->nl; ++l) {
        p.in[l] = h->dims[l];
        p.pad[l] = h->pad[l];
        p.woff[l] = h->woff[l];
        p.boff[l] = h->boff[l];
        p.dact_off[l] = doff;
        if (l < h->nl - 1) doff += h->pad[l];
    }
    p.S = h->S;
    p.x = x;
    p.ldx = ldx;
    p.c = h->C ? c : nullptr;
    p.ldc = ldc;
    p.eps = eps;
    p.ldeps = ldeps;
    p.times = times;
    p.atol = atol;
    p.rtol = rtol;
    p.max_trials = max_trials;
    p.B = B;
    p.y = y;
    p.ldy = ldy;
    p.ladj = ladj;
    p.counts = counts;
    p.log = step_log;
    p.W = h->D + (trace != ZK_CNF_TRACE_NONE ? 1 : 0);
    char* ws = (char*)workspace;
    p.ctrl = (unsigned*)ws;
    p.X = (float*)(ws + 256);
    p.Fk = (float*)(ws + 256 + align_up((size_t)2 * p.W * B * 4, 256));
    p.passes = (int)ceil_div(B, (int64_t)g * nt);
    cudaStream_t st = (cudaStream_t)stream;
    ZK_CUDA(cudaMemsetAsync(p.ctrl, 0, cnf::kCtrlSlots * sizeof(unsigned), st));
    void* args[] = {&p};
    ZK_CUDA(cudaLaunchCooperativeKernel((const void*)cnf::cnf_dopri_kernel, dim3(g), dim3(nt), args, s, st));
    return check_launch("cnf_dopri_kernel");
}

}  // extern "C"

namespace {

// per-row floats of the adjoint kernel: x_s and c, act and act' of the hidden layers, three vectors of S, and
// with a trace act'', the tangent, d tau / d pre and eps
int cnf_back_thread_floats(const zk_cnf* h, int trace) {
    return h->D + h->C + 2 * h->hidden_pad + 3 * h->S + (trace ? 3 * h->hidden_pad + h->D : 0);
}

size_t cnf_back_smem(const zk_cnf* h, int trace, int nt) {
    return ((size_t)h->wfloats + cnf::kStages * 2 * cnf::kMaxFreqs + nt + (size_t)(nt + 1) * cnf_back_thread_floats(h, trace)) * 4;
}

size_t cnf_replay_smem(const zk_cnf* h, int nt) {
    return ((size_t)h->wfloats + cnf::kStages * 2 * cnf::kMaxFreqs + (size_t)nt * 2 * h->S) * 4;
}

// threads per CTA by cnf_geometry's rule (the most resident threads per SM by shared memory, ties to more
// threads), and co-resident CTAs of the adjoint kernel
zk_status cnf_back_geometry(const zk_cnf* h, int trace, int* threads, size_t* smem, int* ctas) {
    int best = 0;
    size_t best_smem = 0;
    int64_t best_res = 0;
    for (int nt : cnf::kThreadChoices) {
        const size_t s = cnf_back_smem(h, trace, nt);
        if (s > cnf::kSmemCap) continue;
        const int64_t per_sm = std::min<int64_t>({(int64_t)(cnf::kSmemPerSm / (s + 1024)), 2048 / nt, 32});
        if (per_sm * nt > best_res) {
            best_res = per_sm * nt;
            best = nt;
            best_smem = s;
        }
    }
    if (!best)
        return fail(ZK_EUNSUPPORTED, "cnf_backward: the MLP's backward state does not fit in shared memory (%zu bytes of "
                    "weights, %d floats per row)", (size_t)h->wfloats * 4, cnf_back_thread_floats(h, trace));
    ZK_CUDA(cudaFuncSetAttribute(cnf::cnf_adjoint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)best_smem));
    ZK_CUDA(cudaFuncSetAttribute(cnf::cnf_replay_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)cnf_replay_smem(h, best)));
    int per_sm = 0;
    ZK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cnf::cnf_adjoint_kernel, best, best_smem));
    if (per_sm <= 0) return fail(ZK_EUNSUPPORTED, "cnf_backward: no CTA of %d threads and %zu bytes fits an SM", best, best_smem);
    *threads = best;
    *smem = best_smem;
    *ctas = per_sm * sm_count();
    return ZK_OK;
}

// workspace: the CTA partials, then per chunk row the replayed states, the stage values of f and da/dt, a and
// the context gradient (five 256-byte aligned arrays)
size_t cnf_back_fixed(const zk_cnf* h, int ctas) { return align_up((size_t)ctas * h->wfloats * 4, 256) + 5 * 256; }
size_t cnf_back_row_bytes(const zk_cnf* h, int accepted) {
    return ((size_t)(accepted + 1 + cnf::kStages + cnf::kAdjStages + 1) * h->D + h->C) * 4;
}

size_t cnf_back_ws(const zk_cnf* h, int64_t rows, int trace, int accepted) {
    int nt = 0, g = 0;
    size_t s = 0;
    if (!h || rows < 0 || accepted < 0 || cnf_back_geometry(h, trace != ZK_CNF_TRACE_NONE, &nt, &s, &g) != ZK_OK) return 0;
    return cnf_back_fixed(h, g) + (size_t)rows * cnf_back_row_bytes(h, accepted);
}

}  // namespace

extern "C" {

size_t zk_cnf_backward_workspace_bytes(const zk_cnf* h, int64_t B, int trace, int accepted) {
    return cnf_back_ws(h, B, trace, accepted);
}

size_t zk_cnf_backward_min_workspace_bytes(const zk_cnf* h, int trace, int accepted) {
    int nt = 0, g = 0;
    size_t s = 0;
    if (!h || cnf_back_geometry(h, trace != ZK_CNF_TRACE_NONE, &nt, &s, &g) != ZK_OK) return 0;
    return cnf_back_ws(h, nt, trace, accepted);
}

zk_status zk_cnf_backward_plan(const zk_cnf* h, int64_t B, int trace, int accepted, size_t ws_bytes, int* ctas,
                               int* threads, int64_t* chunk_rows, size_t* smem) {
    ZK_REQUIRE(h && B >= 0 && accepted >= 0, "cnf_backward_plan: bad argument");
    ZK_REQUIRE(trace >= ZK_CNF_TRACE_NONE && trace <= ZK_CNF_TRACE_HUTCHINSON, "cnf_backward_plan: unknown trace %d", trace);
    int nt = 0, g = 0;
    size_t s = 0;
    ZK_TRY(cnf_back_geometry(h, trace != ZK_CNF_TRACE_NONE, &nt, &s, &g));
    const size_t fixed = cnf_back_fixed(h, g), row = cnf_back_row_bytes(h, accepted);
    int64_t rows = 0;
    if (B > 0) {  // whole blocks of nt rows per chunk, so that every row meets the same CTA whatever the chunking
        const size_t least = fixed + (size_t)std::min<int64_t>(B, nt) * row;
        ZK_REQUIRE(ws_bytes >= least, "cnf_backward_plan: workspace of %zu bytes given, %zu needed at least", ws_bytes, least);
        const int64_t fit = (int64_t)((ws_bytes - fixed) / row);
        rows = fit >= B ? B : fit / nt * nt;
    }
    if (ctas) *ctas = g;
    if (threads) *threads = nt;
    if (chunk_rows) *chunk_rows = rows;
    if (smem) *smem = s;
    return ZK_OK;
}

zk_status zk_cnf_backward(const zk_cnf* h, const float* x, int64_t ldx, const float* c, int64_t ldc, int64_t B,
                          const float* step_log, int trials, int accepted, int trace, const float* eps, int64_t ldeps,
                          const float* grad_y, int64_t ldgy, const float* grad_ladj, float* grad_x, int64_t ldgx,
                          float* grad_c, int64_t ldgc, const zk_layer_grads* grads, void* workspace, size_t ws_bytes,
                          zk_stream stream) {
    ZK_REQUIRE(h, "cnf_backward: null handle");
    ZK_REQUIRE(B >= 0, "cnf_backward: B=%lld", (long long)B);
    ZK_REQUIRE(trace >= ZK_CNF_TRACE_NONE && trace <= ZK_CNF_TRACE_HUTCHINSON, "cnf_backward: unknown trace %d", trace);
    ZK_REQUIRE(trials >= 0 && accepted >= 0 && accepted <= trials, "cnf_backward: trials=%d accepted=%d", trials, accepted);
    ZK_REQUIRE(trials == 0 || step_log, "cnf_backward: null step_log");
    ZK_REQUIRE((trace == ZK_CNF_TRACE_NONE) == (grad_ladj == nullptr),
               "cnf_backward: grad_ladj must be NULL iff trace is NONE");
    ZK_REQUIRE((trace == ZK_CNF_TRACE_HUTCHINSON) == (eps != nullptr) && (!eps || ldeps >= h->D),
               "cnf_backward: eps (B, D) must be given iff trace is HUTCHINSON");
    ZK_REQUIRE(!grad_y || ldgy >= h->D, "cnf_backward: ldgy=%lld", (long long)ldgy);
    ZK_REQUIRE(!grad_x || ldgx >= h->D, "cnf_backward: ldgx=%lld", (long long)ldgx);
    ZK_REQUIRE(h->C == 0 || (c && (ldc == 0 || ldc >= h->C)), "cnf_backward: bad context");
    ZK_REQUIRE(!grad_c || h->C == 0 || ldc == 0 || ldgc >= h->C, "cnf_backward: ldgc=%lld", (long long)ldgc);
    ZK_REQUIRE(B == 0 || (x && ldx >= h->D), "cnf_backward: bad x");
    int nt = 0, g = 0;
    size_t s = 0;
    int64_t R = 0;
    ZK_REQUIRE(((uintptr_t)workspace & 255) == 0, "cnf_backward: the workspace must be 256-byte aligned");
    ZK_TRY(zk_cnf_backward_plan(h, B, trace, accepted, ws_bytes, &g, &nt, &R, &s));
    ZK_REQUIRE(B == 0 || workspace, "cnf_backward: null workspace");
    cudaStream_t st = (cudaStream_t)stream;
    const int C = h->C;
    const bool csum = grad_c && C && ldc == 0;
    if (csum) ZK_CUDA(cudaMemsetAsync(grad_c, 0, (size_t)C * 4, st));
    if (B == 0) return ZK_OK;

    char* ws = (char*)workspace;
    float* part = (float*)ws;
    ZK_CUDA(cudaMemsetAsync(part, 0, (size_t)g * h->wfloats * 4, st));
    char* rows = ws + align_up((size_t)g * h->wfloats * 4, 256);
    const int D = h->D;
    float* Xs = (float*)rows;
    float* Fk = (float*)((char*)Xs + align_up((size_t)(accepted + 1) * D * R * 4, 256));
    float* Ka = (float*)((char*)Fk + align_up((size_t)cnf::kStages * D * R * 4, 256));
    float* Aa = (float*)((char*)Ka + align_up((size_t)cnf::kAdjStages * D * R * 4, 256));
    float* Gc = (float*)((char*)Aa + align_up((size_t)D * R * 4, 256));

    cnf::BackParams q{};
    cnf::Params& p = q.m;
    p.w = h->w;
    p.wfloats = h->wfloats;
    p.nl = h->nl;
    p.act = h->act;
    p.D = D;
    p.C = C;
    p.F = h->F;
    p.trace = ZK_CNF_TRACE_NONE;  // the replay integrates x alone
    q.trace = trace;
    int hoff = 0;
    for (int l = 0; l < h->nl; ++l) {
        p.in[l] = h->dims[l];
        p.pad[l] = h->pad[l];
        p.woff[l] = h->woff[l];
        p.boff[l] = h->boff[l];
        q.out[l] = h->dims[l + 1];
        q.hoff[l] = hoff;
        if (l < h->nl - 1) hoff += h->pad[l];
    }
    p.S = h->S;
    p.W = D;
    q.H = h->hidden_pad;
    q.ns = nt + 1;
    q.log = step_log;
    q.trials = trials;
    q.accepted = accepted;
    q.Xs = Xs;
    q.Fk = Fk;
    q.Ka = Ka;
    q.Aa = Aa;
    q.Gc = Gc;
    q.part = part;
    const size_t replay_smem = cnf_replay_smem(h, nt);
    q.gtot = (int)std::min<int64_t>(g, ceil_div(B, nt));
    for (int64_t r0 = 0; r0 < B; r0 += R) {
        const int64_t Rc = std::min<int64_t>(R, B - r0);
        p.B = Rc;
        p.x = x + r0 * ldx;
        p.ldx = ldx;
        p.c = C ? c + (ldc ? r0 * ldc : 0) : nullptr;
        p.ldc = ldc;
        p.eps = eps ? eps + r0 * ldeps : nullptr;
        p.ldeps = ldeps;
        q.gy = grad_y ? grad_y + r0 * ldgy : nullptr;
        q.ldgy = ldgy;
        q.gl = grad_ladj ? grad_ladj + r0 : nullptr;
        q.gx = grad_x ? grad_x + r0 * ldgx : nullptr;
        q.ldgx = ldgx;
        q.gc = grad_c && C && ldc ? grad_c + r0 * ldgc : nullptr;
        q.ldgc = ldgc;
        const int grid = (int)std::min<int64_t>(g, ceil_div(Rc, nt));
        q.passes = (int)ceil_div(Rc, (int64_t)grid * nt);
        q.blk0 = r0 / nt;
        cnf::cnf_replay_kernel<<<grid, nt, replay_smem, st>>>(q);
        ZK_TRY(check_launch("cnf_replay_kernel"));
        cnf::cnf_adjoint_kernel<<<q.gtot, nt, s, st>>>(q);
        ZK_TRY(check_launch("cnf_adjoint_kernel"));
        if (csum) {
            cnf::cnf_context_sum_kernel<<<(C + 127) / 128, 128, 0, st>>>(Gc, Rc, C, grad_c);
            ZK_TRY(check_launch("cnf_context_sum_kernel"));
        }
    }
    if (grads && (grads->grad_weight || grads->grad_bias)) {
        cnf::GradOut go{};
        for (int l = 0; l < h->nl; ++l) {
            go.gw[l] = grads->grad_weight ? grads->grad_weight[l] : nullptr;
            go.gb[l] = grads->grad_bias ? grads->grad_bias[l] : nullptr;
            go.in[l] = h->dims[l];
            go.out[l] = h->dims[l + 1];
            go.pad[l] = h->pad[l];
            go.woff[l] = h->woff[l];
        }
        go.nl = h->nl;
        go.wfloats = h->wfloats;
        go.ctas = g;
        go.part = part;
        cnf::cnf_grad_reduce_kernel<<<(h->wfloats + 255) / 256, 256, 0, st>>>(go);
        ZK_TRY(check_launch("cnf_grad_reduce_kernel"));
    }
    return ZK_OK;
}

}  // extern "C"
