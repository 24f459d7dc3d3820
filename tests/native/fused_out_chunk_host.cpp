// Host replay of the output-chunk path of fused_layer_kernel (zuko_b200/csrc/fused_layer.cu): the pack's column
// order of an output chunk and the quad exchange that gives each consumer thread its (row, slot)'s parameters, both
// from zuko_b200/csrc/fused_out_chunk.cuh.
//
// For every chunk of a packed output layer it fills a 64-row chunk of the output layer with values that name their
// (sample row, unpacked output row), or a pad marker, lays them out as the m64nNL wgmma accumulator fragment of a
// consumer warpgroup, and runs the kernel's `assemble` for all 128 threads at once: a warp shuffle is replayed by
// re-running every lane until what each lane sends no longer changes (the exchanges are at most two deep).  Each
// lane's values are then held against the staging order the chunk's parameters are evaluated in.

#include <stdio.h>

#include <vector>

#include "../../zuko_b200/csrc/fused_out_chunk.cuh"

namespace {

using namespace zk;

constexpr int FK = 64;
constexpr float PAD = -1.f;  // value of a packed column that holds no parameter

float encode(int row, int unpacked) { return (float)(row * 65536 + unpacked); }

template <int P, int DPC, int NL>
int check(int D, char* msg, int n) {
    using S = outchunk::Shape<P, DPC>;
    constexpr int NA = NL / 2;
    const int n_last = (D + DPC - 1) / DPC;
    std::vector<int> lr(n_last * FK);
    outchunk::last_rows(D, P, DPC, n_last, lr.data());
    // the pack permutes rows only within a chunk, and only into the columns its MMAs cover
    std::vector<int> seen(D * P, 0);
    for (int ch = 0; ch < n_last; ++ch)
        for (int c = 0; c < FK; ++c) {
            const int u = lr[ch * FK + c];
            if (u < 0) continue;
            if (u >= D * P || u / P / DPC != ch || c >= S::NCOL || c >= NL) {
                snprintf(msg, n, "chunk %d column %d holds output row %d", ch, c, u);
                return 1;
            }
            ++seen[u];
        }
    for (int u = 0; u < D * P; ++u)
        if (seen[u] != 1) {
            snprintf(msg, n, "output row %d packed %d times", u, seen[u]);
            return 2;
        }
    std::vector<int> evals(64 * D, 0);  // (row, dim) -> lanes that evaluate it
    for (int ch = 0; ch < n_last; ++ch) {
        // the accumulator fragment of the chunk: a[t][4 i + 2 hh + e] = D[16 w + l / 4 + 8 hh][8 i + 2 (l % 4) + e]
        static float a[128][NA];
        for (int t = 0; t < 128; ++t)
            for (int i = 0; i < NL / 8; ++i)
                for (int hh = 0; hh < 2; ++hh)
                    for (int e = 0; e < 2; ++e) {
                        const int w = t / 32, l = t % 32;
                        const int row = 16 * w + l / 4 + 8 * hh, c = 8 * i + 2 * (l % 4) + e;
                        const int u = lr[ch * FK + c];
                        a[t][4 * i + 2 * hh + e] = u < 0 ? PAD : encode(row, u);
                    }
        // lockstep replay of the shuffles: sent[t][k] = what thread t passed to its k-th exchange
        std::vector<std::vector<float>> sent(128), next(128);
        static float v[128][S::NV];
        for (int pass = 0;; ++pass) {
            for (int t = 0; t < 128; ++t) {
                next[t].clear();
                int k = 0;
                outchunk::assemble<P, DPC>(a[t], t % 32, [&](float mine, int mask) {
                    next[t].push_back(mine);
                    const std::vector<float>& o = sent[t ^ mask];
                    const float got = k < (int)o.size() ? o[k] : PAD;
                    ++k;
                    return got;
                }, v[t]);
            }
            if (next == sent) break;
            if (pass == 4) {
                snprintf(msg, n, "exchange does not settle");
                return 3;
            }
            sent = next;
        }
        for (int t = 0; t < 128; ++t) {
            const int l = t % 32, row = 16 * (t / 32) + outchunk::row(l), slot = outchunk::slot(l);
            // staging order: value NV * slot + j of the chunk is parameter (NV slot + j) % P of dim ch DPC + (...) / P
            for (int j = 0; j < S::NV; ++j) {
                const int k = S::NV * slot + j;
                if (k >= S::NP) break;  // RQS with 16 bins: slot 1 evaluates nothing
                const int d = ch * DPC + k / P;
                if (d >= D) continue;   // absent dim of a partial last chunk: not evaluated
                if (v[t][j] != encode(row, d * P + k % P)) {
                    snprintf(msg, n, "chunk %d thread %d (row %d, slot %d) value %d: %.0f, expected row %d param %d of dim %d",
                             ch, t, row, slot, j, (double)v[t][j], row, k % P, d);
                    return 4;
                }
                if (k % P == 0) ++evals[row * D + d];
            }
        }
    }
    for (int i = 0; i < 64 * D; ++i)
        if (evals[i] != 1) {
            snprintf(msg, n, "row %d dim %d evaluated %d times", i / D, i % D, evals[i]);
            return 5;
        }
    return 0;
}

}  // namespace

// P, DPC: an RQS layer with 8 bins (23, 2), 16 bins (47, 1) or an affine layer (2, 32); D its features.  Returns 0 or
// a failure code with its description in msg.
extern "C" int out_chunk_check(int P, int DPC, int D, char* msg, int n) {
    if (P == 23 && DPC == 2) return check<23, 2, 48>(D, msg, n);
    if (P == 47 && DPC == 1) return check<47, 1, 48>(D, msg, n);
    if (P == 2 && DPC == 32) return check<2, 32, 64>(D, msg, n);
    snprintf(msg, n, "no such chunk shape");
    return -1;
}
