// Host replay of the weight-ring protocol of fused_layer_kernel (zuko_b200/csrc/fused_layer.cu): one TMA producer
// and two consumer warpgroups exchanging 64 x 64 weight tiles through a ring of `full` / `empty` mbarrier pairs.
//
// The producer and consumer tile sequences below are the kernel's loops, restated step by step for both row-tile
// modes:
//   64 rows:  two rings of n_stages / 2 slots; chunk ch goes to consumer ch % 2, which releases each slot as soon
//             as its (synchronous) MMAs are done;
//   128 rows: one ring of n_stages slots whose `empty` barriers expect two arrivals; both consumers take every
//             slot; a hidden-layer slot is released once the next tile has been issued (one tile late), and the
//             slots of an output-layer chunk are released together once the chunk's MMAs are done.
// A random scheduler interleaves the three agents and the TMA completions, with the mbarrier parity semantics of
// sm_90 (try_wait.parity(x) passes once the phase of parity x has completed).  It checks that every consumer
// wait hands over exactly the tile that consumer expects, that no slot is refilled before all its consumers
// released it, that releases name the slot the consumer holds, and that the replay never deadlocks.

#include <stdint.h>
#include <stdio.h>

#include <random>
#include <vector>

namespace {

struct Tile {
    int l, ch, kb;
    bool operator==(const Tile& o) const { return l == o.l && ch == o.ch && kb == o.kb; }
};

enum { OP_ACQ, OP_REL };
struct Op {
    int kind;
    int slot;
    uint32_t parity;  // OP_ACQ: the parity the consumer waits on
    Tile tile;        // OP_ACQ: the tile it expects in the slot
};

struct Ring {  // one consumer's (or the producer's) walk over a ring of slots [s0, s0 + n)
    int s0, n, s = 0;
    uint32_t ph = 0;
    Ring(int s0_, int n_) : s0(s0_), n(n_), s(s0_) {}
    void advance() {
        if (++s == s0 + n) { s = s0; ph ^= 1; }
    }
};

struct Barrier {
    int count, pending = 0;
    uint32_t phase = 0;  // completed phases
    bool passes(uint32_t parity) const { return (phase & 1u) != parity; }
    void arrive() {
        if (++pending == count) { pending = 0; ++phase; }
    }
};

struct Problem {
    const uint8_t* kbmask;  // [L][128]
    int L, KB0, nch, n_last, rows, n_stages, n_tiles;
    bool bit(int l, int ch, int kb) const { return (kbmask[l * 128 + ch] >> kb) & 1u; }
};

// the producer's tile order for one row tile (fused_layer_kernel, warpgroup 0)
std::vector<Tile> producer_tiles(const Problem& P) {
    std::vector<Tile> t;
    for (int l = 0; l < P.L - 1; ++l) {
        const int KB = (l == 0) ? P.KB0 : P.nch;
        for (int kb = 0; kb < KB; ++kb)
            for (int ch = 0; ch < P.nch; ++ch)
                if (P.bit(l, ch, kb)) t.push_back({l, ch, kb});
    }
    for (int ch = 0; ch < P.n_last; ++ch)
        for (int kb = 0; kb < P.nch; ++kb)
            if (P.bit(P.L - 1, ch, kb)) t.push_back({P.L - 1, ch, kb});
    return t;
}

// the ring operations of consumer warpgroup cw over all row tiles (fused_layer_kernel, consumers)
std::vector<Op> consumer_ops(const Problem& P, int cw) {
    const bool wide = P.rows == 128;
    const int NR = wide ? P.n_stages : P.n_stages / 2;
    Ring r(wide ? 0 : cw * NR, NR);
    std::vector<Op> ops;
    auto acquire = [&](int l, int ch, int kb) {
        ops.push_back({OP_ACQ, r.s, r.ph, {l, ch, kb}});
        const int s = r.s;
        r.advance();
        return s;
    };
    auto release = [&](int s) { ops.push_back({OP_REL, s, 0, {}}); };
    for (int t = 0; t < P.n_tiles; ++t) {
        for (int l = 0; l < P.L - 1; ++l) {
            const int KB = (l == 0) ? P.KB0 : P.nch;
            if (wide) {
                int held = -1;
                for (int kb = 0; kb < KB; ++kb)
                    for (int q = 0; q < 4; ++q) {
                        if (q >= P.nch || !P.bit(l, q, kb)) continue;
                        const int s = acquire(l, q, kb);
                        if (held >= 0) release(held);
                        held = s;
                    }
                if (held >= 0) release(held);
            } else {
                for (int kb = 0; kb < KB; ++kb)
                    for (int ch = 0; ch < P.nch; ++ch)
                        if (P.bit(l, ch, kb) && (ch & 1) == cw) release(acquire(l, ch, kb));
            }
        }
        if (wide) {
            for (int ch = 0; ch < P.n_last; ++ch) {
                std::vector<int> held;
                for (int kb = 0; kb < P.nch; ++kb)
                    if (P.bit(P.L - 1, ch, kb)) held.push_back(acquire(P.L - 1, ch, kb));
                for (int s : held) release(s);
            }
        } else {
            for (int ch = 0; ch < P.n_last; ++ch)
                for (int kb = 0; kb < P.nch; ++kb)
                    if (P.bit(P.L - 1, ch, kb) && (ch & 1) == cw) release(acquire(P.L - 1, ch, kb));
        }
    }
    return ops;
}

struct Slot {
    Tile tile{-1, -1, -1};
    int releases_needed = 0;  // consumers that have yet to release the current content
    bool filled = false;      // the TMA of the current content has completed
    bool holder[2] = {false, false};
};

}  // namespace

// 0: the replay completed and every check held; 1: deadlock; 2: a consumer was handed the wrong tile; 3: a slot was
// refilled before its consumers released it; 4: a release of a slot the consumer does not hold; 5: bad arguments.
// `msg` (may be null) receives a one-line description of the first failure.
extern "C" int ring_replay(const uint8_t* kbmask, int L, int KB0, int nch, int n_last, int rows, int n_stages,
                           int n_tiles, unsigned seed, char* msg, int msg_len) {
    auto fail = [&](int code, const char* what, int a = 0, int b = 0) {
        if (msg && msg_len > 0) snprintf(msg, (size_t)msg_len, "%s (%d, %d)", what, a, b);
        return code;
    };
    if (L < 2 || nch < 1 || nch > 8 || KB0 < 1 || n_last < 1 || n_last > 128 || (rows != 64 && rows != 128) ||
        n_stages < 2 || n_stages > 8 || (rows == 64 && n_stages % 2) || n_tiles < 1)
        return fail(5, "bad arguments");
    const Problem P{kbmask, L, KB0, nch, n_last, rows, n_stages, n_tiles};
    const bool wide = rows == 128;
    const int NR = wide ? n_stages : n_stages / 2;

    // producer: (tile, ring) per load, over all row tiles
    std::vector<Tile> per_tile = producer_tiles(P), prod;
    for (int t = 0; t < n_tiles; ++t) prod.insert(prod.end(), per_tile.begin(), per_tile.end());
    std::vector<Op> cons[2] = {consumer_ops(P, 0), consumer_ops(P, 1)};

    std::vector<Barrier> full(n_stages, Barrier{1}), empty(n_stages, Barrier{wide ? 2 : 1});
    std::vector<Slot> slots(n_stages);
    Ring pr[2] = {Ring(0, NR), Ring(NR, NR)};
    size_t pi = 0, ci[2] = {0, 0};
    std::vector<int> in_flight;  // slots whose TMA has been issued and has not completed
    std::mt19937 rng(seed);

    while (pi < prod.size() || ci[0] < cons[0].size() || ci[1] < cons[1].size() || !in_flight.empty()) {
        // runnable agents: 0 producer, 1-2 consumers, 3 a TMA completion
        int ready[4], n = 0;
        if (pi < prod.size()) {
            const Ring& r = pr[wide ? 0 : (prod[pi].ch & 1)];
            if (empty[r.s].passes(r.ph ^ 1)) ready[n++] = 0;
        }
        for (int c = 0; c < 2; ++c) {
            if (ci[c] >= cons[c].size()) continue;
            const Op& op = cons[c][ci[c]];
            if (op.kind == OP_REL || full[op.slot].passes(op.parity)) ready[n++] = 1 + c;
        }
        if (!in_flight.empty()) ready[n++] = 3;
        if (n == 0) return fail(1, "deadlock: producer at load / consumers at op", (int)pi, (int)(ci[0] * 100000 + ci[1]));
        const int who = ready[rng() % n];
        if (who == 0) {
            const Tile& t = prod[pi++];
            Ring& r = pr[wide ? 0 : (t.ch & 1)];
            Slot& sl = slots[r.s];
            if (sl.releases_needed != 0 || sl.holder[0] || sl.holder[1])
                return fail(3, "slot refilled before its consumers released it", r.s, (int)pi);
            sl.tile = t;
            sl.filled = false;
            sl.releases_needed = wide ? 2 : 1;
            in_flight.push_back(r.s);
            r.advance();
        } else if (who == 3) {
            const size_t k = rng() % in_flight.size();
            const int s = in_flight[k];
            in_flight.erase(in_flight.begin() + (long)k);
            slots[s].filled = true;
            full[s].arrive();  // arrive.expect_tx + complete_tx: the phase completes with the bytes
        } else {
            const int c = who - 1;
            const Op& op = cons[c][ci[c]++];
            Slot& sl = slots[op.slot];
            if (op.kind == OP_ACQ) {
                if (!sl.filled || !(sl.tile == op.tile) || sl.holder[c])
                    return fail(2, "consumer handed the wrong tile: consumer / slot", c, op.slot);
                sl.holder[c] = true;
            } else {
                if (!sl.holder[c] || sl.releases_needed <= 0)
                    return fail(4, "release of a slot the consumer does not hold: consumer / slot", c, op.slot);
                sl.holder[c] = false;
                --sl.releases_needed;
                empty[op.slot].arrive();
            }
        }
    }
    for (const Slot& sl : slots)
        if (sl.holder[0] || sl.holder[1] || sl.releases_needed) return fail(4, "a slot is still held at the end");
    return 0;
}
