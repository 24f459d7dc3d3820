// Host replay of the weight-ring protocol of fused_layer_kernel (zuko_b200/csrc/fused_layer.cu) on 128-row tiles, with
// the output layer's chunks multiplied in pairs: one TMA producer and two consumer warpgroups exchanging 64 x 64 weight
// tiles through one ring of n_stages `full` / `empty` mbarrier pairs whose `empty` barriers expect two arrivals.
//
// The producer and consumer tile sequences below are the kernel's loops, restated step by step:
//   producer: hidden layers K block by K block, each over its chunks; the output layer chunk by chunk, each over its
//             K blocks (unchanged by the pairing);
//   consumer: hidden layers one tile at a time, a slot released once the next tile has been issued (one tile late);
//             the output layer's chunks in pairs (2j, 2j + 1) (the last pair of an odd n_last has no chunk B), a pair's
//             tiles (A's, then B's) one stream with the same one-tile-late release, the last one released after the
//             pair's full wait.
// A random scheduler interleaves the three agents and the TMA completions, with the mbarrier parity semantics of
// sm_90 (try_wait.parity(x) passes once the phase of parity x has completed).  It checks that every consumer wait
// hands over exactly the tile that consumer expects, that no slot is refilled before both consumers released it,
// that releases name a slot the consumer holds, that a consumer never holds more than two slots, and that the replay
// never deadlocks.

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
    int L, KB0, nch, n_last, n_stages, n_tiles;
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

// the ring operations of one consumer warpgroup over all row tiles (both walk the same sequence)
std::vector<Op> consumer_ops(const Problem& P) {
    int s = 0;
    uint32_t ph = 0;
    std::vector<Op> ops;
    int held = -1;
    // mbar_wait on the next slot, the tile's MMAs issued, wait_group 1, the previous tile's slot released
    auto take = [&](int l, int ch, int kb) {
        ops.push_back({OP_ACQ, s, ph, {l, ch, kb}});
        if (held >= 0) ops.push_back({OP_REL, held, 0, {}});
        held = s;
        if (++s == P.n_stages) { s = 0; ph ^= 1; }
    };
    auto drain = [&]() {  // wait_group 0, the last slot released
        if (held >= 0) ops.push_back({OP_REL, held, 0, {}});
        held = -1;
    };
    for (int t = 0; t < P.n_tiles; ++t) {
        for (int l = 0; l < P.L - 1; ++l) {
            const int KB = (l == 0) ? P.KB0 : P.nch;
            for (int kb = 0; kb < KB; ++kb)
                for (int q = 0; q < 4; ++q)
                    if (q < P.nch && P.bit(l, q, kb)) take(l, q, kb);
            drain();
        }
        for (int ch = 0; ch < P.n_last; ch += 2) {
            const bool has_b = ch + 1 < P.n_last;
            for (int kb = 0; kb < P.nch; ++kb)
                if (P.bit(P.L - 1, ch, kb)) take(P.L - 1, ch, kb);
            for (int kb = 0; kb < P.nch; ++kb)
                if (has_b && P.bit(P.L - 1, ch + 1, kb)) take(P.L - 1, ch + 1, kb);
            drain();
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
// refilled before its consumers released it; 4: a release of a slot the consumer does not hold, or a slot still held
// at the end; 5: bad arguments; 6: a consumer held more than two slots.  `msg` (may be null) receives a one-line
// description of the first failure.  `max_held` (may be null) receives the most slots one consumer held at once.
extern "C" int pair_ring_replay(const uint8_t* kbmask, int L, int KB0, int nch, int n_last, int n_stages, int n_tiles,
                                unsigned seed, char* msg, int msg_len, int* max_held) {
    auto fail = [&](int code, const char* what, int a = 0, int b = 0) {
        if (msg && msg_len > 0) snprintf(msg, (size_t)msg_len, "%s (%d, %d)", what, a, b);
        return code;
    };
    if (L < 2 || nch < 1 || nch > 4 || KB0 < 1 || KB0 > 8 || n_last < 1 || n_last > 128 || n_stages < 2 ||
        n_stages > 8 || n_tiles < 1)
        return fail(5, "bad arguments");
    const Problem P{kbmask, L, KB0, nch, n_last, n_stages, n_tiles};

    std::vector<Tile> per_tile = producer_tiles(P), prod;
    for (int t = 0; t < n_tiles; ++t) prod.insert(prod.end(), per_tile.begin(), per_tile.end());
    const std::vector<Op> ops = consumer_ops(P);

    std::vector<Barrier> full(n_stages, Barrier{1}), empty(n_stages, Barrier{2});
    std::vector<Slot> slots(n_stages);
    int ps = 0;
    uint32_t pph = 0;
    size_t pi = 0, ci[2] = {0, 0};
    int n_held[2] = {0, 0}, most = 0;
    std::vector<int> in_flight;  // slots whose TMA has been issued and has not completed
    std::mt19937 rng(seed);

    while (pi < prod.size() || ci[0] < ops.size() || ci[1] < ops.size() || !in_flight.empty()) {
        // runnable agents: 0 producer, 1-2 consumers, 3 a TMA completion
        int ready[4], n = 0;
        if (pi < prod.size() && empty[ps].passes(pph ^ 1)) ready[n++] = 0;
        for (int c = 0; c < 2; ++c) {
            if (ci[c] >= ops.size()) continue;
            const Op& op = ops[ci[c]];
            if (op.kind == OP_REL || full[op.slot].passes(op.parity)) ready[n++] = 1 + c;
        }
        if (!in_flight.empty()) ready[n++] = 3;
        if (n == 0) return fail(1, "deadlock: producer at load / consumers at op", (int)pi, (int)(ci[0] * 100000 + ci[1]));
        const int who = ready[rng() % n];
        if (who == 0) {
            Slot& sl = slots[ps];
            if (sl.releases_needed != 0 || sl.holder[0] || sl.holder[1])
                return fail(3, "slot refilled before its consumers released it", ps, (int)pi);
            sl.tile = prod[pi++];
            sl.filled = false;
            sl.releases_needed = 2;
            in_flight.push_back(ps);
            if (++ps == n_stages) { ps = 0; pph ^= 1; }
        } else if (who == 3) {
            const size_t k = rng() % in_flight.size();
            const int s = in_flight[k];
            in_flight.erase(in_flight.begin() + (long)k);
            slots[s].filled = true;
            full[s].arrive();  // arrive.expect_tx + complete_tx: the phase completes with the bytes
        } else {
            const int c = who - 1;
            const Op& op = ops[ci[c]++];
            Slot& sl = slots[op.slot];
            if (op.kind == OP_ACQ) {
                if (!sl.filled || !(sl.tile == op.tile) || sl.holder[c])
                    return fail(2, "consumer handed the wrong tile: consumer / slot", c, op.slot);
                sl.holder[c] = true;
                if (++n_held[c] > most) most = n_held[c];
                if (most > 2) return fail(6, "a consumer holds more than two slots: consumer / slot", c, op.slot);
            } else {
                if (!sl.holder[c] || sl.releases_needed <= 0)
                    return fail(4, "release of a slot the consumer does not hold: consumer / slot", c, op.slot);
                sl.holder[c] = false;
                --n_held[c];
                --sl.releases_needed;
                empty[op.slot].arrive();
            }
        }
    }
    for (const Slot& sl : slots)
        if (sl.holder[0] || sl.holder[1] || sl.releases_needed) return fail(4, "a slot is still held at the end");
    if (max_held) *max_held = most;
    return 0;
}
