"""CPU checks of the flow-level edge table (tests/test_gpu_flow_edges.py): restating the branches of api.cu's
flow_forward_chunk and flow_inverse_chunk, the case table reaches every cell; and the restated row-chunk search
(largest_fitting_rows with its 1024-row granule) equals a brute-force search."""

import numpy as np
import pytest
from test_gpu_flow_edges import CASES, GRANULE, LAYERS, case_params, largest_fitting_rows, token


def cells(name, ctx, fused):
    """The branches one run of a case takes, restated from flow_forward_chunk (log_prob and forward) and
    flow_inverse_chunk (inverse with log_prob)."""
    members, base = CASES[name]
    T = len(members)
    out = set()
    if T == 0:
        return {("empty", base)}
    for i, m in enumerate(members):
        tok, inv = token(m)
        kind, fwd_fused, seq, fp32 = LAYERS[tok]
        last, ar_path = i == T - 1, ("ar_fused" if fwd_fused and fused else "ar_unfused")
        if inv:
            if not fused:
                out.add(("inverted_refused_unfused",))
                continue
            where = "last" if last else ("first" if i == 0 else "middle")
            out.add(("inverted", where))
            if last and base == "normal":
                out.add(("inverted_last_fuses_base", "copy" if i > 0 else "first"))
            if last and base == "box":
                out.add(("inverted_last_box",))
            out.add(("inverse_runs_forward", "fp32" if fp32 else tok))
            continue
        if i == 0 and kind in ("perm", "rot"):
            out.add(("ladj_fill", kind))
        if last:
            if base == "box":
                out.add(("box_after", kind))
            elif kind == "ar":
                out.add(("fuses_base", "ar_fp32" if fp32 else ar_path))
            elif kind == "ew":
                out.add(("fuses_base", "ew_table"))
            elif kind == "ewc":
                out.add(("fuses_base", f"ew_{ctx}"))
            else:
                out.add(("base_after", kind))
    # inverse + log_prob (no inverted member): the layers from the last to the first
    if not any(token(m)[1] for m in members):
        seeded = False
        for i in range(T - 1, -1, -1):
            tok = token(members[i])[0]
            kind, _, seq, _ = LAYERS[tok]
            done = kind == "ar" and seq and fused
            can_seed = not seeded and i == T - 1 and base != "box"
            if not seeded and not can_seed:
                out.add(("seed_box",))
                seeded = True
            if done:
                if can_seed:
                    out.add(("seed_in_kernel",))
                seeded = True
            else:
                if not seeded:
                    out.add(("seed_apart", "sweep" if kind == "ar" else kind))
                    seeded = True
                out.add(("ladj_skip" if kind in ("perm", "rot") else "ladj_forward", "sweep" if kind == "ar" else kind))
    for m in members:
        if LAYERS[token(m)[0]][0] in ("ar", "cpl", "ewc") and ctx == "bcast":
            out.add(("bcast", LAYERS[token(m)[0]][0]))
    return out


REQUIRED = (
    {("fuses_base", k) for k in ("ar_fused", "ar_unfused", "ar_fp32", "ew_table", "ew_rows", "ew_bcast")}
    | {("base_after", k) for k in ("cpl", "clip", "perm", "rot")}
    | {("box_after", k) for k in ("ar", "cpl", "perm")}
    | {("inverted", w) for w in ("first", "middle", "last")}
    | {("inverted_last_fuses_base", "copy"), ("inverted_last_fuses_base", "first"), ("inverted_last_box",)}
    | {("inverse_runs_forward", k) for k in ("ar", "fp32", "circ")}
    | {("inverted_refused_unfused",)}
    | {("ladj_fill", "perm"), ("ladj_fill", "rot")}
    | {("empty", "normal"), ("empty", "box")}
    | {("seed_in_kernel",), ("seed_box",), ("seed_apart", "sweep")}
    | {("ladj_forward", k) for k in ("cpl", "ew", "ewc", "clip", "sweep")}
    | {("ladj_skip", "perm"), ("ladj_skip", "rot")}
    | {("bcast", k) for k in ("ar", "cpl", "ewc")}
)  # fmt: skip


def test_case_table_reaches_every_branch():
    reached = set()
    for name, ctx, fused in case_params():
        reached |= cells(name, ctx, fused)
    missing = REQUIRED - reached
    assert not missing, f"branches the case table does not reach: {sorted(missing)}"


def test_every_case_runs_on_both_bases_where_it_matters():
    assert {CASES[n][1] for n in CASES if not CASES[n][0]} == {"normal", "box"}
    only = {CASES[n][1] for n in CASES if CASES[n][0] and {LAYERS[token(m)[0]][0] for m in CASES[n][0]} <= {"perm", "rot"}}
    assert only == {"normal", "box"}
    # a sweep-fallback layer closes a flow on DiagNormal: the first layer the inverse meets seeds apart
    assert any(CASES[n][0][-1] == "sweep" and CASES[n][1] == "normal" for n in CASES)


def brute_force(B, ws, need, granule):
    """The whole batch when it fits; else the largest n < B whose need fits (need non-decreasing: every smaller n fits
    too), then whole granules when that count is at least two granules and the rounded count still fits."""
    if need(B) <= ws:
        return B
    fit = [n for n in range(1, B + 1) if need(n) <= ws]
    if not fit:
        return 0
    lo = max(fit)
    if granule > 1 and lo >= 2 * granule and need(lo // granule * granule) <= ws:
        lo = lo // granule * granule
    return lo


def staircase(seed):
    """A synthetic workspace need: 256-byte granules of a few per-row terms (like a256 of the flow's buffers) plus a
    fixed part, non-decreasing with small bumps at each granule step."""
    rng = np.random.default_rng(seed)
    per_row = rng.integers(1, 80, size=3) * 4
    fixed = int(rng.integers(0, 5000))
    return lambda n: fixed + sum(-(-int(n * p) // 256) * 256 for p in per_row)


@pytest.mark.parametrize("seed", range(6))
def test_largest_fitting_rows_equals_brute_force(seed):
    need = staircase(seed)
    B = 3 * GRANULE + 211
    budgets = sorted({need(n) + k for n in (1, 2, 3, 100, GRANULE - 1, 2 * GRANULE - 1, 2 * GRANULE, 2 * GRANULE + 1, 2 * GRANULE + 517,
                                            3 * GRANULE, B - 1, B) for k in (-1, 0, 1)})  # fmt: skip
    sides = set()
    for ws in budgets:
        for granule in (1, GRANULE):
            got = largest_fitting_rows(B, ws, need, granule)
            assert got == brute_force(B, ws, need, granule), (seed, ws, granule)
            if granule > 1 and 0 < got < B:
                sides.add(got >= 2 * GRANULE)
    assert sides == {False, True}, "both sides of the 2-granule threshold"
    assert largest_fitting_rows(0, 1 << 40, need, GRANULE) == 0
    assert largest_fitting_rows(B, need(1) - 1, need, GRANULE) == 0
