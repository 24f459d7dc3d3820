"""GPU tests of the fused layer kernel (fused_layer.cu) at its tile-plan, instantiation, chunk, batch and stride
edges, against the fp64 oracle (oracle/oracle.py).

* `fused_plan_of` restates, from the layer module's masks and options, what fused_layer_prepare and the launcher
  decide: fused_shape's refusals, fused_plan (rows per tile, W ring slots, shared memory), fused_degree_perm, the
  output-row regrouping (last_rows), the zero-tile map (kbmask, n_items) and which of the 36 kernel instantiations
  (bijector {RQS-8, RQS-16, affine} x fast math x general activation x tile {64, 128 / 3 terms, 128 / 1 term}) a
  case selects.  A test without a GPU checks that the shape table reaches every plan cell, refusal, instantiation
  and activation; on the GPU `zk_layer_fused_plan` and `zk_layer_fused_info` must report the same plan.
* Oracle parity on a shape x batch matrix: batches 1, T - 1, T, T + 1, 2T - 1, W - 1, W + 1 and 3W + 77 with T the
  tile rows and W one wave (T x SMs), in both zk_set_fast_math modes, fused and unfused (zk_set_fused_layers(0)).
* Inputs outside the spline's [-5, 5], at +-5 and its float32 neighbours, huge, and exactly on spline knots.
* Where the layer sits in a flow: after and before non-fused layers, under a BoxUniform base, under a DiagNormal base
  with loc != 0 and scale != 1, next to layers of another tile height.
* The C ABI (strided rows, a broadcast context, accumulate, ladj = NULL, B = 0, row chunks) and bitwise properties.

Bars: log_prob and ladj per row |ours - ref64| <= 1e-5 max(1, |ref64|); z per element
|ours - ref64| <= max(4e-5 max(1, |ref64|), 3 |ref32 - ref64|), ref32 being the oracle in float32.  Fused against
unfused at bf16x3: the allclose bars of test_gpu_fused_tiles.py.  bf16x1: err_fused <= 2 err_unfused + 1e-4 against
the oracle."""

import ctypes
from functools import partial

import numpy as np
import pytest
import torch

from cases import O_rqs_knots, rel_err
from oracle import oracle as O
from test_gpu_tcgen05 import FUSED_FLOWS
from zuko_b200 import _engine as E
from zuko_b200.distributions import BoxUniform, DiagNormal
from zuko_b200.flows import MAF, NCSF, NSF, ElementWiseTransform, MaskedAutoregressiveTransform
from zuko_b200.lazy import Flow, UnconditionalDistribution, UnconditionalTransform
from zuko_b200.transforms import MonotonicAffineTransform, MonotonicRQSTransform, SoftclipTransform

SEED = 0
LP_BAR, Z_BAR = 1e-5, 4e-5

A = torch.nn  # activation modules


def _one(t, base=None):
    D = t.features
    base = base or UnconditionalDistribution(DiagNormal, torch.zeros(D), torch.ones(D), buffer=True)
    return Flow([t], base)


def _slope(uni, D, C, hidden):
    if uni == "rqs8":
        t = MaskedAutoregressiveTransform(D, C, univariate=partial(MonotonicRQSTransform, slope=1e-2),
                                          shapes=[(8,), (8,), (7,)], hidden_features=hidden)  # fmt: skip
    else:
        t = MaskedAutoregressiveTransform(D, C, univariate=partial(MonotonicAffineTransform, slope=1e-2), hidden_features=hidden)
    return _one(t)


def _adjacency():
    """D = 16, RQS-16 (one dim per output chunk): dims 0-5 depend on nothing (empty adjacency rows), so their output
    chunks are all-zero tiles; the degree-sorted hidden layers have all-zero (chunk, K block) tiles."""
    D = 16
    adj = torch.tril(torch.ones(D, D, dtype=torch.bool))
    adj[1:6] = torch.eye(D, dtype=torch.bool)[1:6]
    adj[12, :6] = False
    return _one(MaskedAutoregressiveTransform(D, 0, adjacency=adj, univariate=MonotonicRQSTransform,
                                              shapes=[(16,), (16,), (15,)], hidden_features=[256, 256]))  # fmt: skip


def _nsf(D, C, bins, hidden, act=None):
    kw = {} if act is None else {"activation": act}
    return lambda: NSF(D, C, transforms=1, bins=bins, hidden_features=hidden, **kw)


def _maf(D, C, hidden, act=None, **kw):
    if act is not None:
        kw["activation"] = act
    return lambda: MAF(D, C, transforms=1, hidden_features=hidden, **kw)


# name -> (constructor, gemm mode).  The constructors of FUSED_FLOWS are imported; the rest are one-layer flows
# named for the plan cell / edge they reach
NEW = {
    "nsf8c4_h256_L2": (_nsf(8, 4, 8, [256]), "bf16x3"),                       # n_linear 2, RQS 128/4
    "maf12_h128x5": (_maf(12, 0, [128] * 5), "bf16x3"),                     # n_linear 6, affine KBA 2: 128/7
    "nsf12c4_h320": (_nsf(12, 4, 8, [320] * 2), "bf16x3"),                  # RQS KBA 5: 64/6, nch 5 (odd)
    "maf16_h320": (_maf(16, 0, [320] * 2), "bf16x3"),                       # affine KBA 5: 64/6, nch 5
    "maf20_h448": (_maf(20, 0, [448] * 2), "bf16x3"),                       # affine KBA 7: 64/4, nch 7
    "nsf20c300_k16_h64": (_nsf(20, 300, 16, [64] * 2), "bf16x3"),           # KB0 5 > nch 1 at 64 rows
    "nsf40c400_k16_h128": (_nsf(40, 400, 16, [128] * 2), "bf16x3"),         # RQS KBA 7, KB0 7 > nch 2
    "nsf128_k16_h128": (_nsf(128, 0, 16, [128] * 2), "bf16x3"),             # n_last 128 (DPC 1)
    "nsf256_k8_h256": (_nsf(256, 0, 8, [256] * 2), "bf16x3"),               # n_last 128 (DPC 2)
    "maf480c32_h512": (_maf(480, 32, [512]), "bf16x3"),                     # D + C = 512, n_last 15 (odd)
    "nsf16c4_slope": (lambda: _slope("rqs8", 16, 4, [128] * 2), "bf16x3"),  # slope 1e-2: aw, ad
    "maf16c4_slope": (lambda: _slope("affine", 16, 4, [384] * 2), "bf16x3"),
    "adjacency16_k16": (_adjacency, "bf16x3"),                              # zero output chunks, zero hidden tiles
    # every ZK_ACT_* fused, at 64- and 128-row tiles
    "nsf10c2_h128_lrelu": (_nsf(10, 2, 8, [128] * 2, A.LeakyReLU), "bf16x3"),
    "maf16_h384_lrelu": (_maf(16, 0, [384] * 2, A.LeakyReLU), "bf16x3"),
    "nsf12_k16_h192_softplus": (_nsf(12, 0, 16, [192] * 2, A.Softplus), "bf16x3"),
    "nsf16_k16_h384_softplus": (_nsf(16, 0, 16, [384] * 2, A.Softplus), "bf16x3"),
    "maf20c12_h128_sigmoid": (_maf(20, 12, [128] * 2, A.Sigmoid), "bf16x3"),
    "nsf12c4_h448_sigmoid": (_nsf(12, 4, 8, [448] * 2, A.Sigmoid), "bf16x3"),  # RQS KBA 7, nch 7
}  # fmt: skip
# gemm_mode = "bf16x1": the 128-row one-term instantiations, and the 64-row kernel reading n_terms at run time
X1 = {f"{n}_x1": (NEW[n][0], "bf16x1") for n in ("nsf8c4_h256_L2", "nsf10c2_h128_lrelu", "nsf12_k16_h192_softplus",
                                                 "maf20c12_h128_sigmoid", "nsf12c4_h320", "maf20_h448",
                                                 "nsf16_k16_h384_softplus", "maf16_h384_lrelu")}  # fmt: skip
X1.update({f"{n}_x1": (FUSED_FLOWS[n], "bf16x1") for n in ("nsf64_k16_h64", "maf70c100_h128")})
OLD = {n: (FUSED_FLOWS[n], "bf16x3") for n in FUSED_FLOWS}
REFUSED = {
    "maf12_h128x6": (_maf(12, 0, [128] * 6), "bf16x3", "depth"),
    "maf40c30_L1": (_maf(40, 30, []), "bf16x3", "depth"),
    "nsf8_h128_256": (_nsf(8, 0, 8, [128, 256]), "bf16x3", "hidden"),
    "nsf8_h96": (_nsf(8, 0, 8, [96, 96]), "bf16x3", "hidden"),
    "maf481c32_h512": (_maf(481, 32, [512]), "bf16x3", "width"),
    "nsf8_bins4": (_nsf(8, 0, 4, [128, 128]), "bf16x3", "bins"),
    "nsf129_k16_h128": (_nsf(129, 0, 16, [128] * 2), "bf16x3", "chunks"),
    "nsf257_k8_h256": (_nsf(257, 0, 8, [256] * 2), "bf16x3", "chunks"),
    "nsf16c8_h128_fp32": (_nsf(16, 8, 8, [128] * 2), "fp32", "fp32"),
    "maf12c4_h256_residual": (_maf(12, 4, [256, 256], residual=True), "bf16x3", "residual"),
    "ncsf4c3_h128": (lambda: NCSF(4, 3, transforms=1, hidden_features=[128, 128]), "bf16x3", "circular"),
}  # fmt: skip
FUSED = {**OLD, **NEW, **X1}
SHAPES = {**FUSED, **{n: v[:2] for n, v in REFUSED.items()}}


def make_flow(name):
    torch.manual_seed(SEED)
    ctor, mode = SHAPES[name]
    flow = ctor().eval()
    for t in ar_layers(flow):
        t.hyper.gemm_mode = mode
    return flow


def ar_layers(flow):
    return [t for t in flow.transform.transforms if type(t).__name__ == "MaskedAutoregressiveTransform"]


# --------------------------------------------------------------------------- #
# the fused plan, restated
# --------------------------------------------------------------------------- #

FK, MAXKB, MAX_STAGES, WIDE_MAXKB, SMEM_MAX, STAGE = 64, 8, 8, 4, 232448, 16384
ACT_NAMES = {E.ZK_ACT_RELU: "ReLU", E.ZK_ACT_ELU: "ELU", E.ZK_ACT_TANH: "Tanh", E.ZK_ACT_SILU: "SiLU", E.ZK_ACT_GELU: "GELU",
             E.ZK_ACT_LEAKY_RELU: "LeakyReLU", E.ZK_ACT_SOFTPLUS: "Softplus", E.ZK_ACT_SIGMOID: "Sigmoid"}  # fmt: skip


def dpc_p(kind, bins):
    """fused_dpc, fused_p (fused_common.cuh): dims per 64-row output chunk, parameters per dim."""
    return (2 if bins == 8 else 1, 3 * bins - 1) if kind == E.ZK_UNI_RQS else (32, 2)


def tile_plan(KBA, kind, bins):
    """fused_plan: (rows, ring slots, dynamic shared memory) from the A operand's K blocks and the staging width."""
    dpc, P = dpc_p(kind, bins)
    srow = (dpc * P) | 1
    for rows in (128, 64):
        fixed = 1024 + rows // 64 * 2 * KBA * 8192 + 2 * 64 * srow * 4 + 4 * rows * 4 + 2 * MAX_STAGES * 8
        if fixed >= SMEM_MAX:
            continue
        ns = min(MAX_STAGES, (SMEM_MAX - fixed) // STAGE)
        if rows == 128 and (KBA > WIDE_MAXKB or ns < 4):
            continue
        if rows == 64:
            ns &= ~1
        return rows, ns, ns * STAGE + fixed
    return 0, 0, 0


def resolved_mode(t):
    dims = [t.hyper._linears()[0].weight.shape[1]] + [m.weight.shape[0] for m in t.hyper._linears()]
    mode = t.hyper.gemm_mode
    if mode == "auto":
        mode = "bf16x3" if max(dims) >= 64 else "fp32"
    return mode


def fused_plan_of(t):
    """What the engine decides for the autoregressive layer module `t`: dict with why (refusal reason or None)
    and, when it runs fused, rows, slots, smem, the degree permutations, last_rows, kbmask, n_items and the
    instantiation key (without the math mode)."""
    lins = t.hyper._linears()
    L, u = len(lins), t._uni
    D, C = t.features, t.context
    dims = [lins[0].weight.shape[1]] + [m.weight.shape[0] for m in lins]
    mode = resolved_mode(t)
    H = dims[1] if L > 1 else 0
    why = None
    if u["kind"] == E.ZK_UNI_CRQS:
        why = "circular"
    elif mode == "fp32":
        why = "fp32"
    elif any(type(m).__name__ == "Residual" for m in t.hyper):
        why = "residual"
    elif not 2 <= L <= 6:
        why = "depth"
    elif H % 64 or not 64 <= H <= 512 or any(d != H for d in dims[1:L]):
        why = "hidden"
    elif D + C > 512:
        why = "width"
    elif u["kind"] == E.ZK_UNI_RQS and u["bins"] not in (8, 16):
        why = "bins"
    elif u["kind"] not in (E.ZK_UNI_RQS, E.ZK_UNI_AFFINE):
        why = "bijector"
    elif -(-D // dpc_p(u["kind"], u["bins"])[0]) > 128:
        why = "chunks"
    act = t.hyper._activation_code()
    if why:
        return {"why": why, "rows": 0, "L": L, "act": act}
    kind, bins = u["kind"], u["bins"]
    dpc, P = dpc_p(kind, bins)
    masks = [m.mask.numpy().astype(bool) for m in lins]
    # fused_degree_perm: dependency set of every hidden unit, stable sort by its size
    perms, dep = [], masks[0]
    for l in range(L - 1):
        if l > 0:
            dep = (masks[l].astype(np.int64) @ dep.astype(np.int64)) > 0
        perms.append(np.argsort(dep.sum(1), kind="stable"))
    # output rows regrouped into 64-row chunks of whole dims
    n_last = -(-D // dpc)
    last_rows = np.full(n_last * FK, -1, np.int64)
    for ch in range(n_last):
        for j in range(dpc * P):
            d = ch * dpc + j // P
            if d < D:
                last_rows[ch * FK + j] = d * P + j % P
    nch = H // FK
    kbmask = []
    for l in range(L):
        rows_l = last_rows if l == L - 1 else perms[l]
        cols = perms[l - 1] if l > 0 else np.arange(dims[0])
        Mp = masks[l][:, cols]
        nb = -(-dims[l] // FK)
        bits = np.zeros((len(rows_l) // FK, nb), bool)
        for ch in range(len(rows_l) // FK):
            r = rows_l[ch * FK : (ch + 1) * FK]
            r = r[r >= 0]
            if r.size:
                colany = Mp[r].any(0)
                bits[ch] = [colany[kb * FK : (kb + 1) * FK].any() for kb in range(nb)]
        kbmask.append(bits)
    KB0 = -(-dims[0] // FK)
    KBA = max(KB0, nch)
    rows, slots, smem = tile_plan(KBA, kind, bins)
    nt = 1 if mode == "bf16x1" else 3
    uni = f"rqs{bins}" if kind == E.ZK_UNI_RQS else "affine"
    tile = "64" if rows == 64 else f"128x{nt}"
    return {"why": None, "rows": rows, "slots": slots, "smem": smem, "L": L, "H": H, "nch": nch, "KB0": KB0, "KBA": KBA,
            "D": D, "C": C, "n_last": n_last, "perms": perms, "last_rows": last_rows, "kbmask": kbmask,
            "n_items": int(sum(b.sum() for b in kbmask)), "act": act, "gact": act != E.ZK_ACT_RELU,
            "uni": uni, "kind": kind, "bins": bins, "tile": tile, "mode": mode}  # fmt: skip


def instantiation(plan, fast):
    return (plan["uni"], bool(fast), plan["gact"], plan["tile"])


ALL_INSTANTIATIONS = {(u, f, g, tl) for u in ("rqs8", "rqs16", "affine") for f in (True, False) for g in (True, False)
                      for tl in ("64", "128x3", "128x1")}  # fmt: skip
# rows / slots of the plan table, by bijector family and KBA
PLAN_TABLE = {
    "rqs": {1: (128, 8), 2: (128, 8), 3: (128, 6), 4: (128, 4), 5: (64, 6), 6: (64, 6), 7: (64, 4), 8: (64, 4)},
    "affine": {1: (128, 8), 2: (128, 7), 3: (128, 5), 4: (64, 8), 5: (64, 6), 6: (64, 6), 7: (64, 4), 8: (64, 4)},
}

_PLANS = {}


def plans_of(name):
    """Restated plans of every autoregressive layer of the shape (cached: the masks do not change)."""
    if name not in _PLANS:
        _PLANS[name] = [fused_plan_of(t) for t in ar_layers(make_flow(name))]
    return _PLANS[name]


def test_plan_table_and_refusals_are_reached():
    """The shape table reaches every plan cell, refusal, tile-map case, instantiation and activation (no GPU)."""
    for fam, kind, bins in (("rqs", E.ZK_UNI_RQS, 8), ("rqs", E.ZK_UNI_RQS, 16), ("affine", E.ZK_UNI_AFFINE, 0)):
        for kba, cell in PLAN_TABLE[fam].items():
            assert tile_plan(kba, kind, bins)[:2] == cell, (fam, bins, kba)
    assert tile_plan(4, E.ZK_UNI_AFFINE, 0)[2] == 232064  # affine KBA 4 / 6 / 8: 384 bytes short of the limit
    fused = {n: plans_of(n) for n in FUSED}
    cells = {("rqs" if p["kind"] == E.ZK_UNI_RQS else "affine", p["KBA"]) for ps in fused.values() for p in ps}
    assert cells == {(f, k) for f in PLAN_TABLE for k in PLAN_TABLE[f]}, sorted(cells)
    for name, ps in fused.items():
        for p in ps:
            assert p["why"] is None, (name, p["why"])
            fam = "rqs" if p["kind"] == E.ZK_UNI_RQS else "affine"
            assert (p["rows"], p["slots"]) == PLAN_TABLE[fam][p["KBA"]], name
    for name, (_, _, why) in REFUSED.items():
        assert [p["why"] for p in plans_of(name)] == [why], (name, plans_of(name))
    flat = [p for ps in fused.values() for p in ps]
    assert any(p["rows"] == 64 and p["nch"] % 2 for p in flat), "odd hidden-chunk count at 64 rows"
    for rows in (64, 128):
        assert any(p["rows"] == rows and p["KB0"] > p["nch"] for p in flat), f"KB0 > nch at {rows} rows"
    assert {2, 6} <= {p["L"] for p in flat} and {1, 128} <= {p["n_last"] for p in flat}
    assert {p["n_last"] for p in plans_of("nsf256_k8_h256")} == {128}
    assert any((p["kbmask"][-1].sum(1) == 0).any() for p in flat), "an all-zero output chunk"
    assert any((~p["kbmask"][l][:, : (p["KB0"] if l == 0 else p["nch"])]).any() for p in flat for l in range(p["L"] - 1))
    adj = plans_of("adjacency16_k16")[0]
    assert (adj["kbmask"][-1].sum(1) == 0).sum() >= 5 and any((~b).any() for b in adj["kbmask"][:-1])
    # every instantiation is reached by the parity matrix (both math modes, W + 1 rows among its batches)
    reached = {instantiation(p, fast) for ps in fused.values() for p in ps for fast in (True, False)}
    assert reached == ALL_INSTANTIATIONS, sorted(ALL_INSTANTIATIONS - reached)
    assert {p["act"] for p in flat} == set(ACT_NAMES), sorted(ACT_NAMES[a] for a in set(ACT_NAMES) - {p["act"] for p in flat})


def test_degree_perm_is_a_stable_sort_by_dependency_count():
    """The restated permutation on a small layer, against a per-unit walk of the mask graph."""
    t = ar_layers(make_flow("nsf12c4_h320"))[0]
    masks = [m.mask.numpy().astype(bool) for m in t.hyper._linears()]
    p = plans_of("nsf12c4_h320")[0]
    deps = [set(np.nonzero(r)[0]) for r in masks[0]]
    for l, perm in enumerate(p["perms"]):
        if l > 0:
            deps = [set().union(*(deps[k] for k in np.nonzero(r)[0])) for r in masks[l]]
        deg = [len(s) for s in deps]
        assert sorted(range(len(deg)), key=lambda n: deg[n]) == perm.tolist()
    # every output row is produced exactly once by the regrouped chunks
    lr = p["last_rows"]
    assert sorted(lr[lr >= 0].tolist()) == list(range(p["D"] * t.total))


# --------------------------------------------------------------------------- #
# GPU helpers
# --------------------------------------------------------------------------- #


def sm_count():
    n, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    E.check(E.lib().zk_device_info(ctypes.byref(n), ctypes.byref(major), ctypes.byref(minor)))
    return n.value


def query(handle):
    """zk_layer_fused_plan + zk_layer_fused_info: (rows, slots, smem, kind, n_items)."""
    slots, smem = ctypes.c_int(-1), ctypes.c_size_t(0)
    rows = E.lib().zk_layer_fused_plan(handle, ctypes.byref(slots), ctypes.byref(smem))
    info = (ctypes.c_double * 4)()
    kind = E.lib().zk_layer_fused_info(handle, info)
    if not rows:
        return 0, 0, 0, kind, 0
    return rows, slots.value, smem.value, kind, int(info[1])


def want(plan):
    if plan["why"]:
        return 0, 0, 0, 0, 0
    return plan["rows"], plan["slots"], plan["smem"], 1, plan["n_items"]


def dev_t(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)


def cpu(t):
    return t.detach().cpu().numpy().astype(np.float64)


def context_dim(flow):
    return getattr(flow.transform.transforms[0], "context", 0)


def check_z(ours, ref64, ref32, what, rows=None):
    ours, ref64, ref32 = (np.asarray(a, np.float64) for a in (ours, ref64, ref32))
    tol = np.maximum(Z_BAR * np.maximum(np.abs(ref64), 1.0), 3.0 * np.abs(ref32 - ref64))
    with np.errstate(invalid="ignore"):
        bad = ~(np.abs(ours - ref64) <= tol)
    if bad.any():
        r = tuple(np.argwhere(bad)[0])
        row = r[0] if rows is None else rows[r[0]]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} entries off the oracle; first at row {row} {r[1:]}: "
                             f"ours {ours[r]!r} ref64 {ref64[r]!r} ref32 {ref32[r]!r}")  # fmt: skip


def check_row(ours, ref64, what, rows=None, scale=None):
    """Per row |ours - ref64| <= 1e-5 max(1, |ref64|, scale).  The ladj is held to the absolute bar of the row's
    log_prob (scale = |log_prob64|): log_prob = ladj + the base term of z, so both carry the conditioner's rounding
    (bf16x3 GEMMs, ~1e-6 per dim and layer) in the same absolute amount, which a ladj near 0 cannot absorb in a
    relative bar (measured on an H100: 2.3e-5 on a ladj of -0.86, nsf64_k16_h64, 2 layers x 64 dims x 16 bins)."""
    ours, ref64 = np.asarray(ours, np.float64), np.asarray(ref64, np.float64)
    ref_scale = np.maximum(np.abs(ref64), 1.0) if scale is None else np.maximum(np.maximum(np.abs(ref64), 1.0), np.abs(scale))
    with np.errstate(invalid="ignore"):
        bad = ~(np.abs(ours - ref64) <= LP_BAR * ref_scale)
    if bad.any():
        i = int(np.argmax(np.where(bad, np.abs(ours - ref64), -1)))
        row = i if rows is None else rows[i]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} rows off the oracle; worst at row {row}: "
                             f"ours {ours[i]!r} ref64 {ref64[i]!r}")  # fmt: skip


class Fixed:
    """Seeded inputs of one shape whose rows do not depend on the batch (x[:B] for every B), and the oracle on the
    rows checked so far: one shape's oracle is shared by all its batches and math modes."""

    def __init__(self, name, n):
        self.name, self.flow = name, make_flow(name)
        self.spec = O.flowspec_from_module(self.flow)
        D, C = self.spec.loc.shape[0], context_dim(self.flow)
        g = torch.Generator().manual_seed(1234)
        self.x = torch.randn(n, D, generator=g).numpy()
        self.c = torch.randn(n, C, generator=g).numpy() if C else None
        self.known = np.zeros(n, bool)
        self.z64, self.z32 = np.zeros((n, D)), np.zeros((n, D))
        self.ladj64, self.lp64 = np.zeros(n), np.zeros(n)

    def oracle(self, rows):
        new = np.setdiff1d(rows, np.nonzero(self.known)[0])
        if new.size:
            c = None if self.c is None else self.c[new]
            z, ladj = self.spec.forward(self.x[new].astype(np.float64), c)
            self.z64[new], self.ladj64[new] = z, ladj
            self.lp64[new] = self.spec._base_log_prob(z, ladj, np.float64)
            self.z32[new] = self.spec.forward(self.x[new], None if c is None else c.astype(np.float32), np.float32)[0]
            self.known[new] = True
        return self.z64[rows], self.z32[rows], self.ladj64[rows], self.lp64[rows]


_FIXED = {}


def fixed(name, n):
    f = _FIXED.get(name)
    if f is None or f.x.shape[0] < n:
        _FIXED.clear()  # one shape at a time: the matrix runs shape by shape
        f = _FIXED[name] = Fixed(name, n)
    return f


BATCHES = ["1", "T-1", "T", "T+1", "2T-1", "W-1", "W+1", "3W+77"]


def batch_of(key, T, W):
    return {"1": 1, "T-1": T - 1, "T": T, "T+1": T + 1, "2T-1": 2 * T - 1, "W-1": W - 1, "W+1": W + 1, "3W+77": 3 * W + 77}[key]


def oracle_rows(B, T, n_sm, n_random=512):
    """Every row of the first CTA's tiles (tiles 0, G, 2G, ... of the persistent grid of G CTAs), of the last two
    tiles, and n_random rows drawn once below one wave (the same rows for every large batch of a shape)."""
    tiles = -(-B // T)
    grid = min(tiles, n_sm)
    if B <= 6 * T + n_random:
        return np.arange(B)
    first = np.concatenate([np.arange(t * T, min(B, t * T + T)) for t in range(0, tiles, grid)])
    rnd = np.random.default_rng(7).choice(T * n_sm - 1, n_random, replace=False)
    return np.unique(np.concatenate([first, np.arange((tiles - 2) * T, B), rnd]))


@pytest.fixture
def math_mode():
    prev = E.lib().zk_set_fast_math(1)
    yield lambda fast: E.lib().zk_set_fast_math(int(fast))
    E.lib().zk_set_fast_math(prev)


@pytest.fixture
def unfused():
    def run(fn):
        prev = E.lib().zk_set_fused_layers(0)
        try:
            return fn()
        finally:
            E.lib().zk_set_fused_layers(prev)

    return run


def forward_all(flow, x, c, device):
    """log_prob and call_and_ladj (z, ladj) of the flow on device tensors."""
    with torch.no_grad():
        dist = flow(c)
        lp = dist.log_prob(x)
        z, ladj = dist.transform.call_and_ladj(x)
    return lp, z, ladj


# --------------------------------------------------------------------------- #
# path and plan
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_path_and_plan(device, name):
    plans = plans_of(name)
    flow = make_flow(name).to(device)
    layers = ar_layers(flow)
    D, C = flow.transform.transforms[0].features, context_dim(flow)
    g = torch.Generator().manual_seed(5)
    B = 300
    x = torch.randn(B, D, generator=g).numpy()
    c = torch.randn(B, C, generator=g).numpy() if C else None
    xd, cd = dev_t(x, device), (None if c is None else dev_t(c, device))
    with torch.no_grad():
        flow(cd).log_prob(xd[:1])  # packs outside the count
        n0 = E.lib().zk_launch_count()
        lp = flow(cd).log_prob(xd)
        launches = E.lib().zk_launch_count() - n0
    for t, plan in zip(layers, plans, strict=True):
        h = t._zk_layer()
        got = query(h)
        print(f"{name}: zk_layer_fused_plan / info {got}, restated {want(plan)}")
        assert got == want(plan), f"{name}: the engine reports {got}, the restated plan {want(plan)}"
        assert E.lib().zk_layer_fused_tile_rows(h) == plan["rows"]
        assert E.lib().zk_mlp_gemm_mode(t.hyper._handle()) == E.GEMM_MODES[resolved_mode(t)]
    if all(p["why"] is None for p in plans) and len(plans) == len(flow.transform.transforms):
        assert launches == len(plans), f"{name}: {launches} launches for {len(plans)} fused layers"
    else:
        assert launches > len(plans), launches  # per-layer GEMM kernels + the bijector kernel
        spec = O.flowspec_from_module(make_flow(name))
        check_row(cpu(lp), spec.log_prob(x.astype(np.float64), c), f"{name} per-layer kernels log_prob")


# --------------------------------------------------------------------------- #
# oracle parity matrix
# --------------------------------------------------------------------------- #

MATRIX = [(s, b, fast) for s in FUSED for b in BATCHES for fast in (1, 0)]
RANDOM_ROWS = {"nsf256_k8_h256": 256, "maf480c32_h512": 256}
# Softplus activations are all positive (about 0.7 at 0): the hidden sums add |a w| without cancelling, and the fused
# kernel (degree-sorted K order, zero tiles skipped) and the per-layer GEMMs round those split-bf16 sums differently.
# Measured on an H100 80GB HBM3: up to 1.0e-4 apart on the ladj and 7.2e-5 on log_prob (nsf16_k16_h384_softplus,
# B = 25421), both paths within the oracle bar on every checked row.  Other shapes keep atol 2e-5.
UNFUSED_ATOL = {"nsf12_k16_h192_softplus": 2e-4, "nsf16_k16_h384_softplus": 2e-4}


@pytest.mark.gpu
@pytest.mark.parametrize("name,b,fast", MATRIX, ids=[f"{s}-{b}-{'fast' if f else 'ieee'}" for s, b, f in MATRIX])
def test_oracle_parity_matrix(device, math_mode, unfused, name, b, fast):
    math_mode(fast)
    plans = plans_of(name)
    T, n_sm = plans[0]["rows"], sm_count()
    W = T * n_sm
    B = batch_of(b, T, W)
    fx = fixed(name, 3 * W + 77)
    flow = fx.flow.to(device)
    for t, plan in zip(ar_layers(flow), plans, strict=True):  # the instantiation this case is meant to run
        assert query(t._zk_layer()) == want(plan), name
        assert E.lib().zk_mlp_gemm_mode(t.hyper._handle()) == E.GEMM_MODES[plan["mode"]]
    assert E.lib().zk_set_fast_math(fast) == fast
    xd = dev_t(fx.x[:B], device)
    cd = None if fx.c is None else dev_t(fx.c[:B], device)
    lp, z, ladj = (cpu(v) for v in forward_all(flow, xd, cd, device))
    lp_u, z_u, ladj_u = (cpu(v) for v in unfused(lambda: forward_all(flow, xd, cd, device)))
    rows = oracle_rows(B, T, n_sm, RANDOM_ROWS.get(name, 512))
    z64, z32, ladj64, lp64 = fx.oracle(rows)
    what = f"{name} B={B} ({b}, T={T}) {'fast' if fast else 'ieee'}"
    assert np.isfinite(lp).all() and np.isfinite(z).all() and np.isfinite(ladj).all(), what
    if plans[0]["mode"] == "bf16x1":  # a single bf16 product: no better than the per-layer kernels at bf16x1
        for ours, theirs, ref, part in ((lp, lp_u, lp64, "log_prob"), (ladj, ladj_u, ladj64, "ladj"), (z, z_u, z64, "z")):
            err_f, err_u = rel_err(ours[rows], ref), rel_err(theirs[rows], ref)
            assert err_u < 1e-1, (what, part, err_u)
            assert err_f <= 2 * err_u + 1e-4, (what, part, err_f, err_u)
        return
    check_row(lp[rows], lp64, what + " log_prob", rows)
    check_row(ladj[rows], ladj64, what + " ladj", rows, lp64)
    check_z(z[rows], z64, z32, what + " z", rows)
    lp_f, lp_u, ladj_f, ladj_u = (torch.from_numpy(v) for v in (lp, lp_u, ladj, ladj_u))
    atol = UNFUSED_ATOL.get(name, 2e-5)
    assert torch.allclose(lp_f, lp_u, rtol=2e-6, atol=atol), (what, (lp_f - lp_u).abs().max())
    assert torch.allclose(torch.from_numpy(z), torch.from_numpy(z_u), rtol=1e-5, atol=1e-5), what
    assert torch.allclose(ladj_f, ladj_u, rtol=2e-6, atol=atol), (what, (ladj_f - ladj_u).abs().max())


# --------------------------------------------------------------------------- #
# input edges
# --------------------------------------------------------------------------- #

EDGE_SHAPES = ["nsf12c4_h320", "nsf8c4_h256_L2", "nsf128_k16_h128", "nsf16c4_slope", "nsf12c4_h448_sigmoid",
               "maf20_h448", "maf12_h128x5", "maf16c4_slope"]  # fmt: skip
F5 = np.float32(5)
EDGES = np.array([F5, -F5, np.nextafter(F5, np.float32(np.inf)), np.nextafter(-F5, np.float32(-np.inf)), np.nextafter(F5, 0),
                  np.nextafter(-F5, 0), 6, -6, 1e30, -1e30], np.float32)  # fmt: skip


def edge_inputs(flow, B):
    """x of a one-layer flow: the last dim in the order cycles through EDGES on every third row (it feeds no
    conditioner); on the rows after those the first dim in the order (whose phi depends on c only) sits exactly on
    one of its spline's x-knots."""
    t = ar_layers(flow)[0]
    D, C = t.features, t.context
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, D, generator=g).numpy()
    c = torch.randn(B, C, generator=g).numpy() if C else None
    order = t.order.numpy()
    last, first = int(np.argmax(order)), int(np.argmin(order))
    x[::3, last] = EDGES[np.arange(0, B, 3) % EDGES.size]
    layer = O.flowspec_from_module(flow).layers[0]
    if layer.univariate == "rqs":
        P = 3 * layer.bins - 1
        phi = layer.hyper(np.zeros((B, D)), c, np.float64).reshape(B, D, P)[:, first]
        X, _, _ = O_rqs_knots(phi[:, None, :], layer.bins, layer.bound, layer.slope)
        rows = np.arange(1, B, 3)
        x[rows, first] = X[rows, 0, rows % (layer.bins + 1)]
    return x.astype(np.float32), c


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
@pytest.mark.parametrize("name", EDGE_SHAPES)
def test_input_edges(device, math_mode, name, fast):
    math_mode(fast)
    cpu_flow = make_flow(name)
    T = plans_of(name)[0]["rows"]
    B = 3 * T + 5
    x, c = edge_inputs(cpu_flow, B)
    spec = O.flowspec_from_module(cpu_flow)
    z64, ladj64 = spec.forward(x.astype(np.float64), c)
    z32 = spec.forward(x, None if c is None else c.astype(np.float32), np.float32)[0]
    lp64 = spec._base_log_prob(z64, ladj64, np.float64)
    huge = (np.abs(x) > 1e18).any(1)
    # the ladj's absolute bar is that of the row's log_prob with the huge entries at 0 (they feed no conditioner)
    lp_scale = spec.log_prob(np.where(np.abs(x) > 1e18, 0.0, x.astype(np.float64)), c)
    flow = make_flow(name).to(device)
    lp, z, ladj = (cpu(v) for v in forward_all(flow, dev_t(x, device), None if c is None else dev_t(c, device), device))
    what = f"{name} {'fast' if fast else 'ieee'}"
    check_z(z, z64, z32, what + " z")
    check_row(ladj, ladj64, what + " ladj", None, lp_scale)
    check_row(lp[~huge], lp64[~huge], what + " log_prob", np.nonzero(~huge)[0])
    assert np.isneginf(lp[huge]).all(), what  # -0.5 (1e30)^2 overflows float32: the correctly rounded value
    if spec.layers[0].univariate == "rqs":
        # the identity beyond the last knot, bit for bit.  The knots are cumulative fmaf sums in float32, so the last
        # one may round to 5 + 1 ulp and nextafter(5, inf) can still be inside: the kernel follows its own knots
        # there, as the reference's float32 does, and those entries are held to the oracle bar above
        out = np.abs(x) >= 6
        assert out.sum() >= B // 3 * 4 // 10
        i = np.argwhere(out & (z != x))
        assert not i.size, f"{what}: y != x at {i[0]}: x {x[tuple(i[0])]!r} y {z[tuple(i[0])]!r}"


# --------------------------------------------------------------------------- #
# where the layer sits in the flow
# --------------------------------------------------------------------------- #


def _rqs(D, C, hidden, bins=8, **kw):
    return MaskedAutoregressiveTransform(D, C, univariate=MonotonicRQSTransform, shapes=[(bins,), (bins,), (bins - 1,)],
                                         hidden_features=hidden, **kw)  # fmt: skip


def _normal(D, loc=0.0, scale=1.0):
    return UnconditionalDistribution(DiagNormal, torch.zeros(D) + loc, torch.ones(D) * scale, buffer=True)


def _position(kind):
    D, C = 16, 4
    if kind == "after_elementwise":  # accumulates onto the ladj an element-wise layer wrote
        return Flow([ElementWiseTransform(D, 0), _rqs(D, C, [128] * 2)], _normal(D))
    if kind == "between_softclips":  # after a soft clip; y written for the soft clip that follows (log_prob = NULL)
        clip = UnconditionalTransform(SoftclipTransform, bound=11.0)
        return Flow([clip, _rqs(D, C, [256] * 2), UnconditionalTransform(SoftclipTransform, bound=11.0)], _normal(D))
    if kind == "box_uniform":  # the base is not fused: the layer writes y and its ladj
        base = UnconditionalDistribution(BoxUniform, torch.full((D,), -40.0), torch.full((D,), 40.0), buffer=True)
        return Flow([_rqs(D, C, [320] * 2)], base)
    if kind == "diag_normal":  # the DiagNormal term of the kernel with loc != 0, scale != 1
        g = torch.Generator().manual_seed(2)
        base = UnconditionalDistribution(DiagNormal, torch.randn(D, generator=g), torch.randn(D, generator=g).exp(), buffer=True)
        return Flow([MaskedAutoregressiveTransform(D, C, hidden_features=[128] * 2)], base)
    if kind == "mixed_tiles":  # 128-, 64-, 128- and 64-row layers in one flow
        return Flow([_rqs(D, C, [128] * 2), MaskedAutoregressiveTransform(D, C, hidden_features=[512] * 2, order=torch.arange(D).flip(0)),
                     _rqs(D, C, [192] * 2, bins=16), _rqs(D, C, [320] * 2, bins=16, order=torch.arange(D).flip(0))],
                    _normal(D, 0.25, 1.5))  # fmt: skip
    raise ValueError(kind)


POSITION_ROWS = {"after_elementwise": [128], "between_softclips": [128], "box_uniform": [64], "diag_normal": [128],
                 "mixed_tiles": [128, 64, 128, 64]}  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
@pytest.mark.parametrize("B", [1, 127, 3001])
@pytest.mark.parametrize("kind", list(POSITION_ROWS))
def test_flow_position(device, math_mode, kind, B, fast):
    math_mode(fast)
    torch.manual_seed(SEED)
    cpu_flow = _position(kind).eval()
    for t in ar_layers(cpu_flow):
        t.hyper.gemm_mode = "bf16x3"
    spec = O.flowspec_from_module(cpu_flow)
    D, C = 16, 4
    g = torch.Generator().manual_seed(B)
    x, c = torch.randn(B, D, generator=g).numpy(), torch.randn(B, C, generator=g).numpy()
    z64, ladj64 = spec.forward(x.astype(np.float64), c)
    z32 = spec.forward(x, c.astype(np.float32), np.float32)[0]
    lp64 = spec._base_log_prob(z64, ladj64, np.float64)
    torch.manual_seed(SEED)
    flow = _position(kind)
    flow.load_state_dict(cpu_flow.state_dict())
    for t in ar_layers(flow):
        t.hyper.gemm_mode = "bf16x3"
    flow = flow.to(device)
    lp, z, ladj = (cpu(v) for v in forward_all(flow, dev_t(x, device), dev_t(c, device), device))
    assert [E.lib().zk_layer_fused_tile_rows(t._zk_layer()) for t in ar_layers(flow)] == POSITION_ROWS[kind]
    what = f"{kind} B={B} {'fast' if fast else 'ieee'}"
    check_row(lp, lp64, what + " log_prob")
    check_row(ladj, ladj64, what + " ladj", None, lp64)
    check_z(z, z64, z32, what + " z")


# --------------------------------------------------------------------------- #
# C ABI
# --------------------------------------------------------------------------- #

ABI_SHAPES = ["nsf12c4_h320", "nsf8c4_h256_L2", "maf20c12_h128_sigmoid", "maf480c32_h512"]


def layer_forward_abi(h, x, ldx, c, ldc, B, y, ldy, ladj, accumulate, device):
    L = E.lib()
    need = L.zk_layer_workspace_bytes(h, B)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    E.check(L.zk_layer_forward(h, p(x), ldx, p(c), ldc, B, p(y), ldy, p(ladj), accumulate, p(ws), need, E.stream_ptr(device)))
    torch.cuda.synchronize(device)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ABI_SHAPES)
def test_layer_forward_c_abi(device, name):
    flow = make_flow(name).to(device)
    t = ar_layers(flow)[0]
    h = t._zk_layer()
    plan = plans_of(name)[0]
    assert query(h) == want(plan)
    D, C, T = t.features, t.context, plan["rows"]
    B = 2 * T + 7
    fx = Fixed(name, B)
    f32 = dict(device=device, dtype=torch.float32)
    x = dev_t(fx.x, device)
    c = None if fx.c is None else dev_t(fx.c, device)
    y, ladj = torch.full((B, D), float("nan"), **f32), torch.full((B,), float("nan"), **f32)
    layer_forward_abi(h, x, D, c, C, B, y, D, ladj, 0, device)
    z64, z32, ladj64, lp64 = fx.oracle(np.arange(B))
    check_z(cpu(y), z64, z32, f"{name} contiguous z")
    check_row(cpu(ladj), ladj64, f"{name} contiguous ladj", None, lp64)
    # strided, odd leading dimensions: the pads of y stay NaN, the results are bit-identical
    xs = torch.full((B, D + 3), float("nan"), **f32)
    xs[:, :D] = x
    cs = None
    if c is not None:
        cs = torch.full((B, C + 5), float("nan"), **f32)
        cs[:, :C] = c
    ys, ls = torch.full((B, D + 5), float("nan"), **f32), torch.full((B,), float("nan"), **f32)
    layer_forward_abi(h, xs, D + 3, cs, C + 5 if C else 0, B, ys, D + 5, ls, 0, device)
    assert torch.equal(ys[:, :D], y) and torch.equal(ls, ladj), f"{name}: strided rows differ"
    assert torch.isnan(ys[:, D:]).all(), f"{name}: the kernel wrote into the row padding"
    # accumulate = 1 adds to what the ladj buffer holds
    base = torch.randn(B, generator=torch.Generator().manual_seed(9)).to(device)
    la = base.clone()
    layer_forward_abi(h, x, D, c, C, B, torch.empty(B, D, **f32), D, la, 1, device)
    assert torch.equal(la, base + ladj), f"{name}: accumulate = 1 is not T + ladj"
    # ladj = NULL: y only
    yn = torch.full((B, D), float("nan"), **f32)
    layer_forward_abi(h, x, D, c, C, B, yn, D, None, 0, device)
    assert torch.equal(yn, y), f"{name}: ladj = NULL changes y"
    # B = 0 writes nothing
    y0, l0 = torch.full((B, D), float("nan"), **f32), torch.full((B,), float("nan"), **f32)
    layer_forward_abi(h, x, D, c, C, 0, y0, D, l0, 0, device)
    assert torch.isnan(y0).all() and torch.isnan(l0).all()
    if C:  # a broadcast context row (ldc = 0) equals the expanded context
        yb, lb = torch.empty(B, D, **f32), torch.empty(B, **f32)
        layer_forward_abi(h, x, D, c[3].contiguous(), 0, B, yb, D, lb, 0, device)
        ye, le = torch.empty(B, D, **f32), torch.empty(B, **f32)
        layer_forward_abi(h, x, D, c[3].expand(B, C).contiguous(), C, B, ye, D, le, 0, device)
        assert torch.equal(yb, ye) and torch.equal(lb, le), f"{name}: ldc = 0 differs from the expanded context"


ABI_FLOWS = {"mixed_tiles": lambda: _position("mixed_tiles"), "between_softclips": lambda: _position("between_softclips")}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ABI_FLOWS))
def test_flow_forward_strides_and_row_chunks(device, name):
    torch.manual_seed(SEED)
    flow = ABI_FLOWS[name]()
    for t in ar_layers(flow):
        t.hyper.gemm_mode = "bf16x3"
    flow = flow.to(device)
    D, C, B = 16, 4, 2 * 128 * sm_count() + 77
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, D, generator=g).to(device)
    c = torch.randn(B, C, generator=g).to(device)
    f32 = dict(device=device, dtype=torch.float32)
    xs = torch.full((B, D + 3), float("nan"), **f32)
    xs[:, :D] = x
    with torch.no_grad():
        fc = flow(c)._flow_call()[0]
    L = E.lib()
    full_ws = L.zk_flow_workspace_bytes(ctypes.byref(fc.desc), B)
    min_ws = L.zk_flow_min_workspace_bytes(ctypes.byref(fc.desc))
    assert min_ws < full_ws
    out = []
    for ws_bytes, ldx, xin in ((full_ws, D, x.contiguous()), (full_ws, D + 3, xs), (min_ws, D + 3, xs)):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        z = torch.full((B, D + 2), float("nan"), **f32)
        ladj = torch.full((B,), float("nan"), **f32)
        lp = torch.full((B,), float("nan"), **f32)
        st = E.stream_ptr(device)
        E.check(L.zk_flow_forward(ctypes.byref(fc.desc), xin.data_ptr(), ldx, c.data_ptr(), C, B, z.data_ptr(), D + 2,
                                  ladj.data_ptr(), ws.data_ptr(), ws_bytes, st))  # fmt: skip
        E.check(L.zk_flow_log_prob(ctypes.byref(fc.desc), xin.data_ptr(), ldx, c.data_ptr(), C, B, lp.data_ptr(), None,
                                   ws.data_ptr(), ws_bytes, st))  # fmt: skip
        torch.cuda.synchronize(device)
        assert torch.isnan(z[:, D:]).all(), f"{name}: the row padding of z was written"
        out.append((z[:, :D].clone(), ladj.clone(), lp.clone()))
    for got in out[1:]:
        assert all(torch.equal(a, b) for a, b in zip(got, out[0])), f"{name}: strided / row-chunked call differs"
    assert all(torch.isfinite(v).all() for v in out[0])
    with torch.no_grad():
        lp_api = flow(c).log_prob(x)
    assert torch.equal(lp_api, out[0][2])


# --------------------------------------------------------------------------- #
# bitwise properties
# --------------------------------------------------------------------------- #

BIT_SHAPES = ["nsf12c4_h320", "maf20_h448", "nsf20c300_k16_h64", "nsf12c4_h448_sigmoid", "maf20_h448_x1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIT_SHAPES)
def test_bitwise_sub_batches_and_runs(device, name):
    """64-row tiles: a row's results do not depend on where the batch starts or on the run."""
    assert plans_of(name)[0]["rows"] == 64
    flow = make_flow(name).to(device)
    B = 5000
    fx = Fixed(name, B)
    xd = dev_t(fx.x, device)
    cd = None if fx.c is None else dev_t(fx.c, device)
    full = [cpu(v) for v in forward_all(flow, xd, cd, device)]
    again = [cpu(v) for v in forward_all(flow, xd, cd, device)]
    assert all(np.array_equal(a, b) for a, b in zip(full, again)), f"{name}: two runs differ"
    for off, n in ((1, 200), (63, 129), (65, 64), (100, 1), (129, 3000), (B - 77, 77)):
        sub = forward_all(flow, xd[off : off + n], None if cd is None else cd[off : off + n], device)
        for a, b, what in zip(sub, full, ("log_prob", "z", "ladj")):
            assert np.array_equal(cpu(a), b[off : off + n]), f"{name}: rows {off}..{off + n} {what} differ from the full batch"
