"""GPU tests of the dimension-sequential inverse (ar_inverse.cu) at its launch-geometry, step-plan, batch and
stride edges, against the fp64 oracle (oracle/oracle.py, which restates the reference's `passes` sweeps).

* `inverse_plan` restates ar_inverse_pack (per-step hidden-unit counts and their 8-wide / 2-wide tiling,
  the sorted state, the largest step block) and inv_geometry from the module's masks, order and passes.
  The shape table reaches every tile remainder 0-7, L = 1 and L = 7 linear layers, an empty order class
  and every geometry rung (two 128-thread CTAs per SM, one CTA of 32-256 threads, the sweeps).  That is
  checked without a GPU; on the GPU `zk_layer_inverse_geometry` must report the same geometry.
* Oracle parity on a shape x batch matrix: batches 1, T - 1, T, T + 1, W - 1, W + 1 and 3W + 77 with T the
  threads per CTA and W one wave (T x CTAs per SM x SMs), in both zk_set_fast_math modes.
* Inputs outside the spline's [-5, 5], at +-5 and its float32 neighbours, and exactly on spline knots.
* The ladj the kernel accumulates for rsample_and_log_prob, for LazyInverse members and in flows that
  mix sequential layers with sweep-fallback layers.
* Bitwise properties: sub-batches, repeated runs and every ZK_INV_GEOM override that fits.
* The C ABI: strided rows, a broadcast context, B = 0 and row chunks of zk_flow_inverse.

Bar of the sequential kernel, per element: |ours - ref64| <= max(1e-5 max(1, |ref64|), 3 |ref32 - ref64|),
ref32 being the oracle in float32 (the reference's own fp32 conditioning).  Layers that fall back to the
sweeps re-round the conditioner `passes` times and get 5e-5 in the first term (test_gpu_inverse.py)."""

import ctypes
import os
from functools import partial

import numpy as np
import pytest
import torch

from cases import O_rqs_knots
from oracle import oracle as O
from zuko_b200 import _engine as E
from zuko_b200.distributions import DiagNormal
from zuko_b200.flows import MAF, NCSF, NSF, MaskedAutoregressiveTransform
from zuko_b200.lazy import Flow, LazyInverse, UnconditionalDistribution, UnconditionalTransform
from zuko_b200.transforms import MonotonicRQSTransform, PermutationTransform, SoftclipTransform

SEED = 0
SEQ_BAR, SWEEP_BAR = 1e-5, 5e-5


def _one(t):
    D = t.features
    return Flow([t], UnconditionalDistribution(DiagNormal, torch.zeros(D), torch.ones(D), buffer=True))


def _adjacency():
    A = torch.tril(torch.ones(5, 5, dtype=torch.bool))
    A[3, 0] = A[4, 1] = False
    return _one(MaskedAutoregressiveTransform(5, 2, adjacency=A, hidden_features=[32, 32]))


def _bins(K):
    return lambda: NSF(6, 2, transforms=1, bins=K, hidden_features=[32, 32])


# name -> one-layer flow.  The geometry table: cfg4 is NSF(64, 0, bins=16) with the hidden widths below
GEOMETRY = {
    "cfg4_h64": lambda: NSF(64, 0, transforms=1, bins=16),
    **{f"cfg4_h{h}": (lambda h=h: NSF(64, 0, transforms=1, bins=16, hidden_features=[h, h])) for h in (96, 128, 160, 168, 456, 464)},
    "cfg2": lambda: NSF(16, 8, transforms=1, bins=8, hidden_features=[256] * 3),
    "cfg3": lambda: MAF(32, 0, transforms=1, hidden_features=[512] * 4),
    "cfg5": lambda: NSF(64, 16, transforms=1, bins=16, hidden_features=[512] * 3),
    # every step finalises k units per hidden layer: remainders k mod 8 (two 8-wide tiles for k = 8)
    **{f"maf8_k{k}": (lambda k=k: MAF(8, 3, transforms=1, hidden_features=[8 * k, 8 * k])) for k in range(1, 9)},
    # L = 7: per-step counts 1..6, remainders 1-6 in one layer stack
    "nsf8_L7": lambda: NSF(8, 0, transforms=1, hidden_features=[7, 14, 21, 28, 35, 42]),
}
EXTRA = {
    "maf1c3": lambda: MAF(1, 3, transforms=1),  # one feature: an element-wise layer, no autoregressive inverse
    "nsf5_passes4": lambda: NSF(5, 0, transforms=1, passes=4, hidden_features=[32, 32]),  # classes {0, 0, 1, 1, 2}
    "maf6_passes1": lambda: MAF(6, 3, transforms=1, passes=1),
    "maf6_L1": lambda: MAF(6, 3, transforms=1, hidden_features=[]),
    "nsf256": lambda: NSF(256, 0, transforms=1, bins=8, hidden_features=[256, 256]),
    "maf5_randperm": lambda: MAF(5, 2, transforms=1, randperm=True, hidden_features=[24]),
    "ncsf4c3": lambda: NCSF(4, 3, transforms=1, hidden_features=[32, 32]),
    **{f"act_{a.__name__.lower()}": (lambda a=a: NSF(5, 2, transforms=1, hidden_features=[32, 32], activation=a))
       for a in (torch.nn.ELU, torch.nn.Tanh, torch.nn.SiLU, torch.nn.GELU, torch.nn.LeakyReLU, torch.nn.Softplus, torch.nn.Sigmoid)},
}  # fmt: skip
FALLBACK = {
    "nsf8_L8": lambda: NSF(8, 0, transforms=1, hidden_features=[16] * 7),
    "nsf6_bins4": _bins(4),
    "nsf6_bins12": _bins(12),
    "maf5_residual": lambda: MAF(5, 2, transforms=1, residual=True, hidden_features=[32, 32]),
    "maf5_adjacency": _adjacency,
}
SHAPES = {**GEOMETRY, **EXTRA, **FALLBACK}

# what each fallback shape is refused for (inverse_plan's reason)
REFUSED = {"nsf8_L8": "depth", "nsf6_bins4": "bins", "nsf6_bins12": "bins", "maf5_residual": "residual",
           "maf5_adjacency": "no order", "cfg4_h464": "state", "cfg3": "state", "cfg5": "state"}  # fmt: skip


def make_flow(name):
    torch.manual_seed(SEED)
    return SHAPES[name]().eval()


# --------------------------------------------------------------------------- #
# the step plan and launch geometry, restated
# --------------------------------------------------------------------------- #

TILE = 8


def inverse_plan(t):
    """ar_inverse_pack + inv_geometry (ar_inverse.cu) restated for the layer module `t`.  Returns a dict:
    path ("kernel" / "sweeps" / "none": not an autoregressive layer), why (refusal), L, steps (per step:
    hidden units finalised per layer, their n8 / n2 tiles, dims of the class), state_floats, max_step_words,
    and for the kernel path threads, per_thread, smem, ctas (per SM, by the rule of inv_geometry)."""
    if type(t).__name__ != "MaskedAutoregressiveTransform":
        return {"path": "none", "why": type(t).__name__}
    lins = t.hyper._linears()
    L, u = len(lins), t._uni
    kind = E.ZK_UNI_RQS if u["kind"] == E.ZK_UNI_CRQS else u["kind"]
    why = None
    if t.order is None:
        why = "no order"
    elif not 1 <= L <= 7:
        why = "depth"
    elif any(type(m).__name__ == "Residual" for m in t.hyper):
        why = "residual"
    elif kind == E.ZK_UNI_RQS and u["bins"] not in (8, 16):
        why = "bins"
    elif kind not in (E.ZK_UNI_RQS, E.ZK_UNI_AFFINE):
        why = "bijector"
    if why:
        return {"path": "sweeps", "why": why, "L": L}
    D, C, P, passes = t.features, t.context, u["total"], t.passes
    order = t.order.numpy().astype(np.int64)
    masks = [m.mask.numpy().astype(bool) for m in lins]
    dims = [D + C] + [int(m.weight.shape[0]) for m in lins]
    fin = [np.concatenate([order + 1, np.zeros(C, np.int64)])]  # step at which each input is final
    ready = []
    for mk in masks:  # 1 + the largest order class a unit depends on
        ready.append(np.where(mk, fin[-1][None, :], 0).max(1) if mk.shape[1] else np.zeros(mk.shape[0], np.int64))
        fin.append(ready[-1])
    assert (ready[-1].reshape(D, P).max(1) <= order).all(), "not a pure order-class structure"
    PT = -(-P // TILE)
    steps, words = [], []
    for p in range(passes):
        n = [int((ready[l] == p).sum()) for l in range(L - 1)]
        n8 = [k // TILE + (k % TILE > 4) for k in n]
        n2 = [(k % TILE + 1) // 2 if 1 <= k % TILE <= 4 else 0 for k in n]
        K = [int((fin[l] <= p).sum()) for l in range(L)]
        nd = int((order == p).sum())
        w = (3 * L + 3) & ~3  # header
        w += -(-sum(a * TILE + b * 2 for a, b in zip(n8, n2)) // 4) * 4  # destinations
        w += -(-2 * nd // 4) * 4  # dims
        w += sum(a * (K[l] + 1) * TILE + b * (-(-(K[l] + 1) * 2 // 4) * 4) for l, (a, b) in enumerate(zip(n8, n2)))
        w += nd * (K[L - 1] + 1) * PT * TILE
        steps.append({"units": n, "n8": n8, "n2": n2, "dims": nd, "K": K})
        words.append(w)
    state = D + C + sum(dims[1:L])
    plan = {"path": "kernel", "why": None, "L": L, "steps": steps, "state_floats": state, "max_step_words": max(words)}
    per_sample, wbytes, budget = 4 * state, 4 * max(words) + 16, 226 * 1024
    plan["fits"] = lambda T, R: per_sample * T * R + wbytes <= budget
    if per_sample * 128 + wbytes <= 112 * 1024:
        return {**plan, "threads": 128, "per_thread": 1, "smem": per_sample * 128 + wbytes, "ctas": 2}
    T = min(256, (budget - min(budget, wbytes)) // per_sample // 32 * 32)
    if T < 32:
        return {**plan, "path": "sweeps", "why": "state"}
    return {**plan, "threads": T, "per_thread": 1, "smem": per_sample * T + wbytes, "ctas": 1}


def layer_of(flow):
    ts = flow.transform.transforms
    assert len(ts) == 1
    return ts[0]


# geometry the issue's table expects: threads per CTA and CTAs per SM, or None for the sweeps
EXPECTED = {"cfg4_h64": (128, 2), "cfg4_h96": (192, 1), "cfg4_h128": (160, 1), "cfg4_h160": (128, 1), "cfg4_h168": (96, 1),
            "cfg4_h456": (32, 1), "cfg4_h464": None, "cfg2": (32, 1), "cfg3": None, "cfg5": None,
            **{f"maf8_k{k}": (128, 2) for k in range(1, 9)}, "nsf8_L7": (128, 2)}  # fmt: skip


def test_plan_reaches_every_case():
    """The shape table really reaches each case of the pack and the geometry (no GPU needed)."""
    plans = {name: inverse_plan(layer_of(make_flow(name))) for name in SHAPES}
    kernel = {k: p for k, p in plans.items() if p["path"] == "kernel"}
    for name, want in EXPECTED.items():
        p = plans[name]
        got = None if p["path"] != "kernel" else (p["threads"], p["ctas"])
        assert got == want, f"{name}: plan {got}, table {want}"
    rems = {k % TILE for p in kernel.values() for s in p["steps"] for k in s["units"] if k}
    assert rems == set(range(TILE)), f"tile remainders reached: {sorted(rems)}"
    for name in (f"maf8_k{k}" for k in range(1, 9)):  # exactly k units per step and hidden layer
        k = int(name[-1])
        assert all(s["units"] == [k, k] for s in kernel[name]["steps"][1:]), name
    assert {p["L"] for p in kernel.values()} >= {1, 7}
    assert any(s["dims"] == 0 for p in kernel.values() for s in p["steps"]), "no empty order class"
    assert kernel["nsf5_passes4"]["steps"][3]["dims"] == 0
    assert kernel["nsf256"]["threads"] == 64 and len(kernel["nsf256"]["steps"]) == 256
    rungs = {(p["threads"], p["ctas"]) for p in kernel.values()}
    assert (128, 2) in rungs and {192, 160, 128, 96, 32} <= {T for T, n in rungs if n == 1}, rungs
    for name, why in REFUSED.items():
        assert plans[name]["path"] == "sweeps" and plans[name]["why"] == why, (name, plans[name]["why"])
    assert plans["maf1c3"]["path"] == "none"


# --------------------------------------------------------------------------- #
# GPU helpers
# --------------------------------------------------------------------------- #


def sm_count():
    n, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    E.check(E.lib().zk_device_info(ctypes.byref(n), ctypes.byref(major), ctypes.byref(minor)))
    return n.value


def query(handle):
    """zk_layer_inverse_geometry: (threads, samples per thread, smem) or None."""
    T, R, smem = ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_size_t(0)
    ok = E.lib().zk_layer_inverse_geometry(handle, ctypes.byref(T), ctypes.byref(R), ctypes.byref(smem))
    return (T.value, R.value, smem.value) if ok else None


def dev_t(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)


def cpu(t):
    return t.detach().cpu().numpy().astype(np.float64)


def context_dim(flow):
    return getattr(flow.transform.transforms[0], "context", 0)


def misses(ours, ref64, ref32, rtol):
    ours, ref64, ref32 = (np.asarray(a, np.float64) for a in (ours, ref64, ref32))
    tol = np.maximum(rtol * np.maximum(np.abs(ref64), 1.0), 3.0 * np.abs(ref32 - ref64))
    with np.errstate(invalid="ignore"):
        return ~(np.abs(ours - ref64) <= tol)


def check(ours, ref64, ref32, rtol, what, rows=None):
    bad = misses(ours, ref64, ref32, rtol)
    if bad.any():
        i = np.argwhere(bad)[0]
        r = tuple(i)
        row = r[0] if rows is None else rows[r[0]]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} entries off the oracle; first at row {row} "
                             f"{r[1:]}: ours {ours[r]!r} ref64 {ref64[r]!r} ref32 {ref32[r]!r}")  # fmt: skip


class Fixed:
    """Seeded inputs of one shape whose rows do not depend on the batch (z[:B] for every B), and the
    oracle on the rows checked so far: one shape's oracle is shared by all its batches and math modes."""

    def __init__(self, name, n):
        self.name, self.flow = name, make_flow(name)
        self.spec = O.flowspec_from_module(self.flow)
        D, C = layer_of(self.flow).features, context_dim(self.flow)
        g = torch.Generator().manual_seed(1234)
        if name.startswith("ncsf"):
            self.z = ((torch.rand(n, D, generator=g) * 2 - 1) * 3.1).numpy()
        else:
            self.z = torch.randn(n, D, generator=g).numpy()
        self.c = torch.randn(n, C, generator=g).numpy() if C else None
        self.known = np.zeros(n, bool)
        self.x64, self.x32 = np.zeros((n, D)), np.zeros((n, D))
        self.lp64, self.lp32 = np.zeros(n), np.zeros(n)

    def oracle(self, rows):
        new = np.setdiff1d(rows, np.nonzero(self.known)[0])
        if new.size:
            c = None if self.c is None else self.c[new]
            self.x64[new], self.lp64[new] = self.spec.inverse_and_log_prob(self.z[new].astype(np.float64), c)
            self.x32[new], self.lp32[new] = self.spec.inverse_and_log_prob(self.z[new], None if c is None else c.astype(np.float32), np.float32)
            self.known[new] = True
        return self.x64[rows], self.x32[rows], self.lp64[rows], self.lp32[rows]


_FIXED = {}


def fixed(name, n):
    f = _FIXED.get(name)
    if f is None or f.z.shape[0] < n:
        _FIXED.clear()  # one shape at a time: the matrix runs shape by shape
        f = _FIXED[name] = Fixed(name, n)
    return f


def geometry(plan):
    """(T, CTAs per SM, samples per CTA) of the batch edges; the sweeps have no CTA: 128 rows stand in."""
    if plan["path"] != "kernel":
        return 128, 1, 128
    return plan["threads"], plan["ctas"], plan["threads"] * plan["per_thread"]


BATCHES = ["1", "T-1", "T", "T+1", "W-1", "W+1", "3W+77"]


def batch_of(key, T, W):
    return {"1": 1, "T-1": T - 1, "T": T, "T+1": T + 1, "W-1": W - 1, "W+1": W + 1, "3W+77": 3 * W + 77}[key]


def oracle_rows(B, S, W, n_random=512):
    """Every row of the first CTA and of the last two, and n_random rows drawn once below W - 1 (the same
    rows for every large batch of a shape, so that the oracle is evaluated once)."""
    if B <= 4 * S + n_random:
        return np.arange(B)
    last = -(-B // S) * S
    rnd = np.random.default_rng(7).choice(W - 1, n_random, replace=False)
    return np.unique(np.concatenate([np.arange(S), np.arange(max(0, last - 2 * S), B), rnd]))


def assert_round_trip(spec, flow, z, c, x, device, what, fast):
    """t(t.inv(z)) equals z as torch.allclose(atol=1e-4) has it, on every row (test_gpu_inverse.py).  A row
    beyond that must be one on which the oracle's own float32 round trip drifts about as far: an affine
    layer's exp(scale) reaches 1e3, so x and the next dimensions' shifts reach 1e3 too, and a batch of 1e5
    rows meets such rows.  "As far" is 3x in IEEE mode.  In fast-math mode exp is the MUFU approximation,
    whose error is 2 + floor(1.173 |s|) ulp (CUDA C++ Programming Guide, intrinsic functions), about 10 ulp
    at the affine's |s| <= 6.9, against the oracle's correctly rounded exp: 12x there (measured on an H100
    80GB HBM3: 9.4x on one row of maf6_L1 at B = 101453)."""
    factor = 12.0 if fast else 3.0
    with torch.no_grad():
        zz = cpu(flow(None if c is None else dev_t(c, device)).transform(dev_t(x, device)))
    err = np.abs(zz - z)
    assert np.isfinite(err).all(), what
    tol = 1e-4 + 1e-5 * np.abs(z)
    far = np.nonzero((err > tol).any(-1))[0]
    if far.size:
        cf = None if c is None else c[far].astype(np.float32)
        z32 = spec.forward(spec.inverse(z[far], cf, np.float32), cf, np.float32)[0]
        ref = np.abs(z32 - z[far])
        worse = (err[far] > np.maximum(tol[far], factor * ref)).any(-1)
        err = err.max(-1)
        ref = ref.max(-1)
        assert not worse.any(), (f"{what}: round trip {err[far][worse].max():.3e} on {int(worse.sum())} rows "
                                 f"(first {far[worse][0]}), the oracle's fp32 round trip {ref[worse].max():.3e}")  # fmt: skip


def run_inverse(flow, z, c, device, with_log_prob=True):
    zd, cd = dev_t(z, device), (None if c is None else dev_t(c, device))
    with torch.no_grad():
        call, ctx = flow(cd)._flow_call()
        if with_log_prob:
            x, lp = call.inverse(zd, ctx, with_log_prob=True)
            return x, lp
        return call.inverse(zd, ctx), None


@pytest.fixture
def math_mode(request):
    prev = E.lib().zk_set_fast_math(1)
    yield lambda fast: E.lib().zk_set_fast_math(int(fast))
    E.lib().zk_set_fast_math(prev)


# --------------------------------------------------------------------------- #
# b. path and geometry
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_path_and_geometry(device, name):
    flow = make_flow(name)
    plan = inverse_plan(layer_of(flow))
    flow = flow.to(device)
    t = layer_of(flow)
    h = t._zk_layer()
    got = query(h)
    want = None if plan["path"] != "kernel" else (plan["threads"], plan["per_thread"], plan["smem"])
    print(f"{name}: zk_layer_inverse_geometry {got}, plan {want}")
    assert got == want, f"{name}: the engine reports {got}, the restated plan {want}"
    assert E.lib().zk_layer_sequential_inverse(h) == (plan["path"] == "kernel")
    D, C = t.features, context_dim(flow)
    g = torch.Generator().manual_seed(5)
    B = 300
    z = torch.randn(B, D, generator=g).numpy()
    c = torch.randn(B, C, generator=g).numpy() if C else None
    zd, cd = dev_t(z, device), (None if c is None else dev_t(c, device))
    with torch.no_grad():
        flow(cd).transform.inv(zd[:1])  # packs outside the count
        n0 = E.lib().zk_launch_count()
        x = flow(cd).transform.inv(zd)
        launches = E.lib().zk_launch_count() - n0
    if plan["path"] == "kernel":
        assert launches == 1, launches
    if plan["path"] == "sweeps":
        assert launches > 1, launches  # `passes` conditioner + bijector sweeps
        if name in ("cfg3", "cfg5", "cfg4_h464"):  # the oracle's sweeps cost `passes` wide MLPs: a row subset
            rows = np.arange(0, B, 7)
            z, c, x = z[rows], (None if c is None else c[rows]), x[torch.as_tensor(rows, device=device)]
        spec = O.flowspec_from_module(make_flow(name))
        x64 = spec.inverse(z.astype(np.float64), c)
        x32 = spec.inverse(z, None if c is None else c.astype(np.float32), np.float32)
        check(cpu(x), x64, x32, SWEEP_BAR, f"{name} sweeps")


# --------------------------------------------------------------------------- #
# c. oracle parity matrix
# --------------------------------------------------------------------------- #

MATRIX_SHAPES = [n for n in GEOMETRY if n not in ("cfg3", "cfg5", "cfg4_h464")] + list(EXTRA)
MATRIX = [(s, b, fast) for s in MATRIX_SHAPES for b in BATCHES for fast in (1, 0)]
# nsf256 runs 256 sweeps of a 256-wide conditioner per oracle row
RANDOM_ROWS = {"nsf256": 128}


@pytest.mark.gpu
@pytest.mark.parametrize("name,b,fast", MATRIX, ids=[f"{s}-{b}-{'fast' if f else 'ieee'}" for s, b, f in MATRIX])
def test_oracle_parity_matrix(device, math_mode, name, b, fast):
    math_mode(fast)
    plan = inverse_plan(layer_of(make_flow(name)))
    T, ctas, S = geometry(plan)
    W = T * ctas * sm_count()
    B = batch_of(b, T, W)
    fx = fixed(name, 3 * W + 77)
    flow = fx.flow.to(device)
    z, c = fx.z[:B], (None if fx.c is None else fx.c[:B])
    x, lp = run_inverse(flow, z, c, device)
    x, lp = cpu(x), cpu(lp)
    rows = oracle_rows(B, S, W, RANDOM_ROWS.get(name, 512))
    x64, x32, lp64, lp32 = fx.oracle(rows)
    bar = SEQ_BAR if plan["path"] != "sweeps" else SWEEP_BAR
    what = f"{name} B={B} ({b}, T={T}) {'fast' if fast else 'ieee'}"
    assert np.isfinite(x).all() and np.isfinite(lp).all(), what
    check(x[rows], x64, x32, bar, what + " x", rows)
    check(lp[rows], lp64, lp32, bar, what + " log_prob", rows)
    assert_round_trip(fx.spec, flow, z, c, x, device, what, fast)


# --------------------------------------------------------------------------- #
# d. input edges
# --------------------------------------------------------------------------- #

EDGE_SHAPES = ["cfg4_h64", "cfg4_h456", "cfg2", "nsf8_L7", "maf8_k3", "nsf6_bins4"]


def edge_inputs(name, flow, B):
    """z x 4 (many entries outside [-5, 5], where the spline is the identity); entries at +-5 and their float32
    neighbours; entries of the order-class-0 dimensions exactly on a y-knot (their phi depends on c only)."""
    t = layer_of(flow)
    D, C = t.features, context_dim(flow)
    g = torch.Generator().manual_seed(11)
    z = (torch.randn(B, D, generator=g) * 4).numpy()
    c = torch.randn(B, C, generator=g).numpy() if C else None
    f5 = np.float32(5)
    edges = np.array([f5, -f5, np.nextafter(f5, 0), np.nextafter(-f5, 0), np.nextafter(f5, 9), np.nextafter(-f5, -9)], np.float32)
    z[::3, :] = edges[(np.arange(0, B, 3)[:, None] + np.arange(D)) % edges.size]
    layer = O.flowspec_from_module(flow).layers[0]
    if layer.univariate == "rqs":
        cls0 = np.nonzero(t.order.numpy() == 0)[0]
        P = 3 * layer.bins - 1
        phi = layer.hyper(np.zeros((B, D)), c, np.float64).reshape(B, D, P)[:, cls0]
        _, Y, _ = O_rqs_knots(phi, layer.bins, layer.bound, layer.slope)
        rows = np.arange(1, B, 3)
        k = np.broadcast_to((rows % (layer.bins + 1))[:, None, None], (rows.size, cls0.size, 1))
        z[rows[:, None], cls0[None, :]] = np.take_along_axis(Y[rows], k, 2)[..., 0]
    return z.astype(np.float32), c


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
@pytest.mark.parametrize("name", EDGE_SHAPES)
def test_input_edges(device, math_mode, name, fast):
    math_mode(fast)
    cpu_flow = make_flow(name)
    plan = inverse_plan(layer_of(cpu_flow))
    T = geometry(plan)[0]
    B = 2 * T + 3
    z, c = edge_inputs(name, cpu_flow, B)
    spec = O.flowspec_from_module(cpu_flow)
    x64, lp64 = spec.inverse_and_log_prob(z.astype(np.float64), c)
    x32, lp32 = spec.inverse_and_log_prob(z, None if c is None else c.astype(np.float32), np.float32)
    flow = make_flow(name).to(device)
    x, lp = run_inverse(flow, z, c, device)
    bar = SEQ_BAR if plan["path"] == "kernel" else SWEEP_BAR
    check(cpu(x), x64, x32, bar, f"{name} x")
    check(cpu(lp), lp64, lp32, bar, f"{name} log_prob")
    assert_round_trip(spec, flow, z, c, cpu(x), device, f"{name} input edges", fast)


# --------------------------------------------------------------------------- #
# e. ladj paths
# --------------------------------------------------------------------------- #


def _mixed(first_sequential):
    """D = 64 members: sequential layers (hidden [64, 64]: two 128-thread CTAs), sweep fallbacks (4 bins;
    hidden [464, 464]), a permutation and a soft clip.  The LAST member is the first the inverse runs: a
    sequential one folds the base density into its kernel, a sweep one seeds it apart."""
    D = 64
    seq = lambda: MaskedAutoregressiveTransform(D, 0, univariate=MonotonicRQSTransform, shapes=[(16,), (16,), (15,)])  # noqa: E731
    bins4 = lambda: MaskedAutoregressiveTransform(D, 0, univariate=partial(MonotonicRQSTransform, slope=1e-3),  # noqa: E731
                                                  shapes=[(4,), (4,), (3,)], order=torch.arange(D).flip(0))  # fmt: skip
    wide = lambda: MaskedAutoregressiveTransform(D, 0, hidden_features=[464, 464], univariate=MonotonicRQSTransform,  # noqa: E731
                                                 shapes=[(16,), (16,), (15,)])  # fmt: skip
    perm = UnconditionalTransform(PermutationTransform, torch.randperm(D), buffer=True)
    clip = UnconditionalTransform(SoftclipTransform, bound=11.0)
    layers = [wide(), clip, seq(), perm, bins4(), seq()] if first_sequential else [seq(), perm, seq(), clip, wide(), bins4()]
    return Flow(layers, UnconditionalDistribution(DiagNormal, torch.zeros(D) + 0.25, torch.ones(D) * 1.5, buffer=True))


LADJ_FLOWS = {
    "nsf64_k16_x3": lambda: NSF(64, 0, transforms=3, bins=16),  # base folded into the first inverted layer, then accumulated
    "nsf16c8_h256_x2": lambda: NSF(16, 8, transforms=2, bins=8, hidden_features=[256] * 3),
    "mixed_seq_first": lambda: _mixed(True),
    "mixed_sweep_first": lambda: _mixed(False),
    "ncsf4c3_x2": lambda: NCSF(4, 3, transforms=2, hidden_features=[32, 32]),  # BoxUniform base
}


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 127, 129, 300])
@pytest.mark.parametrize("name", list(LADJ_FLOWS))
def test_rsample_and_log_prob_ladj(device, name, B):
    torch.manual_seed(SEED)
    cpu_flow = LADJ_FLOWS[name]().eval()
    spec = O.flowspec_from_module(cpu_flow)
    D = spec.loc.shape[0]
    C = getattr(cpu_flow.transform.transforms[0], "context", 0)
    g = torch.Generator().manual_seed(B)
    z = ((torch.rand(B, D, generator=g) * 2 - 1) * 3.1 if name.startswith("ncsf") else torch.randn(B, D, generator=g)).numpy()
    c = torch.randn(B, C, generator=g).numpy() if C else None
    x64, lp64 = spec.inverse_and_log_prob(z.astype(np.float64), c)
    x32, lp32 = spec.inverse_and_log_prob(z, None if c is None else c.astype(np.float32), np.float32)
    torch.manual_seed(SEED)
    flow = LADJ_FLOWS[name]().to(device)
    flow.load_state_dict(cpu_flow.state_dict())
    x, lp = run_inverse(flow, z, c, device)
    bar = SWEEP_BAR if name.startswith("mixed") else SEQ_BAR
    check(cpu(x), x64, x32, bar, f"{name} B={B} x")
    check(cpu(lp), lp64, lp32, bar, f"{name} B={B} log_prob")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, "T-1", "T+1", "3T+5"])
@pytest.mark.parametrize("hidden", [64, 168, 456])
def test_lazy_inverse_members_ladder(device, hidden, B):
    """IAF stack (zuko/lazy.py:81-98) on the geometry ladder: the member's kernel accumulates minus the layer's
    forward ladj (sign -1) and the last member the base density of its OUTPUT (base = 2)."""
    D, n = 64, 2
    torch.manual_seed(SEED)
    layers = [MaskedAutoregressiveTransform(D, 0, hidden_features=[hidden, hidden], univariate=MonotonicRQSTransform,
                                            shapes=[(16,), (16,), (15,)], order=torch.arange(D) if i % 2 == 0 else torch.arange(D).flip(0))
              for i in range(n)]  # fmt: skip
    base = lambda: UnconditionalDistribution(DiagNormal, torch.zeros(D) + 0.25, torch.ones(D) * 1.5, buffer=True)  # noqa: E731
    spec = O.flowspec_from_module(Flow(layers, base()).eval())
    T = inverse_plan(layers[0])["threads"]
    B = {"T-1": T - 1, "T+1": T + 1, "3T+5": 3 * T + 5}.get(B, B)
    x = torch.randn(B, D, generator=torch.Generator().manual_seed(B)).numpy()

    def ref(dtype):
        u, total = x.astype(dtype), np.zeros(B, dtype)
        for layer in spec.layers:  # u_{l+1} = layer_l^-1(u_l), ladj_member = -ladj_layer(u_{l+1})
            u = layer.inverse(u, None, dtype)
            total = total - layer.forward(u, None, dtype)[1]
        return O.diag_normal_log_prob(u, spec.loc, spec.scale, total, dtype)

    iaf = Flow([LazyInverse(t) for t in layers], base()).to(device)
    with torch.no_grad():
        dist = iaf()
        assert dist._flow_call()[0]._inverted == [True] * n
        for t in layers:
            assert query(t._zk_layer())[0] == T
        n0 = E.lib().zk_launch_count()
        lp = dist.log_prob(dev_t(x, device))
        assert E.lib().zk_launch_count() - n0 == n
    check(cpu(lp), ref(np.float64), ref(np.float32), SEQ_BAR, f"IAF hidden={hidden} B={B}")


# --------------------------------------------------------------------------- #
# f. bitwise properties
# --------------------------------------------------------------------------- #

BIT_SHAPES = ["cfg4_h64", "cfg2", "maf8_k3", "nsf8_L7", "act_elu", "ncsf4c3"]


@pytest.fixture
def inv_geom():
    """Sets ZK_INV_GEOM (read by every launch); restores the environment."""
    prev = os.environ.get("ZK_INV_GEOM")

    def put(v):
        if v is None:
            os.environ.pop("ZK_INV_GEOM", None)
        else:
            os.environ["ZK_INV_GEOM"] = v

    yield put
    put(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIT_SHAPES)
def test_bitwise_sub_batches_runs_and_geometries(device, inv_geom, name):
    inv_geom(None)
    cpu_flow = make_flow(name)
    plan = inverse_plan(layer_of(cpu_flow))
    T = plan["threads"]
    flow = make_flow(name).to(device)
    h = layer_of(flow)._zk_layer()
    B = 3 * 512 + 77
    fx = Fixed(name, B)
    z, c = fx.z, fx.c
    full = [cpu(v) for v in run_inverse(flow, z, c, device)]
    again = [cpu(v) for v in run_inverse(flow, z, c, device)]
    assert all(np.array_equal(a, b) for a, b in zip(full, again)), "two runs differ"
    for off in (1, T - 3, T, 2 * T, T + 5):  # aligned and unaligned to the CTA
        n = min(2 * T + 1, B - off)
        sub = run_inverse(flow, z[off : off + n], None if c is None else c[off : off + n], device)
        for a, b, what in zip(sub, full, ("x", "log_prob")):
            assert np.array_equal(cpu(a), b[off : off + n]), f"{name}: rows {off}..{off + n} {what} differ from the full batch"
    r2 = layer_of(cpu_flow)._uni["kind"] != E.ZK_UNI_SOSP
    tried = []
    for Tq in (32, 64, 96, 256):
        for R in (1, 2) if r2 else (1,):
            if not plan["fits"](Tq, R):
                continue
            inv_geom(f"{Tq}x{R}")
            assert query(h)[:2] == (Tq, R), f"ZK_INV_GEOM={Tq}x{R} did not take effect: {query(h)}"
            got = [cpu(v) for v in run_inverse(flow, z, c, device)]
            # every sample runs the same fmaf sequence in every geometry
            for a, b, what in zip(got, full, ("x", "log_prob")):
                assert np.array_equal(a, b), f"{name}: {what} under {Tq}x{R} differs from the default {T}x1 (max {np.abs(a - b).max():.3e})"
            tried.append((Tq, R))
    inv_geom(None)
    assert query(h)[:2] == (T, 1)
    print(f"{name}: overrides {tried}")
    assert tried


# --------------------------------------------------------------------------- #
# g. C ABI
# --------------------------------------------------------------------------- #

ABI_SHAPES = ["cfg4_h64", "cfg2", "maf8_k5", "ncsf4c3", "maf6_L1"]


def layer_inverse_abi(h, y, ldy, c, ldc, B, x, ldx, device):
    L = E.lib()
    need = L.zk_layer_workspace_bytes(h, B)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    E.check(L.zk_layer_inverse(h, p(y), ldy, p(c), ldc, B, p(x), ldx, p(ws), need, E.stream_ptr(device)))
    torch.cuda.synchronize(device)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ABI_SHAPES)
def test_layer_inverse_c_abi(device, name):
    flow = make_flow(name).to(device)
    t = layer_of(flow)
    h = t._zk_layer()
    assert E.lib().zk_layer_sequential_inverse(h) == 1
    D, C = t.features, context_dim(flow)
    T = query(h)[0]
    B = 2 * T + 7
    fx = Fixed(name, B)
    f32 = dict(device=device, dtype=torch.float32)
    y = dev_t(fx.z, device)
    c = None if fx.c is None else dev_t(fx.c, device)
    ref = torch.full((B, D), float("nan"), **f32)
    layer_inverse_abi(h, y, D, c, C, B, ref, D, device)
    x64 = fx.oracle(np.arange(B))[0]
    x32 = fx.x32[:B]
    check(cpu(ref), x64, x32, SEQ_BAR, f"{name} contiguous")
    # strided rows: the pads of x stay NaN, the results are bit-identical
    ys = torch.full((B, D + 3), float("nan"), **f32)
    ys[:, :D] = y
    cs = None
    if c is not None:
        cs = torch.full((B, C + 2), float("nan"), **f32)
        cs[:, :C] = c
    xs = torch.full((B, D + 5), float("nan"), **f32)
    layer_inverse_abi(h, ys, D + 3, cs, C + 2 if C else 0, B, xs, D + 5, device)
    assert torch.equal(xs[:, :D], ref), f"{name}: strided rows differ"
    assert torch.isnan(xs[:, D:]).all(), f"{name}: the kernel wrote into the row padding"
    # B = 0 writes nothing
    x0 = torch.full((B, D), float("nan"), **f32)
    layer_inverse_abi(h, y, D, c, C, 0, x0, D, device)
    assert torch.isnan(x0).all()
    if C:  # a broadcast context row (ldc = 0) equals the expanded context
        xb = torch.full((B, D), float("nan"), **f32)
        layer_inverse_abi(h, y, D, c[3].contiguous(), 0, B, xb, D, device)
        xe = torch.full((B, D), float("nan"), **f32)
        layer_inverse_abi(h, y, D, c[3].expand(B, C).contiguous(), C, B, xe, D, device)
        assert torch.equal(xb, xe), f"{name}: ldc = 0 differs from the expanded context"


def flow_inverse_abi(fc, z, ldz, c, ldc, B, x, ldx, lp, ws_bytes, device):
    L = E.lib()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    E.check(L.zk_flow_inverse(ctypes.byref(fc.desc), p(z), ldz, p(c), ldc, B, p(x), ldx, p(lp), p(ws), ws_bytes, E.stream_ptr(device)))
    torch.cuda.synchronize(device)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["nsf64_k16_x3", "nsf16c8_h256_x2", "mixed_sweep_first", "ncsf4c3_x2"])
def test_flow_inverse_strides_and_row_chunks(device, name):
    torch.manual_seed(SEED)
    flow = LADJ_FLOWS[name]().to(device)
    D = flow.transform.transforms[0].features
    C = getattr(flow.transform.transforms[0], "context", 0)
    B = 261
    g = torch.Generator().manual_seed(3)
    z = ((torch.rand(B, D, generator=g) * 2 - 1) * 3.1) if name.startswith("ncsf") else torch.randn(B, D, generator=g)
    c = torch.randn(B, C, generator=g).to(device) if C else None
    f32 = dict(device=device, dtype=torch.float32)
    zs = torch.full((B, D + 3), float("nan"), **f32)
    zs[:, :D] = z.to(device)
    with torch.no_grad():
        fc = flow(c)._flow_call()[0]
    L = E.lib()
    full_ws = L.zk_flow_workspace_bytes(ctypes.byref(fc.desc), B)
    min_ws = L.zk_flow_min_workspace_bytes(ctypes.byref(fc.desc))
    assert min_ws < full_ws
    out = []
    for ws_bytes, ldz, zin in ((full_ws, D, zs[:, :D].contiguous()), (full_ws, D + 3, zs), (min_ws, D + 3, zs)):
        x = torch.full((B, D + 2), float("nan"), **f32)
        lp = torch.full((B,), float("nan"), **f32)
        flow_inverse_abi(fc, zin, ldz, c, C, B, x, D + 2, lp, ws_bytes, device)
        assert torch.isnan(x[:, D:]).all(), f"{name}: the row padding of x was written"
        out.append((x[:, :D].clone(), lp.clone()))
    for x, lp in out[1:]:
        assert torch.equal(x, out[0][0]) and torch.equal(lp, out[0][1]), f"{name}: strided / row-chunked call differs"
    assert torch.isfinite(out[0][0]).all() and torch.isfinite(out[0][1]).all()
