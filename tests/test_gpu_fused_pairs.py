"""GPU tests of the fused layer kernel's output layer on 128-row tiles, where the output chunks are multiplied and
evaluated in pairs (A, B) = (2j, 2j + 1) (fused_layer.cu), against the fp64 oracle (oracle/oracle.py) at the bars of
test_gpu_fused_edges.py.

The one-layer flows below are chosen for the pair edges: an odd n_last (the last pair has no chunk B) with the last
chunk holding a single dim, n_last = 1, adjacent chunks of 1 and 4 non-zero K-block tiles and pairs of 4 + 4 tiles
(more than the flagship shape's four-slot ring holds, so slots roll over inside a pair and across pair boundaries),
and the affine 128-row instantiation, in bf16x3 and bf16x1 and in both math modes.  The batches end in partial tiles
(1, 127, 129 and 2^17 + 1 rows, the last over several waves of the persistent grid).  Also: strided x / y,
accumulate and ladj = NULL through the C ABI, the log_prob of a flow's last layer, and bit-identical rows whether a
row runs alone or inside a larger batch."""

import numpy as np
import pytest
import torch

from cases import rel_err
from oracle import oracle as O
from test_gpu_fused_edges import (
    _one,
    _rqs,
    ar_layers,
    check_row,
    check_z,
    context_dim,
    cpu,
    dev_t,
    forward_all,
    fused_plan_of,
    layer_forward_abi,
    math_mode,  # noqa: F401  (fixture)
    oracle_rows,
    query,
    sm_count,
    unfused,  # noqa: F401  (fixture)
    want,
)
from zuko_b200.flows import MAF, NSF

SEED = 0

# output order of the 16 dims: chunks (two dims each) whose dims come first or last in the order alternate, so that
# adjacent chunks have 1 and 4 non-zero K-block tiles in both orders, and chunks 6, 7 (orders 6 - 9) have 2 and 3
MIXED_ORDER = torch.tensor([0, 1, 14, 15, 12, 13, 2, 3, 4, 5, 10, 11, 6, 7, 8, 9])

BASE = {
    "nsf9c4_h256": lambda: NSF(9, 4, transforms=1, bins=8, hidden_features=[256] * 2),  # n_last 5, chunk 4: one dim
    "nsf2c3_h128": lambda: NSF(2, 3, transforms=1, bins=8, hidden_features=[128] * 2),  # n_last 1
    "nsf16c8_h256x3": lambda: NSF(16, 8, transforms=1, bins=8, hidden_features=[256] * 3),  # flagship layer: 4 + 4 pair
    "nsf16c8_h256x3_mixed": lambda: _one(_rqs(16, 8, [256] * 3, order=MIXED_ORDER)),  # 1 + 4 and 4 + 1 pairs
    "maf65_h192": lambda: MAF(65, 0, transforms=1, hidden_features=[192] * 2),  # affine: n_last 3, chunk 2: one dim
    "maf80c8_h128": lambda: MAF(80, 8, transforms=1, hidden_features=[128] * 2),  # affine: n_last 3, 16 dims last
}
SHAPES = {**{n: (c, "bf16x3") for n, c in BASE.items()}, **{f"{n}_x1": (c, "bf16x1") for n, c in BASE.items()}}
BATCHES = [1, 127, 129, (1 << 17) + 1]


def make_flow(name):
    torch.manual_seed(SEED)
    ctor, mode = SHAPES[name]
    flow = ctor().eval()
    for t in ar_layers(flow):
        t.hyper.gemm_mode = mode
    return flow


_PLANS = {}


def plan_of(name):
    if name not in _PLANS:
        (_PLANS[name],) = [fused_plan_of(t) for t in ar_layers(make_flow(name))]
    return _PLANS[name]


def pairs_of(plan):
    """Tiles per output chunk, grouped in the kernel's pairs (an odd n_last ends in a pair with an empty B)."""
    tiles = [int(v) for v in plan["kbmask"][-1][:, : plan["nch"]].sum(1)]
    return [(tiles[i], tiles[i + 1] if i + 1 < len(tiles) else None) for i in range(0, len(tiles), 2)]


def test_shapes_reach_the_pair_edges():
    """Every shape runs 128-row tiles, and together they reach the pair edges named in the module docstring (no
    GPU)."""
    plans = {n: plan_of(n) for n in SHAPES}
    for n, p in plans.items():
        assert p["why"] is None and p["rows"] == 128, (n, p["why"], p["rows"])
    assert {p["tile"] for p in plans.values()} == {"128x3", "128x1"}
    assert {p["uni"] for p in plans.values()} == {"rqs8", "affine"}
    for n in ("nsf9c4_h256", "maf65_h192"):  # odd n_last, last chunk one dim
        p = plans[n]
        dpc = 2 if p["uni"] == "rqs8" else 32
        assert p["n_last"] % 2 == 1 and p["D"] % 2 == 1 and p["D"] - (p["n_last"] - 1) * dpc == 1, n
        assert pairs_of(p)[-1][1] is None
    assert plans["nsf2c3_h128"]["n_last"] == 1
    flag = plans["nsf16c8_h256x3"]
    assert flag["slots"] == 4 and (4, 4) in pairs_of(flag), pairs_of(flag)
    mixed = plans["nsf16c8_h256x3_mixed"]
    assert mixed["slots"] == 4 and {(1, 4), (4, 1)} <= set(pairs_of(mixed)), pairs_of(mixed)


class Inputs:
    """Seeded rows of one shape (x[:B] for every B) and the fp64 / fp32 oracle on the rows checked so far."""

    def __init__(self, name, n):
        self.flow = make_flow(name)
        self.spec = O.flowspec_from_module(self.flow)
        D, C = self.spec.loc.shape[0], context_dim(self.flow)
        g = torch.Generator().manual_seed(4321)
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


_INPUTS = {}


def inputs(name):
    if name not in _INPUTS:
        _INPUTS.clear()  # one shape at a time: the matrix runs shape by shape
        _INPUTS[name] = Inputs(name, max(BATCHES))
    return _INPUTS[name]


MATRIX = [(n, b, fast) for n in SHAPES for b in BATCHES for fast in (1, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,fast", MATRIX, ids=[f"{n}-{b}-{'fast' if f else 'ieee'}" for n, b, f in MATRIX])
def test_pairs_against_the_oracle(device, math_mode, unfused, name, B, fast):  # noqa: F811
    math_mode(fast)
    plan = plan_of(name)
    fx = inputs(name)
    flow = fx.flow.to(device)
    (t,) = ar_layers(flow)
    assert query(t._zk_layer()) == want(plan), name
    xd = dev_t(fx.x[:B], device)
    cd = None if fx.c is None else dev_t(fx.c[:B], device)
    lp, z, ladj = (cpu(v) for v in forward_all(flow, xd, cd, device))
    rows = oracle_rows(B, 128, sm_count())
    z64, z32, ladj64, lp64 = fx.oracle(rows)
    what = f"{name} B={B} {'fast' if fast else 'ieee'}"
    assert np.isfinite(lp).all() and np.isfinite(z).all() and np.isfinite(ladj).all(), what
    if plan["mode"] == "bf16x1":  # one bf16 product: held to what the per-layer kernels reach at bf16x1
        lp_u, z_u, ladj_u = (cpu(v) for v in unfused(lambda: forward_all(flow, xd, cd, device)))
        for ours, theirs, ref, part in ((lp, lp_u, lp64, "log_prob"), (ladj, ladj_u, ladj64, "ladj"), (z, z_u, z64, "z")):
            err_f, err_u = rel_err(ours[rows], ref), rel_err(theirs[rows], ref)
            assert err_u < 1e-1, (what, part, err_u)
            assert err_f <= 2 * err_u + 1e-4, (what, part, err_f, err_u)
        return
    check_row(lp[rows], lp64, what + " log_prob", rows)
    check_row(ladj[rows], ladj64, what + " ladj", rows, lp64)
    check_z(z[rows], z64, z32, what + " z", rows)


ABI_SHAPES = ["nsf9c4_h256", "nsf16c8_h256x3_mixed", "maf65_h192", "nsf9c4_h256_x1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ABI_SHAPES)
def test_pairs_strides_accumulate_and_null_ladj(device, name):
    flow = make_flow(name).to(device)
    (t,) = ar_layers(flow)
    h = t._zk_layer()
    assert query(h) == want(plan_of(name))
    D, C, B = t.features, t.context, 3 * 128 + 1
    fx = inputs(name)
    f32 = dict(device=device, dtype=torch.float32)
    x = dev_t(fx.x[:B], device)
    c = None if fx.c is None else dev_t(fx.c[:B], device)
    y, ladj = torch.full((B, D), float("nan"), **f32), torch.full((B,), float("nan"), **f32)
    layer_forward_abi(h, x, D, c, C, B, y, D, ladj, 0, device)
    if plan_of(name)["mode"] == "bf16x3":
        z64, z32, ladj64, lp64 = fx.oracle(np.arange(B))
        check_z(cpu(y), z64, z32, f"{name} z")
        check_row(cpu(ladj), ladj64, f"{name} ladj", None, lp64)
    # strided rows with odd leading dimensions: the pads of y stay NaN, the results are bit-identical
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


BIT_SHAPES = ["nsf9c4_h256", "nsf16c8_h256x3_mixed", "maf65_h192", "nsf16c8_h256x3_x1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIT_SHAPES)
def test_pairs_rows_do_not_depend_on_the_batch(device, name):
    """A row's log_prob, z and ladj have the same bits alone, in a sub-batch starting anywhere in a tile, and in the
    full batch; and two runs agree."""
    flow = make_flow(name).to(device)
    B = 2 * 128 * sm_count() + 333
    fx = inputs(name)
    xd = dev_t(fx.x[:B], device)
    cd = None if fx.c is None else dev_t(fx.c[:B], device)
    full = [cpu(v) for v in forward_all(flow, xd, cd, device)]
    again = [cpu(v) for v in forward_all(flow, xd, cd, device)]
    assert all(np.array_equal(a, b) for a, b in zip(full, again)), f"{name}: two runs differ"
    for off, n in ((0, 1), (5, 1), (127, 1), (1, 200), (63, 129), (129, 3000), (B - 77, 77)):
        sub = forward_all(flow, xd[off : off + n], None if cd is None else cd[off : off + n], device)
        for a, b, what in zip(sub, full, ("log_prob", "z", "ladj")):
            assert np.array_equal(cpu(a), b[off : off + n]), f"{name}: rows {off}..{off + n} {what} differ from the full batch"
