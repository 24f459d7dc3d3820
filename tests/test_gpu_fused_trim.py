"""Tests of what the fused layer kernel (fused_layer.cu) leaves out: the k16 steps of layer 0 past D + C, the columns of
the layer-0 operand it no longer stages, and the padding rows of an RQS output chunk (48 of 64 rows multiplied).

* Without a GPU: issued MACs per row and weight bytes streamed per row tile restated from masks and shapes (the plan
  comes from `fused_plan_of` of test_gpu_fused_edges.py); the table reaches every k-step count 1..4 of layer 0's last
  K block, both output widths, both tile heights and both GEMM modes.  On the GPU `zk_layer_fused_info` and
  `zk_layer_fused_stream_bytes` must report the same.
* On the GPU, per shape: oracle parity at the bars of test_gpu_fused_edges.py on more than two waves of tiles (every
  CTA restages its layer-0 operand over one that held hidden activations), and the rows of the last wave evaluated
  alone (first tile of a CTA: the unstaged columns hold something else) give bitwise the same z, ladj and log_prob.
* Rows read as float4 and rows read element by element (odd leading dimension) give bitwise the same results.
* A 128-row layer and a 64-row layer that compute the same function (the second has 300 more context columns, fed
  zeros) agree bitwise."""

import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O
from test_gpu_fused_edges import (Fixed, ar_layers, check_row, check_z, cpu, dev_t, dpc_p, forward_all, fused_plan_of,
                                  layer_forward_abi, oracle_rows, sm_count)  # fmt: skip
from zuko_b200 import _engine as E
from zuko_b200.flows import MAF, NSF

FK = 64


def _nsf(D, C, bins, hidden):
    return lambda: NSF(D, C, transforms=1, bins=bins, hidden_features=hidden)


# K0 = D + C -> (D, C): rows a float4 can read (D, C multiples of 4) and rows it cannot
K0_DC = {16: (16, 0), 17: (12, 5), 31: (16, 15), 32: (24, 8), 33: (33, 0), 48: (16, 32), 64: (40, 24), 65: (20, 45), 80: (64, 16)}
KS0 = {16: 1, 17: 2, 31: 2, 32: 2, 33: 3, 48: 3, 64: 4, 65: 1, 80: 1}
SHAPES = {}
for _k0, (_d, _c) in K0_DC.items():
    for _rows, _h in ((128, [128] * 2), (64, [320] * 2)):
        for _mode in ("bf16x3", "bf16x1"):
            SHAPES[f"k{_k0}_t{_rows}_{_mode}"] = (_nsf(_d, _c, 16 if _k0 == 48 else 8, _h), _mode, _rows, _k0)
BENCHED = {
    "flagship": (lambda: NSF(16, 8, transforms=1, bins=8, hidden_features=[256] * 3), "bf16x3", 128, 24),
    "cfg3_layer": (lambda: MAF(32, 0, transforms=1, hidden_features=[512] * 4), "bf16x3", 64, 32),
    "cfg5_layer": (lambda: NSF(64, 16, transforms=1, bins=16, hidden_features=[512] * 3), "bf16x3", 64, 80),
}
ALL = {**BENCHED, **SHAPES}


def make_flow(name):
    torch.manual_seed(0)
    flow = ALL[name][0]().eval()
    for t in ar_layers(flow):
        t.hyper.gemm_mode = ALL[name][1]
    return flow


def issued_and_streamed(plan):
    """(MACs issued per row, weight bytes streamed per row tile, k16 steps of layer 0's last K block, output width) of
    a restated plan: a hidden tile is 64 wide and 64 deep, except layer 0's last K block, multiplied over the 16-wide
    steps that hold inputs (and loaded whole); an output tile is NL = DPC * P rounded up to 8 wide."""
    dpc, P = dpc_p(plan["kind"], plan["bins"])
    nl = -(-dpc * P // 8) * 8
    K0, KB0, L = plan["D"] + plan["C"], plan["KB0"], plan["L"]
    ks0 = -(-(K0 - FK * (KB0 - 1)) // 16)
    nt = 1 if plan["mode"] == "bf16x1" else 3
    planes = 1 if nt == 1 else 2
    macs = nbytes = 0
    for l, bits in enumerate(plan["kbmask"]):
        for ch, kb in zip(*np.nonzero(bits)):
            n = nl if l == L - 1 else FK
            k = 16 * ks0 if (l == 0 and kb == KB0 - 1) else FK
            macs += n * k * nt
            nbytes += n * FK * 2 * planes
    return macs, nbytes, ks0, nl


def test_issued_work_restated():
    """The formulas on the benchmarked layers and the K0 table (no GPU)."""
    plans = {n: fused_plan_of(ar_layers(make_flow(n))[0]) for n in ALL}
    for n, (_, mode, rows, k0) in ALL.items():
        assert plans[n]["why"] is None and plans[n]["rows"] == rows and plans[n]["mode"] == mode, n
        assert plans[n]["D"] + plans[n]["C"] == k0, n
    # flagship: 4 layer-0 tiles at two k steps, 20 hidden tiles, 20 output tiles 48 wide: 444 m64n64k16 equivalents
    # where every tile whole is 528, and 624 KB of weights where whole tiles are 704 KB
    macs, nbytes, ks0, nl = issued_and_streamed(plans["flagship"])
    assert plans["flagship"]["n_items"] == 44 and (ks0, nl) == (2, 48)
    assert macs == 3 * 1024 * (4 * 2 + 20 * 4 + 20 * 3) == 444 * 1024 and nbytes == 624 * 1024
    assert 44 * 3 * FK * FK == 528 * 1024 and 44 * 16384 == 704 * 1024
    # cfg3: affine chunks are 64 wide, only layer 0 (K0 = 32: two k steps of four) shrinks
    p3 = plans["cfg3_layer"]
    macs, nbytes, ks0, nl = issued_and_streamed(p3)
    assert (ks0, nl) == (2, 64) and nbytes == p3["n_items"] * 16384
    assert macs == 3 * FK * FK * p3["n_items"] - 3 * FK * 32 * int(p3["kbmask"][0][:, 0].sum())
    # cfg5: 64 one-dim output chunks 48 wide; K0 = 80 leaves one k step in layer 0's second K block
    p5 = plans["cfg5_layer"]
    macs, nbytes, ks0, nl = issued_and_streamed(p5)
    n_out, n_l0 = int(p5["kbmask"][-1].sum()), int(p5["kbmask"][0][:, 1].sum())
    assert (ks0, nl, p5["n_last"]) == (1, 48, 64) and n_out > p5["n_items"] // 2
    assert macs == 3 * FK * (FK * p5["n_items"] - 16 * n_out - 48 * n_l0) and nbytes == 16384 * p5["n_items"] - 4096 * n_out
    got = {n: issued_and_streamed(plans[n]) for n in SHAPES}
    assert {n: got[n][2] for n in SHAPES} == {n: KS0[SHAPES[n][3]] for n in SHAPES}
    assert {v[2] for v in got.values()} == {1, 2, 3, 4} and {v[3] for v in got.values()} == {48}
    for n in SHAPES:  # never more than whole tiles, and bf16x1 a third of the MACs and half of the bytes
        whole = plans[n]["n_items"] * FK * FK
        assert got[n][0] < whole * (1 if n.endswith("x1") else 3)
        if n.endswith("x3"):
            x1 = got[n[:-1] + "1"]
            assert got[n][0] == 3 * x1[0] and got[n][1] == 2 * x1[1]


@pytest.fixture
def fast_math():
    prev = E.lib().zk_set_fast_math(1)
    yield
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


class Rows(Fixed):
    """Seeded inputs of one shape of this file and the oracle on the rows asked for."""

    def __init__(self, name, n):
        self.name, self.flow = name, make_flow(name)
        self.spec = O.flowspec_from_module(self.flow)
        t = ar_layers(self.flow)[0]
        g = torch.Generator().manual_seed(1234)
        self.x = torch.randn(n, t.features, generator=g).numpy()
        self.c = torch.randn(n, t.context, generator=g).numpy() if t.context else None
        self.known = np.zeros(n, bool)
        self.z64, self.z32 = np.zeros((n, t.features)), np.zeros((n, t.features))
        self.ladj64, self.lp64 = np.zeros(n), np.zeros(n)


def pack(flow, device):
    """The layer handle of a one-layer flow on the device, packed."""
    t = ar_layers(flow)[0]
    with torch.no_grad():
        flow(None if not t.context else torch.zeros(1, t.context, device=device)).log_prob(torch.zeros(1, t.features, device=device))
    return t._zk_layer()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ALL))
def test_queries_report_the_restated_work(device, name):
    flow = make_flow(name)
    plan = fused_plan_of(ar_layers(flow)[0])
    h = pack(flow.to(device), device)
    info = (ctypes.c_double * 4)()
    assert E.lib().zk_layer_fused_info(h, info) == 1
    macs, nbytes, _, _ = issued_and_streamed(plan)
    got = (int(info[1]), info[2], int(E.lib().zk_layer_fused_stream_bytes(h)))
    print(f"{name}: tiles, issued MACs per row, streamed bytes per row tile {got}")
    assert got == (plan["n_items"], float(macs), nbytes), (name, got, (plan["n_items"], macs, nbytes))


@pytest.mark.gpu
def test_unfused_layer_streams_nothing(device):
    flow = NSF(8, 0, transforms=1, bins=4, hidden_features=[128, 128]).eval().to(device)  # 4 bins: per-layer kernels
    assert E.lib().zk_layer_fused_stream_bytes(pack(flow, device)) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_parity_over_waves_and_last_wave_alone(device, fast_math, unfused, name):
    _, mode, T, _ = SHAPES[name]
    n_sm = sm_count()
    W = T * n_sm
    B = 2 * W + W // 2 + 37  # a CTA's third tile restages over the A operand of its second
    fx = Rows(name, B)
    flow = fx.flow.to(device)
    assert E.lib().zk_layer_fused_tile_rows(pack(flow, device)) == T
    xd = dev_t(fx.x, device)
    cd = None if fx.c is None else dev_t(fx.c, device)
    lp, z, ladj = forward_all(flow, xd, cd, device)
    rows = oracle_rows(B, T, n_sm)
    z64, z32, ladj64, lp64 = fx.oracle(rows)
    if mode == "bf16x1":  # a single bf16 product: no better than the per-layer kernels at bf16x1
        lp_u, z_u, ladj_u = unfused(lambda: forward_all(flow, xd, cd, device))
        for ours, theirs, ref in ((lp, lp_u, lp64), (ladj, ladj_u, ladj64), (z, z_u, z64)):
            err = [float(np.max(np.abs(cpu(v)[rows] - ref) / np.maximum(np.abs(ref), 1.0))) for v in (ours, theirs)]
            assert err[0] <= 2 * err[1] + 1e-4, (name, err)
    else:
        check_row(cpu(lp)[rows], lp64, name + " log_prob", rows)
        check_row(cpu(ladj)[rows], ladj64, name + " ladj", rows, lp64)
        check_z(cpu(z)[rows], z64, z32, name + " z", rows)
    lp1, z1, ladj1 = forward_all(flow, xd[2 * W :], None if cd is None else cd[2 * W :], device)
    assert torch.equal(z1, z[2 * W :]) and torch.equal(ladj1, ladj[2 * W :]) and torch.equal(lp1, lp[2 * W :]), \
        f"{name}: the last wave alone differs from the last wave of the batch"  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["k32_t128_bf16x3", "k64_t128_bf16x1", "k80_t64_bf16x3", "k16_t64_bf16x3"])
def test_vector_and_scalar_staging_agree(device, name):
    flow = make_flow(name).to(device)
    h = pack(flow, device)
    t = ar_layers(flow)[0]
    D, C, T = t.features, t.context, SHAPES[name][2]
    B = T * sm_count() + 3 * T + 5
    g = torch.Generator().manual_seed(3)
    f32 = dict(device=device, dtype=torch.float32)
    x, c = torch.randn(B, D, generator=g).to(device), (torch.randn(B, C, generator=g).to(device) if C else None)
    y, ladj = torch.empty(B, D, **f32), torch.empty(B, **f32)
    layer_forward_abi(h, x, D, c, C, B, y, D, ladj, 0, device)  # float4 rows
    for pad_x, pad_c in ((1, 0), (0, 2), (4, 4)):  # odd ldx, ldc not a multiple of 4, padded rows that stay float4
        if pad_c and not C:
            continue
        xs = torch.full((B, D + pad_x), float("nan"), **f32)
        xs[:, :D] = x
        cs = None
        if C:
            cs = torch.full((B, C + pad_c), float("nan"), **f32)
            cs[:, :C] = c
        ys, ls = torch.empty(B, D, **f32), torch.empty(B, **f32)
        layer_forward_abi(h, xs, D + pad_x, cs, C + pad_c if C else 0, B, ys, D, ls, 0, device)
        assert torch.equal(ys, y) and torch.equal(ls, ladj), f"{name}: rows padded by {pad_x}, {pad_c} differ"
    if D > 4:  # a base address that is not 16-byte aligned
        xo = torch.empty(B * D + 1, **f32)[1:].view(B, D).copy_(x)
        ys, ls = torch.empty(B, D, **f32), torch.empty(B, **f32)
        layer_forward_abi(h, xo, D, c, C, B, ys, D, ls, 0, device)
        assert torch.equal(ys, y) and torch.equal(ls, ladj), f"{name}: unaligned x differs"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16x3", "bf16x1"])
def test_tile_heights_agree_bitwise(device, mode):
    """NSF(12, 4) at hidden 128 runs 128-row tiles; with 300 more context columns (K0 = 316, five K blocks) the same
    network runs 64-row tiles.  Fed zeros there, it adds products with a zero factor only."""
    D, C, X = 12, 4, 300
    torch.manual_seed(0)
    small = NSF(D, C, transforms=1, bins=8, hidden_features=[128] * 2).eval()
    large = NSF(D, C + X, transforms=1, bins=8, hidden_features=[128] * 2).eval()
    ts, tl = ar_layers(small)[0], ar_layers(large)[0]
    with torch.no_grad():
        for a, b in zip(ts.hyper._linears(), tl.hyper._linears(), strict=True):
            k = a.weight.shape[1]
            assert torch.equal(a.mask, b.mask[:, :k])
            b.weight[:, :k] = a.weight
            b.bias.copy_(a.bias)
    for t in (ts, tl):
        t.hyper.gemm_mode = mode
    small, large = small.to(device), large.to(device)
    assert E.lib().zk_layer_fused_tile_rows(pack(small, device)) == 128
    assert E.lib().zk_layer_fused_tile_rows(pack(large, device)) == 64
    B = 128 * sm_count() + 200
    g = torch.Generator().manual_seed(4)
    x, c = torch.randn(B, D, generator=g).to(device), torch.randn(B, C, generator=g).to(device)
    c_wide = torch.cat([c, torch.zeros(B, X, device=device)], 1)
    for a, b in zip(forward_all(small, x, c, device), forward_all(large, x, c_wide, device), strict=True):
        assert torch.equal(a, b), "128-row and 64-row tiles differ"
