"""GPU tests of the backward pass at its batch-slice, tile-padding and row-chunk edges, against the
fp64 gradient oracle (oracle/oracle_grad.py) on EVERY row with full parameter tensors.

* The tensor-core conditioner backward (api_backward.cu: tc_forward_save / tc_mlp_backward) cuts
  the batch of its wgrad GEMM into S slices of Bs = pad64(ceil(B / S)) rows and pads each slice's
  output rows to roundup128(N).  The matrix below runs batches around the 64-row tiles, the
  S = 1 -> 2 transition, a last slice of one row, empty last slices and an S capped by the SM count,
  on widths that are not multiples of 64, a short last 128-column chunk, an input of three K
  blocks, a coupling flow with n_a != n_b and a broadcast context.
* The single-term bf16 mode (gemm_mode="bf16x1") and the inverse direction on the same shapes.
* Row chunking of zk_flow_backward / zk_flow_inverse_backward through the C ABI with small
  workspaces (1-row chunks, and chunks that are not multiples of 64).

Rows at a ReLU kink or spline knot (cases.relu_kink_rows) get zero weight in both the engine's loss
and the oracle's.  Bar: max|ours - ref| <= 5e-5 * max|ref| per tensor (INV_BAR in the inverse
direction)."""

import ctypes

import numpy as np
import pytest
import torch

from cases import build_flow, oracle_named_grads, relu_kink_rows
from oracle import oracle as O
from oracle import oracle_grad as OG
from test_gpu_backward import INV_BAR, _flow_grads, _inverse_grads, close, cpu, dev_t
from zuko_b200 import _engine as E
from zuko_b200.flows import MAF, NICE, NSF

pytestmark = pytest.mark.gpu

BAR = 5e-5

# name -> (constructor, broadcast context).  Seeded with SEED; cfg2_nsf is the golden one.
SEED = 0
SHAPES = {
    # input 8 (one padded K block); N = 115 < one 128-column chunk
    "nsf5": (lambda: NSF(5, 3, transforms=2, hidden_features=[64, 64]), False),
    # hidden widths not multiples of 64 (dgrad gate on Np = 128 and 192); N = 138: 10-column tail chunk
    "nsf6_odd": (lambda: NSF(6, 2, transforms=2, bins=8, hidden_features=[96, 160]), False),
    # D + C = 129: three K blocks with a 1-column tail; N = 130
    "maf65": (lambda: MAF(65, 64, transforms=1, hidden_features=[128]), False),
    # odd D: the coupling splits n_a = 4 / n_b = 3 (and 3 / 4)
    "nice7": (lambda: NICE(7, 3, transforms=2, hidden_features=[64, 64]), False),
    # one broadcast context row: the column sum of the context part of the input gradient
    "nsf5_row": (lambda: NSF(5, 3, transforms=2, hidden_features=[64, 64]), True),
    # hidden 512: the wgrad slice count of its 512 x 512 layer is capped by the SM count
    "nsf5_wide": (lambda: NSF(5, 3, transforms=2, hidden_features=[512, 512]), False),
    "cfg2_nsf": (None, False),
}


def make_flow(shape):
    ctor, _ = SHAPES[shape]
    if ctor is None:
        return build_flow(shape)
    torch.manual_seed(SEED)
    return ctor().eval()


def conditioners(flow):
    return [t.hyper for t in flow.transform.transforms if getattr(t, "hyper", None) is not None]


def assert_tensor_core_path(flow, mode=E.ZK_GEMM_BF16X3):
    """mlp_uses_tc (api_backward.cu): split-bf16 handle, ReLU, no residual block."""
    hypers = conditioners(flow)
    assert hypers
    for h in hypers:
        assert E.lib().zk_mlp_gemm_mode(h._handle()) == mode
        assert h._activation_code() == E.ZK_ACT_RELU and h._layer_flags() is None


def linear_dims(flow):
    """(N, K) of every linear layer of every conditioner."""
    return [(m.weight.shape[0], m.weight.shape[1]) for h in conditioners(flow) for m in h._linears()]


def sm_count():
    n, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    E.check(E.lib().zk_device_info(ctypes.byref(n), ctypes.byref(major), ctypes.byref(minor)))
    return n.value


def slice_plan(N, K, B, sms):
    """tc_plan's batch slices of one linear layer (api_backward.cu), restated only to pick batches
    that reach its edges: (S, Bs, rows of the last slice (<= 0: empty), S allowed by the SM count)."""
    sm = -(-N // 128) * 128
    tiles = (sm // 128) * -(-K // 128)
    s_sm = -(-2 * sms // tiles)
    S = max(1, min(s_sm, B // 512))
    Bs = -(-(-(-B // S)) // 64) * 64
    return S, Bs, B - (S - 1) * Bs, s_sm


# plan-derived batches (132 SMs): the case each must hit
PLAN_BATCHES = {
    "one_row": 4609,  # the last slice holds exactly one row
    "empty": 5121,  # (S - 1) * Bs >= B: the last slice is empty
    "sm_capped": 20000,  # S = ceil(2 SMs / tiles) < B / 512 on a 512 x 512 layer
}
PLAN_HITS = {
    "one_row": lambda S, Bs, last, s_sm, B: last == 1,
    "empty": lambda S, Bs, last, s_sm, B: last <= 0,
    "sm_capped": lambda S, Bs, last, s_sm, B: S == s_sm < B // 512,
}


def batch_of(flow, b):
    """The batch of a test case: an int, or a PLAN_BATCHES key whose case the restated plan must hit."""
    if isinstance(b, int):
        return b
    B, sms = PLAN_BATCHES[b], sm_count()
    plans = [(N, K, *slice_plan(N, K, B, sms)) for N, K in linear_dims(flow)]
    print(f"B={B} on {sms} SMs: (N, K, S, Bs, last-slice rows, SM-allowed S) = {plans}")
    assert any(PLAN_HITS[b](*p[2:], B) for p in plans), f"{b}: B={B} no longer reaches that case of the slice plan: {plans}"
    return B


def inputs(shape, flow, B, seed):
    D = flow.base.loc.shape[0]
    C = flow.transform.transforms[0].context
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, generator=gen).numpy()
    c = None
    if C:
        c = torch.randn(C, generator=gen).numpy() if SHAPES[shape][1] else torch.randn(B, C, generator=gen).numpy()
    gg = {"g": torch.randn(B, generator=gen).numpy(), "gz": torch.randn(B, D, generator=gen).numpy(),
          "gl": torch.randn(B, generator=gen).numpy()}  # fmt: skip
    return x, c, gg


def zero_rows(gg, rows):
    for v in gg.values():
        v[rows] = 0.0
    return gg


def oracle_grads(spec, cpu_flow, x, c, gg, mode):
    kw = dict(g_log_prob=gg["g"]) if mode == "lp" else dict(g_z=gg["gz"], g_ladj=gg["gl"])
    ogx, ogc, lgs = OG.flow_backward(spec, x, c, **kw)
    return ogx, ogc, oracle_named_grads(cpu_flow, lgs)


def assert_grads(got, ref, bar, what):
    gx, gc, pg = got
    ogx, ogc, opg = ref
    close(gx, ogx, bar, f"{what} d/dx")
    if ogc is not None:
        assert gc.shape == ogc.shape
        close(gc, ogc, bar, f"{what} d/dc")
    assert set(pg) == set(opg), f"{what}: parameters {sorted(set(pg) ^ set(opg))}"
    for k in opg:
        close(pg[k], opg[k], bar, f"{what} d/d{k}")


def grad_errors(got, ref):
    """Relative error (to max|ref|) of every tensor."""
    out = {}
    for k, a, b in [("x", got[0], ref[0]), ("c", got[1], ref[1])] + [(k, got[2][k], ref[2][k]) for k in ref[2]]:
        if b is not None:
            out[k] = float(np.abs(np.asarray(a, np.float64) - b).max()) / max(float(np.abs(b).max()), 1e-30)
    return out


# --------------------------------------------------------------------------- #
# A. tensor-core backward: shape x batch
# --------------------------------------------------------------------------- #

SMALL_BATCHES = [1, 2, 63, 64, 65, 127, 129, 511, 512, 513, 1024, 1025]
TWO_TRANSFORM = ["nsf5", "nsf6_odd", "maf65", "nice7", "nsf5_row"]
MATRIX = ([(s, b) for s in TWO_TRANSFORM for b in SMALL_BATCHES + ["one_row", "empty"]]
          + [("cfg2_nsf", b) for b in SMALL_BATCHES] + [("nsf5_wide", "sm_capped")])  # fmt: skip


@pytest.mark.parametrize("mode", ["lp", "tr"])
@pytest.mark.parametrize("shape,b", MATRIX)
def test_tensor_core_backward_vs_oracle(device, shape, b, mode):
    cpu_flow = make_flow(shape)
    flow = make_flow(shape).to(device)
    assert_tensor_core_path(flow)
    B = batch_of(flow, b)
    x, c, gg = inputs(shape, flow, B, seed=B)
    spec = O.flowspec_from_module(cpu_flow)
    zero_rows(gg, relu_kink_rows(spec, x, c))
    what = f"{shape} B={B} {mode}"
    tc = _flow_grads(flow, x, c, mode, gg, device)
    assert_grads(tc, oracle_grads(spec, cpu_flow, x, c, gg, mode), BAR, what)
    if b == "empty":  # fixed-order reductions: two runs agree bit for bit
        again = _flow_grads(flow, x, c, mode, gg, device)
        assert np.array_equal(tc[0], again[0]) and (c is None or np.array_equal(tc[1], again[1]))
        assert all(np.array_equal(tc[2][k], again[2][k]) for k in tc[2])
    prev = E.lib().zk_set_tc_backward(0)
    try:
        f32 = _flow_grads(flow, x, c, mode, gg, device)
    finally:
        E.lib().zk_set_tc_backward(prev)
    close(tc[0], f32[0], 2e-5, f"{what} d/dx tc vs fp32")
    if c is not None:  # a broadcast row is a sum over the batch, like a parameter gradient
        close(tc[1], f32[1], 5e-5 if c.ndim == 1 else 2e-5, f"{what} d/dc tc vs fp32")
    assert set(tc[2]) == set(f32[2])
    for k in f32[2]:
        close(tc[2][k], f32[2][k], 5e-5, f"{what} d/d{k} tc vs fp32")


# --------------------------------------------------------------------------- #
# B. single-term bf16 conditioner (gemm_mode="bf16x1")
# --------------------------------------------------------------------------- #

# worst over the gradient tensors of max|ours - ref| / max|ref|, measured on an H100 80GB HBM3 (SXM) at
# a 700 W power limit: nsf5 1.6e-1 (B = 513) / 1.6e-1 (5121), cfg2_nsf 2.3e-1 / 1.2e-1 (bf16x3 on the
# same inputs: 1.0e-5..1.4e-5).  One bf16 term carries ~4e-3 of relative error per operand, and it moves
# many more hidden units across their ReLU kink than the kink filter (tuned for bf16x3) removes.
BF16X1_BAR = 0.7


@pytest.mark.parametrize("b", [513, "empty"])
@pytest.mark.parametrize("shape", ["nsf5", "cfg2_nsf"])
def test_bf16x1_backward(device, shape, b, record_property):
    cpu_flow = make_flow(shape)
    x3 = make_flow(shape).to(device)
    x1 = make_flow(shape)
    for h in conditioners(x1):
        h.gemm_mode = "bf16x1"
    x1 = x1.to(device)
    assert_tensor_core_path(x3)
    assert_tensor_core_path(x1, E.ZK_GEMM_BF16X1)
    B = batch_of(x1, b)
    x, c, gg = inputs(shape, x1, B, seed=B + 1)
    spec = O.flowspec_from_module(cpu_flow)
    zero_rows(gg, relu_kink_rows(spec, x, c))
    ref = oracle_grads(spec, cpu_flow, x, c, gg, "lp")
    got1 = _flow_grads(x1, x, c, "lp", gg, device)
    got3 = _flow_grads(x3, x, c, "lp", gg, device)
    assert np.isfinite(got1[0]).all() and (c is None or np.isfinite(got1[1]).all())
    assert all(np.isfinite(v).all() for v in got1[2].values())
    e1, e3 = grad_errors(got1, ref), grad_errors(got3, ref)
    w1, w3 = max(e1.values()), max(e3.values())
    record_property("bf16x1_err", w1)
    record_property("bf16x3_err", w3)
    print(f"{shape} B={B}: worst error bf16x1 {w1:.3e} ({max(e1, key=e1.get)}), bf16x3 {w3:.3e} ({max(e3, key=e3.get)})")
    assert w1 > w3, "the single-term path is not less accurate than the three-term one: did it run?"
    assert w1 <= BF16X1_BAR, f"bf16x1 worst error {w1:.3e} (bar {BF16X1_BAR:.1e})"


# --------------------------------------------------------------------------- #
# C. inverse direction (zk_flow_inverse_backward)
# --------------------------------------------------------------------------- #


@pytest.mark.parametrize("mode", ["inv", "invlp"])
@pytest.mark.parametrize("B", [1, 65, 513, 5121])
@pytest.mark.parametrize("shape", ["nsf5", "nsf6_odd", "nsf5_row"])
def test_inverse_backward_vs_oracle(device, shape, B, mode):
    cpu_flow = make_flow(shape)
    flow = make_flow(shape).to(device)
    assert_tensor_core_path(flow)
    z, c, gg = inputs(shape, flow, B, seed=B + 2)
    spec = O.flowspec_from_module(cpu_flow)
    z64 = z.astype(np.float64)
    xs = spec.inverse(z64, c)
    w, wl = gg["gz"], gg["g"]
    kink = relu_kink_rows(spec, xs, c)  # non-smooth rows, judged at the sample
    w[kink], wl[kink] = 0.0, 0.0
    x, gz, gc, pg = _inverse_grads(flow, z, c, mode, w, wl, device)
    ogz, ogc, lgs = OG.flow_inverse_backward(spec, z64, c, g_x=w, g_log_prob=wl if mode == "invlp" else None)
    what = f"{shape} B={B} {mode}"
    close(x, xs, 1e-4, f"{what} sample")
    assert_grads((gz, gc, pg), (ogz, ogc, oracle_named_grads(cpu_flow, lgs)), INV_BAR, what)


# --------------------------------------------------------------------------- #
# D. row chunking through the C ABI
# --------------------------------------------------------------------------- #


def chunk_workspace(ws_for, desc, rows, B):
    """Bytes that hold a chunk of exactly `rows` rows (the chunk planner takes the largest row count that
    fits); `rows` moves up until the workspace for one more row is larger."""
    while ws_for(ctypes.byref(desc), rows + 1) <= ws_for(ctypes.byref(desc), rows):
        rows += 1
    ws = ws_for(ctypes.byref(desc), rows)
    assert all(ws_for(ctypes.byref(desc), r) > ws for r in range(rows + 1, B + 1))
    return rows, ws


def _abi_call(fc, inverse, B, x, c, ldc, g, ws_bytes, device):
    """One zk_flow_(inverse_)backward call on caller-owned buffers.  grad_c is pre-filled with NaN
    (the flow-level calls overwrite it)."""
    L = E.lib()
    D, C = fc.D, fc.C
    f32 = dict(device=device, dtype=torch.float32)
    gx = torch.full((B, D), float("nan"), **f32)
    gc = None if C == 0 else torch.full((C,) if ldc == 0 else (B, C), float("nan"), **f32)
    need = [True] * len(fc._params)
    structs, pg, tables, keep = fc._grad_structs(need, f32)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    if inverse:
        st = L.zk_flow_inverse_backward(ctypes.byref(fc.desc), p(x), D, p(c), ldc, B, p(g["gz"]), D, p(g["g"]), p(g["z"]), D,
                                        p(gx), D, p(gc), C, structs, p(ws), ws_bytes, E.stream_ptr(device))  # fmt: skip
    else:
        st = L.zk_flow_backward(ctypes.byref(fc.desc), p(x), D, p(c), ldc, B, p(g["gz"]), D, p(g["gl"]), p(g["g"]), p(gx), D,
                                p(gc), C, structs, p(ws), ws_bytes, E.stream_ptr(device))  # fmt: skip
    E.check(st)
    torch.cuda.synchronize(device)
    fc._split_tables(pg, tables, need)
    del keep
    return cpu(gx), (None if gc is None else cpu(gc)), [cpu(t) for t in pg]


@pytest.mark.parametrize("inverse", [False, True], ids=["forward", "inverse"])
@pytest.mark.parametrize("shape", ["nsf5", "nsf5_row"])
@pytest.mark.parametrize("chunk", ["one_row", "hundred"])
def test_row_chunks_through_c_abi(device, shape, chunk, inverse):
    L = E.lib()
    cpu_flow = make_flow(shape)
    flow = make_flow(shape).to(device)
    spec = O.flowspec_from_module(cpu_flow)
    probe = torch.zeros(3, device=device) if SHAPES[shape][1] else torch.zeros(1, 3, device=device)
    fc = flow(probe)._flow_call()[0]
    ws_for = L.zk_flow_inverse_backward_workspace_bytes if inverse else L.zk_flow_backward_workspace_bytes
    min_ws = (L.zk_flow_inverse_backward_min_workspace_bytes if inverse else L.zk_flow_backward_min_workspace_bytes)(ctypes.byref(fc.desc))
    if chunk == "one_row":
        B = 37
        assert min_ws == ws_for(ctypes.byref(fc.desc), 1) < ws_for(ctypes.byref(fc.desc), 2)
        rows, small = 1, min_ws
    else:
        rows, small = chunk_workspace(ws_for, fc.desc, 100, 1100)
        B = 10 * rows + 37  # ten chunks and a tail that is not a multiple of 64
    x, c, gg = inputs(shape, flow, B, seed=B + 3)
    if inverse:  # x is the sample of z = gg["gz"]; the upstream gradients are fresh rows
        gen = torch.Generator().manual_seed(B + 4)
        gg = {"z": gg["gz"], "gz": torch.randn(B, fc.D, generator=gen).numpy(), "g": gg["g"]}
        with torch.no_grad():
            x = cpu(flow(None if c is None else dev_t(c, device)).transform.inv(dev_t(gg["z"], device)))
    zero_rows({k: v for k, v in gg.items() if k != "z"}, relu_kink_rows(spec, x, c))
    dev = {k: dev_t(v, device) for k, v in gg.items()}
    xt, ct = dev_t(x, device), (None if c is None else dev_t(c, device))
    ldc = 0 if (c is not None and c.ndim == 1) else fc.C
    full = _abi_call(fc, inverse, B, xt, ct, ldc, dev, ws_for(ctypes.byref(fc.desc), B), device)
    part = _abi_call(fc, inverse, B, xt, ct, ldc, dev, small, device)
    what = f"{shape} {'inverse' if inverse else 'forward'} B={B} in {rows}-row chunks"
    assert np.isfinite(full[0]).all() and np.isfinite(part[0]).all()
    close(part[0], full[0], 1e-6, f"{what}: grad_x")
    if c is not None:
        assert np.isfinite(part[1]).all() and np.isfinite(full[1]).all(), f"{what}: grad_c not overwritten"
        close(part[1], full[1], 1e-6 if ldc else 5e-5, f"{what}: grad_c")
    for a, b in zip(part[2], full[2], strict=True):
        close(a, b, 5e-5, f"{what}: parameter gradient")
