"""GPU tests of the per-layer conditioner (zk_mlp_forward) and the fp32 conditioner backward at their tile,
padding, residual, activation, batch and stride edges, against the fp64 oracle (oracle.Conditioner,
oracle.Layer / FlowSpec, oracle_grad).

* Forward: the tensor-core GEMM (linear_tc_kernel<false|true>, mlp_tcgen05.cu) behind split_input_kernel and
  the bf16 hi / lo ping-pong planes of tc_forward, and the exact-order fp32 GEMM (linear_fp32_kernel,
  mlp_simt.cu).  `forward_plan` restates, per handle and batch, the resolved GEMM mode, the instantiation
  each layer runs, its 128-column chunks and their tail, its 64-wide K blocks against the 3-stage ring and its
  tiles against the SM count; a CPU test checks that the case table reaches every cell.  Large batches are
  compared with the oracle on a subset of rows (every row within 2 of a 128-row tile edge, the first and last
  tile, 512 random rows); every row is checked bit for bit against the prefix calls and for finiteness.
* Layers that always run the per-layer conditioner: coupling layers and element-wise layers with context.
* The fp32 conditioner backward (mlp_forward_save / mlp_backward in api_backward.cu with the sliced wgrad and
  two-stage column sums of backward.cu): residual blocks, non-ReLU activations, fp32 handles, a ReLU
  tensor-core handle with zk_set_tc_backward(0), coupling and element-wise layers, at batches picked from the
  restated slice plans (`wgrad_plan`, `colsum_plan`).

Bars: conditioner outputs max|ours - ref| <= 2e-6 (fp32), 3e-5 (bf16x3), 3e-2 (bf16x1) of max|ref|; coupling and
element-wise flows: log_prob / ladj 3e-5 (LAYER_LP_BAR), z 4e-5 (test_gpu_fused_edges.py), GF log_prob 1e-5,
inverses 1e-4; gradients
max|ours - ref| <= 5e-5 max|ref| per tensor, rows at a ReLU kink or spline knot given zero weight
(cases.relu_kink_rows)."""

import ctypes
from functools import partial

import numpy as np
import pytest
import torch

import gf_reference as GFR
from cases import oracle_named_grads, relu_kink_rows
from oracle import oracle as O
from oracle import oracle_grad as OG
from test_gpu_backward import _flow_grads, close, cpu, dev_t
from test_gpu_backward_abi import LayerCase
from test_gpu_fused_edges import check_row, check_z
from zuko_b200 import _engine as E
from zuko_b200.distributions import DiagNormal
from zuko_b200.flows import GF, MAF, NICE, NSF, ElementWiseTransform, RealNVP
from zuko_b200.lazy import Flow, UnconditionalDistribution
from zuko_b200.transforms import MonotonicRQSTransform

NAN = float("nan")
H100_SMS = 132  # H100 SXM
BARS = {"fp32": 2e-6, "bf16x3": 3e-5, "bf16x1": 3e-2}
GRAD_BAR = 5e-5
INV_BAR = 1e-4

# internal activation codes of zk_mlp_desc.layer_act (0 none, 1 ReLU, else ZK_ACT_*) -> oracle names
ACT_NAMES = {1: "ReLU", E.ZK_ACT_ELU: "ELU", E.ZK_ACT_TANH: "Tanh", E.ZK_ACT_SILU: "SiLU", E.ZK_ACT_GELU: "GELU",
             E.ZK_ACT_LEAKY_RELU: "LeakyReLU", E.ZK_ACT_SOFTPLUS: "Softplus", E.ZK_ACT_SIGMOID: "Sigmoid"}  # fmt: skip
ALL_ACTS = [E.ZK_ACT_RELU, E.ZK_ACT_ELU, E.ZK_ACT_TANH, E.ZK_ACT_SILU, E.ZK_ACT_GELU, E.ZK_ACT_LEAKY_RELU,
            E.ZK_ACT_SOFTPLUS, E.ZK_ACT_SIGMOID]  # fmt: skip


def cdiv(a, b):
    return -(-a // b)


def pad64(k):
    return cdiv(k, 64) * 64


def sm_count():
    n, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    E.check(E.lib().zk_device_info(ctypes.byref(n), ctypes.byref(major), ctypes.byref(minor)))
    return n.value


# --------------------------------------------------------------------------- #
# 1. case table and restated plans
# --------------------------------------------------------------------------- #


def plain(K0, hidden, N, mode, act=E.ZK_ACT_RELU):
    """Plain conditioner: the activation `act` (ZK_ACT_*) after every layer but the last."""
    return {"dims": [K0, *hidden, N], "mode": mode, "act": act, "lact": None, "lres": None}


def residual(K0, widths, N, mode, act, blocks):
    """Residual conditioner: linear layers K0 -> widths[0] -> ... -> N; layer i in `blocks` closes a block opened
    by layer i - 1 (activation `act` inside, none after the sum); every other hidden layer is followed by `act`."""
    dims = [K0, *widths, N]
    n = len(dims) - 1
    code = 1 if act == E.ZK_ACT_RELU else act
    lact = [0 if (i + 1 in blocks or i in blocks or i == n - 1) else code for i in range(n)]
    for i in blocks:
        lact[i - 1] = code
    lres = [1 if i in blocks else 0 for i in range(n)]
    return {"dims": dims, "mode": mode, "act": act, "lact": lact, "lres": lres}


CASES = {
    # ---- tensor cores, plain: widths / tails / K blocks / activations ----
    "k1_h64_n1_auto": plain(1, [64], 1, "auto"),  # widest dim exactly 64: AUTO picks bf16x3
    "k63_h96x2_n2_tanh": plain(63, [96, 96], 2, "bf16x3", E.ZK_ACT_TANH),
    "k64_h192_n63_gelu_x1": plain(64, [192], 63, "bf16x1", E.ZK_ACT_GELU),
    "k65_h640x2_n64": plain(65, [640, 640], 64, "bf16x3"),  # 5 column chunks, 10 K blocks
    "k129_h1000_n65_lrelu": plain(129, [1000], 65, "bf16x3", E.ZK_ACT_LEAKY_RELU),  # 8 chunks, 104-column tail
    "k1000_h1024_n127_softplus": plain(1000, [1024], 127, "bf16x3", E.ZK_ACT_SOFTPLUS),  # 16 K blocks
    "k8_h64x4_n128_sigmoid": plain(8, [64] * 4, 128, "bf16x3", E.ZK_ACT_SIGMOID),  # 5 linear layers
    "k24_h256_n368_x1": plain(24, [256], 368, "bf16x1"),
    "k24_h96_n129_silu": plain(24, [96], 129, "bf16x3", E.ZK_ACT_SILU),  # 1-column tail chunk
    "k129_n368_single": plain(129, [], 368, "bf16x3"),  # one linear layer, no activation
    "k1000_h640_n1_elu": plain(1000, [640], 1, "bf16x3", E.ZK_ACT_ELU),
    # ---- fp32 CUDA-core kernel: every activation ----
    "fp32_relu": plain(65, [640, 640], 64, "fp32"),
    "fp32_elu": plain(1, [64], 1, "fp32", E.ZK_ACT_ELU),
    "fp32_tanh": plain(63, [96, 96], 2, "fp32", E.ZK_ACT_TANH),
    "fp32_silu": plain(24, [96], 129, "fp32", E.ZK_ACT_SILU),
    "fp32_gelu": plain(64, [192], 63, "fp32", E.ZK_ACT_GELU),
    "fp32_lrelu": plain(129, [1000], 65, "fp32", E.ZK_ACT_LEAKY_RELU),
    "fp32_softplus": plain(8, [64] * 4, 128, "fp32", E.ZK_ACT_SOFTPLUS),
    "fp32_sigmoid": plain(1000, [1024], 127, "fp32", E.ZK_ACT_SIGMOID),
    "auto_narrow": plain(4, [32, 32], 8, "auto"),  # widest dim < 64: AUTO picks fp32
    # ---- residual blocks ----
    "res_at2_h96": residual(65, [96, 96, 96], 2, "bf16x3", E.ZK_ACT_RELU, [2]),  # earliest closing layer, ReLU inside
    "res_h160_96_gelu": residual(63, [160, 96, 96, 96], 65, "bf16x3", E.ZK_ACT_GELU, [3]),  # block 96 != first 160
    "res2_h192_elu": residual(24, [192] * 5, 368, "bf16x3", E.ZK_ACT_ELU, [2, 4]),  # two back to back
    "res3_h160_silu_x1": residual(8, [160] * 7, 129, "bf16x1", E.ZK_ACT_SILU, [2, 4, 6]),  # three, bf16x1
    "res_fp32_at2_h96": residual(65, [96, 96, 96], 2, "fp32", E.ZK_ACT_RELU, [2]),
    "res2_fp32_h160_tanh": residual(24, [160] * 5, 63, "fp32", E.ZK_ACT_TANH, [2, 4]),
}


def resolved_mode(spec):
    """tc_pack's rule (sm_90): AUTO takes bf16x3 once the widest layer dimension is at least 64."""
    if spec["mode"] == "auto":
        return "bf16x3" if max(spec["dims"]) >= 64 else "fp32"
    return spec["mode"]


def layer_acts(spec):
    """Internal activation code per linear layer (zk_mlp_create)."""
    n = len(spec["dims"]) - 1
    if spec["lact"] is not None:
        return list(spec["lact"]), list(spec["lres"])
    code = 1 if spec["act"] == E.ZK_ACT_RELU else spec["act"]
    return [code] * (n - 1) + [0], [0] * n


def forward_plan(spec, B, sms):
    """What zk_mlp_forward runs for this handle and batch: (mode, per linear layer a dict)."""
    mode = resolved_mode(spec)
    dims = spec["dims"]
    lact, lres = layer_acts(spec)
    n = len(dims) - 1
    layers = []
    for i in range(n):
        K, N = dims[i], dims[i + 1]
        last = i == n - 1
        res = bool(lres[i]) and not last
        L = {"act": lact[i], "res": res, "K": K, "N": N}
        if mode == "fp32":
            L["inst"] = "fp32"
        else:
            L["inst"] = "true" if (lact[i] > 1 or res) else "false"
            Kp = pad64(K)
            L["chunks"] = cdiv(N, 128)
            t = N % 128
            L["tail"] = "0" if t == 0 else ("1-64" if t <= 64 else "65-127")
            L["kblocks"] = str(Kp // 64) if Kp // 64 <= 3 else ">3"
            tiles = cdiv(B, 128) * L["chunks"]
            L["tiles"] = "fewer" if tiles < sms else ("equal" if tiles == sms else "more")
        layers.append(L)
    return mode, layers


def launches(spec):
    n = len(spec["dims"]) - 1
    return n if resolved_mode(spec) == "fp32" else n + 1


def wgrad_slices_max(N, K, sms):
    S = min(64, max(1, cdiv(8 * sms, cdiv(N, 64) * cdiv(K, 64))))
    while S > 1 and S * N * K * 4 > (256 << 20):
        S //= 2
    return S


def wgrad_plan(N, K, B, sms):
    """launch_wgrad_fp32 (backward.cu): (slices, rows per slice, rows of the last slice, slice cap)."""
    cap = wgrad_slices_max(N, K, sms)
    S = min(cap, cdiv(B, 64))
    rows = cdiv(cdiv(B, S), 16) * 16
    S = cdiv(B, rows)
    return S, rows, B - (S - 1) * rows, cap


def colsum_plan(B):
    """launch_colsum_add (backward.cu): (slices, rows per slice)."""
    S = min(64, cdiv(B, 256))
    rows = cdiv(B, S)
    return cdiv(B, rows), rows


def fwd_batches(sms):
    T = 128 * sms
    return [0, 1, 63, 64, 127, 128, 129, T - 1, T, T + 1, 3 * T + 77]


def forward_cells(table, sms):
    cells = set()
    for spec in table.values():
        n = len(spec["dims"]) - 1
        cells.add(("n_linear", "1" if n == 1 else ("2" if n == 2 else (">=5" if n >= 5 else "3-4"))))
        lact, lres = layer_acts(spec)
        mode = resolved_mode(spec)
        for B in fwd_batches(sms):
            if B == 0:
                continue
            _, layers = forward_plan(spec, B, sms)
            for L in layers:
                cells.add(("inst", L["inst"], mode))
                kernel = "fp32" if mode == "fp32" else "tc"
                if L["act"]:
                    cells.add(("act", E.ZK_ACT_RELU if L["act"] == 1 else L["act"], kernel))
                if mode != "fp32":
                    cells |= {("tail", L["tail"]), ("kblocks", L["kblocks"]), ("tiles", L["tiles"])}
        blocks = [i for i in range(n) if lres[i]]
        if blocks:
            w = [spec["dims"][i] for i in blocks]
            cells.add(("res", "mode", mode))
            cells.add(("res", "inside", "relu" if lact[blocks[0] - 1] == 1 else "general"))
            if blocks[0] == 2:
                cells.add(("res", "closed_at_2"))
            run = best = 1
            for a, b in zip(blocks, blocks[1:]):
                run = run + 1 if b - a == 2 else 1
                best = max(best, run)
            cells.add(("res", f"back_to_back_{best}"))
            cells |= {("res", "width", wd) for wd in w if wd % 64}
            if any(wd != spec["dims"][1] for wd in w):
                cells.add(("res", "width_differs_from_first"))
    return cells


REQUIRED_FORWARD_CELLS = (
    {("inst", i, m) for i in ("false", "true") for m in ("bf16x3", "bf16x1")} | {("inst", "fp32", "fp32")}
    | {("tail", t) for t in ("0", "1-64", "65-127")}
    | {("kblocks", k) for k in ("1", "2", "3", ">3")}
    | {("tiles", t) for t in ("fewer", "equal", "more")}
    | {("n_linear", n) for n in ("1", "2", ">=5")}
    | {("act", a, k) for a in ALL_ACTS for k in ("fp32", "tc")}
    | {("res", "closed_at_2"), ("res", "back_to_back_2"), ("res", "back_to_back_3"), ("res", "width", 96),
       ("res", "width", 160), ("res", "width_differs_from_first"), ("res", "inside", "relu"), ("res", "inside", "general")}
    | {("res", "mode", m) for m in ("fp32", "bf16x3", "bf16x1")}
)  # fmt: skip


# backward: flows whose conditioner backward runs the fp32 kernels (mlp_uses_tc is false, or tc backward is off)
A = torch.nn
RQS8 = dict(univariate=partial(MonotonicRQSTransform, slope=1e-3), shapes=[(8,), (8,), (7,)])
RQS16 = dict(univariate=partial(MonotonicRQSTransform, slope=1e-3), shapes=[(16,), (16,), (15,)])


def _one(*layers):
    D = layers[0].features
    return Flow(list(layers), UnconditionalDistribution(DiagNormal, torch.zeros(D), torch.ones(D), buffer=True))


# name -> (constructor, broadcast context, tensor-core backward switched off)
BWD_FLOWS = {
    "res_maf_at2_h96": (lambda: MAF(5, 3, transforms=2, hidden_features=[96, 96], residual=True), False, False),
    "res_nsf_h160_96_96_elu": (lambda: NSF(4, 2, transforms=1, hidden_features=[160, 96, 96], residual=True, activation=A.ELU), False, False),
    "res_maf_h192x3_gelu": (lambda: MAF(6, 0, transforms=1, hidden_features=[192] * 3, residual=True, activation=A.GELU), False, False),
    "res_nsf_h64x4_silu": (lambda: NSF(3, 2, transforms=1, hidden_features=[64] * 4, residual=True, activation=A.SiLU), False, False),
    "maf_elu": (lambda: MAF(4, 2, transforms=1, hidden_features=[64, 64], activation=A.ELU), False, False),
    "maf_tanh": (lambda: MAF(4, 2, transforms=1, hidden_features=[64, 64], activation=A.Tanh), False, False),
    "nsf_silu": (lambda: NSF(4, 2, transforms=1, hidden_features=[64, 64], activation=A.SiLU), False, False),
    "maf_gelu": (lambda: MAF(4, 2, transforms=1, hidden_features=[96], activation=A.GELU), False, False),
    "nsf_lrelu": (lambda: NSF(4, 2, transforms=1, hidden_features=[64, 64], activation=A.LeakyReLU), False, False),
    "maf_softplus": (lambda: MAF(4, 2, transforms=1, hidden_features=[64, 64], activation=A.Softplus), False, False),
    "maf_sigmoid": (lambda: MAF(4, 2, transforms=1, hidden_features=[64, 64], activation=A.Sigmoid), False, False),
    "nsf_fp32": (lambda: NSF(5, 3, transforms=2, hidden_features=[64, 64]), False, False),
    "nsf_tc_off": (lambda: NSF(5, 3, transforms=1, hidden_features=[96, 160]), False, True),
    "nice7_c3": (lambda: NICE(7, 3, transforms=2, hidden_features=[64]), False, True),
    "realnvp7_rqs_row": (lambda: RealNVP(7, 3, transforms=2, hidden_features=[64], **RQS8), True, True),
    "ew_affine_c3": (lambda: _one(ElementWiseTransform(4, 3, hidden_features=[64])), False, False),
    "ew_rqs_row": (lambda: _one(ElementWiseTransform(4, 3, hidden_features=[64], **RQS8)), True, False),
}
FP32_MODE_FLOWS = {"nsf_fp32"}

# slice-plan batches (132 SMs) -> the cell each must reach on some linear layer of the flow
SLICE_BATCHES = {
    "s1": 64,  # wgrad: S = 1 (one slice of 64 rows)
    "s2_last17": 65,  # wgrad: S = 1 -> 2; last slice of 17 rows
    "last1": 193,  # wgrad: last slice of 1 row
    "last15": 207,  # wgrad: last slice of 15 rows
    "last16": 208,  # wgrad: last slice of 16 rows
    "colsum_256k_m1": 511,  # colsum: 256 k - 1
    "colsum_256k_p1": 513,  # colsum: 256 k + 1
    "wgrad_cap": 5000,  # wgrad: S at wgrad_slices_max < ceil(B / 64)
    "colsum_cap": 16641,  # colsum: B > 64 * 256, S = 64
}
SLICE_HITS = {
    "s1": lambda w, c: w[0] == 1,
    "s2_last17": lambda w, c: w[0] == 2 and w[2] == 17,
    "last1": lambda w, c: w[2] == 1,
    "last15": lambda w, c: w[2] == 15,
    "last16": lambda w, c: w[2] == 16,
    "colsum_256k_m1": lambda w, c: True,
    "colsum_256k_p1": lambda w, c: True,
    "wgrad_cap": lambda w, c: w[3] < cdiv(w[4], 64),
    "colsum_cap": lambda w, c: c[0] == 64 and w[4] > 64 * 256,
}
# every flow at the cheap batches, a few at the large ones
BWD_MATRIX = ([(f, b) for f in BWD_FLOWS for b in ["s1", "s2_last17", "last1", "last15", "last16", "colsum_256k_p1"]]
              + [(f, b) for f in ["res_maf_at2_h96", "res_nsf_h160_96_96_elu", "nsf_lrelu", "nice7_c3", "ew_rqs_row"]
                 for b in ["colsum_256k_m1", "wgrad_cap"]]
              + [(f, "colsum_cap") for f in ["res_maf_h192x3_gelu", "realnvp7_rqs_row"]])  # fmt: skip


def make_bwd_flow(name, seed=0):
    torch.manual_seed(seed)
    flow = BWD_FLOWS[name][0]().eval()
    if name in FP32_MODE_FLOWS:
        for h in conditioners(flow):
            h.gemm_mode = "fp32"
    return flow


def conditioners(flow):
    return [t.hyper for t in flow.transform.transforms if getattr(t, "hyper", None) is not None]


def linear_dims(flow):
    return [(m.weight.shape[0], m.weight.shape[1]) for h in conditioners(flow) for m in h._linears()]


def slice_cells(flow, B, sms):
    """(wgrad plan + (B,), colsum plan) of every launch the fp32 backward makes at this batch."""
    out = []
    for N, K in linear_dims(flow):
        w = (*wgrad_plan(N, K, B, sms), B)
        out.append((w, colsum_plan(B)))
    return out


def slice_batch(flow, key, sms):
    B = SLICE_BATCHES[key]
    plans = slice_cells(flow, B, sms)
    if key.startswith("colsum_256k"):
        assert (B + (1 if key.endswith("m1") else -1)) % 256 == 0
    assert any(SLICE_HITS[key](w, c) for w, c in plans), f"{key}: B={B} no longer reaches its slice-plan cell: {plans}"
    return B


def test_case_table_reaches_every_cell():
    """CPU: the restated plans over the case tables reach every cell the GPU tests are meant to cover."""
    cells = forward_cells(CASES, H100_SMS)
    missing = REQUIRED_FORWARD_CELLS - cells
    assert not missing, f"forward cells no case reaches: {sorted(map(str, missing))}"
    assert {resolved_mode(CASES["k1_h64_n1_auto"]), resolved_mode(CASES["auto_narrow"])} == {"bf16x3", "fp32"}
    reached = set()
    for name, b in BWD_MATRIX:
        slice_batch(make_bwd_flow(name), b, H100_SMS)
        reached.add(b)
    assert reached == set(SLICE_BATCHES), sorted(set(SLICE_BATCHES) - reached)


# --------------------------------------------------------------------------- #
# 2. zk_mlp_forward through the C ABI
# --------------------------------------------------------------------------- #


class Mlp:
    """A zk_mlp handle over seeded weights (1/sqrt(K) scale) and its fp64 oracle."""

    def __init__(self, name, device, seed=0):
        self.spec = spec = CASES[name]
        self.name, self.device = name, device
        dims = spec["dims"]
        self.n = len(dims) - 1
        rng = np.random.default_rng(seed)
        self.W = [(rng.standard_normal((dims[i + 1], dims[i])) / np.sqrt(dims[i])).astype(np.float32) for i in range(self.n)]
        self.b = [(0.1 * rng.standard_normal(dims[i + 1])).astype(np.float32) for i in range(self.n)]
        keep = [torch.from_numpy(a).to(device) for a in self.W + self.b]
        W = (ctypes.c_void_p * self.n)(*[t.data_ptr() for t in keep[: self.n]])
        Bv = (ctypes.c_void_p * self.n)(*[t.data_ptr() for t in keep[self.n :]])
        la = lr = None
        if spec["lact"] is not None:
            la, lr = (ctypes.c_int * self.n)(*spec["lact"]), (ctypes.c_int * self.n)(*spec["lres"])
        d = (ctypes.c_int * (self.n + 1))(*dims)
        desc = E.MlpDesc(self.n, d, W, Bv, None, E.GEMM_MODES[spec["mode"]], spec["act"], la, lr)
        self.h = ctypes.c_void_p()
        torch.cuda.synchronize(device)
        E.check(E.lib().zk_mlp_create(ctypes.byref(desc), ctypes.byref(self.h)))
        del keep
        lact, lres = layer_acts(spec)
        if spec["lact"] is None:
            self.oracle = O.Conditioner([w.astype(np.float64) for w in self.W], [b.astype(np.float64) for b in self.b],
                                        [None] * self.n, ACT_NAMES[1 if spec["act"] == 0 else spec["act"]])  # fmt: skip
        else:
            names = [ACT_NAMES.get(a) for a in lact]
            self.oracle = O.Conditioner([w.astype(np.float64) for w in self.W], [b.astype(np.float64) for b in self.b],
                                        [None] * self.n, ACT_NAMES[lact[1] or 1], names, [bool(r) for r in lres])  # fmt: skip

    def destroy(self):
        E.lib().zk_mlp_destroy(self.h)

    @property
    def mode(self):
        return resolved_mode(self.spec)

    def ws_bytes(self, B):
        return E.lib().zk_mlp_workspace_bytes(self.h, B)

    def call(self, x, ldx, dx, c, ldc, dc, B, out, ldo, ws=None, ws_bytes=None, check=True):
        """One zk_mlp_forward; x / c / out / ws are device tensors or raw addresses."""
        p = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
        if ws is None:
            need = self.ws_bytes(B)
            ws = torch.empty(max(need, 1), dtype=torch.uint8, device=self.device)
            ws_bytes = need
        st = E.lib().zk_mlp_forward(self.h, p(x), ldx, dx, p(c), ldc, dc, B, p(out), ldo, p(ws), ws_bytes,
                                    E.stream_ptr(self.device))  # fmt: skip
        torch.cuda.synchronize(self.device)
        if check:
            E.check(st)
        return st


@pytest.fixture
def mlp(device):
    made = []

    def make(name, seed=0):
        m = Mlp(name, device, seed)
        made.append(m)
        return m

    yield make
    for m in made:
        m.destroy()


def check_rows(B, seed=0):
    """Rows compared with the oracle: all of a small batch; else every row within 2 of a 128-row tile edge, the
    first and last tile and 512 random rows."""
    if B <= 1024:
        return np.arange(B)
    edges = np.arange(0, B + 128, 128)
    near = (edges[:, None] + np.arange(-2, 2)[None, :]).reshape(-1)
    last0 = (B - 1) // 128 * 128
    rng = np.random.default_rng(seed)
    rows = np.concatenate([near, np.arange(128), np.arange(last0, B), rng.integers(0, B, 512)])
    return np.unique(rows[(rows >= 0) & (rows < B)])


def split_k(K0):
    """(dx, dc) of a K0-wide input: about a third context."""
    dc = K0 // 3
    return K0 - dc, dc


def assert_close_rows(m, got, inp, rows, what, scale=None):
    """max|ours - ref| over `rows` <= bar * max|ref| (of `scale`, the reference over a larger batch of the same
    inputs, when given: one output of a one-row batch is no scale for the GEMM's rounding)."""
    ref = m.oracle(inp[rows].astype(np.float64), None, np.float64)
    err = float(np.abs(np.asarray(got, np.float64)[rows] - ref).max())
    scale = max(float(np.abs(ref).max()) if scale is None else scale, 1e-30)
    assert err <= BARS[m.mode] * scale, f"{what}: max err {err:.3e} of max|ref| {scale:.3e} ({m.mode}, bar {BARS[m.mode]:.0e})"
    return float(np.abs(ref).max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_mlp_forward_vs_oracle(device, mlp, name):
    m = mlp(name)
    sms = sm_count()
    L = E.lib()
    assert L.zk_mlp_gemm_mode(m.h) == E.GEMM_MODES[m.mode]
    K0, N = m.spec["dims"][0], m.spec["dims"][-1]
    dx, dc = split_k(K0)
    batches = fwd_batches(sms)
    Bmax = batches[-1]
    rng = np.random.default_rng(1)
    inp = rng.standard_normal((Bmax, K0), dtype=np.float32)
    x = torch.from_numpy(np.ascontiguousarray(inp[:, :dx])).to(device)
    c = torch.from_numpy(np.ascontiguousarray(inp[:, dx:])).to(device) if dc else None
    full = torch.full((Bmax + 1, N), NAN, device=device)
    m.call(x, dx, dx, c, dc, dc, Bmax, full, N)
    full_h = cpu(full)
    assert np.isfinite(full_h[:Bmax]).all(), f"{name}: non-finite outputs"
    assert np.isnan(full_h[Bmax]).all(), f"{name}: wrote past row B"
    scale = assert_close_rows(m, full_h, inp, check_rows(Bmax), f"{name} B={Bmax}")
    mode, layers = forward_plan(m.spec, Bmax, sms)
    print(f"{name} on {sms} SMs: {mode} {[(l['inst'], l.get('tail'), l.get('kblocks'), l.get('tiles')) for l in layers]}")
    for B in batches[:-1]:
        out = torch.full((B + 1, N), NAN, device=device)
        n0 = L.zk_launch_count()
        m.call(x, dx, dx, c, dc, dc, B, out, N)
        assert L.zk_launch_count() - n0 == (launches(m.spec) if B else 0), f"{name} B={B}: launch count"
        got = cpu(out)
        assert np.isnan(got[B]).all(), f"{name} B={B}: wrote past row B"
        assert np.array_equal(got[:B], full_h[:B]), f"{name}: the first {B} rows differ from the batch of {Bmax}"
        if B:
            assert_close_rows(m, got, inp, check_rows(B), f"{name} B={B}", scale)


LAYOUT_CASES = ["k63_h96x2_n2_tanh", "k129_h1000_n65_lrelu", "res2_h192_elu", "res3_h160_silu_x1", "fp32_gelu",
                "res_fp32_at2_h96", "k24_h96_n129_silu"]  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("name", LAYOUT_CASES)
def test_mlp_forward_layouts(device, mlp, name):
    """x and c as column slices of one padded buffer (ldx > dx, ldc > dc), one context row (ldc = 0), context-only
    (dx = 0) and x-only (dc = 0) inputs, and ldo > N with NaN in the pads: values equal the contiguous call bit for
    bit, and every pad comes back NaN."""
    m = mlp(name)
    K0, N = m.spec["dims"][0], m.spec["dims"][-1]
    dx, dc = split_k(K0)
    B = 128 * sm_count() + 129
    rng = np.random.default_rng(2)
    inp = rng.standard_normal((B, K0), dtype=np.float32)
    x = torch.from_numpy(np.ascontiguousarray(inp[:, :dx])).to(device)
    c = torch.from_numpy(np.ascontiguousarray(inp[:, dx:])).to(device) if dc else None
    ref = torch.full((B, N), NAN, device=device)
    m.call(x, dx, dx, c, dc, dc, B, ref, N)
    ref_h = cpu(ref)
    assert_close_rows(m, ref_h, inp, check_rows(B), f"{name} contiguous")
    # one buffer: [x | 3 NaN | c | 5 NaN], and out with 7 NaN pad columns and 3 NaN rows past B
    ld = K0 + 8
    buf = torch.full((B, ld), NAN, device=device)
    buf[:, :dx] = x
    if dc:
        buf[:, dx + 3 : dx + 3 + dc] = c
    ldo = N + 7
    out = torch.full((B + 3, ldo), NAN, device=device)
    cptr = buf.data_ptr() + 4 * (dx + 3) if dc else None
    m.call(buf, ld, dx, cptr, ld if dc else 0, dc, B, out, ldo)
    got = cpu(out)
    assert np.array_equal(got[:B, :N], ref_h), f"{name}: strided x / c / out differ from the contiguous call"
    pads = out[:B, N:].contiguous().view(torch.int32)
    assert (pads == torch.tensor([NAN], device=device).view(torch.int32)).all() and torch.isnan(out[B:]).all(), f"{name}: pads written"
    if dc:
        # one context row (ldc = 0) equals that row repeated
        row = c[5].contiguous()
        o1 = torch.full((B, N), NAN, device=device)
        m.call(x, dx, dx, row, 0, dc, B, o1, N)
        o2 = torch.full((B, N), NAN, device=device)
        m.call(x, dx, dx, row.expand(B, dc).contiguous(), dc, dc, B, o2, N)
        assert torch.equal(o1, o2), f"{name}: ldc = 0 differs from the repeated context row"
        inp_row = inp.copy()
        inp_row[:, dx:] = inp[5, dx:]
        assert_close_rows(m, cpu(o1), inp_row, check_rows(B), f"{name} ldc = 0")
    # all of the input as context (dx = 0, how the element-wise layers call it) and all of it as x (dc = 0)
    allin = torch.from_numpy(inp).to(device)
    o3 = torch.full((B, N), NAN, device=device)
    m.call(None, 0, 0, allin, K0, K0, B, o3, N)
    o4 = torch.full((B, N), NAN, device=device)
    m.call(allin, K0, K0, None, 0, 0, B, o4, N)
    assert torch.equal(o3, ref) and torch.equal(o4, ref), f"{name}: dx = 0 / dc = 0 differ from the split input"


WS_CASES = ["k65_h640x2_n64", "res2_h192_elu", "k129_n368_single", "fp32_tanh", "res3_h160_silu_x1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", WS_CASES)
def test_mlp_forward_workspace(device, mlp, name):
    """Exactly zk_mlp_workspace_bytes(B) suffices and the bytes past it stay untouched; one byte less is
    refused; a base offset by 256 bytes gives the same result.  Offsets of 128, 16 and 4 bytes are refused with
    ZK_EINVAL before anything is launched on a tensor-core handle (bf16 planes in 256-byte granules, 16-byte stores,
    128B-swizzled TMA boxes) and give the same result on an fp32 one."""
    m = mlp(name)
    K0, N = m.spec["dims"][0], m.spec["dims"][-1]
    B = 128 * sm_count() + 1
    inp = torch.from_numpy(np.random.default_rng(3).standard_normal((B, K0), dtype=np.float32)).to(device)
    need = m.ws_bytes(B)
    assert need > 0 or m.n == 1
    ref = torch.full((B, N), NAN, device=device)
    m.call(inp, K0, K0, None, 0, 0, B, ref, N)
    ws = torch.full((need + 512,), 0xA5, dtype=torch.uint8, device=device)
    out = torch.full((B, N), NAN, device=device)
    m.call(inp, K0, K0, None, 0, 0, B, out, N, ws=ws, ws_bytes=need)
    assert torch.equal(out, ref)
    assert (ws[need:] == 0xA5).all(), f"{name}: wrote past the workspace size it asked for"
    if need:
        n0 = E.lib().zk_launch_count()
        st = m.call(inp, K0, K0, None, 0, 0, B, out, N, ws=ws, ws_bytes=need - 1, check=False)
        assert st == E.ZK_EINVAL and E.lib().zk_launch_count() == n0
    for off in (256, 128, 16, 4):
        ws = torch.full((need + 512,), 0xA5, dtype=torch.uint8, device=device)
        o = torch.full((B, N), NAN, device=device)
        n0 = E.lib().zk_launch_count()
        st = m.call(inp, K0, K0, None, 0, 0, B, o, N, ws=ws.data_ptr() + off, ws_bytes=need, check=False)
        if off < 256 and m.mode != "fp32":
            assert st == E.ZK_EINVAL, f"{name}: a workspace {off} bytes off returned {st}"
            assert E.lib().zk_launch_count() == n0 and torch.isnan(o).all()
            continue
        E.check(st)
        assert torch.equal(o, ref), f"{name}: workspace offset by {off} bytes changes the result"
        assert (ws[off + need :] == 0xA5).all()


# --------------------------------------------------------------------------- #
# 3. layers that always run the per-layer conditioner
# --------------------------------------------------------------------------- #

LAYER_FLOWS = {
    "nice2_h64": (lambda: NICE(2, 0, transforms=2, hidden_features=[64]), "none"),
    "nice3_c2_h640": (lambda: NICE(3, 2, transforms=2, hidden_features=[640]), "rows"),
    "nice7_c3_row": (lambda: NICE(7, 3, transforms=2, hidden_features=[64]), "row"),
    "realnvp7_rqs8_c3": (lambda: RealNVP(7, 3, transforms=2, hidden_features=[64], **RQS8), "rows"),
    "realnvp7_rqs16_randmask": (lambda: RealNVP(7, 0, transforms=2, randmask=True, hidden_features=[640], **RQS16), "none"),
    "realnvp3_rqs8_row_h640": (lambda: RealNVP(3, 4, transforms=2, hidden_features=[640], **RQS8), "row"),
    "ew_affine_c3": (lambda: _one(ElementWiseTransform(4, 3, hidden_features=[64])), "rows"),
    "ew_rqs8_c5_h640": (lambda: _one(ElementWiseTransform(3, 5, hidden_features=[640], **RQS8)), "rows"),
    "ew_rqs16_row": (lambda: _one(ElementWiseTransform(4, 3, hidden_features=[64], **RQS16)), "row"),
}
LAYER_BATCHES = [1, 127, 129, 4097]


def make_layer_flow(name, seed=0):
    torch.manual_seed(seed)
    return LAYER_FLOWS[name][0]().eval()


def layer_inputs(name, D, C, B, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, generator=gen).numpy()
    kind = LAYER_FLOWS[name][1]
    c = None if kind == "none" else (torch.randn(C, generator=gen).numpy() if kind == "row" else torch.randn(B, C, generator=gen).numpy())
    return x, c


# per row |ours - ref64| <= LAYER_LP_BAR max(1, |ref64|, |log_prob64|) for log_prob and ladj of the coupling and
# element-wise flows: their phi comes from a bf16x3 GEMM (3e-5 of the output scale) and the spline / affine maps
# amplify it on rows far in the tails.  Worst measured on an H100 80GB HBM3 (SXM) at a 700 W power limit, B = 4097
# default-initialised flows: 2.2e-5 (ew_rqs8_c5_h640), 1.4e-5 (ew_affine_c3), 1.0e-5 (realnvp7_rqs16_randmask).
LAYER_LP_BAR = 3e-5


def check_lp(ours, ref64, what, scale=None):
    ours, ref64 = np.asarray(ours, np.float64), np.asarray(ref64, np.float64)
    s = np.maximum(np.abs(ref64), 1.0) if scale is None else np.maximum(np.maximum(np.abs(ref64), 1.0), np.abs(scale))
    err = np.abs(ours - ref64) / s
    assert np.isfinite(ours).all() and err.max() <= LAYER_LP_BAR, f"{what}: worst {err.max():.3e} at row {int(err.argmax())}"


@pytest.fixture
def fast_math():
    prev = E.lib().zk_set_fast_math(1)
    yield lambda fast: E.lib().zk_set_fast_math(int(fast))
    E.lib().zk_set_fast_math(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [True, False], ids=["fast", "ieee"])
@pytest.mark.parametrize("name", list(LAYER_FLOWS))
def test_layer_flows_vs_oracle(device, fast_math, name, fast):
    cpu_flow = make_layer_flow(name)
    spec = O.flowspec_from_module(cpu_flow)
    flow = make_layer_flow(name).to(device)
    fast_math(fast)
    D = spec.layers[0].features
    C = flow.transform.transforms[0].context
    for B in LAYER_BATCHES:
        x, c = layer_inputs(name, D, C, B, seed=B)
        xd, cd = dev_t(x, device), (None if c is None else dev_t(c, device))
        with torch.no_grad():
            dist = flow(cd)
            lp = cpu(dist.log_prob(xd))
            z, ladj = (cpu(v) for v in dist.transform.call_and_ladj(xd))
            xi = cpu(dist.transform.inv(dev_t(z, device)))
        z64, ladj64 = spec.forward(x.astype(np.float64), c)
        z32 = spec.forward(x, None if c is None else c.astype(np.float32), np.float32)[0]
        lp64 = spec._base_log_prob(z64, ladj64, np.float64)
        what = f"{name} B={B} {'fast' if fast else 'ieee'}"
        check_lp(lp, lp64, what + " log_prob")
        check_lp(ladj, ladj64, what + " ladj", lp64)
        check_z(z, z64, z32, what + " z")
        xr = spec.inverse(z.astype(np.float64), c)
        err = np.abs(xi - xr) / np.maximum(np.abs(xr), 1.0)
        assert err.max() <= INV_BAR, f"{what} inverse: {err.max():.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("row", [False, True], ids=["rows", "row"])
def test_gf_with_context_vs_reference(device, row):
    """GF(D, C): element-wise Gaussianization layers whose parameters come from the conditioner (one shared row
    when the context is one row)."""
    D, C, K = 3, 4, 8
    torch.manual_seed(0)
    flow = GF(D, C, transforms=3, components=K, hidden_features=[96]).eval()
    ref = GFR.Flow({k: v.numpy() for k, v in flow.state_dict().items()}, D, C, K)
    flow = flow.to(device)
    for B in [1, 129, 4097]:
        gen = torch.Generator().manual_seed(B)
        x = torch.randn(B, D, generator=gen).numpy()
        c = torch.randn(C, generator=gen).numpy() if row else torch.randn(B, C, generator=gen).numpy()
        with torch.no_grad():
            lp = cpu(flow(dev_t(c, device)).log_prob(dev_t(x, device)))
        check_row(lp, ref.log_prob(x.astype(np.float64), c.astype(np.float64)), f"GF B={B} log_prob")


def _layer_abi(h, x, ldx, c, ldc, B, y, ldy, ladj, device, inverse=False):
    L = E.lib()
    need = L.zk_layer_workspace_bytes(h, B)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
    p = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
    if inverse:
        E.check(L.zk_layer_inverse(h, p(x), ldx, p(c), ldc, B, p(y), ldy, p(ws), need, E.stream_ptr(device)))
    else:
        E.check(L.zk_layer_forward(h, p(x), ldx, p(c), ldc, B, p(y), ldy, p(ladj), 0, p(ws), need, E.stream_ptr(device)))
    torch.cuda.synchronize(device)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["nice3_c2_h640", "realnvp7_rqs8_c3", "ew_rqs8_c5_h640", "ew_rqs16_row"])
def test_layer_abi_strided(device, name):
    """zk_layer_forward / zk_layer_inverse on x, y and c rows padded with NaN: the pads stay NaN and the values
    equal the contiguous call bit for bit."""
    flow = make_layer_flow(name).to(device)
    t = flow.transform.transforms[0]
    D, C = t.features, t.context
    B = 128 * 3 + 77
    x, c = layer_inputs(name, D, C, B, seed=7)
    with torch.no_grad():
        probe = None if c is None else dev_t(c if c.ndim == 1 else c[:1], device)
        fc = flow(probe)._flow_call()[0]
    h = fc._handles[0]
    f32 = dict(device=device, dtype=torch.float32)
    ldc = 0 if (c is not None and c.ndim == 1) else C
    xd, cd = dev_t(x, device), (None if c is None else dev_t(c, device))
    y0, l0 = torch.full((B, D), NAN, **f32), torch.full((B,), NAN, **f32)
    _layer_abi(h, xd, D, cd, ldc, B, y0, D, l0, device)
    xs = torch.full((B, D + 3), NAN, **f32)
    xs[:, :D] = xd
    cs = cd
    ldcs = ldc
    if ldc:
        cs = torch.full((B, C + 5), NAN, **f32)
        cs[:, :C] = cd
        ldcs = C + 5
    ys, ls = torch.full((B + 2, D + 4), NAN, **f32), torch.full((B,), NAN, **f32)
    _layer_abi(h, xs, D + 3, cs, ldcs, B, ys, D + 4, ls, device)
    assert torch.equal(ys[:B, :D], y0) and torch.equal(ls, l0), f"{name}: strided forward differs"
    assert torch.isnan(ys[:B, D:]).all() and torch.isnan(ys[B:]).all(), f"{name}: forward wrote into the pads"
    xi0 = torch.full((B, D), NAN, **f32)
    _layer_abi(h, y0, D, cd, ldc, B, xi0, D, None, device, inverse=True)
    xis = torch.full((B + 2, D + 6), NAN, **f32)
    _layer_abi(h, ys, D + 4, cs, ldcs, B, xis, D + 6, None, device, inverse=True)
    assert torch.equal(xis[:B, :D], xi0), f"{name}: strided inverse differs"
    assert torch.isnan(xis[:B, D:]).all() and torch.isnan(xis[B:]).all(), f"{name}: inverse wrote into the pads"
    spec = O.flowspec_from_module(make_layer_flow(name))
    xr = spec.layers[0].inverse(cpu(y0), c)
    assert (np.abs(cpu(xi0) - xr) / np.maximum(np.abs(xr), 1.0)).max() <= INV_BAR


# --------------------------------------------------------------------------- #
# 4. fp32 conditioner backward
# --------------------------------------------------------------------------- #


def assert_fp32_backward_path(name, flow):
    """mlp_uses_tc (api_backward.cu) is false for every conditioner but the element-wise ones (which always take
    the fp32 backward), or the tensor-core backward is switched off for a flow whose handles would use it."""
    tc_off = BWD_FLOWS[name][2]
    uses = []
    for t in flow.transform.transforms:
        h = getattr(t, "hyper", None)
        if h is None or type(t).__name__ == "ElementWiseTransform":
            continue
        uses.append(E.lib().zk_mlp_gemm_mode(h._handle()) != E.ZK_GEMM_FP32 and h._activation_code() == E.ZK_ACT_RELU
                    and h._layer_flags() is None)  # fmt: skip
    assert all(uses) if tc_off else not any(uses), f"{name}: mlp_uses_tc = {uses}"


@pytest.mark.gpu
@pytest.mark.parametrize("name,b", BWD_MATRIX)
def test_fp32_conditioner_backward_vs_oracle(device, name, b):
    cpu_flow = make_bwd_flow(name)
    flow = make_bwd_flow(name).to(device)
    B = slice_batch(flow, b, sm_count())
    spec = O.flowspec_from_module(cpu_flow)
    D = spec.layers[0].features
    C = flow.transform.transforms[0].context
    gen = torch.Generator().manual_seed(B)
    x = torch.randn(B, D, generator=gen).numpy()
    c = None
    if C:
        c = torch.randn(C, generator=gen).numpy() if BWD_FLOWS[name][1] else torch.randn(B, C, generator=gen).numpy()
    gg = {"g": torch.randn(B, generator=gen).numpy(), "gz": torch.randn(B, D, generator=gen).numpy(),
          "gl": torch.randn(B, generator=gen).numpy()}  # fmt: skip
    for v in gg.values():
        v[relu_kink_rows(spec, x, c)] = 0.0
    tc_off = BWD_FLOWS[name][2]
    prev = E.lib().zk_set_tc_backward(0) if tc_off else None
    try:
        assert_fp32_backward_path(name, flow)
        for mode in ("lp", "tr"):
            got = _flow_grads(flow, x, c, mode, gg, device)
            kw = dict(g_log_prob=gg["g"]) if mode == "lp" else dict(g_z=gg["gz"], g_ladj=gg["gl"])
            ogx, ogc, lgs = OG.flow_backward(spec, x, c, **kw)
            ref = oracle_named_grads(cpu_flow, lgs)
            what = f"{name} B={B} {mode}"
            close(got[0], ogx, GRAD_BAR, f"{what} d/dx")
            if ogc is not None:
                close(got[1], ogc, GRAD_BAR, f"{what} d/dc")
            assert set(got[2]) == set(ref), f"{what}: parameters {sorted(set(got[2]) ^ set(ref))}"
            for k in ref:
                close(got[2][k], ref[k], GRAD_BAR, f"{what} d/d{k}")
    finally:
        if tc_off:
            E.lib().zk_set_tc_backward(prev)


class CondLayerCase(LayerCase):
    """LayerCase (test_gpu_backward_abi.py) over member 0 of a BWD_FLOWS flow."""

    def __init__(self, name, device, B, broadcast):  # noqa: super().__init__ builds from its own table
        cpu_flow = make_bwd_flow(name)
        self.flow = make_bwd_flow(name).to(device)
        spec = O.flowspec_from_module(cpu_flow)
        self.layer = spec.layers[0]
        self.D, self.C = spec.layers[0].features, self.flow.transform.transforms[0].context
        self.broadcast = broadcast and self.C > 0
        gen = torch.Generator().manual_seed(B)
        c = None
        if self.C:
            c = torch.randn(self.C, generator=gen).numpy() if self.broadcast else torch.randn(B, self.C, generator=gen).numpy()
        self.x, self.c = torch.randn(B, self.D, generator=gen).numpy(), c
        self.gy = torch.randn(B, self.D, generator=gen).numpy()
        self.gl = torch.randn(B, generator=gen).numpy()
        kink = relu_kink_rows(O.FlowSpec([self.layer], spec.loc, spec.scale), self.x, c)
        self.gy[kink], self.gl[kink] = 0.0, 0.0
        self.conditioned = self.layer.hyper is not None and self.C > 0
        probe = None if c is None else dev_t(c if self.broadcast else c[:1], device)
        self.fc = self.flow(probe)._flow_call()[0]
        self.handle, self.src = self.fc._handles[0], self.fc._sources[0]
        self.B, self.device = B, device


ABI_BWD = [("res_nsf_h160_96_96_elu", False), ("nice7_c3", False), ("nice7_c3", True), ("realnvp7_rqs_row", True),
           ("ew_affine_c3", False), ("ew_rqs_row", True), ("maf_sigmoid", False)]  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("name,broadcast", ABI_BWD)
def test_layer_backward_abi(device, name, broadcast):
    """zk_layer_backward with strided x / c / grad_y / grad_x / grad_c (NaN pads), a broadcast context (grad_c one
    summed row), the element-wise one-row path, and accumulation into non-zero gradient buffers."""
    case = CondLayerCase(name, device, 513, broadcast)
    D, C = case.D, case.C
    ogx, ogc, ref = case.oracle()
    _, gx, gc, pg = case.call(ldx=D + 3, ldg=D + 2, ldc=C + 2, ldgc=C + 3)
    assert np.isnan(gx[:, D:]).all(), f"{name}: grad_x pad written"
    close(gx[:, :D], ogx, GRAD_BAR, f"{name} grad_x")
    if case.conditioned:
        if case.broadcast:
            close(gc, ogc, GRAD_BAR, f"{name} grad_c (one summed row)")
        else:
            assert np.isnan(gc[:, C:]).all(), f"{name}: grad_c pad written"
            close(gc[:, :C], ogc, GRAD_BAR, f"{name} grad_c")
    assert set(pg) == set(ref)
    for k in ref:
        close(pg[k], ref[k], GRAD_BAR, f"{name} d/d{k}")
    # += into buffers that already hold T: T + g
    bufs = case.grad_buffers()
    T = {k: torch.randn(v.shape, generator=torch.Generator().manual_seed(3)).to(device) for k, v in bufs[0].items()}
    for k, v in bufs[0].items():
        v.copy_(T[k])
    gc0 = None
    if case.conditioned:
        gc0 = np.random.default_rng(4).standard_normal(C if case.broadcast else (case.B, C)).astype(np.float32)
    _, gx2, gc2, pg2 = case.call(bufs=bufs, gc_fill=0.0 if gc0 is None else gc0)
    close(gx2[:, :D], ogx, GRAD_BAR, f"{name} grad_x (second call)")
    for k in ref:
        close(pg2[k] - cpu(T[k]), ref[k], GRAD_BAR, f"{name} d/d{k} accumulated")
    if gc0 is not None:
        close((gc2 if case.broadcast else gc2[:, :C]) - gc0, ogc, GRAD_BAR, f"{name} grad_c accumulated")
