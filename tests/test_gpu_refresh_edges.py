"""GPU tests of the in-place weight refresh (zk_layer_update_weights, zk_gmm_update_weights) at every packed copy it
brings up to date: `mask * W` and the biases, the bf16 planes of the per-layer GEMMs, the fused kernel's permuted
planes and biases, the backward transposes and bf16 backward planes (rebuilt on the next backward) and the sequential
inverse's step-ordered stream (rebuilt on the next inverse).

* `CASES` is one handle per case, taken from the existing shape tables (test_gpu_fused_edges.SHAPES, cases.build_flow,
  gmm_cases): fused autoregressive layers on both tile plans, every bijector the fused kernel takes, a trimmed first K
  block, an odd output-chunk count, all-zero tiles, a non-ReLU activation and bf16x1; autoregressive layers off the
  fused kernel (fp32 GEMMs, residual, circular, Bernstein, SOSP, passes < D, the sweep fallback); a coupling layer
  with n_a != n_b; an element-wise layer with a context; a permutation folded into the next autoregressive layer.
  Every case asserts its path with the query APIs first.  tests/test_refresh_host.py checks on the CPU that the
  table reaches every refresh and rebuild row of the handle caches.
* `SEQUENCES` change the weights of a live handle the way an optimizer does, after a forward only, after a backward
  and an inverse, twice in a row, biases only, weights only, with large values in masked-out entries, around a
  sweeps / sequential inverse switch, before an inverse backward, through load_state_dict, and on a side stream.
  The fused cases and the coupling, element-wise and folded cases run every sequence; the cases in SHORT run the
  five that differ in what the refresh must rebuild ((b), (d), (f), (g), (i)).
* After each sequence every path the case has must equal a handle built fresh from `state_dict()` bit for bit
  (forward and log_prob fused and unfused, the sequential inverse and the sweeps, the forward and inverse backward;
  after (b), (d) and (j) the backward also with the tensor-core backward off), and the fp64 oracle at the new weights within the bars of the edge
  files: log_prob 1e-5 max(1, |ref|) per row from the fused kernel, 3e-5 from the per-layer kernels (bf16x1: no
  worse than twice the per-layer kernels' error + 1e-4), the inverse 1e-4, gradients 5e-5 of max|ref| (inverse
  direction 1e-4); GMM log_prob 2e-5, gradients 5e-5.  The forward and the inverse go to the oracle after every
  sequence, the gradients after (b), (d), (f) and (i), where rows at a ReLU kink or a spline knot get zero weight
  (cases.relu_kink_rows).  Bernstein and SOSP layers are compared with the fresh handle only: the oracle has no
  model of them (their own files test them against the reference).
* The C ABI: NULL bias arrays and entries keep the current biases; refusals queue nothing and change nothing; the
  launch count of the backward after a refresh."""

from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Callable

import numpy as np
import pytest
import torch

import gmm_cases as GC
import test_gpu_fused_edges as FE
import zuko_b200 as zuko
from cases import build_flow, oracle_named_grads, relu_kink_rows
from oracle import oracle as O
from oracle import oracle_grad as OG
from test_gpu_gmm_edges import kink_rows as gmm_kink_rows
from test_gpu_gmm_edges import oracle as gmm_oracle
from zuko_b200 import _engine as E
from zuko_b200.distributions import DiagNormal
from zuko_b200.flows import BPF, NICE, SOSPF, MaskedAutoregressiveTransform
from zuko_b200.flows._packed import PackedLayerMixin
from zuko_b200.lazy import Flow, UnconditionalDistribution, UnconditionalTransform
from zuko_b200.transforms import PermutationTransform, RotationTransform, SoftclipTransform

# test_gpu_fused_edges (fused log_prob), test_gpu_conditioner_edges (per-layer kernels' log_prob, the inverse,
# gradients), test_gpu_backward (inverse-direction gradients), test_gpu_gmm_edges (D <= 16)
LP_BAR, LAYER_LP_BAR, INV_BAR, GRAD_BAR, INV_GRAD_BAR = 1e-5, 3e-5, 1e-4, 5e-5, 1e-4
GMM_LP_BAR, GMM_GRAD_BAR = 2e-5, 5e-5
B = 300  # above two 128-row tiles and four 64-row tiles


# --------------------------------------------------------------------------- #
# the case table
# --------------------------------------------------------------------------- #


def _seeded(ctor, seed=0):
    def build():
        torch.manual_seed(seed)
        return ctor().eval()

    return build


def _perm_ar():
    """A permutation, an autoregressive layer and the inverse permutation: the two permutations fold away (no gather
    kernel), so inference calls run the layer re-indexed by the first one."""
    D = 6
    perm = torch.tensor([3, 0, 5, 1, 4, 2])
    layers = [UnconditionalTransform(PermutationTransform, perm, buffer=True),
              MaskedAutoregressiveTransform(D, 2, hidden_features=[128, 128]),
              UnconditionalTransform(PermutationTransform, torch.argsort(perm), buffer=True)]  # fmt: skip
    return Flow(layers, UnconditionalDistribution(DiagNormal, torch.zeros(D), torch.ones(D), buffer=True))


@dataclass(frozen=True)
class Case:
    build: Callable  # () -> the flow on the CPU, eval mode, seeded
    kind: str  # member kind of the conditioned layers: "ar", "coupling", "elementwise"
    rows: int  # zk_layer_fused_tile_rows of the autoregressive layers (0: not the fused kernel)
    seq_inverse: int  # zk_layer_sequential_inverse of the autoregressive layers
    mode: str  # conditioner gemm mode as zk_mlp_gemm_mode reports it
    oracle: bool = True  # the fp64 oracle models the bijector
    grad_oracle: bool = True  # gradients against the oracle (bf16x1 has no useful gradient bar)
    bf16x1: bool = False
    folded: bool = False  # a permutation in front: the inference calls run the re-indexed handle
    tc: bool = True  # the backward takes the tensor-core path (bf16 planes, plain ReLU)

    def tc_settings(self, seq: str) -> tuple:
        """zk_set_tc_backward values the backward runs with: off as well (the fp32 transposes) where the backward
        has the tensor-core path, after the sequences that rebuild the backward pack from a backward already run."""
        return (1, 0) if self.tc and seq in TC_OFF else (1,)


CASES = {
    # fused autoregressive layers
    "affine_t64": Case(lambda: FE.make_flow("maf16_h320"), "ar", 64, 1, "bf16x3"),
    "rqs8_t128_trimmed_k": Case(lambda: FE.make_flow("nsf8c4_h256_L2"), "ar", 128, 1, "bf16x3"),
    "rqs16_t128_odd_n_last": Case(lambda: FE.make_flow("nsf7_k16_h128"), "ar", 128, 1, "bf16x3"),
    "rqs8_t64_odd_chunks": Case(lambda: FE.make_flow("nsf12c4_h320"), "ar", 64, 1, "bf16x3"),
    "adjacency16_k16": Case(lambda: FE.make_flow("adjacency16_k16"), "ar", 128, 0, "bf16x3"),  # sweep fallback
    "lrelu_t128": Case(lambda: FE.make_flow("nsf10c2_h128_lrelu"), "ar", 128, 1, "bf16x3", tc=False),
    "bf16x1_t128": Case(lambda: FE.make_flow("nsf8c4_h256_L2_x1"), "ar", 128, 1, "bf16x1", grad_oracle=False, bf16x1=True),
    # autoregressive layers off the fused kernel
    "fp32": Case(lambda: FE.make_flow("nsf16c8_h128_fp32"), "ar", 0, 1, "fp32", tc=False),
    "residual": Case(lambda: FE.make_flow("maf12c4_h256_residual"), "ar", 0, 0, "bf16x3", tc=False),
    "ncsf": Case(lambda: FE.make_flow("ncsf4c3_h128"), "ar", 0, 1, "bf16x3"),
    "bpf": Case(_seeded(lambda: BPF(3, 2, transforms=1, hidden_features=[64, 64])), "ar", 0, 1, "bf16x3", oracle=False),
    "sospf": Case(_seeded(lambda: SOSPF(3, 2, transforms=1, hidden_features=[64, 64])), "ar", 0, 1, "bf16x3", oracle=False),
    "passes2": Case(lambda: build_flow("nsf5_passes2"), "ar", 0, 1, "bf16x3"),
    # other conditioned layers
    "coupling_4_3": Case(_seeded(lambda: NICE(7, 3, transforms=2, hidden_features=[64, 64])), "coupling", 0, 0, "bf16x3"),
    "elementwise_ctx": Case(lambda: build_flow("nsf1_elementwise"), "elementwise", 0, 0, "fp32", tc=False),
    "perm_then_ar": Case(_seeded(_perm_ar), "ar", 128, 1, "bf16x3", folded=True),
}  # fmt: skip

# name -> (gmm_cases name, gemm mode of the conditioner)
GMM = {
    "gmm_rows_fp32": ("full_untied", "fp32"),
    "gmm_rows_tc": ("full_untied", "bf16x3"),
    "gmm_bcast_fp32": ("bcast", "fp32"),
    "gmm_bcast_tc": ("bcast", "bf16x3"),
}

# (a) .. (k); (j) has its own test
SEQUENCES = ["a_forward_only", "b_backward_inverse", "c_twice", "d_biases_adam", "e_weights_only", "f_masked_entries",
             "g_sweeps_then_sequential", "h_inverse_backward", "i_load_state_dict", "k_side_stream"]  # fmt: skip
GMM_SEQUENCES = ["a_forward_only", "b_backward_inverse", "c_twice", "d_biases_adam", "e_weights_only",
                 "i_load_state_dict", "k_side_stream"]  # fmt: skip


# layers off the fused kernel whose bijector or conditioner differs only past the refresh: the sequences that
# differ in what the refresh must rebuild (the others run on every other case)
SHORT = {"residual", "ncsf", "bpf", "sospf", "passes2", "adjacency16_k16", "lrelu_t128", "bf16x1_t128"}
SHORT_SEQUENCES = ["b_backward_inverse", "d_biases_adam", "f_masked_entries", "g_sweeps_then_sequential",
                   "i_load_state_dict"]  # fmt: skip


def sequences_of(name: str) -> list[str]:
    case = CASES[name]
    out = []
    for s in SHORT_SEQUENCES if name in SHORT else SEQUENCES:
        if s == "f_masked_entries" and case.kind != "ar":
            continue  # no masked-out entries
        if s == "g_sweeps_then_sequential" and not case.seq_inverse:
            continue
        out.append(s)
    return out


FLOW_MATRIX = [(n, s) for n in CASES for s in sequences_of(n)]
# sequences whose gradients also go to the fp64 oracle (every sequence compares them with a fresh handle bit for bit)
GRAD_ORACLE = {"b_backward_inverse", "d_biases_adam", "f_masked_entries", "i_load_state_dict"}
TC_OFF = {"b_backward_inverse", "d_biases_adam", "j_new_order"}


def conditioned(flow) -> list:
    return [t for t in flow.transform.transforms if isinstance(t, PackedLayerMixin) and getattr(t, "hyper", None) is not None]


def rebuilds_on_load(t) -> bool:
    """load_state_dict copies buffers in place too: a layer whose state holds a mask or an order buffer rebuilds."""
    return any(name.endswith(("mask", "order")) for name, _ in t.named_buffers())


# --------------------------------------------------------------------------- #
# helpers
# --------------------------------------------------------------------------- #


def cpu(t):
    return None if t is None else t.detach().cpu().numpy().astype(np.float64)


def dev_t(a, device, grad=False):
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
    return t.requires_grad_() if grad else t


class Switch:
    """zk_set_fused_layers / zk_set_tc_backward for one block."""

    def __init__(self, fn, on):
        self.fn, self.on = fn, on

    def __enter__(self):
        self.prev = self.fn(int(self.on))

    def __exit__(self, *exc):
        self.fn(self.prev)


def fused(on):
    return Switch(E.lib().zk_set_fused_layers, on)


def tc_backward(on):
    return Switch(E.lib().zk_set_tc_backward, on)


def inputs(flow, seed=11):
    D = next(t.features for t in flow.transform.transforms if hasattr(t, "features"))
    C = max(getattr(t, "context", 0) for t in flow.transform.transforms)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, generator=g).numpy()
    z = torch.randn(B, D, generator=g).numpy()
    c = torch.randn(B, C, generator=g).numpy() if C else None
    w = (torch.rand(B, generator=g) + 0.5).numpy().astype(np.float64)
    wx = torch.randn(B, D, generator=g).numpy().astype(np.float64)
    return x, z, c, w, wx


def cpu_copy(case: Case, flow):
    """The case's CPU module holding the live flow's state."""
    other = case.build()
    other.load_state_dict({k: v.detach().cpu() for k, v in flow.state_dict().items()})
    return other


def fresh(case: Case, flow, device):
    return cpu_copy(case, flow).to(device)


def param_grads(flow):
    return [cpu(p.grad) for _, p in flow.named_parameters()]


def paths(flow, x, z, c, w, wx, device, tcs=(1, 0)) -> dict:
    """Every result the flow's handles produce on the inputs, as fp64 arrays."""
    xd, zd = dev_t(x, device), dev_t(z, device)
    cd = None if c is None else dev_t(c, device)
    out = {}
    with torch.no_grad():
        for on in (1, 0):
            with fused(on):
                d = flow(cd)
                out[f"log_prob/fused={on}"] = cpu(d.log_prob(xd))
                zz, ladj = d.transform.call_and_ladj(xd)
                out[f"z/fused={on}"], out[f"ladj/fused={on}"] = cpu(zz), cpu(ladj)
                out[f"inverse/fused={on}"] = cpu(d.transform.inv(zd))
    for tc in tcs:
        with tc_backward(tc):
            for p in flow.parameters():
                p.grad = None
            xg = dev_t(x, device, grad=True)
            cg = None if c is None else dev_t(c, device, grad=True)
            (dev_t(w, device) * flow(cg).log_prob(xg)).sum().backward()
            out[f"grad_x/tc={tc}"], out[f"grad_c/tc={tc}"] = cpu(xg.grad), cpu(None if cg is None else cg.grad)
            for k, g in enumerate(param_grads(flow)):
                out[f"grad_p{k}/tc={tc}"] = g
            for p in flow.parameters():
                p.grad = None
            zg = dev_t(z, device, grad=True)
            cg = None if c is None else dev_t(c, device, grad=True)
            call, ctx = flow(cg)._flow_call()
            xi, lpi = call.inverse(zg, ctx, with_log_prob=True)
            ((dev_t(wx, device) * xi).sum() + (dev_t(w, device) * lpi).sum()).backward()
            out[f"inv_x/tc={tc}"], out[f"inv_lp/tc={tc}"] = cpu(xi), cpu(lpi)
            out[f"inv_grad_z/tc={tc}"], out[f"inv_grad_c/tc={tc}"] = cpu(zg.grad), cpu(None if cg is None else cg.grad)
            for k, g in enumerate(param_grads(flow)):
                out[f"inv_grad_p{k}/tc={tc}"] = g
    for p in flow.parameters():
        p.grad = None
    return out


def assert_same(got: dict, want: dict, what: str):
    assert got.keys() == want.keys()
    for k in want:
        a, b = got[k], want[k]
        if b is None:
            assert a is None, f"{what}: {k}"
            continue
        assert a is not None and a.shape == b.shape, f"{what}: {k}"
        if not np.array_equal(a, b, equal_nan=True):
            bad = np.argwhere(a != b)
            raise AssertionError(f"{what}: {k} differs from a freshly built handle in {len(bad)} of {a.size} entries; "
                                 f"first at {tuple(bad[0])}: {a[tuple(bad[0])]!r} vs {b[tuple(bad[0])]!r}")  # fmt: skip


def close(ours, ref, bar, what):
    ours, ref = np.asarray(ours, np.float64), np.asarray(ref, np.float64)
    scale = max(float(np.abs(ref).max()), 1e-30)
    err = float(np.abs(ours - ref).max()) / scale
    assert np.isfinite(ours).all() and err <= bar, f"{what}: max err {err:.3e} of max|ref| {scale:.3e} (bar {bar:.0e})"
    return err


def row_err(ours, ref):
    return float(np.max(np.abs(ours - ref) / np.maximum(np.abs(ref), 1.0)))


def weights_for(case: Case, flow, x, z, c, kinks: bool):
    """Per-row gradient weights, with the rows at a kink or knot zeroed (at the flow's current weights) when the
    gradients go to the oracle."""
    _, _, _, w, wx = inputs(flow)
    if kinks:
        spec = O.flowspec_from_module(cpu_copy(case, flow))
        bad = relu_kink_rows(spec, x, c) | relu_kink_rows(spec, spec.inverse(z.astype(np.float64), c), c)
        w, wx = w.copy(), wx.copy()
        w[bad], wx[bad] = 0.0, 0.0
    return w, wx


def report(path: str, err: float, what: str):
    print(f"oracle error {path}: {err:.2e} ({what})")


def check_oracle(case: Case, flow, got: dict, x, z, c, w, wx, what: str, grads: bool, tcs: tuple):
    """The live results against the fp64 oracle at the flow's current weights (each error printed for -s runs)."""
    host = cpu_copy(case, flow)
    spec = O.flowspec_from_module(host)
    x64, z64 = x.astype(np.float64), z.astype(np.float64)
    lp = spec.log_prob(x64, c)
    if case.bf16x1:
        e_f, e_u = row_err(got["log_prob/fused=1"], lp), row_err(got["log_prob/fused=0"], lp)
        assert e_f <= 2 * e_u + 1e-4, f"{what}: bf16x1 fused log_prob error {e_f:.3e}, per-layer kernels {e_u:.3e}"
    else:
        for on in (1, 0):
            e, bar = row_err(got[f"log_prob/fused={on}"], lp), (LP_BAR if on and case.rows else LAYER_LP_BAR)
            report("log_prob " + ("fused kernel" if bar == LP_BAR else "per-layer kernels"), e, what)
            assert e <= bar, f"{what}: log_prob (fused={on}) {e:.3e} off the oracle (bar {bar:.0e})"
    xs = spec.inverse(z64, c)
    if case.bf16x1:
        e_s, e_w = row_err(got["inverse/fused=1"], xs), row_err(got["inverse/fused=0"], xs)
        assert e_s <= 2 * e_w + 1e-4, f"{what}: bf16x1 sequential inverse error {e_s:.3e}, sweeps {e_w:.3e}"
    else:
        for on in (1, 0):
            e = close(got[f"inverse/fused={on}"], xs, INV_BAR, f"{what}: inverse (fused={on})")
            report("inverse " + ("sequential" if on and case.seq_inverse else "sweeps"), e, what)
    if not (grads and case.grad_oracle):
        return
    names = [n for n, _ in host.named_parameters()]
    ogx, ogc, lgs = OG.flow_backward(spec, x, c, g_log_prob=w)
    opg = oracle_named_grads(host, lgs)
    ogz, oic, ilgs = OG.flow_inverse_backward(spec, z64, c, g_x=wx, g_log_prob=w)
    oipg = oracle_named_grads(host, ilgs)
    for tc in tcs:
        fwd = [close(got[f"grad_x/tc={tc}"], ogx, GRAD_BAR, f"{what}: d/dx (tc={tc})")]
        inv = [close(got[f"inv_grad_z/tc={tc}"], ogz, INV_GRAD_BAR, f"{what}: inverse d/dz (tc={tc})")]
        if ogc is not None:
            fwd.append(close(got[f"grad_c/tc={tc}"], ogc, GRAD_BAR, f"{what}: d/dc (tc={tc})"))
            inv.append(close(got[f"inv_grad_c/tc={tc}"], oic, INV_GRAD_BAR, f"{what}: inverse d/dc (tc={tc})"))
        for k, n in enumerate(names):
            fwd.append(close(got[f"grad_p{k}/tc={tc}"].reshape(-1), opg[n], GRAD_BAR, f"{what}: d/d{n} (tc={tc})"))
            inv.append(close(got[f"inv_grad_p{k}/tc={tc}"].reshape(-1), oipg[n], INV_GRAD_BAR,
                             f"{what}: inverse d/d{n} (tc={tc})"))  # fmt: skip
        kind = "tensor-core" if (tc and case.tc) else "fp32"
        report(f"backward ({kind})", max(fwd), what)
        report(f"inverse backward ({kind})", max(inv), what)


def assert_path(case: Case, flow):
    """The case runs where its name says: fused tile rows, sequential inverse and GEMM mode from the query APIs."""
    for t in conditioned(flow):
        h = t._zk_layer()
        # the mode the conditioner module resolves to, read from its stand-alone zk_mlp handle (no query reads the
        # conditioner inside a layer handle; both are packed from the same zk_mlp_desc by zk_mlp_create)
        assert E.lib().zk_mlp_gemm_mode(t.hyper._handle()) == E.GEMM_MODES[case.mode]
        if case.kind == "ar":
            assert E.lib().zk_layer_fused_tile_rows(h) == case.rows
            info = (ctypes.c_double * 4)()
            assert E.lib().zk_layer_fused_info(h, info) == (1 if case.rows else 0)
            assert E.lib().zk_layer_sequential_inverse(h) == case.seq_inverse
        else:
            assert E.lib().zk_layer_fused_tile_rows(h) == 0 and E.lib().zk_layer_sequential_inverse(h) == 0


def step(flow, which="all", seed=0):
    """An in-place parameter update that bumps _version, as an optimizer step does."""
    g = torch.Generator().manual_seed(1000 + seed)
    with torch.no_grad():
        for n, p in flow.named_parameters():
            if (which == "weights" and not n.endswith("weight")) or (which == "biases" and not n.endswith("bias")):
                continue
            p.add_(0.01 * torch.randn(p.shape, generator=g).to(p.device))


def adam_biases(flow, seed=0):
    """(d): weights frozen with requires_grad_(False), one Adam step on the rest."""
    g = torch.Generator().manual_seed(2000 + seed)
    frozen = [p for n, p in flow.named_parameters() if n.endswith("weight")]
    for p in frozen:
        p.requires_grad_(False)
    live = [p for p in flow.parameters() if p.requires_grad]
    opt = torch.optim.Adam(live, lr=1e-2)
    for p in live:
        p.grad = torch.randn(p.shape, generator=g).to(p.device)
    opt.step()  # every bias moves by about lr
    for p in live:
        p.grad = None
    for p in frozen:
        p.requires_grad_(True)


def mask_noise(flow):
    """(f): large values added in place to the masked-out weight entries (bumps _version)."""
    n = 0
    with torch.no_grad():
        for t in conditioned(flow):
            for m in t.hyper._linears():
                mask = getattr(m, "mask", None)
                if mask is not None and not bool(mask.all()):
                    m.weight.add_(1e3 * (~mask.bool()).to(m.weight.dtype))
                    n += 1
    assert n > 0, "no masked-out entries"


def other_checkpoint(case: Case, flow) -> dict:
    """A second checkpoint of the same structure (same masks and order): the case perturbed."""
    other = case.build()
    step(other, seed=77)
    return other.state_dict()


# --------------------------------------------------------------------------- #
# A. flow cases x refresh sequences
# --------------------------------------------------------------------------- #


def run_sequence(case: Case, seq: str, flow, device, x, z, c):
    """Applies the sequence to the live flow; returns the expected kind per conditioned layer: "refresh" (same
    OwnedLayer, generation + n) or "rebuild" (a new OwnedLayer)."""
    xd, zd = dev_t(x, device), dev_t(z, device)
    cd = None if c is None else dev_t(c, device)
    layers = conditioned(flow)
    refs = [t._zk_layer_ref() for t in layers]
    gens = [r.generation for r in refs]
    if seq == "a_forward_only":
        with torch.no_grad():
            flow(cd).log_prob(xd)
        step(flow)
    elif seq in ("b_backward_inverse", "k_side_stream", "g_sweeps_then_sequential", "h_inverse_backward"):
        (-flow(cd).log_prob(xd).mean()).backward()
        with torch.no_grad():
            flow(cd).transform.inv(zd)
        for p in flow.parameters():
            p.grad = None
        step(flow)
    elif seq == "c_twice":
        (-flow(cd).log_prob(xd).mean()).backward()
        for p in flow.parameters():
            p.grad = None
        step(flow, seed=1)
        for t in layers:
            t._zk_layer_ref()  # first refresh, no engine call before the second
        step(flow, seed=2)
    elif seq == "d_biases_adam":
        (-flow(cd).log_prob(xd).mean()).backward()
        for p in flow.parameters():
            p.grad = None
        adam_biases(flow)
    elif seq == "e_weights_only":
        (-flow(cd).log_prob(xd).mean()).backward()
        for p in flow.parameters():
            p.grad = None
        step(flow, "weights")
    elif seq == "f_masked_entries":
        (-flow(cd).log_prob(xd).mean()).backward()
        with torch.no_grad():
            flow(cd).transform.inv(zd)
        for p in flow.parameters():
            p.grad = None
        mask_noise(flow)
    elif seq == "i_load_state_dict":
        (-flow(cd).log_prob(xd).mean()).backward()
        with torch.no_grad():
            flow(cd).transform.inv(zd)
        for p in flow.parameters():
            p.grad = None
        flow.load_state_dict(other_checkpoint(case, flow))
    else:
        raise AssertionError(seq)
    if seq == "g_sweeps_then_sequential":  # the first inverse after the step runs the sweeps: the step-ordered pack is
        # rebuilt from there (layer_inverse_impl rebuilds before it looks at zk_set_fused_layers), and the
        # sequential inverse in paths() must then run on that rebuilt pack
        with torch.no_grad(), fused(0):
            flow(cd).transform.inv(zd)
    if seq == "h_inverse_backward":  # the first call after the step is zk_flow_inverse_backward
        call, ctx = flow(cd)._flow_call()
        xi, lpi = call.inverse(dev_t(z, device, grad=True), ctx, with_log_prob=True)
        (xi.sum() + lpi.sum()).backward()
        for p in flow.parameters():
            p.grad = None
    kinds = []
    for t, r, g0 in zip(layers, refs, gens):
        now = t._zk_layer_ref()
        if seq == "i_load_state_dict" and rebuilds_on_load(t):
            assert now is not r and now.generation == 0, f"{seq}: {type(t).__name__} was not rebuilt"
            kinds.append("rebuild")
        else:
            assert now is r, f"{seq}: {type(t).__name__} was rebuilt, not refreshed"
            assert now.generation == g0 + (2 if seq == "c_twice" else 1)
            kinds.append("refresh")
    return kinds


def reindexed(flow):
    return [v[1] for t in conditioned(flow) for v in t.__dict__.get("_zk_reindexed", {}).values()]


@pytest.mark.gpu
@pytest.mark.parametrize("name,seq", FLOW_MATRIX)
def test_refresh_sequence(device, name, seq):
    case = CASES[name]
    flow = case.build().to(device)
    assert_path(case, flow)
    x, z, c, _, _ = inputs(flow)
    what = f"{name} {seq}"
    side = torch.cuda.Stream(device) if seq == "k_side_stream" else None
    with torch.cuda.stream(side) if side is not None else torch.cuda.stream(torch.cuda.current_stream(device)):
        if case.folded:
            with torch.no_grad():
                flow(dev_t(c, device)).log_prob(dev_t(x, device))
            before = reindexed(flow)
            assert before, "the inference call did not run the re-indexed handle"
        run_sequence(case, seq, flow, device, x, z, c)
        grads = case.oracle and case.grad_oracle and seq in GRAD_ORACLE
        tcs = case.tc_settings(seq)
        w, wx = weights_for(case, flow, x, z, c, kinks=grads)
        ref = fresh(case, flow, device)
        want = paths(ref, x, z, c, w, wx, device, tcs)
        if seq == "b_backward_inverse":  # no atomics on these paths: a fresh handle repeats itself bit for bit
            assert_same(paths(ref, x, z, c, w, wx, device, tcs), want, f"{what}: fresh handle run twice")
        got = paths(flow, x, z, c, w, wx, device, tcs)
        if case.folded:
            assert not any(r is b for r in reindexed(flow) for b in before), "the re-indexed handle was served stale"
    if side is not None:
        torch.cuda.synchronize(device)
    assert_same(got, want, what)
    if case.oracle:
        check_oracle(case, flow, got, x, z, c, w, wx, what, grads, tcs)


def _maf_randperm():
    return zuko.flows.MAF(5, 2, transforms=2, randperm=True, hidden_features=[128, 128])


@pytest.mark.gpu
def test_load_state_dict_with_new_order_rebuilds(device):
    """(j): MAF(randperm=True) checkpoints of other seeds carry other orders and masks: a new handle."""
    case = Case(_seeded(_maf_randperm, 7), "ar", 128, 1, "bf16x3")
    flow = case.build().to(device)
    other = _seeded(_maf_randperm, 8)()
    assert any(not torch.equal(a.order.cpu(), b.order) for a, b in zip(conditioned(flow), conditioned(other)))
    x, z, c, _, _ = inputs(flow)
    with torch.no_grad():
        flow(dev_t(c, device)).log_prob(dev_t(x, device))
    refs = [t._zk_layer_ref() for t in conditioned(flow)]
    flow.load_state_dict(other.state_dict())
    assert all(t._zk_layer_ref() is not r for t, r in zip(conditioned(flow), refs))
    assert_path(case, flow)
    tcs = case.tc_settings("j_new_order")
    w, wx = weights_for(case, flow, x, z, c, kinks=True)
    got = paths(flow, x, z, c, w, wx, device, tcs)
    assert_same(got, paths(fresh(case, flow, device), x, z, c, w, wx, device, tcs), "randperm load_state_dict")
    check_oracle(case, flow, got, x, z, c, w, wx, "randperm load_state_dict", True, tcs)


# --------------------------------------------------------------------------- #
# B. the generation guard
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rqs8_t128_trimmed_k", "coupling_4_3", "elementwise_ctx", "fp32"])
def test_graph_across_a_refresh_raises(device, name):
    case = CASES[name]
    flow = case.build().to(device)
    x, z, c, _, _ = inputs(flow)
    cd = dev_t(c, device)
    lp = flow(cd).log_prob(dev_t(x, device, grad=True))
    call, ctx = flow(cd)._flow_call()
    xi, lpi = call.inverse(dev_t(z, device, grad=True), ctx, with_log_prob=True)
    step(flow)
    with torch.no_grad():
        flow(cd).log_prob(dev_t(x, device))  # refreshes in place
    with pytest.raises(RuntimeError, match="refreshed in place"):
        lp.sum().backward()
    with pytest.raises(RuntimeError, match="refreshed in place"):
        (xi.sum() + lpi.sum()).backward()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GMM))
def test_gmm_graph_across_a_refresh_raises(device, name):
    gmm, x, c, _ = make_gmm(name, device)
    lp = gmm(c).log_prob(x.requires_grad_())
    step(gmm)
    with torch.no_grad():
        gmm(c).log_prob(x)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        lp.sum().backward()


# --------------------------------------------------------------------------- #
# C. GMM cases x refresh sequences
# --------------------------------------------------------------------------- #


def make_gmm(name, device, seed=None):
    src, mode = GMM[name]
    gmm = GC.build(zuko, src)
    if seed is not None:
        step(gmm, seed=seed)
    gmm.hyper.gemm_mode = mode
    x, c, w = GC.inputs(src)
    return gmm.to(device), x.to(device), c.to(device), w.to(device)


def gmm_handle(gmm):
    return gmm.__dict__["_zk_cache"][2].value


def gmm_paths(gmm, x, c, w) -> dict:
    out = {}
    with torch.no_grad():
        out["log_prob"] = cpu(gmm(c).log_prob(x))
        torch.manual_seed(5)
        out["sample"] = cpu(gmm(c).sample((17,)))
    for tc in (1, 0):
        with tc_backward(tc):
            for p in gmm.parameters():
                p.grad = None
            xg, cg = x.clone().requires_grad_(), c.clone().requires_grad_()
            (w * gmm(cg).log_prob(xg)).sum().backward()
            out[f"grad_x/tc={tc}"], out[f"grad_c/tc={tc}"] = cpu(xg.grad), cpu(cg.grad)
            for k, g in enumerate(param_grads(gmm)):
                out[f"grad_p{k}/tc={tc}"] = g
    for p in gmm.parameters():
        p.grad = None
    return out


def gmm_fresh(name, gmm, device):
    src, mode = GMM[name]
    other = GC.build(zuko, src)
    other.load_state_dict({k: v.detach().cpu() for k, v in gmm.state_dict().items()})
    other.hyper.gemm_mode = mode
    return other.to(device)


@pytest.mark.gpu
@pytest.mark.parametrize("seq", GMM_SEQUENCES)
@pytest.mark.parametrize("name", list(GMM))
def test_gmm_refresh_sequence(device, name, seq):
    side = torch.cuda.Stream(device) if seq == "k_side_stream" else None
    with torch.cuda.stream(side) if side is not None else torch.cuda.stream(torch.cuda.current_stream(device)):
        gmm, x, c, w = make_gmm(name, device)
        assert E.lib().zk_mlp_gemm_mode(gmm.hyper._handle()) == E.GEMM_MODES[GMM[name][1]]
        if seq == "a_forward_only":
            with torch.no_grad():
                gmm(c).log_prob(x)
        else:
            (-gmm(c).log_prob(x).mean()).backward()
            with torch.no_grad():
                gmm(c).sample((3,))
            for p in gmm.parameters():
                p.grad = None
        h = gmm_handle(gmm)
        if seq == "c_twice":
            step(gmm, seed=1)
            gmm.handle(gmm.params())
            step(gmm, seed=2)
        elif seq == "d_biases_adam":
            adam_biases(gmm)
        elif seq == "e_weights_only":
            step(gmm, "weights")
        elif seq == "i_load_state_dict":
            gmm.load_state_dict(make_gmm(name, "cpu", seed=77)[0].state_dict())
        else:
            step(gmm)
        gmm.handle(gmm.params())
        assert gmm_handle(gmm) == h, f"{seq}: the GMM handle was rebuilt, not refreshed"
        wk = w.clone()
        if GMM[name][1] != "fp32":  # as test_gpu_gmm_edges: a broadcast row runs its conditioner in fp32, no kinks
            wk[torch.from_numpy(gmm_kink_rows(gmm, cpu(c), x.shape[0])).to(device)] = 0.0
        ref = gmm_fresh(name, gmm, device)
        want = gmm_paths(ref, x, c, wk)
        assert_same(gmm_paths(ref, x, c, wk), want, f"{name} {seq}: fresh handle run twice")
        got = gmm_paths(gmm, x, c, wk)
    if side is not None:
        torch.cuda.synchronize(device)
    assert_same(got, want, f"{name} {seq}")
    o = gmm_oracle(gmm, cpu(x), cpu(c), cpu(wk))
    e = row_err(got["log_prob"], o.lp)
    report("GMM log_prob", e, f"{name} {seq}")
    assert e <= GMM_LP_BAR, f"{name} {seq}: log_prob {e:.3e} off the oracle"
    for tc in (1, 0):
        errs = [close(got[f"grad_x/tc={tc}"], o.gx, GMM_GRAD_BAR, f"{name} {seq} d/dx"),
                close(got[f"grad_c/tc={tc}"], o.gc, GMM_GRAD_BAR, f"{name} {seq} d/dc")]  # fmt: skip
        for k, r in enumerate(o.params):
            errs.append(close(got[f"grad_p{k}/tc={tc}"], r, GMM_GRAD_BAR, f"{name} {seq} d/dparam{k}"))
        report("GMM backward", max(errs), f"{name} {seq} tc={tc}")


# --------------------------------------------------------------------------- #
# D. the C ABI directly
# --------------------------------------------------------------------------- #


def ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def abi_flow(device):
    case = CASES["rqs8_t128_trimmed_k"]
    flow = case.build().to(device)
    x, z, c, _, _ = inputs(flow)
    with torch.no_grad():
        flow(dev_t(c, device)).transform.inv(dev_t(z, device))  # the step-ordered pack exists
    return case, flow, x, z, c


def forward_paths(flow, x, z, c, device):
    xd, zd, cd = dev_t(x, device), dev_t(z, device), (None if c is None else dev_t(c, device))
    out = {}
    with torch.no_grad():
        for on in (1, 0):
            with fused(on):
                d = flow(cd)
                out[f"log_prob/fused={on}"] = cpu(d.log_prob(xd))
                out[f"inverse/fused={on}"] = cpu(d.transform.inv(zd))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("bias", ["null_array", "null_entries"])
def test_layer_update_keeps_null_biases(device, bias):
    """zk_layer_update_weights with a NULL bias array, or NULL entries for some layers: those biases stay."""
    case, flow, x, z, c = abi_flow(device)
    t = conditioned(flow)[0]
    lins = t.hyper._linears()
    g = torch.Generator().manual_seed(3)
    W = [(m.weight.detach() + 0.05 * torch.randn(m.weight.shape, generator=g).to(device)).contiguous() for m in lins]
    Bn = [(m.bias.detach() + 0.05 * torch.randn(m.bias.shape, generator=g).to(device)).contiguous() for m in lins]
    sent = [None] * len(lins) if bias == "null_array" else [Bn[i] if i % 2 == 0 else None for i in range(len(lins))]
    st = E.lib().zk_layer_update_weights(t._zk_layer(), ptrs(W), None if bias == "null_array" else ptrs(sent),
                                         E.stream_ptr(device))  # fmt: skip
    assert st == E.ZK_OK
    torch.cuda.synchronize(device)
    got = forward_paths(flow, x, z, c, device)  # the module's versions did not move: the handle serves as updated
    ref = cpu_copy(case, flow)
    with torch.no_grad():
        for m, w, b in zip(ref.transform.transforms[0].hyper._linears(), W, sent):
            m.weight.copy_(w.cpu())
            if b is not None:
                m.bias.copy_(b.cpu())
    assert_same(got, forward_paths(ref.to(device), x, z, c, device), f"update with {bias}")


@pytest.mark.gpu
@pytest.mark.parametrize("bias", ["null_array", "null_entries"])
def test_gmm_update_keeps_null_biases(device, bias):
    gmm, x, c, w = make_gmm("gmm_rows_tc", device)
    h = gmm.handle(gmm.params())
    lins = gmm.hyper._linears()
    g = torch.Generator().manual_seed(4)
    W = [(m.weight.detach() + 0.05 * torch.randn(m.weight.shape, generator=g).to(device)).contiguous() for m in lins]
    Bn = [(m.bias.detach() + 0.05 * torch.randn(m.bias.shape, generator=g).to(device)).contiguous() for m in lins]
    sent = [None] * len(lins) if bias == "null_array" else [Bn[i] if i % 2 == 0 else None for i in range(len(lins))]
    st = E.lib().zk_gmm_update_weights(h, ptrs(W), None if bias == "null_array" else ptrs(sent), E.stream_ptr(device))
    assert st == E.ZK_OK
    with torch.no_grad():
        got = cpu(gmm(c).log_prob(x))
    ref = gmm_fresh("gmm_rows_tc", gmm, "cpu")
    with torch.no_grad():
        for m, wt, b in zip(ref.hyper._linears(), W, sent):
            m.weight.copy_(wt.cpu())
            if b is not None:
                m.bias.copy_(b.cpu())
    ref = ref.to(device)
    with torch.no_grad():
        assert np.array_equal(got, cpu(ref(c).log_prob(x)))


def _no_conditioner_flow():
    D = 4
    torch.manual_seed(5)
    layers = [UnconditionalTransform(SoftclipTransform, bound=11.0),
              UnconditionalTransform(PermutationTransform, torch.tensor([2, 0, 3, 1]), buffer=True),
              UnconditionalTransform(RotationTransform, torch.randn(D, D), buffer=True),
              zuko.flows.ElementWiseTransform(D, 0)]  # fmt: skip
    return Flow(layers, UnconditionalDistribution(DiagNormal, torch.zeros(D), torch.ones(D), buffer=True))


REFUSALS = ["null_handle", "null_weights", "last_weight_null", "softclip", "permutation", "rotation", "table",
            "gmm_null_weights", "gmm_last_weight_null", "gmm_unconditional"]  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("what", REFUSALS)
def test_update_refusals_change_nothing(device, what):
    """Each refusal returns a status, launches nothing and leaves the next forward bit-identical."""
    L = E.lib()
    s = E.stream_ptr(device)
    if what.startswith("gmm"):
        gmm, x, c, _ = make_gmm("gmm_rows_tc", device)
        if what == "gmm_unconditional":
            torch.manual_seed(6)
            gmm = zuko.mixtures.GMM(3, components=3).to(device)
            c = None
        run = lambda: cpu(gmm(c).log_prob(x))  # noqa: E731
        with torch.no_grad():
            before = run()
        h = gmm.handle(gmm.params())
        lins = gmm.hyper._linears() if hasattr(gmm, "hyper") else []
        W = [(m.weight.detach() * 1.5).contiguous() for m in lins] or [torch.ones(8, device=device)]
        if what == "gmm_last_weight_null":
            W[-1] = None
        call = lambda: L.zk_gmm_update_weights(h, None if what == "gmm_null_weights" else ptrs(W), None, s)  # noqa: E731
    elif what in ("softclip", "permutation", "rotation", "table"):
        flow = _no_conditioner_flow().to(device)
        x = torch.randn(B, 4, generator=torch.Generator().manual_seed(1)).to(device)
        run = lambda: cpu(flow().log_prob(x))  # noqa: E731
        with torch.no_grad():
            before = run()
        hs = flow()._flow_call()[0]._handles
        assert len(hs) == 4
        h = hs[["softclip", "permutation", "rotation", "table"].index(what)]
        one = torch.ones(8, device=device)
        call = lambda: L.zk_layer_update_weights(h, ptrs([one]), None, s)  # noqa: E731
    else:
        case, flow, xn, zn, cn = abi_flow(device)
        run = lambda: forward_paths(flow, xn, zn, cn, device)  # noqa: E731
        before = run()
        t = conditioned(flow)[0]
        W = [(m.weight.detach() * 1.5).contiguous() for m in t.hyper._linears()]
        if what == "last_weight_null":
            W[-1] = None
        h = None if what == "null_handle" else t._zk_layer()
        call = lambda: L.zk_layer_update_weights(h, None if what == "null_weights" else ptrs(W), None, s)  # noqa: E731
    torch.cuda.synchronize(device)
    n0 = L.zk_launch_count()
    st = call()
    assert st != E.ZK_OK, f"{what}: accepted"
    assert L.zk_launch_count() == n0, f"{what}: the refusal launched kernels"
    with torch.no_grad():
        after = run()
    if isinstance(before, dict):
        assert_same(after, before, what)
    else:
        assert np.array_equal(after, before), what


def backward_launches(flow, x, c, device):
    xd = dev_t(x, device, grad=True)
    lp = flow(dev_t(c, device)).log_prob(xd)
    n0 = E.lib().zk_launch_count()
    lp.sum().backward()
    torch.cuda.synchronize(device)
    n = E.lib().zk_launch_count() - n0
    for p in flow.parameters():
        p.grad = None
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("when", ["before_first_backward", "after_a_backward"])
@pytest.mark.parametrize("name", ["rqs8_t128_trimmed_k", "fp32"])
def test_backward_launch_count_after_refresh(device, name, when):
    """The first backward after a refresh rebuilds the transposes once; the next launches exactly as many kernels as
    a backward on a handle that was never refreshed."""
    case = CASES[name]
    steady = case.build().to(device)
    flow = case.build().to(device)
    x, z, c, _, _ = inputs(flow)
    first = backward_launches(steady, x, c, device)
    n_steady = backward_launches(steady, x, c, device)
    assert first > n_steady  # the first backward builds the transposes
    if when == "after_a_backward":
        assert backward_launches(flow, x, c, device) == first
    else:
        with torch.no_grad():
            flow(dev_t(c, device)).log_prob(dev_t(x, device))
    step(flow)
    n1 = backward_launches(flow, x, c, device)
    n2 = backward_launches(flow, x, c, device)
    assert n1 == first, f"first backward after the refresh: {n1} launches, a first backward {first}"
    assert n2 == n_steady, f"second backward after the refresh: {n2} launches, a steady backward {n_steady}"
