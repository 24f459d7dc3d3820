"""GPU tests of the tensor-core (wgmma) conditioner path against the fp64 oracle and the
fp32 CUDA-core path."""

import ctypes

import numpy as np
import pytest
import torch

import zuko_b200 as zuko
from cases import assert_log_prob_parity, build_flow, load, rel_err
from oracle import oracle as O
from zuko_b200 import _engine as E

pytestmark = pytest.mark.gpu


def _oracle_mlp(net, x):
    cond = O.conditioner_from_module(net)
    return cond(x.numpy().astype(np.float64), None, np.float64)


def _masked(adj_shape, hidden, seed=0):
    torch.manual_seed(seed)
    out_f, in_f = adj_shape
    adjacency = torch.rand(out_f, in_f) < 0.6
    adjacency[:, 0] = True
    return zuko.nn.MaskedMLP(adjacency, hidden)


SHAPES = [
    ((368, 24), [256, 256, 256]),  # BASELINE config 2 conditioner
    ((69, 8), [64, 64]),           # N not a multiple of 16, K padded 8 -> 64
    ((64, 32), [512, 512]),        # two N chunks per hidden layer
    ((6, 100), [96]),              # hidden width 96 -> padded to 128 for the next K
    ((300, 64), []),               # single linear layer
]


@pytest.mark.parametrize("shape,hidden", SHAPES)
@pytest.mark.parametrize("B", [1, 127, 128, 129, 1000, 40000])
def test_tcgen05_mlp_vs_oracle(device, shape, hidden, B):
    net = _masked(shape, hidden)
    net.gemm_mode = "bf16x3"
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B, shape[1], generator=g)
    ref = _oracle_mlp(net, x)
    out = net.to(device)(x.to(device))
    assert E.lib().zk_mlp_gemm_mode(net._handle()) == E.ZK_GEMM_BF16X3
    out = out.detach().cpu().numpy().astype(np.float64)
    scale = np.abs(ref).max()
    err = np.abs(out - ref).max() / scale
    # split-bf16 (3 MMAs, fp32 accumulate): ~2^-16 per product term; bound 3e-5 of the output scale
    assert err < 3e-5, err
    # and the fp32 CUDA-core path agrees with both
    net32 = _masked(shape, hidden)
    net32.gemm_mode = "fp32"
    out32 = net32.to(device)(x.to(device)).detach().cpu().numpy().astype(np.float64)
    assert np.abs(out32 - ref).max() / scale < 2e-6


def test_bf16x1_is_available_but_inexact(device):
    net = _masked((368, 24), [256, 256, 256])
    net.gemm_mode = "bf16x1"
    x = torch.randn(4096, 24, generator=torch.Generator().manual_seed(1))
    ref = _oracle_mlp(net, x)
    out = net.to(device)(x.to(device)).detach().cpu().numpy().astype(np.float64)
    err = np.abs(out - ref).max() / np.abs(ref).max()
    assert 1e-4 < err < 3e-2, err  # single bf16 MMA: ~2^-8 per operand


@pytest.mark.parametrize("name", ["cfg2_nsf", "cfg3_maf", "cfg4_nsf", "cfg5_nsf", "nsf35_row", "nice35"])
def test_flow_parity_on_tensor_cores(device, name):
    """The BASELINE configs with the conditioner forced onto the tensor cores (bf16x3): log_prob within
    1e-5 relative of the reference."""
    g = load(f"flow_{name}")
    flow = build_flow(name, g)
    for t in flow.transform.transforms:
        t.hyper.gemm_mode = "bf16x3"
    flow = flow.to(device)
    c = None if "c" not in g else torch.from_numpy(g["c"]).to(device)
    lp = flow(c).log_prob(torch.from_numpy(g["x"]).to(device))
    assert E.lib().zk_mlp_gemm_mode(flow.transform.transforms[0].hyper._handle()) == E.ZK_GEMM_BF16X3
    assert_log_prob_parity(lp.detach().cpu().numpy(), g, rtol=1e-5)


RES_SHAPES = [
    ((368, 24), [256, 256, 256], torch.nn.ReLU),   # cfg2's conditioner with residual blocks: L, R(L a L), R, R, L
    ((64, 40), [512, 512], torch.nn.ELU),          # two N chunks per layer, general activation inside the block
    ((69, 8), [96, 160, 160], torch.nn.SiLU),      # widths change: Linear 96, Linear 160 + block, block (padded K 192)
]


@pytest.mark.parametrize("shape,hidden,act", RES_SHAPES)
@pytest.mark.parametrize("B", [1, 129, 5000])
def test_residual_mlp_on_tensor_cores(device, shape, hidden, act, B):
    """MaskedMLP(residual=True) (zuko/nn.py:195-199, 297-309) on the tensor-core GEMM kernels: the second layer of a
    block adds the block's input, read back from the bf16 hi / lo planes the kernel overwrites in place."""
    def make():
        torch.manual_seed(5)
        adjacency = torch.rand(*shape) < 0.6
        adjacency[:, 0] = True
        return zuko.nn.MaskedMLP(adjacency, hidden, activation=act, residual=True)

    net = make()
    assert any(isinstance(m, zuko.nn.Residual) for m in net)
    net.gemm_mode = "bf16x3"
    x = torch.randn(B, shape[1], generator=torch.Generator().manual_seed(B))
    ref = _oracle_mlp(net, x)
    out = net.to(device)(x.to(device)).detach().cpu().numpy().astype(np.float64)
    assert E.lib().zk_mlp_gemm_mode(net._handle()) == E.ZK_GEMM_BF16X3
    scale = np.abs(ref).max()
    assert np.abs(out - ref).max() / scale < 3e-5
    net32 = make()
    net32.gemm_mode = "fp32"
    out32 = net32.to(device)(x.to(device)).detach().cpu().numpy().astype(np.float64)
    assert np.abs(out32 - ref).max() / scale < 2e-6


@pytest.mark.parametrize("name", ["res_nsf_relu", "res_nsf_mixed"])
def test_residual_goldens_on_tensor_cores(device, name):
    """The reference's residual flows (tests/golden/make_golden_res.py) with the conditioner forced onto
    the tensor cores: log_prob within 1e-5 of the reference, gradients still flow (fp32 backward kernels)."""
    g = load(f"flow_{name}")
    flow = build_flow(name, g)
    for t in flow.transform.transforms:
        t.hyper.gemm_mode = "bf16x3"
    flow = flow.to(device)
    c = None if "c" not in g else torch.from_numpy(g["c"]).to(device)
    x = torch.from_numpy(g["x"]).to(device)
    lp = flow(c).log_prob(x)
    assert E.lib().zk_mlp_gemm_mode(flow.transform.transforms[0].hyper._handle()) == E.ZK_GEMM_BF16X3
    assert_log_prob_parity(lp.detach().cpu().numpy(), g, rtol=1e-5)
    (-lp.mean()).backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in flow.parameters())


def test_wide_residual_flow_vs_oracle(device):
    """A residual MAF wide enough for `auto` to pick the tensor cores (hidden 256): per-layer GEMM kernels (the
    fused layer kernels refuse residual blocks), log_prob and the sweep inverse against the fp64 oracle."""
    torch.manual_seed(21)
    flow_cpu = zuko.flows.MAF(12, 4, transforms=2, hidden_features=[256, 256], residual=True)
    spec = O.flowspec_from_module(flow_cpu)
    gen = torch.Generator().manual_seed(2)
    x, c = torch.randn(3000, 12, generator=gen), torch.randn(3000, 4, generator=gen)
    flow = flow_cpu.to(device)
    with torch.no_grad():
        lp = flow(c.to(device)).log_prob(x.to(device))
        assert E.lib().zk_mlp_gemm_mode(flow.transform.transforms[0].hyper._handle()) == E.ZK_GEMM_BF16X3
        info = (ctypes.c_double * 4)()
        assert E.lib().zk_layer_fused_info(flow.transform.transforms[0]._zk_layer(), info) == 0  # per-layer GEMM kernels
        ref = spec.log_prob(x.numpy(), c.numpy())
        assert rel_err(lp.cpu().numpy(), ref) < 1e-5
        xr = flow(c.to(device)).transform.inv(flow(c.to(device)).transform(x.to(device)))
        assert (xr.cpu() - x).abs().max().item() < 1e-4


def test_auto_mode_picks_tensor_cores_for_wide_layers(device):
    wide = _masked((368, 24), [256, 256]).to(device)
    tiny = _masked((8, 4), [32, 32]).to(device)
    assert E.lib().zk_mlp_gemm_mode(wide._handle()) == E.ZK_GEMM_BF16X3
    assert E.lib().zk_mlp_gemm_mode(tiny._handle()) == E.ZK_GEMM_FP32


# --------------------------------------------------------------------------- #
# fully fused layer kernel (conditioner + bijector + ladj in one launch)
# --------------------------------------------------------------------------- #

FUSED_FLOWS = {
    "nsf16c8_h256": lambda: zuko.flows.NSF(16, 8, transforms=2, bins=8, hidden_features=[256] * 3),   # cfg2 shape
    "nsf64_k16_h64": lambda: zuko.flows.NSF(64, 0, transforms=2, bins=16),                             # cfg4 shape
    "nsf5c3_h192": lambda: zuko.flows.NSF(5, 3, transforms=3, bins=8, hidden_features=[192, 192]),     # hidden width 192, odd D with DPC = 2
    "nsf7_k16_h128": lambda: zuko.flows.NSF(7, 0, transforms=2, bins=16, hidden_features=[128, 128]),  # 16 bins: one dim per output chunk (DPC = 1)
    "maf32_h256": lambda: zuko.flows.MAF(32, 0, transforms=2, hidden_features=[256] * 2),              # affine, 32 dims / chunk
    "maf70c100_h128": lambda: zuko.flows.MAF(70, 100, transforms=2, hidden_features=[128] * 2),        # K0 = 170 -> 3 K blocks, 3 affine chunks
    # ---- hidden width 384 / 512: four accumulators per warpgroup, activations overwritten in place ----
    "maf32_h512x4": lambda: zuko.flows.MAF(32, 0, transforms=2, hidden_features=[512] * 4),            # cfg3 shape
    "nsf64c16_k16_h512": lambda: zuko.flows.NSF(64, 16, transforms=2, bins=16, hidden_features=[512] * 3),  # cfg5 shape
    "nsf24_k8_h512": lambda: zuko.flows.NSF(24, 0, transforms=2, bins=8, hidden_features=[512, 512]),  # degree classes not aligned to chunks
    "nsf10c3_h384": lambda: zuko.flows.NSF(10, 3, transforms=3, bins=8, hidden_features=[384, 384]),   # 3 chunks / 6 K blocks
    "maf100c28_h512": lambda: zuko.flows.MAF(100, 28, transforms=2, hidden_features=[512] * 2),        # K0 = 128, 2 affine chunks
    # ---- non-ReLU activations (nn.py:264-265; general-activation instantiation) ----
    "maf32_h512_elu": lambda: zuko.flows.MAF(32, 0, transforms=2, hidden_features=[512] * 2, activation=torch.nn.ELU),
    "nsf16c8_h256_silu": lambda: zuko.flows.NSF(16, 8, transforms=2, bins=8, hidden_features=[256] * 2, activation=torch.nn.SiLU),
    "nsf12_h256_tanh": lambda: zuko.flows.NSF(12, 0, transforms=2, bins=8, hidden_features=[256, 256], activation=torch.nn.Tanh),
    "maf24c4_h384_gelu": lambda: zuko.flows.MAF(24, 4, transforms=2, hidden_features=[384] * 2, activation=torch.nn.GELU),
    # ---- ... and at hidden width 64 - 192, the library's default widths ----
    "maf8_h64_tanh": lambda: zuko.flows.MAF(8, 0, transforms=2, activation=torch.nn.Tanh),
    "nsf5c3_h192_elu": lambda: zuko.flows.NSF(5, 3, transforms=2, bins=8, hidden_features=[192, 192], activation=torch.nn.ELU),
    "nsf20_k16_h64_silu": lambda: zuko.flows.NSF(20, 0, transforms=2, bins=16, activation=torch.nn.SiLU),
}
WIDE_FLOWS = ["maf32_h512x4", "nsf64c16_k16_h512", "nsf24_k8_h512", "nsf10c3_h384", "maf100c28_h512",
              "maf32_h512_elu", "nsf16c8_h256_silu", "nsf12_h256_tanh", "maf24c4_h384_gelu"]
ONE_LAUNCH_FLOWS = WIDE_FLOWS + ["maf8_h64_tanh", "nsf5c3_h192_elu", "nsf20_k16_h64_silu"]


@pytest.fixture
def unfused():
    def run(fn):
        prev = E.lib().zk_set_fused_layers(0)
        try:
            return fn()
        finally:
            E.lib().zk_set_fused_layers(prev)

    return run


@pytest.mark.parametrize("name", list(FUSED_FLOWS))
@pytest.mark.parametrize("B", [1, 100, 128, 777, 20000])
def test_fused_layer_matches_unfused_and_oracle(device, unfused, name, B):
    torch.manual_seed(11)
    flow_cpu = FUSED_FLOWS[name]().eval()
    spec = O.flowspec_from_module(flow_cpu)
    D = flow_cpu.base.loc.shape[0]
    C = flow_cpu.transform.transforms[0].context
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B, D, generator=g)
    c = torch.randn(B, C, generator=g) if C else None
    flow = FUSED_FLOWS[name]()
    flow.load_state_dict(flow_cpu.state_dict())
    flow = flow.to(device)
    xd, cd = x.to(device), (None if c is None else c.to(device))
    from zuko_b200.flows._packed import PackedLayerMixin  # noqa: F401

    dist = flow(cd)
    lp_f = dist.log_prob(xd)
    z_f, ladj_f = dist.transform.call_and_ladj(xd)
    lp_u = unfused(lambda: flow(cd).log_prob(xd))
    z_u, ladj_u = unfused(lambda: flow(cd).transform.call_and_ladj(xd))
    ref = spec.log_prob(x.numpy(), None if c is None else c.numpy())
    assert rel_err(lp_f.detach().cpu().numpy(), ref) < 1e-5
    assert rel_err(lp_u.detach().cpu().numpy(), ref) < 1e-5
    # same arithmetic (split-bf16 GEMMs, same bijector math): fused and unfused agree to rounding
    assert torch.allclose(lp_f, lp_u, rtol=2e-6, atol=2e-5)
    assert torch.allclose(z_f, z_u, rtol=1e-5, atol=1e-5)
    assert torch.allclose(ladj_f, ladj_u, rtol=2e-6, atol=2e-5)


@pytest.mark.parametrize("name", ONE_LAUNCH_FLOWS)
def test_wide_layers_run_as_one_kernel_each(device, name):
    """Hidden width 384 / 512, and non-ReLU conditioners of every fused width: ONE launch per flow layer (no
    per-layer GEMM fallback), and a ragged batch (partial tile) gives the rows of the full batch bit for bit."""
    torch.manual_seed(5)
    flow = FUSED_FLOWS[name]().to(device)
    D = flow.base.loc.shape[0]
    C = flow.transform.transforms[0].context
    B = 256 * 3 + 129
    x = torch.randn(B, D, device=device)
    c = torch.randn(B, C, device=device) if C else None
    with torch.no_grad():
        lp = flow(c).log_prob(x)  # packs
        n0 = E.lib().zk_launch_count()
        lp = flow(c).log_prob(x)
        assert E.lib().zk_launch_count() - n0 == len(flow.transform.transforms)
        lp_part = flow(None if c is None else c[:300]).log_prob(x[:300])
    assert torch.equal(lp[:300], lp_part)


def test_fused_layer_broadcast_context_and_launch_count(device):
    torch.manual_seed(3)
    flow = zuko.flows.NSF(16, 8, transforms=4, bins=8, hidden_features=[256] * 3).to(device)
    x = torch.randn(4096, 16, device=device)
    c_row = torch.randn(8, device=device)
    lp_row = flow(c_row).log_prob(x)
    lp_full = flow(c_row.expand(4096, 8).contiguous()).log_prob(x)
    assert torch.equal(lp_row, lp_full)
    n0 = E.lib().zk_launch_count()
    flow(c_row).log_prob(x)
    assert E.lib().zk_launch_count() - n0 == 4  # ONE kernel per flow layer, base log-prob fused into the last
