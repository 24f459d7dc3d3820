"""GPU tests of the fused layer kernel's row tiles: 128-row tiles (two consumer warpgroups sharing every streamed
weight tile) for the shapes whose A operands and weight ring fit shared memory, 64-row tiles for the rest.  Batch
sizes sit at the tile edges, at one and several tiles per CTA of the persistent grid."""

import ctypes

import pytest
import torch

import zuko_b200 as zuko
from cases import rel_err
from oracle import oracle as O
from test_gpu_tcgen05 import FUSED_FLOWS
from zuko_b200 import _engine as E

pytestmark = pytest.mark.gpu

# rows per tile of every FUSED_FLOWS shape: 128 unless the two A operands (2 x 2 planes x KBA x 8 KB), the output
# staging and a ring of four 16 KB slots exceed 227 KB (KBA > 4: hidden width 384 / 512; the affine staging is
# wider, so MAF at KBA = 4 keeps 64-row tiles)
TILE_ROWS = {
    "nsf16c8_h256": 128, "nsf64_k16_h64": 128, "nsf5c3_h192": 128, "nsf7_k16_h128": 128, "maf32_h256": 64,
    "maf70c100_h128": 128, "maf32_h512x4": 64, "nsf64c16_k16_h512": 64, "nsf24_k8_h512": 64, "nsf10c3_h384": 64,
    "maf100c28_h512": 64, "maf32_h512_elu": 64, "nsf16c8_h256_silu": 128, "nsf12_h256_tanh": 128,
    "maf24c4_h384_gelu": 64, "maf8_h64_tanh": 128, "nsf5c3_h192_elu": 128, "nsf20_k16_h64_silu": 128,
}  # fmt: skip
WIDE = ["nsf16c8_h256", "nsf64_k16_h64", "nsf5c3_h192", "nsf7_k16_h128", "maf70c100_h128", "nsf12_h256_tanh"]
# batch sizes as functions of the SM count S: partial tiles, a tile whose second half lies past the batch, one
# tile per CTA and CTAs that loop over several tiles
BATCHES = {
    "1": lambda S: 1, "63": lambda S: 63, "64": lambda S: 64, "65": lambda S: 65, "127": lambda S: 127,
    "128": lambda S: 128, "129": lambda S: 129, "255": lambda S: 255, "S*128-1": lambda S: S * 128 - 1,
    "S*128+1": lambda S: S * 128 + 1, "3*S*128+77": lambda S: 3 * S * 128 + 77,
}  # fmt: skip


def _sm_count(device) -> int:
    return torch.cuda.get_device_properties(device).multi_processor_count


def _flow_and_inputs(name, B, device, seed):
    torch.manual_seed(11)
    flow_cpu = FUSED_FLOWS[name]().eval()
    D = flow_cpu.base.loc.shape[0]
    C = flow_cpu.transform.transforms[0].context
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, generator=g)
    c = torch.randn(B, C, generator=g) if C else None
    flow = FUSED_FLOWS[name]()
    flow.load_state_dict(flow_cpu.state_dict())
    return flow_cpu, flow.to(device), x, c


@pytest.fixture
def unfused():
    def run(fn):
        prev = E.lib().zk_set_fused_layers(0)
        try:
            return fn()
        finally:
            E.lib().zk_set_fused_layers(prev)

    return run


def test_tile_rows_follow_the_shape(device):
    assert set(TILE_ROWS) == set(FUSED_FLOWS)
    for name, rows in TILE_ROWS.items():
        _, flow, x, c = _flow_and_inputs(name, 4, device, 0)
        with torch.no_grad():
            flow(None if c is None else c.to(device)).log_prob(x.to(device))  # packs
        for t in flow.transform.transforms:
            assert E.lib().zk_layer_fused_tile_rows(t._zk_layer()) == rows, name
            assert E.lib().zk_layer_fused_info(t._zk_layer(), (ctypes.c_double * 4)()) == 1, name


def test_unfused_layers_report_no_tile(device, unfused):
    flow = FUSED_FLOWS["nsf16c8_h256"]().to(device)
    x, c = torch.randn(8, 16, device=device), torch.randn(8, 8, device=device)
    with torch.no_grad():
        flow(c).log_prob(x)
    assert E.lib().zk_layer_fused_tile_rows(None) == 0
    flow_res = zuko.flows.MAF(12, 4, transforms=1, hidden_features=[256, 256], residual=True).to(device)
    with torch.no_grad():
        flow_res(c[:, :4]).log_prob(x[:, :12])
    assert E.lib().zk_layer_fused_tile_rows(flow_res.transform.transforms[0]._zk_layer()) == 0


@pytest.mark.parametrize("name", WIDE)
@pytest.mark.parametrize("batch", list(BATCHES))
def test_wide_tiles_match_unfused_and_oracle(device, unfused, name, batch):
    B = BATCHES[batch](_sm_count(device))
    flow_cpu, flow, x, c = _flow_and_inputs(name, B, device, B)
    spec = O.flowspec_from_module(flow_cpu)
    xd, cd = x.to(device), (None if c is None else c.to(device))
    with torch.no_grad():
        lp_f = flow(cd).log_prob(xd)
        z_f, ladj_f = flow(cd).transform.call_and_ladj(xd)
        lp_u = unfused(lambda: flow(cd).log_prob(xd))
        z_u, ladj_u = unfused(lambda: flow(cd).transform.call_and_ladj(xd))
    assert E.lib().zk_layer_fused_tile_rows(flow.transform.transforms[0]._zk_layer()) == 128
    ref = spec.log_prob(x.numpy(), None if c is None else c.numpy())
    assert rel_err(lp_f.cpu().numpy(), ref) < 1e-5
    assert rel_err(lp_u.cpu().numpy(), ref) < 1e-5
    assert torch.allclose(lp_f, lp_u, rtol=2e-6, atol=2e-5)
    assert torch.allclose(z_f, z_u, rtol=1e-5, atol=1e-5)
    assert torch.allclose(ladj_f, ladj_u, rtol=2e-6, atol=2e-5)


@pytest.mark.parametrize("name", WIDE)
def test_wide_tiles_rows_do_not_depend_on_the_batch(device, name):
    """One launch per flow layer, and every row of a sub-batch (aligned or not to the 128-row tiles) equals the
    same row of the full batch bit for bit."""
    S = _sm_count(device)
    B = 3 * S * 128 + 77
    _, flow, x, c = _flow_and_inputs(name, B, device, 7)
    xd, cd = x.to(device), (None if c is None else c.to(device))
    with torch.no_grad():
        lp = flow(cd).log_prob(xd)
        n0 = E.lib().zk_launch_count()
        lp = flow(cd).log_prob(xd)
        assert E.lib().zk_launch_count() - n0 == len(flow.transform.transforms)
        for lo, hi in [(0, 300), (0, 129), (64, 1000), (191, 192), (B - 200, B)]:
            part = flow(None if cd is None else cd[lo:hi]).log_prob(xd[lo:hi])
            assert torch.equal(lp[lo:hi], part), (lo, hi)


@pytest.mark.parametrize("batch", ["1", "129", "S*128+1", "3*S*128+77"])
def test_wide_tiles_single_bf16_term(device, unfused, batch):
    """gemm_mode = "bf16x1": the 128-row instantiations that stream one 8 KB plane per ring slot and issue one MMA
    per k step.  Their error against the fp64 oracle is that of a single bf16 product, the same as the per-layer
    GEMM kernels' at bf16x1, and a row's result does not depend on the batch it sits in."""
    B = BATCHES[batch](_sm_count(device))
    flow_cpu, flow, x, c = _flow_and_inputs("nsf16c8_h256", B, device, B)
    for t in flow.transform.transforms:
        t.hyper.gemm_mode = "bf16x1"
    xd, cd = x.to(device), c.to(device)
    with torch.no_grad():
        lp_f = flow(cd).log_prob(xd)
        lp_u = unfused(lambda: flow(cd).log_prob(xd))
        for t in flow.transform.transforms:
            assert E.lib().zk_mlp_gemm_mode(t.hyper._handle()) == E.ZK_GEMM_BF16X1
            assert E.lib().zk_layer_fused_tile_rows(t._zk_layer()) == 128
        part = flow(cd[B // 3 :]).log_prob(xd[B // 3 :])
    assert torch.equal(lp_f[B // 3 :], part)
    ref = O.flowspec_from_module(flow_cpu).log_prob(x.numpy(), c.numpy())
    err_f, err_u = rel_err(lp_f.cpu().numpy(), ref), rel_err(lp_u.cpu().numpy(), ref)
    assert err_u < 1e-1, err_u  # a single bf16 MMA: ~2^-8 per operand, through two flow layers
    assert err_f < 2 * err_u + 1e-4, (err_f, err_u)
