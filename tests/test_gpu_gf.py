"""GPU tests of the Gaussianization flow (GF) and of GaussianizationTransform against the reference's goldens
(tests/golden/make_golden_gf.py).

Value bar: ``|ours - ref64| <= max(1e-5 * max(|ref64|, 1), 2 * |ref32 - ref64|)``; the reference's own fp32
path is poor in the tails, so the fp32 term is what the engine is measured against there.  The inverse is a
bisection whose decisions near a tie may differ from the reference's: its absolute term also allows two final
intervals, ``2 * (2 bound / 2^n)``.  A flow's inverse chains four bisections and three rotations, and in the tails of
a layer it amplifies the fp32 error of that layer's input: there, as for the stress set of the other flows
(cases.assert_log_prob_parity), at most 1% of the elements may miss the per-element bar, provided the engine is no
less accurate than the reference's own fp32 inverse in distribution (max within 10x, 99th percentile and median
within 2x).  Both settings of ``zk_set_fast_math`` are held to the same bar."""

import math

import numpy as np
import pytest
import torch

from cases import assert_param_grads, load
from test_gf_host import GF_CASES, UNIT_TAGS, build_gf
from zuko_b200 import _engine as E
from zuko_b200.transforms import GaussianizationTransform

pytestmark = pytest.mark.gpu
UG = load("units_gf")


@pytest.fixture(params=[1, 0], ids=["fast", "ieee"])
def fast_math(request):
    prev = E.lib().zk_set_fast_math(request.param)
    yield request.param
    E.lib().zk_set_fast_math(prev)


def dev_t(a, device, grad=False):
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
    return t.requires_grad_() if grad else t


def cpu(t):
    return t.detach().cpu().numpy().astype(np.float64)


def misses(ours, ref64, ref32, atol=0.0):
    ours, ref64, ref32 = (np.asarray(a, np.float64) for a in (ours, ref64, ref32))
    tol = np.maximum(np.maximum(1e-5 * np.maximum(np.abs(ref64), 1.0), 2.0 * np.abs(ref32 - ref64)), atol)
    return np.abs(ours - ref64) > tol


def check(ours, ref64, ref32, what, atol=0.0):
    bad = misses(ours, ref64, ref32, atol)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} misses, first at {i}: ours={np.asarray(ours)[i]!r} ref64={ref64[i]!r} ref32={ref32[i]!r}")


def interval(bound=10.0, eps=1e-6):
    return 2 * bound / 2 ** math.ceil(math.log2(2 * bound / eps))


@pytest.mark.parametrize("name", list(GF_CASES))
def test_flow_values(device, fast_math, name):
    g = load(f"flow_{name}")
    flow = build_gf(name).to(device)
    c = g.get("c")
    ct = None if c is None else dev_t(c, device)
    with torch.no_grad():
        lp = flow(ct).log_prob(dev_t(g["x"], device))
        z, ladj = flow(ct).transform.call_and_ladj(dev_t(g["x"], device))
        ci = None if c is None else (ct if c.ndim == 1 else ct[: g["zin"].shape[0]])
        xi = flow(ci).transform.inv(dev_t(g["zin"], device))
    check(cpu(lp), g["log_prob64"], g["log_prob32"], f"{name} log_prob")
    check(cpu(z), g["z64"], g["z32"], f"{name} z")
    check(cpu(ladj), g["ladj64"], g["ladj32"], f"{name} ladj")
    check_inverse(cpu(xi), g["xinv64"], g["xinv32"], f"{name} inverse")


def check_inverse(ours, ref64, ref32, what):
    bad = misses(ours, ref64, ref32, atol=2 * interval())
    if not bad.any():
        return
    assert bad.mean() <= 0.01, f"{what}: {int(bad.sum())} of {bad.size} elements miss the bar"
    err, ref_err = np.abs(ours - ref64), np.abs(ref32.astype(np.float64) - ref64)
    floor = 2 * interval()
    assert err.max() <= max(10 * ref_err.max(), floor), (what, err.max(), ref_err.max())
    for q in (99, 50):
        assert np.percentile(err, q) <= max(2 * np.percentile(ref_err, q), floor), (what, q)


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_bijector_alone(device, fast_math, tag):
    shift, scale = dev_t(UG[f"{tag}_shift"], device), dev_t(UG[f"{tag}_scale"], device)
    bound, eps = float(UG[f"{tag}_bound"]), float(UG[f"{tag}_eps"])
    t = GaussianizationTransform(shift, scale, bound=bound, eps=eps)
    with torch.no_grad():
        y, ladj = t.call_and_ladj(dev_t(UG[f"{tag}_x"], device))
        z = dev_t(UG[f"{tag}_z"], device)
        x = t.inv(z)
        back = t(x)
    check(cpu(y), UG[f"{tag}_y64"], UG[f"{tag}_y32"], f"{tag} y")
    check(cpu(ladj), UG[f"{tag}_ladj64"], UG[f"{tag}_ladj32"], f"{tag} ladj")
    check(cpu(x), UG[f"{tag}_xinv64"], UG[f"{tag}_xinv32"], f"{tag} inverse", atol=2 * interval(bound, eps))
    # beyond the range of f: the reference's edge of the search interval
    zr = UG[f"{tag}_z"]
    edge = bound - interval(bound, eps) / 2
    out = np.abs(UG[f"{tag}_xinv64"]) == edge  # the reference found no x: y is beyond the range of f
    assert out.any()
    np.testing.assert_allclose(cpu(x)[out], np.sign(zr[out]) * edge, rtol=0, atol=2 * interval(bound, eps))
    # round trip inside the range: x is resolved to its final interval, so f(x) to slope * interval
    inside = ~out & (np.abs(cpu(x)) < bound - 1.0)
    with torch.no_grad():
        slope = np.exp(cpu(t.call_and_ladj(x)[1]))[inside]
    err = np.abs(cpu(back) - zr)[inside]
    assert np.all(err <= slope * 2 * interval(bound, eps) + 1e-5 * np.maximum(np.abs(zr[inside]), 1.0))


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_bijector_gradients(device, tag):
    shift = dev_t(UG[f"{tag}_shift"], device, grad=True)
    scale = dev_t(UG[f"{tag}_scale"], device, grad=True)
    x = dev_t(UG[f"{tag}_x"], device, grad=True)
    t = GaussianizationTransform(shift, scale)
    y, ladj = t.call_and_ladj(x)
    ((dev_t(UG[f"{tag}_gy"], device) * y).sum() + (dev_t(UG[f"{tag}_gl"], device) * ladj).sum()).backward()
    for ours, key in ((x.grad, "gx"), (shift.grad, "gshift"), (scale.grad, "gscale")):
        ref = UG[f"{tag}_{key}"]
        err = np.abs(cpu(ours) - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err <= 5e-5, f"{tag} {key}: {err:.2e}"


def named_param_grads(flow):
    return {n: cpu(p.grad).reshape(-1) for n, p in flow.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("mode", ["lp", "tr"])
@pytest.mark.parametrize("name", ["gf53", "gf35_row", "gf6_uncond"])
def test_flow_gradients(device, name, mode):
    gg = load(f"grad_{name}")
    g = load(f"flow_{name}")
    rows = int(gg["rows"])
    c = g.get("c")
    if c is not None and c.ndim == 2:
        c = c[:rows]
    flow = build_gf(name).to(device)
    xt = dev_t(g["x"][:rows], device, grad=True)
    ct = None if c is None else dev_t(c, device, grad=True)
    if mode == "lp":
        (dev_t(gg["g"], device) * flow(ct).log_prob(xt)).sum().backward()
    else:
        z, ladj = flow(ct).transform.call_and_ladj(xt)
        ((dev_t(gg["gz"], device) * z).sum() + (dev_t(gg["gl"], device) * ladj).sum()).backward()
    pre = f"{mode}/"
    for ours, key in ((xt.grad, "gx"), (None if ct is None else ct.grad, "gc")):
        if ours is None:
            continue
        ref = gg[pre + key]
        bar = max(5e-5, 3 * float(gg.get(f"{pre}err32/{key}", 0.0)))
        err = np.abs(cpu(ours) - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err <= bar, f"{name} {mode} d/d{key}: {err:.2e} (bar {bar:.1e})"
    named = named_param_grads(flow)
    assert any(k.endswith(".A") for k in named), "no gradient reached the rotation generators"
    assert_param_grads(named, gg, pre, 5e-5, name, ref32_factor=3.0)


@pytest.mark.parametrize("mode", ["inv", "invlp"])
@pytest.mark.parametrize("name", ["gf53", "gf35_row"])
def test_inverse_direction_gradients(device, name, mode):
    """invgrad_gf6_uncond is not compared: its inverse is ill-conditioned on some rows (d/dz reaches 8.9e4 in fp64),
    and those rows dominate every summed parameter gradient."""
    gg = load(f"invgrad_{name}")
    c = load(f"flow_{name}").get("c")
    if c is not None and c.ndim == 2:
        c = c[: int(gg["rows"])]
    flow = build_gf(name).to(device)
    zt = dev_t(gg["z"], device, grad=True)
    ct = None if c is None else dev_t(c, device, grad=True)
    d = flow(ct)
    if mode == "inv":
        x = d.transform.inv(zt)
        loss = (dev_t(gg["w"], device) * x).sum()
    else:
        call, ctx = d._flow_call()
        x, lp = call.inverse(zt, ctx, with_log_prob=True)
        loss = (dev_t(gg["w"], device) * x).sum() + (dev_t(gg["wl"], device) * lp).sum()
    loss.backward()
    pre = f"{mode}/"
    for ours, key in ((zt.grad, "gx"), (None if ct is None else ct.grad, "gc")):
        if ours is None:
            continue
        ref = gg[pre + key]
        err = np.abs(cpu(ours) - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err <= 1e-4, f"{name} {mode} d/d{key}: {err:.2e}"
    assert_param_grads(named_param_grads(flow), gg, pre, 1e-4, name)


@pytest.mark.parametrize("name", ["gf53", "gf6_uncond"])
def test_log_prob_runs_engine_kernels_only(device, name):
    """Launches of one log_prob: per element-wise layer its conditioner's linear layers (exact-order fp32 GEMM,
    one kernel each) and one bijector kernel (the last one also adds the base density), one per rotation."""
    g = load(f"flow_{name}")
    flow = build_gf(name)
    expected = 0
    for t in flow.transform.transforms:
        if hasattr(t, "hyper"):
            t.hyper.gemm_mode = "fp32"
            expected += len(t.hyper._linears()) + 1
        elif hasattr(t, "phi"):
            expected += 1
        else:
            expected += 1  # rotation
    flow = flow.to(device)
    c = g.get("c")
    ct = None if c is None else dev_t(c, device)
    x = dev_t(g["x"], device)
    with torch.no_grad():
        flow(ct).log_prob(x)  # packs the layers
        torch.cuda.synchronize()
        n0 = E.lib().zk_launch_count()
        lp = flow(ct).log_prob(x)
        launches = E.lib().zk_launch_count() - n0
    assert launches == expected, (launches, expected)
    check(cpu(lp), g["log_prob64"], g["log_prob32"], f"{name} log_prob (fp32 GEMM)")


def test_accelerate_engine_built_gf(device):
    import zuko_b200 as zuko

    g = load("flow_gf53")
    acc = zuko.accelerate(build_gf("gf53").to(device))
    with torch.no_grad():
        lp = acc(dev_t(g["c"], device)).log_prob(dev_t(g["x"], device))
    check(cpu(lp), g["log_prob64"], g["log_prob32"], "accelerated gf53 log_prob")
