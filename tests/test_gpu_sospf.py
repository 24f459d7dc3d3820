"""GPU tests of the sum-of-squares polynomial flow (SOSPF) and of its bijector against the reference's goldens
(tests/golden/make_golden_sospf.py).

Value bar: the one of tests/test_gpu_gf.py, ``|ours - ref64| <= max(1e-5 * max(|ref64|, 1), 2 * |ref32 - ref64|)``,
with two final bisection intervals added to the absolute term of an inverse.  A flow's inverse chains bisections
and soft clips; the inverse of a soft clip can put a value far beyond +-10, where the next bisection saturates, and
the fp32 error of a layer's input is amplified where g is small.  So, as for GF, at most 1% of the inverse elements
may miss the per-element bar, provided the engine is no less accurate than the reference's own fp32 inverse in
distribution.  Both settings of ``zk_set_fast_math`` are held to the same bar."""

import ctypes

import numpy as np
import pytest
import torch

import sospf_reference as R
from cases import assert_param_grads, load
from test_gpu_gf import check, check_inverse, cpu, dev_t, fast_math, interval, named_param_grads  # noqa: F401
from test_sospf_host import SOSPF_CASES, UNIT_TAGS, build_sospf, reference_of
from zuko_b200 import _engine as E
from zuko_b200.transforms import ShiftedSOSPTransform, SOSPolynomialTransform

pytestmark = pytest.mark.gpu
US = load("units_sospf")


def context(g, device, rows=None):
    c = g.get("c")
    if c is None:
        return None, None
    if c.ndim == 2 and rows is not None:
        c = c[:rows]
    return c, dev_t(c, device)


@pytest.mark.parametrize("name", list(SOSPF_CASES))
def test_flow_values(device, fast_math, name):
    g = load(f"flow_{name}")
    flow = build_sospf(name).to(device)
    _, ct = context(g, device)
    _, ci = context(g, device, g["zin"].shape[0])
    with torch.no_grad():
        lp = flow(ct).log_prob(dev_t(g["x"], device))
        z, ladj = flow(ct).transform.call_and_ladj(dev_t(g["x"], device))
        xi = flow(ci).transform.inv(dev_t(g["zin"], device))
    check(cpu(lp), g["log_prob64"], g["log_prob32"], f"{name} log_prob")
    check(cpu(z), g["z64"], g["z32"], f"{name} z")
    check(cpu(ladj), g["ladj64"], g["ladj32"], f"{name} ladj")
    check_inverse(cpu(xi), g["xinv64"], g["xinv32"], f"{name} inverse")


def unit_transform(tag, device, grad=False):
    a = dev_t(US[f"{tag}_a"], device, grad)
    if bool(US[f"{tag}_shifted"]):
        const = dev_t(US[f"{tag}_const"], device, grad)
        return ShiftedSOSPTransform(a, const), a, const
    return SOSPolynomialTransform(a), a, None


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_bijector_alone(device, fast_math, tag):
    t, _, _ = unit_transform(tag, device)
    with torch.no_grad():
        y, ladj = t.call_and_ladj(dev_t(US[f"{tag}_x"], device))
        x = t.inv(dev_t(US[f"{tag}_z"], device))
    check(cpu(y), US[f"{tag}_y64"], US[f"{tag}_y32"], f"{tag} y")
    check(cpu(ladj), US[f"{tag}_ladj64"], US[f"{tag}_ladj32"], f"{tag} ladj")
    check_inverse(cpu(x), US[f"{tag}_xinv64"], US[f"{tag}_xinv32"], f"{tag} inverse")
    # beyond the range of f: the reference's edge of the search interval
    edge = 10.0 - interval() / 2
    out = np.abs(US[f"{tag}_xinv64"]) == edge
    assert out.any()
    np.testing.assert_allclose(cpu(x)[out], np.sign(US[f"{tag}_xinv64"][out]) * edge, rtol=0, atol=2 * interval())


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_bijector_gradients(device, tag):
    x = dev_t(US[f"{tag}_x"], device, grad=True)
    t, a, const = unit_transform(tag, device, grad=True)
    y, ladj = t.call_and_ladj(x)
    ((dev_t(US[f"{tag}_gy"], device) * y).sum() + (dev_t(US[f"{tag}_gl"], device) * ladj).sum()).backward()
    for ours, key in ((x.grad, "gx"), (a.grad, "ga"), (None if const is None else const.grad, "gconst")):
        if ours is None:
            continue
        ref = US[f"{tag}_{key}"]
        err = np.abs(cpu(ours) - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err <= 5e-5, f"{tag} {key}: {err:.2e}"


@pytest.mark.parametrize("mode", ["lp", "tr"])
@pytest.mark.parametrize("name", ["sospf53", "sospf35_row", "sospf6_uncond"])
def test_flow_gradients(device, name, mode):
    gg = load(f"grad_{name}")
    g = load(f"flow_{name}")
    rows = int(gg["rows"])
    c, _ = context(g, device, rows)
    flow = build_sospf(name).to(device)
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
    assert_param_grads(named_param_grads(flow), gg, pre, 5e-5, name, ref32_factor=3.0)


@pytest.mark.parametrize("mode", ["inv", "invlp"])
@pytest.mark.parametrize("name", ["sospf53", "sospf35_row"])
def test_inverse_direction_gradients(device, name, mode):
    gg = load(f"invgrad_{name}")
    c, _ = context(load(f"flow_{name}"), device, int(gg["rows"]))
    flow = build_sospf(name).to(device)
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


def test_inverse_paths(device):
    """The default shape (3 polynomials of degree 4) inverts with the dimension-sequential kernel, other shapes
    with the sweeps; no SOSP layer runs as the fused layer kernel."""
    for name, seq in (("sospf53", 1), ("sospf35_row", 1), ("sospf6_uncond", 0)):
        flow = build_sospf(name).to(device)
        for t in flow.transform.transforms[::2]:
            h = t._zk_layer()
            assert E.lib().zk_layer_sequential_inverse(h) == seq, name
            assert E.lib().zk_layer_fused_tile_rows(h) == 0, name
            assert E.lib().zk_layer_fused_info(h, (ctypes.c_double * 4)()) == 0, name


@pytest.mark.parametrize("name", ["sospf53", "sospf35_row", "sospf16_wide"])
def test_sequential_inverse_agrees_with_sweeps(device, fast_math, name):
    g = load(f"flow_{name}")
    flow = build_sospf(name).to(device)
    _, ci = context(g, device, g["zin"].shape[0])
    z = dev_t(g["zin"], device)
    with torch.no_grad():
        seq = cpu(flow(ci).transform.inv(z))
        prev = E.lib().zk_set_fused_layers(0)
        try:
            sweep = cpu(flow(ci).transform.inv(z))
        finally:
            E.lib().zk_set_fused_layers(prev)
    diff = np.abs(seq - sweep)
    far = diff > 1e-4 * np.maximum(np.abs(sweep), 1.0) + 2 * interval()
    assert far.mean() <= 0.01, (name, int(far.sum()), float(diff.max()))
    assert np.median(diff) <= 2 * interval()


@pytest.mark.parametrize("name", ["sospf53", "sospf35_row", "sospf16_wide"])
def test_rsample_log_prob_matches_log_prob(device, fast_math, name):
    """The log-density fused into the sequential inverse equals log_prob of the returned sample, on the rows the
    fp64 restatement round-trips itself (elsewhere a bisection saturates and the sample is not the preimage)."""
    g = load(f"flow_{name}")
    flow = build_sospf(name).to(device)
    c, ci = context(g, device, g["zin"].shape[0])
    zin = g["zin"]
    ref = reference_of(name, build_sospf(name))
    back, _ = ref.call_and_ladj(ref.inverse(zin, c), c)
    ok = np.abs(back - zin).max(-1) < 1e-6
    assert ok.mean() > 0.5
    with torch.no_grad():
        call, ctx = flow(ci)._flow_call()
        x, lp = call.inverse(dev_t(zin, device), ctx, with_log_prob=True)
        lp2 = flow(ci).log_prob(x)
    lp, lp2 = cpu(lp)[ok], cpu(lp2)[ok]
    assert np.max(np.abs(lp - lp2) / np.maximum(np.abs(lp2), 1.0)) < 1e-4


def test_accelerate_sospf(device):
    """accelerate() on a flow with the reference's module names and state dict (softclip insertions included)."""
    import zuko_b200 as zuko

    g = load("flow_sospf53")
    src = build_sospf("sospf53").to(device)
    sd = {k: torch.from_numpy(v).to(device) for k, v in g.items() if k.startswith("sd/")}
    src.load_state_dict({k[3:]: v for k, v in sd.items()})
    acc = zuko.accelerate(src)
    assert list(acc.state_dict()) == [str(k) for k in g["sd_keys"]]
    with torch.no_grad():
        lp = acc(dev_t(g["c"], device)).log_prob(dev_t(g["x"], device))
    check(cpu(lp), g["log_prob64"], g["log_prob32"], "accelerated sospf53 log_prob")
