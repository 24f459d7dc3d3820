"""GPU tests of the Bernstein polynomial flow (BPF) and of its bijector against the reference's goldens
(tests/golden/make_golden_bpf.py).

Value bar: the one of tests/test_gpu_sospf.py, ``|ours - ref64| <= max(1e-5 * max(|ref64|, 1), 2 * |ref32 - ref64|)``,
with two final bisection intervals added to the absolute term of an inverse (check_inverse).  Gradients: 1e-4 of
the largest entry, on the rows whose fp32 t = (x + B) / 2B takes the same branch as the fp64 golden (at the branch
boundary the precisions disagree and the gradient jumps).  Both settings of ``zk_set_fast_math`` are held to the
same bars."""

import ctypes

import numpy as np
import pytest
import torch

import bpf_reference as R
from cases import assert_param_grads, load
from test_bpf_host import BPF_CASES, UNIT_TAGS, build_bpf, reference_of, same_branch
from test_gpu_gf import check, check_inverse, cpu, dev_t, fast_math, interval, named_param_grads  # noqa: F401
from zuko_b200 import _engine as E
from zuko_b200.lazy import Flow, LazyInverse
from zuko_b200.transforms import BoundedBernsteinTransform

pytestmark = pytest.mark.gpu
US = load("units_bpf")


def context(g, device, rows=None):
    c = g.get("c")
    if c is None:
        return None, None
    if c.ndim == 2 and rows is not None:
        c = c[:rows]
    return c, dev_t(c, device)


@pytest.mark.parametrize("name", list(BPF_CASES))
def test_flow_values(device, fast_math, name):
    g = load(f"flow_{name}")
    flow = build_bpf(name).to(device)
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
    u = dev_t(US[f"{tag}_u"], device, grad)
    return BoundedBernsteinTransform(u, bound=float(US[f"{tag}_bound"]), eps=float(US[f"{tag}_eps"])), u


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_bijector_alone(device, fast_math, tag):
    t, _ = unit_transform(tag, device)
    bound = float(US[f"{tag}_bound"])
    with torch.no_grad():
        y, ladj = t.call_and_ladj(dev_t(US[f"{tag}_x"], device))
        x = t.inv(dev_t(US[f"{tag}_z"], device))
    check(cpu(y), US[f"{tag}_y64"], US[f"{tag}_y32"], f"{tag} y")
    check(cpu(ladj), US[f"{tag}_ladj64"], US[f"{tag}_ladj32"], f"{tag} ladj")
    check_inverse(cpu(x), US[f"{tag}_xinv64"], US[f"{tag}_xinv32"], f"{tag} inverse")
    # the linear branches: ladj 0, and y beyond [-B, B] inverts with the reference's fp32 operations exactly
    xs = US[f"{tag}_x"]
    lin = np.abs(xs) >= bound + 1e-3
    assert lin.any()
    np.testing.assert_array_equal(cpu(ladj)[lin], 0.0)
    np.testing.assert_array_equal(cpu(y)[lin], US[f"{tag}_y32"][lin])
    out = np.abs(US[f"{tag}_z"]) >= bound
    np.testing.assert_array_equal(cpu(x)[out], US[f"{tag}_xinv32"][out])


def test_linear_branch_offset_and_jump(device):
    """x -+ 2B eps beyond the bounds (not the identity), and the jump of about 2B eps at them."""
    t = BoundedBernsteinTransform(dev_t(US["d16_u"][0], device))
    x = torch.tensor([-7.0, -5.0, 5.0, 7.0], device=device)
    with torch.no_grad():
        y = cpu(t(x))
    np.testing.assert_allclose(y - cpu(x), [-1.0014e-5, -1.0014e-5, 1.0014e-5, 1.0014e-5], rtol=0, atol=5e-7)
    y_in = torch.tensor([-5.0 + 5e-6, 5.0 - 5e-6], device=device)  # inside the jump: bisection lands at the bounds
    with torch.no_grad():
        xi = cpu(t.inv(y_in))
    assert np.all(np.abs(np.abs(xi) - 5.0) < 2e-5)


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_bijector_gradients(device, tag):
    x = dev_t(US[f"{tag}_x"], device, grad=True)
    t, u = unit_transform(tag, device, grad=True)
    y, ladj = t.call_and_ladj(x)
    ((dev_t(US[f"{tag}_gy"], device) * y).sum() + (dev_t(US[f"{tag}_gl"], device) * ladj).sum()).backward()
    ok = same_branch(US[f"{tag}_x"], float(US[f"{tag}_bound"]), float(US[f"{tag}_eps"]))
    gx = US[f"{tag}_gx"]
    err = np.abs(cpu(x.grad) - gx)[ok].max() / np.abs(gx).max()
    assert err <= 1e-4, f"{tag} gx: {err:.2e}"
    gu = US[f"{tag}_gu"]
    scale = np.abs(gu).max() or 1.0  # degree 0: the softmax of one entry has no gradient
    if bool(US[f"{tag}_batched"]):
        err = np.abs(cpu(u.grad) - gu)[ok].max() / scale
        assert err <= 1e-4, f"{tag} gu: {err:.2e}"
    elif ok.all():
        err = np.abs(cpu(u.grad) - gu).max() / scale
        assert err <= 1e-4, f"{tag} gu: {err:.2e}"


@pytest.mark.parametrize("mode", ["lp", "tr"])
@pytest.mark.parametrize("name", ["bpf53", "bpf35_row", "bpf6_uncond"])
def test_flow_gradients(device, name, mode):
    gg = load(f"grad_{name}")
    g = load(f"flow_{name}")
    rows = int(gg["rows"])
    c, _ = context(g, device, rows)
    flow = build_bpf(name).to(device)
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
        bar = max(1e-4, 3 * float(gg.get(f"{pre}err32/{key}", 0.0)))
        err = np.abs(cpu(ours) - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err <= bar, f"{name} {mode} d/d{key}: {err:.2e} (bar {bar:.1e})"
    assert_param_grads(named_param_grads(flow), gg, pre, 1e-4, name, ref32_factor=3.0)


@pytest.mark.parametrize("mode", ["inv", "invlp"])
@pytest.mark.parametrize("name", ["bpf53", "bpf35_row", "bpf6_uncond"])
def test_inverse_direction_gradients(device, name, mode):
    gg = load(f"invgrad_{name}")
    c, _ = context(load(f"flow_{name}"), device, int(gg["rows"]))
    flow = build_bpf(name).to(device)
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


def test_inverse_paths_and_geometry(device):
    """Degree 16 inverts with the dimension-sequential kernel (one sample per thread), other degrees with the
    sweeps; no BPF layer runs as the fused layer kernel."""
    for name, seq in (("bpf53", 1), ("bpf35_row", 1), ("bpf16_wide", 1), ("bpf6_uncond", 0), ("bpf42_b3", 0)):
        flow = build_bpf(name).to(device)
        for t in flow.transform.transforms:
            h = t._zk_layer()
            T, R_, smem = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_size_t(0)
            got = E.lib().zk_layer_inverse_geometry(h, ctypes.byref(T), ctypes.byref(R_), ctypes.byref(smem))
            assert got == seq, name
            if got:
                assert R_.value == 1 and T.value >= 32 and smem.value > 0, (name, T.value, R_.value)
            assert E.lib().zk_layer_sequential_inverse(h) == seq, name
            assert E.lib().zk_layer_fused_tile_rows(h) == 0, name
            assert E.lib().zk_layer_fused_info(h, (ctypes.c_double * 4)()) == 0, name


@pytest.mark.parametrize("name", ["bpf53", "bpf35_row", "bpf16_wide"])
def test_sequential_inverse_agrees_with_sweeps(device, fast_math, name):
    g = load(f"flow_{name}")
    flow = build_bpf(name).to(device)
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


@pytest.mark.parametrize("name", ["bpf53", "bpf35_row", "bpf16_wide", "bpf6_uncond"])
def test_rsample_log_prob_matches_log_prob(device, fast_math, name):
    """The log-density accumulated by the inverse equals log_prob of the returned sample, on the rows the fp64
    restatement round-trips itself."""
    g = load(f"flow_{name}")
    flow = build_bpf(name).to(device)
    c, ci = context(g, device, g["zin"].shape[0])
    zin = g["zin"]
    ref = reference_of(name, build_bpf(name))
    back, _ = ref.call_and_ladj(ref.inverse(zin, c), c)
    ok = np.abs(back - zin).max(-1) < 1e-5
    assert ok.mean() > 0.5
    with torch.no_grad():
        call, ctx = flow(ci)._flow_call()
        x, lp = call.inverse(dev_t(zin, device), ctx, with_log_prob=True)
        lp2 = flow(ci).log_prob(x)
    lp, lp2 = cpu(lp)[ok], cpu(lp2)[ok]
    assert np.max(np.abs(lp - lp2) / np.maximum(np.abs(lp2), 1.0)) < 1e-4


def test_lazy_inverse_member(device):
    """An inverted BPF layer inside one flow: log_prob through the sequential kernel's ladj equals the fp64
    restatement run the other way."""
    bpf = build_bpf("bpf53")
    ref = reference_of("bpf53", bpf)
    ref.layers = ref.layers[:1]
    flow = Flow([LazyInverse(bpf.transform.transforms[0])], bpf.base).to(device)
    g = load("flow_bpf53")
    x, c = g["x"][:64], g["c"][:64]
    z = ref.inverse(x, c)  # the inverted member maps x to f^-1(x)
    back, ladj = ref.call_and_ladj(z, c)
    ok = np.abs(back - x).max(-1) < 1e-5
    u = (z - ref.loc) / ref.scale
    lp_ref = -ladj + (-0.5 * u**2 - np.log(ref.scale) - 0.5 * np.log(2 * np.pi)).sum(-1)
    with torch.no_grad():
        lp = cpu(flow(dev_t(c, device)).log_prob(dev_t(x, device)))
    assert ok.mean() > 0.5
    assert np.max(np.abs(lp - lp_ref)[ok] / np.maximum(np.abs(lp_ref[ok]), 1.0)) < 1e-4


@pytest.mark.parametrize("degree", [16, 7])
def test_entry_points_strided_shared_and_empty(device, degree):
    """zk_bernstein_forward / inverse / backward on strided rows (pads untouched; NaN-padded parameter rows, phi_ld =
    D P + 5), a shared row (phi_ld = 0) and B = 0, against the fp64 restatement."""
    L, st = E.lib(), E.stream_ptr(device)
    B, D, P, bound, eps = 37, 3, degree + 1, 4.0, 1e-5
    g = torch.Generator().manual_seed(degree)
    x = torch.randn(B, D, generator=g) * 2.5
    u = torch.randn(B, D * P, generator=g)
    ldx, ldp = D + 3, D * P + 5
    xd = torch.full((B, ldx), float("nan"), device=device)
    xd[:, :D] = x.to(device)
    ud = torch.full((B, ldp), float("nan"), device=device)
    ud[:, : D * P] = u.to(device)
    yd = torch.full((B, ldx), float("nan"), device=device)
    ladj = torch.zeros(B, device=device)
    E.check(L.zk_bernstein_forward(xd.data_ptr(), ldx, ud.data_ptr(), ldp, B, D, degree, bound, eps, yd.data_ptr(), ldx,
                                   ladj.data_ptr(), 0, st))  # fmt: skip
    y64, l64 = R.forward(x.double().numpy(), u.double().numpy().reshape(B, D, P), bound, eps)
    np.testing.assert_allclose(cpu(yd[:, :D]), y64, rtol=0, atol=2e-5 * bound)
    np.testing.assert_allclose(cpu(ladj), l64.sum(-1), rtol=0, atol=1e-4)
    assert torch.isnan(yd[:, D:]).all()
    xi = torch.full((B, ldx), float("nan"), device=device)
    E.check(L.zk_bernstein_inverse(yd.data_ptr(), ldx, ud.data_ptr(), ldp, B, D, degree, bound, eps, xi.data_ptr(), ldx, st))
    np.testing.assert_allclose(cpu(xi[:, :D]), x.numpy(), rtol=0, atol=1e-4)
    assert torch.isnan(xi[:, D:]).all()
    # shared row
    u0 = u[0].to(device).contiguous()
    ys = torch.empty(B, D, device=device)
    E.check(L.zk_bernstein_forward(xd.data_ptr(), ldx, u0.data_ptr(), 0, B, D, degree, bound, eps, ys.data_ptr(), D, None, 0, st))
    ys64, _ = R.forward(x.double().numpy(), u[0].double().numpy().reshape(D, P), bound, eps)
    np.testing.assert_allclose(cpu(ys), ys64, rtol=0, atol=2e-5 * bound)
    # backward: per-sample and shared, against the restatement
    gy = torch.randn(B, D, generator=g)
    gl = torch.randn(B, generator=g)
    gyd, gld = gy.to(device), gl.to(device)
    gx = torch.empty(B, D, device=device)
    gphi = torch.zeros(B, D * P, device=device)
    E.check(L.zk_bernstein_backward(xd.data_ptr(), ldx, ud.data_ptr(), ldp, B, D, degree, bound, eps, gyd.data_ptr(), D,
                                    gld.data_ptr(), gx.data_ptr(), D, gphi.data_ptr(), None, 0, st))  # fmt: skip
    rgx, rgu = R.grad(x.double().numpy(), u.double().numpy().reshape(B, D, P), gy.double().numpy(),
                      np.broadcast_to(gl.double().numpy()[:, None], (B, D)), bound, eps)  # fmt: skip
    assert np.abs(cpu(gx) - rgx).max() <= 1e-4 * np.abs(rgx).max()
    assert np.abs(cpu(gphi).reshape(B, D, P) - rgu).max() <= 1e-4 * np.abs(rgu).max()
    need = L.zk_univariate_backward_workspace_bytes(B, D, P, 0)
    ws = torch.empty(max(need, 1) // 4 + 1, device=device)
    gsh = torch.zeros(D * P, device=device)
    E.check(L.zk_bernstein_backward(xd.data_ptr(), ldx, u0.data_ptr(), 0, B, D, degree, bound, eps, gyd.data_ptr(), D,
                                    gld.data_ptr(), gx.data_ptr(), D, gsh.data_ptr(), ws.data_ptr(), ws.numel() * 4, st))  # fmt: skip
    _, rgs = R.grad(x.double().numpy(), u[0].double().numpy().reshape(D, P), gy.double().numpy(),
                    np.broadcast_to(gl.double().numpy()[:, None], (B, D)), bound, eps)  # fmt: skip
    rgs = rgs.sum(0).reshape(-1)
    assert np.abs(cpu(gsh) - rgs).max() <= 1e-4 * np.abs(rgs).max()
    # B = 0 writes nothing
    E.check(L.zk_bernstein_forward(xd.data_ptr(), ldx, ud.data_ptr(), ldp, 0, D, degree, bound, eps, yd.data_ptr(), ldx, None, 0, st))
    E.check(L.zk_bernstein_inverse(yd.data_ptr(), ldx, ud.data_ptr(), ldp, 0, D, degree, bound, eps, xi.data_ptr(), ldx, st))
    torch.cuda.synchronize(device)
    # out-of-range arguments are refused
    assert L.zk_bernstein_forward(xd.data_ptr(), ldx, ud.data_ptr(), ldp, B, D, 60, bound, eps, yd.data_ptr(), ldx, None, 0, st) != 0


def test_accelerate_bpf(device):
    """accelerate() on a flow with the reference's module names and state dict."""
    import zuko_b200 as zuko

    g = load("flow_bpf53")
    src = build_bpf("bpf53").to(device)
    sd = {k: torch.from_numpy(v).to(device) for k, v in g.items() if k.startswith("sd/")}
    src.load_state_dict({k[3:]: v for k, v in sd.items()})
    acc = zuko.accelerate(src)
    assert list(acc.state_dict()) == [str(k) for k in g["sd_keys"]]
    with torch.no_grad():
        lp = acc(dev_t(g["c"], device)).log_prob(dev_t(g["x"], device))
    check(cpu(lp), g["log_prob64"], g["log_prob32"], "accelerated bpf53 log_prob")
