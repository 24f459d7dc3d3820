"""GPU tests of the CNF backward (zk_cnf_backward: the adaptive checkpoint adjoint of zuko/utils.py:556-593).
Every gradient is compared with the fp64 restatement (tests/cnf_adjoint_reference.py) replaying the engine's
OWN forward step log, at 1e-4 of each tensor's largest entry; on the default cases whose trial sequence matches
the reference's fp32 run, also with the reference's fp32 gradients (tests/golden/make_golden_cnf_grad.py)."""

import ctypes

import numpy as np
import pytest
import torch

import cnf_adjoint_reference as A
import cnf_reference as R
from cases import load
from test_cnf_grad_host import GOPS, back_plan, gap, golden_grads, relmax
from test_cnf_host import CASES, DEFAULT, field_of
from test_gpu_cnf import Engine
from zuko_b200 import _engine as E
from zuko_b200.accel import accelerate
from zuko_b200.flows import CNF

pytestmark = pytest.mark.gpu
BAR = 1e-4
# ReLU / LeakyReLU: f is piecewise linear, so its Jacobian jumps where a pre-activation changes sign, and an fp32
# trajectory crosses a kink at a slightly different point than the fp64 replay of its steps: fp32-sized input
# noise moves the fp64 gradients themselves by up to 1.5e-3 (test_cnf_grad_host.py::
# test_piecewise_linear_gradients_jump_under_fp32_noise), against ~1e-6 for the smooth activations
KINK_BAR = 5e-3
WORST: dict = {}


def backward(eng, x, c, lg, counts, trace, eps=None, gy=None, gl=None, ldc=None, ws_bytes=None, grads_init=None,
             direction=+1, x_view=None, gy_view=None, gx_view=None):  # fmt: skip
    """One zk_cnf_backward call: (gx, gc, [gW], [gb])."""
    dev = eng.dev
    lib = E.lib()
    h = eng.t._cnf_handle()
    x = x_view if x_view is not None else torch.as_tensor(x, dtype=torch.float32, device=dev)
    B, D = x.shape[0], eng.D
    cc = None if c is None else torch.as_tensor(c, dtype=torch.float32, device=dev)
    if cc is not None and ldc is None:
        ldc = cc.stride(0) if cc.dim() == 2 else 0
    ee = None if eps is None else torch.as_tensor(eps, dtype=torch.float32, device=dev)
    gyt = gy_view if gy_view is not None else (None if gy is None else torch.as_tensor(gy, dtype=torch.float32, device=dev))
    glt = None if gl is None else torch.as_tensor(gl, dtype=torch.float32, device=dev)
    gx = gx_view if gx_view is not None else torch.empty(B, D, device=dev)
    gc = None
    if cc is not None:
        gc = torch.full((B, eng.C) if ldc else (eng.C,), float("nan"), device=dev)
    lins = eng.t.ode._linears()
    if grads_init is None:
        gW = [torch.zeros_like(m.weight) for m in lins]
        gb = [torch.zeros_like(m.bias) for m in lins]
    else:
        gW, gb = [g.clone() for g in grads_init[0]], [g.clone() for g in grads_init[1]]
    wp = (ctypes.c_void_p * len(lins))(*[g.data_ptr() for g in gW])
    bp = (ctypes.c_void_p * len(lins))(*[g.data_ptr() for g in gb])
    lg_ = E.LayerGrads()
    lg_.grad_weight, lg_.grad_bias = wp, bp
    trials, acc = counts
    log = torch.as_tensor(np.asarray(lg, np.float32).reshape(-1, 4), device=dev)
    need = lib.zk_cnf_backward_workspace_bytes(h, B, trace, acc) if ws_bytes is None else ws_bytes
    ws = torch.empty(max(need, 256), dtype=torch.uint8, device=dev)
    E.check(lib.zk_cnf_backward(
        h, x.data_ptr(), x.stride(0), None if cc is None else cc.data_ptr(), ldc or 0, B, log.data_ptr(), trials, acc,
        trace, None if ee is None else ee.data_ptr(), 0 if ee is None else ee.stride(0),
        None if gyt is None else gyt.data_ptr(), 0 if gyt is None else gyt.stride(0), None if glt is None else glt.data_ptr(),
        gx.data_ptr(), gx.stride(0), None if gc is None else gc.data_ptr(), eng.C, ctypes.byref(lg_), ws.data_ptr(), need,
        E.stream_ptr(dev)))  # fmt: skip
    torch.cuda.synchronize()
    return gx, gc, gW, gb


def as_np(t):
    return None if t is None else t.double().cpu().numpy()


def check_against_restatement(eng, field, inp, c, lg, trace, eps, gy, gl, out, tag, bar=BAR):
    ref = A.adjoint(field, inp, c, lg, trace, eps, gy, gl)
    gx, gc, gW, gb = out
    errs = {"x": relmax(as_np(gx), ref["x"])}
    if c is not None:
        rc = ref["c"] if np.ndim(c) == 2 else ref["c"].sum(0)
        errs["c"] = relmax(as_np(gc), rc)
    for i in range(len(gW)):
        errs[f"W{i}"] = relmax(as_np(gW[i]), ref["W"][i])
        errs[f"b{i}"] = relmax(as_np(gb[i]), ref["b"][i])
    worst = max(errs.values())
    WORST[tag] = worst
    assert worst <= bar, (tag, errs)
    return ref


@pytest.fixture(scope="module")
def engines(device):
    out = {}
    for name in CASES:
        g = load(f"cnfgrad_{name}")
        torch.manual_seed(0)
        flow = CASES[name]().eval()
        flow.load_state_dict({k[3:]: torch.as_tensor(v) for k, v in g.items() if k.startswith("sd/")})
        out[name] = (Engine(flow, device), g)
    return out


def op_inputs(g, op, y=None):
    """(trace, input, direction, eps, gy, gl) of a golden op; lp's gy needs the forward's y."""
    trace, key, direction = GOPS[op]
    eps = g["hut_eps_32"] if op == "hut" else None
    if op == "lp":
        w = g["w"].astype(np.float64)
        return trace, g[key], direction, eps, None if y is None else -w[:, None] * y, w
    return trace, g[key], direction, eps, g["gy"], (g["gl"] if trace else None)


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("op", list(GOPS))
def test_against_restatement_of_own_log_and_reference(engines, name, op):
    eng, g = engines[name]
    c = g.get("c")
    trace, inp, direction, eps, _, _ = op_inputs(g, op)
    y, ladj, counts, lg = eng.run(inp, c, trace, direction, eps)
    trace, inp, direction, eps, gy, gl = op_inputs(g, op, y.double().cpu().numpy())
    out = backward(eng, inp, c, lg, counts, trace, eps, gy, gl)
    check_against_restatement(eng, field_of(g), inp.astype(np.float64), c, lg, trace, eps, gy, gl, out, f"{name}-{op}")
    gold = g[f"log_{op}_32"]
    if name not in DEFAULT or counts != (len(gold), int(gold[:, 3].sum())) or op == "hut":
        return
    # the reference's own fp32 gradients, at twice the fp32-fp64 gap of its gradient computation (the largest
    # over the op's tensors: one adjoint produces them all)
    gx, gc, gW, gb = out
    ours = {"in0": as_np(gx), "in1": as_np(gc)}
    for i in range(len(gW)):
        ours[f"ode.{2 * i}.weight"] = as_np(gW[i])
        ours[f"ode.{2 * i}.bias"] = as_np(gb[i])
    gold = golden_grads(g, op, "32")
    bar = 2 * max(max(gap(g, op, k) for k in gold), BAR)
    for k, v in gold.items():
        if ours.get(k) is not None:
            assert relmax(ours[k], v) <= bar, (k, relmax(ours[k], v), bar)


def _flow(device, D, C, seed=0, scale=1.0, **kw):
    torch.manual_seed(seed)
    flow = CNF(D, C, **kw).eval()
    with torch.no_grad():
        for p in flow.parameters():
            p.mul_(scale)
    return Engine(flow, device)


def _field(eng):
    sd = {k: v.detach().double().cpu().numpy() for k, v in eng.flow.state_dict().items()}
    act = type(eng.t.ode[1]).__name__ if len(eng.t.ode) > 1 else "ReLU"
    return R.Field.from_state_dict(sd, eng.D, eng.C, act)


def _random_case(eng, B, seed=3, trace=R.TRACE_EXACT, direction=+1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, eng.D, generator=g).numpy()
    c = torch.randn(B, eng.C, generator=g).numpy() if eng.C else None
    eps = torch.randn(B, eng.D, generator=g).numpy() if trace == R.TRACE_HUTCHINSON else None
    gy = torch.randn(B, eng.D, generator=g).numpy()
    gl = torch.randn(B, generator=g).numpy() if trace else None
    return x, c, eps, gy, gl


def _run_and_check(eng, B=64, trace=R.TRACE_EXACT, direction=+1, tag="", bar=BAR, **kw):
    x, c, eps, gy, gl = _random_case(eng, B, trace=trace)
    y, ladj, counts, lg = eng.run(x, c, trace, direction, eps)
    out = backward(eng, x, c, lg, counts, trace, eps, gy, gl, **kw)
    check_against_restatement(eng, _field(eng), x.astype(np.float64), c, lg, trace, eps, gy, gl, out, tag, bar)
    return out


@pytest.mark.parametrize("hidden", [[1], [7], [8, 9], [65], []])
def test_hidden_widths_and_one_layer(device, hidden):
    eng = _flow(device, 3, 2, hidden_features=hidden)
    for trace in (R.TRACE_EXACT, R.TRACE_HUTCHINSON, R.TRACE_NONE):
        gx, gc, gW, gb = _run_and_check(eng, 40, trace, tag=f"hidden{hidden}-{trace}")
    if not hidden:  # tau = tr(W0[:, x]) does not depend on x; its weight gradient is diagonal on the x columns
        x, c, eps, gy, gl = _random_case(eng, 40)
        y, ladj, counts, lg = eng.run(x, c, R.TRACE_EXACT)
        _, _, gW0, _ = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, np.zeros_like(gy), gl)
        F2 = 2 * eng.t.freqs.numel()
        blk = as_np(gW0[0])[:, F2 : F2 + 3]
        np.testing.assert_allclose(blk - np.diag(np.diag(blk)), 0.0, atol=1e-6)
        np.testing.assert_allclose(np.diag(blk), np.sum(gl), rtol=1e-5)


@pytest.mark.parametrize("act", ["ReLU", "ELU", "Tanh", "SiLU", "GELU", "LeakyReLU", "Softplus", "Sigmoid"])
@pytest.mark.parametrize("scale", [1.0, 3.0])
def test_activations_and_weights_x3(device, act, scale):
    eng = _flow(device, 3, 2, scale=scale, activation=getattr(torch.nn, act))
    bar = KINK_BAR if act in ("ReLU", "LeakyReLU") else BAR
    _run_and_check(eng, 48, R.TRACE_EXACT, tag=f"{act}-x{scale}", bar=bar)
    _run_and_check(eng, 48, R.TRACE_HUTCHINSON, direction=-1, tag=f"{act}-x{scale}-hut", bar=bar)


def test_chunks_accumulation_repeat_and_batch_edges(device):
    eng = _flow(device, 4, 3)
    B = 300  # not a multiple of any thread count
    x, c, eps, gy, gl = _random_case(eng, B)
    y, ladj, counts, lg = eng.run(x, c, R.TRACE_EXACT)
    one = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl)
    again = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl)
    for a, b in zip([one[0], one[1], *one[2], *one[3]], [again[0], again[1], *again[2], *again[3]], strict=True):
        assert torch.equal(a, b)
    h = eng.t._cnf_handle()
    small = E.lib().zk_cnf_backward_min_workspace_bytes(h, R.TRACE_EXACT, counts[1]) + 40 * (
        E.lib().zk_cnf_backward_workspace_bytes(h, 2, R.TRACE_EXACT, counts[1])
        - E.lib().zk_cnf_backward_workspace_bytes(h, 1, R.TRACE_EXACT, counts[1]))
    rows, nt = ctypes.c_int64(), ctypes.c_int()
    E.check(E.lib().zk_cnf_backward_plan(h, B, R.TRACE_EXACT, counts[1], small, None, ctypes.byref(nt), ctypes.byref(rows),
                                         None))  # fmt: skip
    assert nt.value < rows.value < B and rows.value % nt.value == 0
    # several chunks give the one chunk's bits: every row meets the same CTA, in the same order
    chunked = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl, ws_bytes=small)
    for a, b in zip([one[0], one[1], *one[2], *one[3]], [chunked[0], chunked[1], *chunked[2], *chunked[3]], strict=True):
        assert torch.equal(a, b)
    c1 = c[:1][0]
    _, _, counts1, lg1 = eng.run(x, c1, R.TRACE_EXACT, ldc=0)
    whole = backward(eng, x, c1, lg1, counts1, R.TRACE_EXACT, None, gy, gl, ldc=0)
    parts = backward(eng, x, c1, lg1, counts1, R.TRACE_EXACT, None, gy, gl, ldc=0, ws_bytes=small)
    assert torch.equal(whole[1], parts[1]) and torch.equal(whole[0], parts[0])
    pre = ([torch.randn_like(w) for w in one[2]], [torch.randn_like(b) for b in one[3]])
    acc = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl, grads_init=pre)
    for a, p, o in zip(acc[2] + acc[3], pre[0] + pre[1], one[2] + one[3], strict=True):
        torch.testing.assert_close(a, p + o, rtol=0, atol=1e-5)
    # B = 0: nothing runs, the summed context row is overwritten with 0 (grad_ladj must still be given: a NULL
    # one means "no trace", as in zk_cnf_integrate)
    gx0, gc0, _, _ = backward(eng, x[:0], c[:1], lg, counts, R.TRACE_EXACT, None, None, gl, ldc=0)
    assert gx0.shape == (0, 4) and torch.equal(gc0, torch.zeros(3, device=device))


def test_broadcast_context_and_padded_strides(device):
    eng = _flow(device, 3, 2)
    B = 70
    x, c, eps, gy, gl = _random_case(eng, B)
    c1 = c[:1].copy()
    y, ladj, counts, lg = eng.run(x, c1[0], R.TRACE_EXACT, ldc=0)
    out = backward(eng, x, c1[0], lg, counts, R.TRACE_EXACT, None, gy, gl, ldc=0)
    check_against_restatement(eng, _field(eng), x.astype(np.float64), c1[0], lg, R.TRACE_EXACT, None, gy, gl, out, "bcast")
    # padded x / grad_y / grad_x rows give the same numbers
    dev = device
    xp = torch.zeros(B, 7, device=dev)
    xp[:, :3] = torch.as_tensor(x)
    gyp = torch.zeros(B, 5, device=dev)
    gyp[:, :3] = torch.as_tensor(gy)
    gxp = torch.full((B, 6), 7.0, device=dev)
    padded = backward(eng, None, c1[0], lg, counts, R.TRACE_EXACT, None, None, gl, ldc=0, x_view=xp[:, :3],
                      gy_view=gyp[:, :3], gx_view=gxp[:, :3])  # fmt: skip
    assert torch.equal(padded[0], out[0]) and torch.all(gxp[:, 3:] == 7.0)
    for a, b in zip(padded[2] + padded[3], out[2] + out[3], strict=True):
        assert torch.equal(a, b)


def test_equal_times_is_the_identity(device):
    eng = _flow(device, 3, 2)
    x, c, eps, gy, gl = _random_case(eng, 20)
    tt = torch.tensor([0.5, 0.5], device=device)
    y, ladj, counts, lg = eng.run(x, c, R.TRACE_EXACT, times=tt)
    assert counts == (0, 0)
    gx, gc, gW, gb = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl)
    assert torch.equal(gx, torch.as_tensor(gy, dtype=torch.float32, device=device))
    assert torch.all(gc == 0) and all(torch.all(g == 0) for g in gW + gb)


def test_plan_against_restatement(device):
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    for D, C, hidden, F in [(16, 8, [64, 64, 64], 3), (3, 5, [64, 64, 64], 3), (2, 0, [16], 0), (64, 0, [128, 128], 3),
                            (5, 0, [32, 32, 32], 3), (16, 8, [256, 256], 3)]:  # fmt: skip
        torch.manual_seed(0)
        eng = Engine(CNF(D, C, freqs=F, hidden_features=hidden).eval(), device)
        h = eng.t._cnf_handle()
        for trace in (R.TRACE_NONE, R.TRACE_EXACT):
            want = back_plan(D, C, F, [D + C + 2 * F, *hidden, D], trace)
            ctas, nt, rows, smem = ctypes.c_int(), ctypes.c_int(), ctypes.c_int64(), ctypes.c_size_t()
            st = E.lib().zk_cnf_backward_plan(h, 1000, trace, 10, 1 << 40, ctypes.byref(ctas), ctypes.byref(nt),
                                              ctypes.byref(rows), ctypes.byref(smem))  # fmt: skip
            if want is None:
                assert st == E.ZK_EUNSUPPORTED
                continue
            assert st == 0 and (nt.value, smem.value) == want and rows.value == 1000
            assert ctas.value % sms == 0 and ctas.value >= sms


def test_refusals(device):
    eng = _flow(device, 3, 2)
    lib = E.lib()
    h = eng.t._cnf_handle()
    x, c, eps, gy, gl = _random_case(eng, 16)
    y, ladj, counts, lg = eng.run(x, c, R.TRACE_EXACT)
    with pytest.raises(ValueError, match="grad_ladj"):
        backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, None)
    with pytest.raises(ValueError, match="grad_ladj"):
        backward(eng, x, c, lg, counts, R.TRACE_NONE, None, gy, gl)
    with pytest.raises(ValueError, match="eps"):
        backward(eng, x, c, lg, counts, R.TRACE_HUTCHINSON, None, gy, gl)
    with pytest.raises(ValueError, match="eps"):
        backward(eng, x, c, lg, counts, R.TRACE_EXACT, eps if eps is not None else x, gy, gl)
    with pytest.raises(ValueError, match="accepted"):
        backward(eng, x, c, lg, (counts[0], counts[0] + 1), R.TRACE_EXACT, None, gy, gl)
    with pytest.raises(ValueError, match="workspace"):
        backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl, ws_bytes=256)
    with pytest.raises(ValueError, match="context"):
        backward(eng, x, None, lg, counts, R.TRACE_EXACT, None, gy, gl)
    with pytest.raises(ValueError, match="unknown trace"):
        backward(eng, x, c, lg, counts, 3, None, gy, gl)
    assert lib.zk_cnf_backward_plan(None, 1, 1, 1, 1 << 30, None, None, None, None) == E.ZK_EINVAL
    assert lib.zk_cnf_backward_plan(h, -1, 1, 1, 1 << 30, None, None, None, None) == E.ZK_EINVAL
    assert lib.zk_cnf_backward_plan(h, 1, 1, -1, 1 << 30, None, None, None, None) == E.ZK_EINVAL
    assert lib.zk_cnf_backward_workspace_bytes(None, 1, 1, 1) == 0
    # a backward state beyond shared memory is refused, and the Python layer refuses it at the forward call
    torch.manual_seed(0)
    big = CNF(16, 8, hidden_features=[512, 512], adjoint=True).to(device)
    assert lib.zk_cnf_backward_plan(big.transform._cnf_handle(), 1, 1, 1, 1 << 30, None, None, None, None) == E.ZK_EUNSUPPORTED
    with pytest.raises(NotImplementedError, match="backward state"):
        big(torch.randn(8, 8, device=device)).log_prob(torch.randn(8, 16, device=device))


# --------------------------------------------------------------------------- public API


def _golden_flow(device, name):
    g = load(f"cnfgrad_{name}")
    torch.manual_seed(0)
    flow = CASES[name]()
    flow.load_state_dict({k[3:]: torch.as_tensor(v) for k, v in g.items() if k.startswith("sd/")})
    return flow.to(device), g


def test_training_log_prob_fills_every_parameter_and_context(device):
    flow, g = _golden_flow(device, "cnf35")
    flow.transform.adjoint = True
    flow.train()
    x = torch.as_tensor(g["x"], device=device).requires_grad_()
    c = torch.as_tensor(g["c"], device=device).requires_grad_()
    w = torch.as_tensor(g["w"], device=device)
    (flow(c).log_prob(x) * w).sum().backward()
    gold = golden_grads(g, "lp", "32")
    assert relmax(as_np(x.grad), gold["in0"]) <= 2 * max(gap(g, "lp", "in0"), BAR)
    assert relmax(as_np(c.grad), gold["in1"]) <= 2 * max(gap(g, "lp", "in1"), BAR)
    for k, p in flow.transform.named_parameters():
        assert p.grad is not None, k
        assert relmax(as_np(p.grad), gold[k]) <= 2 * max(gap(g, "lp", k), BAR), k
    # -mean log_prob, the usual loss, with a broadcast context of shape (C,)
    flow.zero_grad()
    cb = torch.as_tensor(g["c"][0], device=device).requires_grad_()
    (flow(cb).log_prob(x.detach()) * w).sum().backward()
    gold = golden_grads(g, "bcast", "32")
    assert cb.grad.shape == (5,)
    assert relmax(as_np(cb.grad), gold["in1"]) <= 2 * max(gap(g, "bcast", "in1"), BAR)


def test_eval_mode_only_x_and_c(device):
    flow, g = _golden_flow(device, "cnf35")
    flow.eval().transform.adjoint = True
    x = torch.as_tensor(g["x"], device=device).requires_grad_()
    c = torch.as_tensor(g["c"], device=device).requires_grad_()
    (flow(c).log_prob(x) * torch.as_tensor(g["w"], device=device)).sum().backward()
    assert all(p.grad is None for p in flow.parameters())
    gold = golden_grads(g, "eval", "32")
    assert relmax(as_np(x.grad), gold["in0"]) <= 2 * max(gap(g, "eval", "in0"), BAR)
    assert relmax(as_np(c.grad), gold["in1"]) <= 2 * max(gap(g, "eval", "in1"), BAR)


def test_reverse_kl_accelerate_and_refusals(device):
    torch.manual_seed(0)
    flow = CNF(3, 2, adjoint=True).to(device).train()
    c = torch.randn(64, 2, device=device)
    x, lp = flow(c).rsample_and_log_prob()
    (lp.mean() + 0.5 * (x**2).sum(-1).mean()).backward()
    for p in flow.parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all()
    # accelerate carries nothing new: the caller sets adjoint on the result, which then trains the same way
    acc = accelerate(flow)
    acc.transform.adjoint = True
    xs = torch.randn(64, 3, device=device)
    flow.zero_grad()
    flow(c).log_prob(xs).sum().backward()
    ref = [p.grad.clone() for p in flow.parameters()]
    acc.zero_grad()
    acc(c).log_prob(xs).sum().backward()
    for a, b in zip([p.grad for p in acc.parameters()], ref, strict=True):
        assert torch.equal(a, b)
    # double backward, times that require grad, and an optimizer step between forward and backward
    xg = xs.clone().requires_grad_()
    (gx,) = torch.autograd.grad((flow(c).transform(xg) ** 2).sum(), xg, create_graph=True)
    with pytest.raises(RuntimeError, match="once_differentiable|twice"):
        gx.sum().backward()
    t = flow(c).transform
    t.t1 = torch.tensor(1.0, device=device, requires_grad=True)
    with pytest.raises(NotImplementedError, match="times"):
        t(xs)
    loss = flow(c).log_prob(xs).sum()
    with torch.no_grad():
        flow.transform.ode[0].weight.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        loss.backward()


def test_adam_curve_against_reference(device):
    g = load("cnfgrad_adam")
    torch.manual_seed(0)
    flow = CNF(2, 1, hidden_features=[16, 16], adjoint=True)
    flow.load_state_dict({k[8:]: torch.as_tensor(v) for k, v in g.items() if k.startswith("adam_sd/")})
    flow = flow.to(device).train()
    x = torch.as_tensor(g["adam_x"], device=device)
    c = torch.as_tensor(g["adam_c"], device=device)
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    losses, accepted = [], []
    for _ in range(20):
        t = flow(c)
        loss = -t.log_prob(x).mean()
        accepted.append(t.transform.stats[1])
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print("adam accepted steps engine", accepted, "reference", g["adam_accepted"].tolist())
    np.testing.assert_allclose(losses, g["adam_loss"], rtol=1e-3)


def test_report_worst():
    """Prints the worst gradient error against the restatement, smooth and piecewise-linear fields apart (DESIGN
    records both)."""
    for label, keep in (("smooth", lambda k: "ReLU" not in k), ("ReLU / LeakyReLU", lambda k: "ReLU" in k)):
        errs = {k: v for k, v in WORST.items() if keep(k)}
        if errs:
            k = max(errs, key=errs.get)
            print(f"worst gradient error vs the fp64 restatement, {label}: {errs[k]:.2e} ({k}) over {len(errs)} checks")
