"""GPU tests of the continuous normalizing flow (zk_cnf_integrate): every result is compared with the fp64
restatement (tests/cnf_reference.py) replaying the engine's OWN step log, the logged controller is recomputed
on the host bit for bit, and the default-init cases must also take the reference's fp32 trial sequence."""

import ctypes

import numpy as np
import pytest
import torch

import cnf_reference as R
from cases import load
from test_cnf_host import CASES, DEFAULT, OPS, field_of, outputs, rel
from zuko_b200 import _engine as E
from zuko_b200.accel import accelerate
from zuko_b200.flows import CNF

pytestmark = pytest.mark.gpu
BAR = 1e-5


class Engine:
    """A zk_cnf handle of a CNF flow and direct zk_cnf_integrate calls with the step log."""

    def __init__(self, flow, device) -> None:
        self.flow = flow.to(device)
        self.t = self.flow.transform
        self.dev = device
        self.D = self.t.ode.out_features
        self.C = self.t.ode.in_features - self.D - 2 * self.t.freqs.numel()

    def run(self, x, c=None, trace=R.TRACE_EXACT, direction=+1, eps=None, times=None, ldc=None, max_trials=1000,
            x_view=None, y_view=None):  # fmt: skip
        dev = self.dev
        x = x_view if x_view is not None else torch.as_tensor(x, dtype=torch.float32, device=dev)
        B = x.shape[0]
        y = y_view if y_view is not None else torch.empty(B, self.D, device=dev)
        ladj = torch.empty(B, device=dev) if trace else None
        counts = torch.zeros(2, dtype=torch.int32, device=dev)
        log = torch.full((max_trials, 4), float("nan"), device=dev)
        tt = torch.tensor([0.0, 1.0] if direction > 0 else [1.0, 0.0], device=dev) if times is None else times
        cc = None if c is None else torch.as_tensor(c, dtype=torch.float32, device=dev)
        if cc is not None and ldc is None:
            ldc = cc.stride(0) if cc.dim() == 2 else 0
        ee = None if eps is None else torch.as_tensor(eps, dtype=torch.float32, device=dev)
        h = self.t._cnf_handle()
        need = E.lib().zk_cnf_workspace_bytes(h, B, trace)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
        E.check(E.lib().zk_cnf_integrate(
            h, x.data_ptr(), x.stride(0), None if cc is None else cc.data_ptr(), ldc or 0, B, tt.data_ptr(),
            self.t.atol, self.t.rtol, trace, None if ee is None else ee.data_ptr(), 0 if ee is None else ee.stride(0),
            max_trials, y.data_ptr(), y.stride(0), None if ladj is None else ladj.data_ptr(), counts.data_ptr(),
            log.data_ptr(), ws.data_ptr(), need, E.stream_ptr(dev)))  # fmt: skip
        n, acc = counts.tolist()
        lg = log[: max(n, 0)].double().cpu().numpy()
        return y, ladj, (n, acc), lg


def check_log(lg, direction, atol, rtol, field=None, x=None, c=None, trace=None, eps=None):
    assert np.all((lg[:, 2] < 1.0) == (lg[:, 3] == 1.0))
    t0, t1 = (0.0, 1.0) if direction > 0 else (1.0, 0.0)
    steps = R.controller(t0, t1, lg[:, 2].astype(np.float32), np.float32)
    assert len(steps) == len(lg)
    for (t, dt, acc), row in zip(steps, lg, strict=True):
        assert (float(t), float(dt), float(acc)) == (row[0], row[1], row[3])
    if field is not None:
        # the error is |x_next - x_star| of two fp32 states a few ulp apart, over tol ~ rtol |x|: its fp32
        # rounding is about ulp(x) / (rtol |x|) ~ 6e-3 per ulp in units of the accept threshold, so small logged
        # errors are compared at 0.05 (8 ulp) absolute, large ones at 1e-2 relative
        errs = R.replay_errors(field, x, c, lg, trace, atol, rtol, eps)
        np.testing.assert_allclose(lg[:, 2], errs, rtol=1e-2, atol=0.05)


@pytest.fixture(scope="module")
def engines(device):
    out = {}
    for name in CASES:
        g = load(f"flow_{name}")
        torch.manual_seed(0)
        flow = CASES[name]().eval()
        flow.load_state_dict({k[3:]: torch.as_tensor(v) for k, v in g.items() if k.startswith("sd/")})
        out[name] = (Engine(flow, device), g)
    return out


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("op", list(OPS))
def test_against_replay_of_own_log_and_reference(engines, name, op):
    eng, g = engines[name]
    trace, key, direction = OPS[op]
    inp = g[key].astype(np.float64)
    c = g.get("c")
    eps = g["hut_eps_32"] if op == "hut" else None
    y, ladj, (n, acc), lg = eng.run(g[key], c, trace, direction, eps)
    assert acc >= 0
    check_log(lg, direction, float(g["atol"]), float(g["rtol"]), field_of(g), inp, c, trace, eps)
    yr, lr = R.replay(field_of(g), inp, c, lg, trace, eps)
    ours = outputs(g, op, y.double().cpu().numpy(), None if ladj is None else ladj.double().cpu().numpy(), inp)
    ref = outputs(g, op, yr, lr, inp)
    for k in ours:
        assert rel(ours[k], ref[k]) <= BAR, k
    # against the reference's own fp32 run.  Not the Hutchinson values: the ladj column is integrated at a
    # tolerance relaxed 100-fold (trace_scale), so the slightly different step sizes of two fp32 runs move the
    # Hutchinson ladj by up to ~1e-4, and the golden's fp64 run draws a different eps, so it gives no gap.
    gold = g[f"log_{op}_32"]
    if name in DEFAULT:
        assert (n, acc) == (len(gold), int(gold[:, 3].sum()))
    if op == "hut":
        return
    for k in ours:
        bar = BAR if name in DEFAULT else 2 * max(float(g[f"gap_{k}"]), BAR)
        assert rel(ours[k], g[f"{k}_32"]) <= bar, k


@pytest.mark.parametrize("name", ["cnf35", "cnf168"])
def test_round_trip(engines, name):
    eng, g = engines[name]
    c = torch.as_tensor(g["c"], device=eng.dev)
    x = torch.as_tensor(g["x"], device=eng.dev)
    with torch.no_grad():
        t = eng.flow(c).transform
        torch.testing.assert_close(t.inv(t(x)), x, atol=1e-4, rtol=0)


def _flow(device, D, C, seed=0, **kw):
    torch.manual_seed(seed)
    return Engine(CNF(D, C, **kw).eval(), device)


def _check_replay(eng, x, c, y, ladj, lg, trace=R.TRACE_EXACT, direction=+1, eps=None):
    sd = {k: v.detach().double().cpu().numpy() for k, v in eng.flow.state_dict().items()}
    act = type(eng.t.ode[1]).__name__ if len(eng.t.ode) > 1 else "ReLU"
    field = R.Field.from_state_dict(sd, eng.D, eng.C, act)
    check_log(lg, direction, eng.t.atol, eng.t.rtol)
    yr, lr = R.replay(field, x, c, lg, trace, eps)
    assert rel(y.double().cpu().numpy(), yr) <= BAR
    if trace:
        assert rel(ladj.double().cpu().numpy(), lr) <= BAR


@pytest.mark.parametrize("B", [1, 7, 300, None])
def test_batch_edges(device, B):
    """B = 1, CTAs that own no rows, and (None) several row passes per thread."""
    eng = _flow(device, 3, 2)
    h = eng.t._cnf_handle()
    ctas, threads, passes, smem = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_size_t()
    E.check(E.lib().zk_cnf_plan(h, 1, 1, ctypes.byref(ctas), ctypes.byref(threads), ctypes.byref(passes), ctypes.byref(smem)))
    if B is None:
        B = 2 * ctas.value * threads.value + 5
    E.check(E.lib().zk_cnf_plan(h, B, 1, ctypes.byref(ctas), ctypes.byref(threads), ctypes.byref(passes), ctypes.byref(smem)))
    assert passes.value == -(-B // (ctas.value * threads.value))
    rng = np.random.default_rng(B)
    x, c = rng.standard_normal((B, 3)), rng.standard_normal((B, 2))
    y, ladj, _, lg = eng.run(x, c)
    _check_replay(eng, x[:64], c[:64], y[:64], ladj[:64], lg)
    _check_replay(eng, x[-64:], c[-64:], y[-64:], ladj[-64:], lg)


@pytest.mark.parametrize("D,C", [(1, 0), (64, 0), (64, 64), (5, 3)])
def test_shapes_and_broadcast_context(device, D, C):
    eng = _flow(device, D, C)
    rng = np.random.default_rng(D)
    B = 96
    x = rng.standard_normal((B, D))
    c1 = rng.standard_normal(C) if C else None
    y, ladj, _, lg = eng.run(x, c1, ldc=0)
    _check_replay(eng, x, c1, y, ladj, lg)


@pytest.mark.parametrize("act", ["ReLU", "ELU", "Tanh", "SiLU", "GELU", "LeakyReLU", "Softplus", "Sigmoid"])
def test_activations_custom_times_reversed(device, act):
    eng = _flow(device, 4, 2, activation=getattr(torch.nn, act))
    rng = np.random.default_rng(3)
    x, c = rng.standard_normal((64, 4)), rng.standard_normal((64, 2))
    times = torch.tensor([0.25, -0.5], device=device)
    y, ladj, _, lg = eng.run(x, c, times=times)
    check_log_t = R.controller(0.25, -0.5, lg[:, 2].astype(np.float32), np.float32)
    assert [(float(a), float(b)) for a, b, _ in check_log_t] == [(r[0], r[1]) for r in lg]
    sd = {k: v.detach().double().cpu().numpy() for k, v in eng.flow.state_dict().items()}
    field = R.Field.from_state_dict(sd, 4, 2, act)
    yr, lr = R.replay(field, x, c, lg, R.TRACE_EXACT)
    assert rel(y.double().cpu().numpy(), yr) <= BAR and rel(ladj.double().cpu().numpy(), lr) <= BAR


def test_strides_and_aliasing(device):
    eng = _flow(device, 5, 3)
    rng = np.random.default_rng(5)
    B = 80
    big = torch.full((B, 11), float("nan"), device=device)
    big[:, 2:7] = torch.as_tensor(rng.standard_normal((B, 5)), dtype=torch.float32, device=device)
    cbig = torch.as_tensor(rng.standard_normal((B, 9)), dtype=torch.float32, device=device)
    x = big[:, 2:7]
    x_host = x.double().cpu().numpy()
    ref_y, ref_l, _, ref_lg = eng.run(x.contiguous(), cbig[:, 4:7].contiguous())
    yv = torch.full((B, 13), float("nan"), device=device)
    y, l, _, lg = eng.run(None, cbig[:, 4:7], x_view=x, y_view=yv[:, 3:8])
    assert torch.equal(yv[:, 3:8], ref_y) and torch.equal(l, ref_l) and np.array_equal(lg, ref_lg)
    assert torch.isnan(yv[:, :3]).all() and torch.isnan(yv[:, 8:]).all()
    y2, l2, _, _ = eng.run(None, cbig[:, 4:7], x_view=x, y_view=x)  # y aliases x
    assert torch.equal(big[:, 2:7], ref_y) and torch.isnan(big[:, :2]).all() and torch.isnan(big[:, 7:]).all()
    _check_replay(eng, x_host, cbig[:, 4:7].double().cpu().numpy(), ref_y, ref_l, ref_lg)


def test_batch_semantics(device):
    eng = _flow(device, 4, 2)
    rng = np.random.default_rng(9)
    B = 500
    x, c = rng.standard_normal((B, 4)), rng.standard_normal((B, 2))
    a = eng.run(x, c)
    b = eng.run(x, c)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and np.array_equal(a[3], b[3])
    perm = rng.permutation(B)
    p = eng.run(x[perm], c[perm])
    assert torch.equal(p[0], a[0][perm]) and torch.equal(p[1], a[1][perm]) and np.array_equal(p[3], a[3])
    y, ladj, (n, acc), _ = eng.run(x, c, max_trials=2)
    assert n == 2 and acc < 0 and torch.isnan(y).all() and torch.isnan(ladj).all()


def test_refuses_beyond_shared_memory(device):
    eng = _flow(device, 16, 8, hidden_features=[128, 128])
    assert eng.run(np.zeros((4, 16)), np.zeros((4, 8)))[2][1] >= 0
    big = _flow(device, 16, 8, hidden_features=[256, 256])
    with pytest.raises(NotImplementedError):
        big.run(np.zeros((4, 16)), np.zeros((4, 8)))
    with pytest.raises(ValueError):  # one byte short of the workspace
        h = eng.t._cnf_handle()
        need = E.lib().zk_cnf_workspace_bytes(h, 4, 1)
        x = torch.zeros(4, 16, device=device)
        ws = torch.empty(need, dtype=torch.uint8, device=device)
        tt = torch.tensor([0.0, 1.0], device=device)
        E.check(E.lib().zk_cnf_integrate(h, x.data_ptr(), 16, torch.zeros(8, device=device).data_ptr(), 0, 4, tt.data_ptr(),
                                         1e-6, 1e-5, 1, None, 0, 100, x.data_ptr(), 16, torch.empty(4, device=device).data_ptr(),
                                         None, None, ws.data_ptr(), need - 1, E.stream_ptr(device)))  # fmt: skip


def test_python_surface(device):
    torch.manual_seed(0)
    flow = CNF(3, 5).to(device).eval()
    g = torch.Generator(device="cpu").manual_seed(4)
    x = torch.randn(128, 3, generator=g).to(device)
    c = torch.randn(128, 5, generator=g).to(device)
    lp = flow(c).log_prob(x)
    acc = accelerate(flow).eval()
    assert torch.equal(acc(c).log_prob(x), lp)
    with torch.no_grad():
        s = flow(c).sample()
        xs, lps = flow(c).rsample_and_log_prob()
    assert s.shape == (128, 3) and xs.shape == (128, 3) and lps.shape == (128,)
    flow.train()
    with pytest.raises(NotImplementedError, match="adjoint"):
        flow(c).log_prob(x)
    with torch.no_grad():
        assert torch.equal(flow(c).log_prob(x), lp)
    t = flow.eval()(c).transform
    t.max_trials = 2
    with pytest.raises(RuntimeError, match="did not reach"):
        t(x)
