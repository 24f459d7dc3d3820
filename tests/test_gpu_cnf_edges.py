"""Tests of the CNF integration kernel (cnf_dopri_kernel, cnf.cu) at its launch-plan, MLP-shape, batch,
time-interval, stride and failure edges, against the fp64 replay of the engine's own step log (tests/cnf_reference.py)
and, for one-layer fields, against the closed form expm.

* `cnf_plan_of` restates in numpy what cnf_geometry decides: the padded widths, the packed weight floats, the
  per-thread floats of each trace mode, the threads per CTA (most resident threads by shared memory, ties to more
  threads), the dynamic shared memory and the refusal.  Tests without a GPU check that the case table reaches 256, 128,
  64 and 32 threads with and without a trace, a tie, the largest hidden width that fits at 32 threads next to the one
  that is refused, and shapes that fit without a trace but not with one; and that hidden (64, 64) fits every D, C <= 64
  at every freqs count.  On the GPU `zk_cnf_plan` must report the same plan.
* Oracle parity: one to sixteen linear layers, hidden widths 1, 7, 8, 9 and 65, D in {1, 7, 8, 9, 64}, C in
  {0, 1, 7, 64}, F in {0, 1, 32}, every activation, weights x3, every trace in both directions; each run's logged t / dt
  recomputed bit for bit by the fp32 controller and its logged errors by the replay.  A one-layer field is affine in the
  state extended by (cos wt, sin wt, 1, c), so its flow is expm(M (t1 - t0)) and its ladj tr(A) (t1 - t0), or
  eps^T A eps (t1 - t0) with Hutchinson's estimate: an oracle that shares no code with the replay.
* Batch mapping: batches tiled from a base block at sizes around the threads per CTA and per grid, on the 256- and
  32-thread plans, must reproduce the base block's step log and its rows bit for bit.
* Time intervals and failure: equal times, one ulp, offset and negative intervals, the sliver step when
  t + (t1 - t) != t1, the trial budget, NaN / inf rows collapsing the step size until t + dt == t, the zero field.
* Contracts: padded strides with NaN pads, the broadcast context, y aliasing x, NULL counts / log, a garbage or
  oversized workspace, both zk_set_fast_math modes, interleaved handles, B = 0, and every refusal of zk_cnf_create,
  zk_cnf_plan and zk_cnf_integrate with the outputs left untouched.  The Python layer: leading dimensions and every
  context form, Hutchinson's eps draw, handle re-packing, stats, and the dtype / device refusals.

Bars, with the worst values measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit.  Values are within
BAR = 1e-5 of the fp64 replay, relative to max(|ref|, 1), in every case (measured 2.5e-6, the Hutchinson run whose
ladj column decides the steps; 1.6e-6 on the weights-x3 flows, 9.6e-7 on the deep weights-x3 Tanh field).  The
closed form is met within EXPM_BAR = 5e-6 (measured 7.2e-7): the engine's own fp32 steps leave the local errors of an
adaptive solver run at rtol 1e-5, which the fp64 controller of the restatement leaves too (4.3e-7 on the same
fields).  The closed-form ladj is met within LADJ_BAR = 2e-6 of the sum of the magnitudes of its terms (measured
1.4e-7): a constant trace integrated by weights that sum to one leaves only fp32 rounding."""

import ctypes

import numpy as np
import pytest
import torch
from scipy.linalg import expm

import cnf_reference as R
from test_cnf_host import rel
from test_gpu_bijector_edges import math_mode  # noqa: F401
from test_gpu_cnf import BAR, Engine, _check_replay, check_log
from zuko_b200 import _engine as E
from zuko_b200.flows import CNF

NAN = float("nan")
PAD = 3
EXPM_BAR = 5e-6
LADJ_BAR = 2e-6
SMEM_CAP, SMEM_PER_SM = 232448, 233472
THREAD_CHOICES = (256, 128, 64, 32)
ACTS = ["ReLU", "ELU", "Tanh", "SiLU", "GELU", "LeakyReLU", "Softplus", "Sigmoid"]
TRACES = {"none": R.TRACE_NONE, "exact": R.TRACE_EXACT, "hut": R.TRACE_HUTCHINSON}


# --------------------------------------------------------------------------- #
# the plan, restated
# --------------------------------------------------------------------------- #


def cnf_plan_of(D, C, F, hidden, trace):
    """What cnf_geometry decides for an MLP D + C + 2F -> hidden... -> D: {"ok": False, ...} when no thread count
    fits, else threads and smem; with the layout (pad, wfloats, S, hidden_pad, floats) and the resident threads of
    every choice that fits."""
    dims = [D + C + 2 * F, *hidden, D]
    nl = len(dims) - 1
    pad = [-(-d // 8) * 8 for d in dims[1:]]
    wfloats = sum(dims[l] * pad[l] + pad[l] for l in range(nl))
    S = max(D + C, *pad)
    hidden_pad = sum(pad[:-1])
    floats = 2 * S + (hidden_pad if trace != R.TRACE_NONE else 0)
    fixed = (wfloats + 7 * 2 * 32 + 32) * 4
    out = {"pad": pad, "wfloats": wfloats, "S": S, "hidden_pad": hidden_pad, "floats": floats, "resident": {}}
    best = 0
    for nt in THREAD_CHOICES:
        smem = fixed + nt * floats * 4
        if smem > SMEM_CAP:
            continue
        res = min(SMEM_PER_SM // (smem + 1024), 2048 // nt, 32) * nt
        out["resident"][nt] = res
        if res > best:
            best, out["threads"], out["smem"] = res, nt, smem
    out["ok"] = best > 0
    return out


# name -> (D, C, F, hidden); the comments give the threads without / with a trace
PLAN_CASES = {
    "tiny": (1, 0, 0, ()),              # 256 / 256, tied with 128 and 64
    "d2_h16": (2, 0, 3, (16, 16)),      # 256 / 256
    "cnf35": (3, 5, 3, (64, 64)),       # 256 / 128, both tied
    "h32": (16, 8, 3, (32, 32)),        # 128 / 64
    "d96": (96, 0, 3, (64, 64)),        # 128 / 64
    "max64": (64, 64, 32, (64, 64)),    # 128 / 64
    "d160": (160, 0, 3, (64, 64)),      # 64 / 64
    "h144": (16, 8, 3, (144, 144)),     # 64 / 32
    "d192": (192, 0, 3, (64, 64)),      # 64 / 32
    "h167": (16, 8, 3, (167, 167)),     # 32 / 32: the widest (h, h) that fits with a trace
    "h168": (16, 8, 3, (168, 168)),     # 32 / refused
    "h176": (16, 8, 3, (176, 176)),     # 32 / refused
    "cnf256": (256, 0, 3, (64, 64)),    # 32 / refused
    "h188": (16, 8, 3, (188, 188)),     # 32 / refused: the widest (h, h) that fits
    "h189": (16, 8, 3, (189, 189)),     # refused / refused
}  # fmt: skip
FAMILIES = (R.TRACE_NONE, R.TRACE_EXACT)


def plan_case(name, trace):
    return cnf_plan_of(*PLAN_CASES[name], trace)


def test_plan_table_reaches_every_cell():
    for trace in FAMILIES:
        threads = {plan_case(n, trace).get("threads") for n in PLAN_CASES}
        assert threads >= {256, 128, 64, 32, None}, (trace, threads)
    ties = [n for n in PLAN_CASES for tr in FAMILIES
            if plan_case(n, tr)["ok"] and list(plan_case(n, tr)["resident"].values()).count(max(plan_case(n, tr)["resident"].values())) > 1]  # fmt: skip
    assert "tiny" in ties and "cnf35" in ties
    assert plan_case("tiny", R.TRACE_NONE)["resident"] == {256: 2048, 128: 2048, 64: 2048, 32: 1024}
    # the widest hidden (h, h) of CNF(16, 8) at 32 threads, and h + 1 refused, with and without a trace
    for tr, widest in ((R.TRACE_NONE, "h188"), (R.TRACE_EXACT, "h167")):
        p = plan_case(widest, tr)
        assert p["threads"] == 32 and p["smem"] <= SMEM_CAP
        D, C, F, (h, _) = PLAN_CASES[widest]
        assert not cnf_plan_of(D, C, F, (h + 1, h + 1), tr)["ok"]
    for name in ("h168", "cnf256", "h188"):
        assert plan_case(name, R.TRACE_NONE)["threads"] == 32 and not plan_case(name, R.TRACE_EXACT)["ok"]
    assert not plan_case("h189", R.TRACE_NONE)["ok"]
    # the Hutchinson trace keeps the same per-thread floats as the exact one
    assert all(plan_case(n, R.TRACE_HUTCHINSON) == plan_case(n, R.TRACE_EXACT) for n in PLAN_CASES)


def test_plan_layout():
    p = cnf_plan_of(3, 5, 3, (64, 65), R.TRACE_EXACT)
    assert p["pad"] == [64, 72, 8]
    assert p["wfloats"] == 14 * 64 + 64 + 64 * 72 + 72 + 65 * 8 + 8
    assert p["S"] == 72 and p["hidden_pad"] == 136 and p["floats"] == 2 * 72 + 136
    assert cnf_plan_of(3, 5, 3, (64, 65), R.TRACE_NONE)["floats"] == 2 * 72
    assert cnf_plan_of(40, 30, 0, (8,), R.TRACE_EXACT)["S"] == 70  # the context row is wider than every layer


def test_default_hidden_fits_every_small_shape():
    """DESIGN §7: hidden (64, 64) fits every D, C <= 64, at any freqs count, with and without a trace."""
    for F in range(33):
        for D in range(1, 65):
            for C in (0, 1, 31, 63, 64):
                for tr in FAMILIES:
                    assert cnf_plan_of(D, C, F, (64, 64), tr)["ok"], (D, C, F, tr)


# --------------------------------------------------------------------------- #
# the closed form of a one-layer field
# --------------------------------------------------------------------------- #


def affine_flow(field, x, c, t0, t1):
    """x(t1) of dx/dt = A x + W_cos cos(w t) + W_sin sin(w t) + W_c c + b: the state extended by (cos wt, sin wt, 1, c)
    evolves by the constant matrix M, so it is expm(M (t1 - t0)) applied to the extended state at t0."""
    (W,), (b,) = field.W, field.b
    D, C, w = field.D, field.C, field.freqs
    F = len(w)
    n = D + 2 * F + 1 + C
    M = np.zeros((n, n))
    M[:D, :D] = W[:, 2 * F : 2 * F + D]
    M[:D, D : D + 2 * F] = W[:, : 2 * F]
    M[:D, D + 2 * F] = b
    M[:D, D + 2 * F + 1 :] = W[:, 2 * F + D :]
    for i in range(F):
        M[D + i, D + F + i] = -w[i]  # d cos(w t) / dt
        M[D + F + i, D + i] = w[i]  # d sin(w t) / dt
    B = x.shape[0]
    cc = np.zeros((B, 0)) if C == 0 else np.broadcast_to(c, (B, C))
    z0 = np.concatenate([x, np.broadcast_to(np.cos(w * t0), (B, F)), np.broadcast_to(np.sin(w * t0), (B, F)),
                         np.ones((B, 1)), cc], axis=1)  # fmt: skip
    return (z0 @ expm(M * (t1 - t0)).T)[:, :D]


def affine_ladj(field, t0, t1, eps=None):
    """(ladj, the sum of the magnitudes of its terms): tr(A) (t1 - t0), or eps^T A eps (t1 - t0) per row."""
    F2 = 2 * len(field.freqs)
    A = field.W[0][:, F2 : F2 + field.D]
    if eps is None:
        return np.trace(A) * (t1 - t0), np.sum(np.abs(np.diag(A))) * abs(t1 - t0)
    terms = eps[:, :, None] * A[None] * eps[:, None, :]
    return terms.sum(axis=(1, 2)) * (t1 - t0), np.abs(terms).sum(axis=(1, 2)) * abs(t1 - t0)


def scaled_err(ours, ref, scale):
    return float(np.max(np.abs(np.asarray(ours, np.float64) - ref) / np.maximum(scale, 1.0)))


# (D, C, F, scale, t0, t1)
AFFINE_CASES = {
    "d3_c2": (3, 2, 3, 1.0, 0.0, 1.0),
    "d8_c0_f0_back": (8, 0, 0, 1.0, 1.0, 0.0),
    "d5_c4_x3": (5, 4, 2, 3.0, -0.5, 0.75),
}


def affine_field_and_inputs(name, seed=0):
    D, C, F, scale, t0, t1 = AFFINE_CASES[name]
    torch.manual_seed(seed)
    flow = CNF(D, C, freqs=F, hidden_features=[]).eval()
    with torch.no_grad():
        for p in flow.parameters():
            p.mul_(scale)
    sd = {k: v.detach().double().numpy() for k, v in flow.state_dict().items()}
    rng = np.random.default_rng(seed + 1)
    B = 48
    x = rng.standard_normal((B, D)).astype(np.float32).astype(np.float64)
    c = rng.standard_normal((B, C)).astype(np.float32).astype(np.float64) if C else None
    eps = rng.standard_normal((B, D)).astype(np.float32).astype(np.float64)
    return flow, R.Field.from_state_dict(sd, D, C, "ReLU"), x, c, eps, t0, t1


@pytest.mark.parametrize("name", list(AFFINE_CASES))
def test_restatement_meets_closed_form(name):
    _, field, x, c, eps, t0, t1 = affine_field_and_inputs(name)
    ref = affine_flow(field, x, c, t0, t1)
    y, ladj, _ = R.integrate(field, x, c, t0, t1, 1e-6, 1e-5, R.TRACE_EXACT)
    assert rel(y, ref) <= EXPM_BAR / 10  # the fp64 controller: 4.3e-7 at most
    assert scaled_err(ladj, *affine_ladj(field, t0, t1)) <= 1e-12
    _, lh, _ = R.integrate(field, x, c, t0, t1, 1e-6, 1e-5, R.TRACE_HUTCHINSON, eps)
    assert scaled_err(lh, *affine_ladj(field, t0, t1, eps)) <= 1e-12


# --------------------------------------------------------------------------- #
# fp32 controller arithmetic
# --------------------------------------------------------------------------- #


def collapse_trials(t0, t1):
    """Trials until t + dt == t when every trial is rejected with an infinite error (factor 0.1 in fp32)."""
    f = np.float32
    t, t1 = f(t0), f(t1)
    dt = f(t1 - t)
    dt = f(np.sign(dt) * min(abs(dt), abs(f(t1 - t))))
    n = 0
    while f(t + dt) != t:
        n += 1
        dt = f(dt * f(0.1))
    return n


def test_collapse_trials():
    assert collapse_trials(1000.0, 1001.0) == 5  # ulp(1000) = 6.1e-5: dt = 1e-5 is absorbed
    n0 = collapse_trials(0.0, 1.0)
    assert 44 <= n0 <= 47  # from 1 through the subnormals to 0
    assert collapse_trials(1.0, 0.0) == collapse_trials(1.0, 2.0)


def sliver_times():
    t0, t1 = np.float32(0.1), np.float32(0.23)
    assert np.float32(t0 + np.float32(t1 - t0)) != t1
    return float(t0), float(t1)


# --------------------------------------------------------------------------- #
# GPU helpers
# --------------------------------------------------------------------------- #


def cpu(t):
    return t.detach().double().cpu().numpy()


def f32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def make(device, D, C, F=3, hidden=(64, 64), act=None, scale=1.0, seed=0, **kw):
    torch.manual_seed(seed)
    if act is not None:
        kw["activation"] = getattr(torch.nn, act)
    flow = CNF(D, C, freqs=F, hidden_features=list(hidden), **kw).eval()
    with torch.no_grad():
        for p in flow.parameters():
            p.mul_(scale)
    return Engine(flow, device)


def field_of(eng):
    sd = {k: v.detach().double().cpu().numpy() for k, v in eng.flow.state_dict().items()}
    act = type(eng.t.ode[1]).__name__ if len(eng.t.ode) > 1 else "ReLU"
    return R.Field.from_state_dict(sd, eng.D, eng.C, act)


def check_controller(lg, t0, t1):
    """The logged t / dt / accept of every trial recomputed bit for bit from the logged errors."""
    assert np.all((lg[:, 2] < 1.0) == (lg[:, 3] == 1.0))
    steps = R.controller(t0, t1, lg[:, 2].astype(np.float32), np.float32)
    assert len(steps) == len(lg)
    assert [(float(t), float(dt), float(a)) for t, dt, a in steps] == [(r[0], r[1], r[3]) for r in lg]


def replay_check(eng, x, c, out, trace, direction=+1, eps=None, times=None, errors=True):
    """The logged controller and (`errors`: when x holds every row of the run) the logged errors, then y and ladj at
    the fp64 replay of the accepted steps; returns the error."""
    y, ladj, (n, acc), lg = out
    assert acc >= 0 and n == len(lg)
    field = field_of(eng)
    if times is None:
        check_log(lg, direction, eng.t.atol, eng.t.rtol, *((field, x, c, trace, eps) if errors else ()))
    else:
        check_controller(lg, *times)
        if errors:
            errs = R.replay_errors(field, x, c, lg, trace, eng.t.atol, eng.t.rtol, eps)
            np.testing.assert_allclose(lg[:, 2], errs, rtol=1e-2, atol=0.05)
    yr, lr = R.replay(field, x, c, lg, trace, eps)
    err = rel(cpu(y), yr)
    if trace:
        err = max(err, rel(cpu(ladj), lr))
    assert err <= BAR, err
    return err


def times_of(t0, t1, device):
    return torch.tensor([t0, t1], dtype=torch.float32, device=device)


def ptr(t):
    return t if t is None or isinstance(t, int) else t.data_ptr()


def raw(eng, x, B, *, ldx=None, c=None, ldc=0, times=None, trace=R.TRACE_EXACT, eps=None, ldeps=None, max_trials=1000,
        y=None, ldy=None, ladj=None, counts=None, log=None, ws=None, ws_bytes=None, h=None, atol=None, rtol=None):  # fmt: skip
    """One zk_cnf_integrate call with every argument in the caller's hands; returns the status."""
    dev = eng.dev
    times = times_of(0.0, 1.0, dev) if times is None else times
    if ws is None:
        need = E.lib().zk_cnf_workspace_bytes(eng.t._cnf_handle(), B, trace)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
        ws_bytes = need if ws_bytes is None else ws_bytes
    return E.lib().zk_cnf_integrate(
        eng.t._cnf_handle() if h is None else h, ptr(x), eng.D if ldx is None else ldx, ptr(c), ldc, B, ptr(times),
        eng.t.atol if atol is None else atol, eng.t.rtol if rtol is None else rtol, trace, ptr(eps),
        eng.D if ldeps is None else ldeps, max_trials, ptr(y), eng.D if ldy is None else ldy, ptr(ladj), ptr(counts),
        ptr(log), ptr(ws), ws.numel() if ws_bytes is None else ws_bytes,
        E.stream_ptr(dev))  # fmt: skip


def plan(h, B, trace):
    out = [ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_size_t(0)]
    st = E.lib().zk_cnf_plan(h, B, trace, *map(ctypes.byref, out))
    return st, tuple(v.value for v in out)


def inputs(eng, B, seed=0, trace=R.TRACE_EXACT):
    rng = np.random.default_rng(seed)
    x = f32(rng.standard_normal((B, eng.D)))
    c = f32(rng.standard_normal((B, eng.C))) if eng.C else None
    eps = f32(rng.standard_normal((B, eng.D))) if trace == R.TRACE_HUTCHINSON else None
    return x, c, eps


# --------------------------------------------------------------------------- #
# 1. the plan on the GPU
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PLAN_CASES))
def test_plan_matches_restatement(device, name):
    D, C, F, hidden = PLAN_CASES[name]
    eng = make(device, D, C, F, hidden)
    h = eng.t._cnf_handle()
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    for trace in TRACES.values():
        want = cnf_plan_of(D, C, F, hidden, trace)
        if not want["ok"]:
            assert plan(h, 1, trace)[0] == E.ZK_EUNSUPPORTED
            x = torch.zeros(4, D, device=device)
            y = torch.full((4, D), NAN, device=device)
            ladj = None if trace == R.TRACE_NONE else torch.full((4,), NAN, device=device)
            eps = torch.zeros(4, D, device=device) if trace == R.TRACE_HUTCHINSON else None
            c = torch.zeros(4, C, device=device) if C else None
            assert raw(eng, x, 4, c=c, ldc=C, trace=trace, eps=eps, y=y, ladj=ladj) == E.ZK_EUNSUPPORTED
            assert torch.isnan(y).all()
            continue
        for B in (0, 1, 1000, 123457):
            st, (ctas, threads, passes, smem) = plan(h, B, trace)
            assert st == E.ZK_OK
            assert (threads, smem) == (want["threads"], want["smem"]), (trace, B)
            assert ctas > 0 and ctas % sms == 0
            assert passes == -(-B // (ctas * threads))


# --------------------------------------------------------------------------- #
# 2. oracle parity at every shape edge
# --------------------------------------------------------------------------- #

# name -> (D, C, F, hidden, activation, scale)
SHAPES = {
    "one_layer": (3, 2, 3, (), None, 1.0),
    "two_layers": (3, 2, 3, (24,), None, 1.0),
    "three_layers_w65": (5, 3, 3, (65, 65), None, 1.0),
    "sixteen_layers": (4, 2, 2, (16,) * 15, None, 1.0),
    "w1": (3, 2, 3, (1, 1), None, 1.0),
    "w7_w9": (4, 1, 3, (7, 9), None, 1.0),
    "w8": (4, 1, 3, (8, 8, 8), None, 1.0),
    "d1_c0_f0": (1, 0, 0, (16, 16), None, 1.0),
    "d7_c1_f1": (7, 1, 1, (32, 32), None, 1.0),
    "d8_c7_f32": (8, 7, 32, (32, 32), None, 1.0),
    "d9_c64_f1": (9, 64, 1, (64, 64), None, 1.0),
    "d64_c64_f32": (64, 64, 32, (64, 64), None, 1.0),
    "stiff": (3, 5, 3, (64, 64), None, 3.0),
    "deep_stiff": (6, 2, 3, (32,) * 4, "Tanh", 3.0),
    **{f"act_{a}": (4, 2, 3, (9, 24), a, 1.0) for a in ACTS},
}


@pytest.fixture(scope="module")
def shape_engines(device):
    return {}


def shape_engine(cache, device, name):
    if name not in cache:
        D, C, F, hidden, act, scale = SHAPES[name]
        cache[name] = make(device, D, C, F, hidden, act, scale)
    return cache[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("trace", ["exact", "hut", "none"])
def test_shapes_against_replay(device, shape_engines, name, trace):
    eng = shape_engine(shape_engines, device, name)
    tr = TRACES[trace]
    B = 48 if eng.D <= 16 else 24
    x, c, eps = inputs(eng, B, seed=len(name), trace=tr)
    direction = -1 if trace == "none" else +1
    out = eng.run(x, c, tr, direction, eps)
    replay_check(eng, x, c, out, tr, direction, eps)
    if SHAPES[name][5] != 1.0:
        lg = out[3]
        assert (lg[:, 3] == 0).sum() >= 2 and len(lg) > 3 * 3  # rejections, and the 3-slot ring wraps


@pytest.mark.gpu
@pytest.mark.parametrize("trace", ["exact", "hut", "none"])
@pytest.mark.parametrize("direction", [+1, -1])
def test_every_trace_both_directions(device, trace, direction):
    eng = make(device, 5, 3, 3, (32, 32, 32), "SiLU")
    tr = TRACES[trace]
    x, c, eps = inputs(eng, 64, seed=direction + 7, trace=tr)
    replay_check(eng, x, c, eng.run(x, c, tr, direction, eps), tr, direction, eps)


@pytest.mark.gpu
def test_hutchinson_error_dominated_by_the_ladj_column(device):
    """eps x 30 makes the trace estimate 900-fold larger: the ladj column then decides the step sizes, so the logged
    errors must fold in that column too."""
    eng = make(device, 3, 2, 3, (32, 32), "ELU", scale=2.0)
    x, c, eps = inputs(eng, 48, seed=3, trace=R.TRACE_HUTCHINSON)
    eps = 30 * eps
    out = eng.run(x, c, R.TRACE_HUTCHINSON, +1, eps)
    field = field_of(eng)
    lg = out[3]
    # the restatement's error ratio without the ladj column is smaller at some trial
    xs = np.asarray(x)
    L = np.zeros(len(xs))
    shrinks = False
    for t, dt, _, acc in lg:
        nxt, err, S = R.dopri(field, xs, L, float(t), float(dt), c, R.TRACE_HUTCHINSON, eps)
        full = R.error_ratio(err, S, nxt, eng.t.atol, eng.t.rtol)
        part = R.error_ratio(err[:, :-1], S[:, :-1], nxt[:, :-1], eng.t.atol, eng.t.rtol)
        shrinks |= part < 0.5 * full
        if acc:
            xs, L = nxt[:, :-1], nxt[:, -1]
    assert shrinks
    replay_check(eng, x, c, out, R.TRACE_HUTCHINSON, +1, eps)


@pytest.mark.gpu
def test_refused_shapes(device):
    with pytest.raises(ValueError, match="freqs=33"):
        make(device, 3, 2, F=33).t._cnf_handle()
    with pytest.raises(NotImplementedError, match="17 linear layers"):
        make(device, 3, 2, hidden=(8,) * 16).t._cnf_handle()
    assert make(device, 3, 2, hidden=(8,) * 15).t._cnf_handle()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(AFFINE_CASES))
def test_one_layer_field_against_closed_form(device, name):
    flow, field, x, c, eps, t0, t1 = affine_field_and_inputs(name)
    eng = Engine(flow, device)
    tt = times_of(t0, t1, device)
    y, ladj, _, lg = eng.run(x, c, R.TRACE_EXACT, times=tt)
    check_controller(lg, t0, t1)
    assert rel(cpu(y), affine_flow(field, x, c, t0, t1)) <= EXPM_BAR
    assert scaled_err(cpu(ladj), *affine_ladj(field, t0, t1)) <= LADJ_BAR
    yh, lh, _, lgh = eng.run(x, c, R.TRACE_HUTCHINSON, eps=eps, times=tt)
    assert rel(cpu(yh), affine_flow(field, x, c, t0, t1)) <= EXPM_BAR
    assert scaled_err(cpu(lh), *affine_ladj(field, t0, t1, eps)) <= LADJ_BAR
    replay_check(eng, x, c, (yh, lh, (len(lgh), int(lgh[:, 3].sum())), lgh), R.TRACE_HUTCHINSON, eps=eps, times=(t0, t1))


# --------------------------------------------------------------------------- #
# 3. batch and row mapping
# --------------------------------------------------------------------------- #

B0 = 29


@pytest.mark.gpu
@pytest.mark.parametrize("name,trace", [("d2_h16", "exact"), ("d2_h16", "hut"), ("h144", "exact"), ("h176", "none")])
def test_tiled_batches_reproduce_the_base_block(device, name, trace):
    D, C, F, hidden = PLAN_CASES[name]
    tr = TRACES[trace]
    eng = make(device, D, C, F, hidden)
    h = eng.t._cnf_handle()
    _, (ctas, nt, _, _) = plan(h, 1, tr)
    assert nt == (256 if name == "d2_h16" else 32)
    x, c, eps = inputs(eng, B0, seed=11, trace=tr)
    base = eng.run(x, c, tr, +1, eps)
    assert base[2][1] >= 0
    sizes = [B0, nt - 1, nt + 1, ctas * nt - 1, ctas * nt + 1, 2 * ctas * nt + 77]
    for B in sizes:
        idx = np.arange(B) % B0
        out = eng.run(x[idx], None if c is None else c[idx], tr, +1, None if eps is None else eps[idx])
        assert np.array_equal(out[3], base[3]), B
        assert torch.equal(out[0], base[0][idx]), B
        if tr:
            assert torch.equal(out[1], base[1][idx]), B
        assert plan(h, B, tr)[1][2] == -(-B // (ctas * nt))
    # rows around every pass boundary of the largest batch, and its last rows, against the replay
    B = sizes[-1]
    rows = np.unique(np.concatenate([np.arange(3), ctas * nt + np.arange(-2, 2), 2 * ctas * nt + np.arange(-2, 2),
                                     B - np.arange(1, 4)]))  # fmt: skip
    idx = rows % B0
    y, ladj = out[0][rows], (out[1][rows] if tr else None)
    replay_check(eng, x[idx], None if c is None else c[idx], (y, ladj, out[2], out[3]), tr, +1,
                 None if eps is None else eps[idx], errors=False)  # fmt: skip


# --------------------------------------------------------------------------- #
# 4. time interval and failure semantics
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
def test_equal_times(device):
    eng = make(device, 4, 2)
    x, c, eps = inputs(eng, 40, seed=1, trace=R.TRACE_HUTCHINSON)
    xt = torch.as_tensor(x, dtype=torch.float32, device=device)
    for tr in TRACES.values():
        y, ladj, counts, lg = eng.run(x, c, tr, eps=eps if tr == R.TRACE_HUTCHINSON else None,
                                      times=times_of(0.5, 0.5, device))  # fmt: skip
        assert torch.equal(y, xt) and counts == (0, 0) and len(lg) == 0
        if tr:
            assert torch.equal(ladj, torch.zeros_like(ladj))
    eng.t.times.fill_(0.5)
    ct = torch.as_tensor(c, dtype=torch.float32, device=device)
    with torch.no_grad():
        t = eng.flow(ct).transform
        z, l = t.call_and_ladj(xt)
        assert torch.equal(z, xt) and torch.equal(l, torch.zeros(40, device=device)) and t.stats == (0, 0)
        assert torch.equal(t.inv(xt), xt)


# (t0, t1, freqs): an offset interval runs without a time embedding, whose fp32 argument w t is coarse there
INTERVALS = {
    "one_ulp": (1.0, float(np.nextafter(np.float32(1.0), np.float32(2.0))), 3),
    "one_ulp_back": (-2.0, float(np.nextafter(np.float32(-2.0), np.float32(0.0))), 3),
    "offset_1000": (1000.0, 1001.0, 0),
    "negative": (-2.5, -3.25, 3),
    "across_zero": (-0.5, 0.75, 3),
    "sliver": (*sliver_times(), 3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(INTERVALS))
def test_time_intervals(device, name):
    t0, t1, F = INTERVALS[name]
    eng = make(device, 3, 2, F, (32, 32))
    x, c, _ = inputs(eng, 48, seed=2)
    out = eng.run(x, c, R.TRACE_EXACT, times=times_of(t0, t1, device))
    replay_check(eng, x, c, out, R.TRACE_EXACT, times=(t0, t1))
    lg = out[3]
    if name.startswith("one_ulp"):
        assert len(lg) == 1 and lg[0, 1] == np.float32(t1) - np.float32(t0)
    if name == "sliver":
        f = np.float32
        acc = lg[lg[:, 3] == 1]
        assert len(acc) >= 2 and f(acc[-2, 0] + acc[-2, 1]) != f(t1) and acc[-1, 1] == f(t1) - f(acc[-1, 0])
        assert abs(acc[-1, 1]) <= 4 * np.spacing(f(t1))


@pytest.mark.gpu
def test_trial_budget(device):
    eng = make(device, 3, 5, scale=2.0)
    x, c, _ = inputs(eng, 64, seed=4)
    y, ladj, (n, acc), lg = eng.run(x, c)
    assert n > 2 and acc >= 0
    y2, l2, counts, lg2 = eng.run(x, c, max_trials=n)
    assert counts == (n, acc) and torch.equal(y2, y) and torch.equal(l2, ladj) and np.array_equal(lg2, lg)
    y3, l3, counts, lg3 = eng.run(x, c, max_trials=n - 1)
    assert counts == (n - 1, -1 - int(lg[: n - 1, 3].sum()))
    assert torch.isnan(y3).all() and torch.isnan(l3).all() and np.array_equal(lg3, lg[: n - 1])


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["x_nan", "x_inf", "c_nan", "eps_nan", "eps_inf"])
@pytest.mark.parametrize("t0", [0.0, 1000.0])
def test_non_finite_row_collapses_the_step(device, where, t0):
    eng = make(device, 3, 2, 3 if t0 == 0 else 0, (16, 16))
    B = 40
    tr = R.TRACE_HUTCHINSON if where.startswith("eps") else R.TRACE_EXACT
    x, c, eps = inputs(eng, B, seed=5, trace=tr)
    x, c = x.copy(), c.copy()
    bad = {"nan": NAN, "inf": float("inf")}[where.split("_")[1]]
    {"x": x, "c": c, "eps": eps}[where.split("_")[0]][17, 1] = bad
    t1 = t0 + 1.0
    y, ladj, (n, acc), lg = eng.run(x, c, tr, eps=eps, times=times_of(t0, t1, device))
    want = collapse_trials(t0, t1)
    assert (n, acc) == (want, -1)
    assert np.all(lg[:, 2] == np.inf) and np.all(lg[:, 3] == 0) and np.all(lg[:, 0] == np.float32(t0))
    check_controller(lg, t0, t1)
    assert torch.isnan(y).all() and torch.isnan(ladj).all()
    if where.startswith("x"):
        eng.t.times.copy_(torch.tensor([t0, t1]))
        with torch.no_grad(), pytest.raises(RuntimeError, match="did not reach"):
            eng.flow(torch.as_tensor(c, dtype=torch.float32, device=device)).transform(
                torch.as_tensor(x, dtype=torch.float32, device=device))


@pytest.mark.gpu
def test_zero_field_takes_one_trial(device):
    eng = make(device, 4, 2, scale=0.0)
    x, c, eps = inputs(eng, 50, seed=6, trace=R.TRACE_HUTCHINSON)
    xt = torch.as_tensor(x, dtype=torch.float32, device=device)
    for tr in TRACES.values():
        y, ladj, counts, lg = eng.run(x, c, tr, eps=eps if tr == R.TRACE_HUTCHINSON else None)
        assert counts == (1, 1) and torch.equal(y, xt) and lg[0, 2] == np.float32(1e-9)
        if tr:
            assert torch.equal(ladj, torch.zeros_like(ladj))


# --------------------------------------------------------------------------- #
# 5. strides, aliasing and contracts
# --------------------------------------------------------------------------- #


def padded(a, device, pad=PAD, fill=NAN):
    """a (B, n) inside a NaN-filled (B, n + 2 pad), as a view at column `pad`."""
    big = torch.full((a.shape[0], a.shape[1] + 2 * pad), fill, device=device)
    big[:, pad : pad + a.shape[1]] = torch.as_tensor(a, dtype=torch.float32, device=device)
    return big, big[:, pad : pad + a.shape[1]]


@pytest.mark.gpu
@pytest.mark.parametrize("trace", list(TRACES))
def test_padded_strides(device, trace):
    tr = TRACES[trace]
    eng = make(device, 5, 3, 3, (24, 24), "GELU")
    B = 70
    x, c, eps = inputs(eng, B, seed=8, trace=tr)
    ref = eng.run(x, c, tr, eps=eps)
    _, xv = padded(x, device)
    _, cv = padded(c, device, pad=2)
    ev = None if eps is None else padded(eps, device, pad=4)[1]
    ybig, yv = padded(np.zeros((B, 5)), device)
    ybig.fill_(NAN)
    y, ladj, counts, lg = eng.run(None, cv, tr, eps=ev, x_view=xv, y_view=yv)
    assert torch.equal(yv, ref[0]) and counts == ref[2] and np.array_equal(lg, ref[3])
    assert torch.isnan(ybig[:, :PAD]).all() and torch.isnan(ybig[:, PAD + 5 :]).all()
    if tr:
        assert torch.equal(ladj, ref[1])


@pytest.mark.gpu
def test_broadcast_context(device):
    eng = make(device, 4, 6)
    B = 60
    x, c, _ = inputs(eng, B, seed=9)
    row = c[:1]
    ref = eng.run(x, np.repeat(row, B, axis=0))
    out = eng.run(x, row[0], ldc=0)
    assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1]) and np.array_equal(out[3], ref[3])


@pytest.mark.gpu
@pytest.mark.parametrize("trace", ["hut", "none"])
def test_y_aliases_x(device, trace):
    tr = TRACES[trace]
    eng = make(device, 5, 3)
    x, c, eps = inputs(eng, 66, seed=10, trace=tr)
    ref = eng.run(x, c, tr, eps=eps)
    xbig, xv = padded(x, device)
    out = eng.run(None, c, tr, eps=eps, x_view=xv, y_view=xv)
    assert torch.equal(xv, ref[0]) and np.array_equal(out[3], ref[3])
    assert torch.isnan(xbig[:, :PAD]).all() and torch.isnan(xbig[:, PAD + 5 :]).all()


@pytest.mark.gpu
def test_optional_outputs_workspace_and_math_mode(device, math_mode):  # noqa: F811
    eng = make(device, 4, 3, 3, (32, 32), "GELU")
    B = 90
    x, c, _ = inputs(eng, B, seed=12)
    math_mode(False)
    ref = eng.run(x, c)
    xt = torch.as_tensor(x, dtype=torch.float32, device=device)
    ct = torch.as_tensor(c, dtype=torch.float32, device=device)
    h = eng.t._cnf_handle()
    need = E.lib().zk_cnf_workspace_bytes(h, B, R.TRACE_EXACT)

    def call(counts=True, log=True, ws_extra=0, fill=None):
        y = torch.full((B, 4), NAN, device=device)
        ladj = torch.full((B,), NAN, device=device)
        cn = torch.zeros(2, dtype=torch.int32, device=device) if counts else None
        lg = torch.full((1000, 4), NAN, device=device) if log else None
        ws = torch.empty(need + ws_extra, dtype=torch.uint8, device=device)
        if fill is not None:
            ws.fill_(fill)
        E.check(raw(eng, xt, B, c=ct, ldc=3, y=y, ladj=ladj, counts=cn, log=lg, ws=ws, ws_bytes=need + ws_extra))
        assert torch.equal(y, ref[0]) and torch.equal(ladj, ref[1])
        if counts:
            assert tuple(cn.tolist()) == ref[2]
        if log:
            n = ref[2][0]
            assert np.array_equal(cpu(lg[:n]), ref[3]) and torch.isnan(lg[n:]).all()

    for counts, log in ((False, True), (True, False), (False, False)):
        call(counts, log)
    call(fill=0xFF)
    call(ws_extra=4096 + 77, fill=0xFF)
    math_mode(True)
    call()
    assert np.array_equal(eng.run(x, c)[3], ref[3])


@pytest.mark.gpu
def test_interleaved_handles(device):
    a, b = make(device, 3, 2, seed=1), make(device, 6, 0, 2, (16, 16, 16), "Tanh", seed=2)
    xa, ca, _ = inputs(a, 50, seed=13)
    xb, _, eb = inputs(b, 30, seed=14, trace=R.TRACE_HUTCHINSON)
    ra, rb = a.run(xa, ca), b.run(xb, None, R.TRACE_HUTCHINSON, eps=eb)
    for _ in range(2):
        ra2, rb2 = a.run(xa, ca), b.run(xb, None, R.TRACE_HUTCHINSON, eps=eb)
        for r, r2 in ((ra, ra2), (rb, rb2)):
            assert torch.equal(r[0], r2[0]) and torch.equal(r[1], r2[1]) and np.array_equal(r[3], r2[3])


@pytest.mark.gpu
def test_empty_batch(device):
    eng = make(device, 3, 2)
    counts = torch.full((2,), 77, dtype=torch.int32, device=device)
    assert E.lib().zk_cnf_workspace_bytes(eng.t._cnf_handle(), 0, 1) > 0
    for tr in TRACES.values():
        ladj = None if tr == R.TRACE_NONE else torch.full((1,), NAN, device=device)
        eps = torch.zeros(1, 3, device=device) if tr == R.TRACE_HUTCHINSON else None
        assert raw(eng, None, 0, trace=tr, eps=eps, ladj=ladj, counts=counts) == E.ZK_OK
        assert E.lib().zk_cnf_integrate(eng.t._cnf_handle(), None, 0, None, 0, 0, ptr(times_of(0, 1, device)), 1e-6, 1e-5,
                                        tr, ptr(eps), 3, 1, None, 0, ptr(ladj), ptr(counts), None, None, 0,
                                        E.stream_ptr(device)) == E.ZK_OK  # fmt: skip
    torch.cuda.synchronize()
    assert counts.tolist() == [77, 77]
    # the Python layer: an empty batch of rows, with per-row, broadcast and no context, exact and Hutchinson
    x0 = torch.zeros(2, 0, 3, device=device)
    with torch.no_grad():
        for c in (torch.zeros(2, 0, 2, device=device), torch.zeros(2, device=device)):
            for exact in (True, False):
                eng.t.exact = exact
                t = eng.flow(c).transform
                z, l = t.call_and_ladj(x0)
                assert z.shape == (2, 0, 3) and l.shape == (2, 0) and t.stats == (0, 0)
                assert t.inv(x0).shape == (2, 0, 3)
        assert make(device, 3, 0).flow().sample((0,)).shape == (0, 3)


# --------------------------------------------------------------------------- #
# 6. refusals
# --------------------------------------------------------------------------- #


def last_error():
    return E.lib().zk_last_error().decode()


@pytest.mark.gpu
def test_integrate_and_plan_refusals(device):
    eng = make(device, 4, 3)
    D, C, B = 4, 3, 8
    h = eng.t._cnf_handle()
    x = torch.zeros(B, D, device=device)
    c = torch.zeros(B, C, device=device)
    eps = torch.zeros(B, D, device=device)
    need = E.lib().zk_cnf_workspace_bytes(h, B, R.TRACE_HUTCHINSON)
    ws = torch.empty(need + 512, dtype=torch.uint8, device=device)
    base = dict(c=c, ldc=C, ws=ws, ws_bytes=need)
    cases = {  # name -> (overrides, status, message)
        "null_handle": (dict(h=ctypes.c_void_p(0)), E.ZK_EINVAL, "null handle"),
        "negative_B": (dict(B=-1), E.ZK_EINVAL, "B=-1"),
        "trace_3": (dict(trace=3), E.ZK_EINVAL, "unknown trace 3"),
        "trace_-1": (dict(trace=-1), E.ZK_EINVAL, "unknown trace -1"),
        "ladj_without_trace": (dict(trace=R.TRACE_NONE), E.ZK_EINVAL, "ladj must be NULL"),
        "no_ladj_with_trace": (dict(ladj=None), E.ZK_EINVAL, "ladj must be NULL"),
        "hutchinson_without_eps": (dict(trace=R.TRACE_HUTCHINSON), E.ZK_EINVAL, "Hutchinson needs eps"),
        "hutchinson_short_ldeps": (dict(trace=R.TRACE_HUTCHINSON, eps=eps, ldeps=D - 1), E.ZK_EINVAL, "Hutchinson"),
        "max_trials_0": (dict(max_trials=0), E.ZK_EINVAL, "max_trials=0"),
        "null_times": (dict(times=0), E.ZK_EINVAL, "null times"),
        "null_x": (dict(x=None), E.ZK_EINVAL, "bad x / y"),
        "null_y": (dict(y=None), E.ZK_EINVAL, "bad x / y"),
        "short_ldx": (dict(ldx=D - 1), E.ZK_EINVAL, "bad x / y"),
        "short_ldy": (dict(ldy=D - 1), E.ZK_EINVAL, "bad x / y"),
        "short_ldc": (dict(ldc=C - 1), E.ZK_EINVAL, "bad context"),
        "null_context": (dict(c=None), E.ZK_EINVAL, "bad context"),
        "null_workspace": (dict(ws=0), E.ZK_EINVAL, "workspace"),
        "workspace_one_byte_short": (dict(ws_bytes=E.lib().zk_cnf_workspace_bytes(h, B, 1) - 1), E.ZK_EINVAL, "workspace"),
        "workspace_misaligned": (dict(ws=ws.data_ptr() + 128), E.ZK_EINVAL, "workspace"),
    }
    for name, (over, status, msg) in cases.items():
        y = torch.full((B, D), NAN, device=device)
        ladj = torch.full((B,), NAN, device=device)
        counts = torch.full((2,), 77, dtype=torch.int32, device=device)
        kw = {**base, "x": x, "y": y, "ladj": ladj, "counts": counts, **over}
        st = raw(eng, kw.pop("x"), kw.pop("B", B), **kw)
        assert st == status, name
        assert msg in last_error(), (name, last_error())
        torch.cuda.synchronize()
        assert torch.isnan(y).all() and torch.isnan(ladj).all() and counts.tolist() == [77, 77], name
    assert plan(None, 1, 1)[0] == E.ZK_EINVAL
    assert plan(h, -1, 1)[0] == E.ZK_EINVAL
    assert plan(h, 1, 3)[0] == E.ZK_EINVAL and "unknown trace 3" in last_error()
    assert E.lib().zk_cnf_workspace_bytes(None, 1, 1) == 0 and E.lib().zk_cnf_workspace_bytes(h, -1, 1) == 0


def create(desc, D, C, F, freqs, out=True):
    h = ctypes.c_void_p()
    st = E.lib().zk_cnf_create(None if desc is None else ctypes.byref(desc), D, C, F, freqs,
                               ctypes.byref(h) if out else None)  # fmt: skip
    if st == E.ZK_OK:
        E.lib().zk_cnf_destroy(h)
    return st


@pytest.mark.gpu
def test_create_refusals(device):
    eng = make(device, 4, 3)
    D, C, F = 4, 3, 3
    fr = eng.t.freqs.contiguous()
    desc, keep = eng.t.ode.mlp_desc()
    n = desc.n_linear
    assert create(desc, D, C, F, fr.data_ptr()) == E.ZK_OK

    def variant(**kw):
        d = E.MlpDesc.from_buffer_copy(desc)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    ones = (ctypes.c_int * n)(*([1] * n))
    zeros = (ctypes.c_int * n)()
    dims = list(desc.dims[: n + 1])
    bad_in, bad_out, bad_hidden = (ctypes.c_int * (n + 1))(*dims), (ctypes.c_int * (n + 1))(*dims), (ctypes.c_int * (n + 1))(*dims)  # fmt: skip
    bad_in[0] += 1
    bad_out[n] += 1
    bad_hidden[1] = 0
    no_w = (ctypes.c_void_p * n)(*desc.weight[:n])
    no_w[1] = None
    mask = (ctypes.c_void_p * n)()
    mask[1] = desc.weight[1]
    keep += [ones, zeros, bad_in, bad_out, bad_hidden, no_w, mask]
    cases = {  # name -> (desc, D, C, F, freqs, status, message)
        "null_desc": (None, D, C, F, fr.data_ptr(), E.ZK_EINVAL, "null argument"),
        "features_0": (desc, 0, C, F, fr.data_ptr(), E.ZK_EINVAL, "features=0"),
        "context_-1": (desc, D, -1, F, fr.data_ptr(), E.ZK_EINVAL, "context=-1"),
        "freqs_33": (desc, D, C, 33, fr.data_ptr(), E.ZK_EINVAL, "freqs=33"),
        "freqs_-1": (desc, D, C, -1, fr.data_ptr(), E.ZK_EINVAL, "freqs=-1"),
        "null_freq_values": (desc, D, C, F, None, E.ZK_EINVAL, "null freq_values"),
        "no_layers": (variant(n_linear=0), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "bad MLP descriptor"),
        "null_dims": (variant(dims=None), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "bad MLP descriptor"),
        "null_weights": (variant(weight=None), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "bad MLP descriptor"),
        "activation_1": (variant(activation=1), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "unknown activation 1"),
        "activation_-1": (variant(activation=-1), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "unknown activation -1"),
        "activation_9": (variant(activation=9), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "unknown activation 9"),
        "layer_act": (variant(layer_act=ones), D, C, F, fr.data_ptr(), E.ZK_EUNSUPPORTED, "residual"),
        "layer_res": (variant(layer_res=zeros), D, C, F, fr.data_ptr(), E.ZK_EUNSUPPORTED, "residual"),
        "input_width": (variant(dims=bad_in), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "do not match"),
        "output_width": (variant(dims=bad_out), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "do not match"),
        "features_mismatch": (desc, D, C + 1, F, fr.data_ptr(), E.ZK_EINVAL, "do not match"),
        "hidden_width_0": (variant(dims=bad_hidden), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "bad layer 0"),
        "null_layer_weight": (variant(weight=no_w), D, C, F, fr.data_ptr(), E.ZK_EINVAL, "bad layer 1"),
        "masked": (variant(mask=mask), D, C, F, fr.data_ptr(), E.ZK_EUNSUPPORTED, "masked"),
    }
    for name, (d, Dd, Cc, Ff, fv, status, msg) in cases.items():
        assert create(d, Dd, Cc, Ff, fv) == status, name
        assert msg in last_error(), (name, last_error())
    assert create(desc, D, C, F, fr.data_ptr(), out=False) == E.ZK_EINVAL
    deep = make(device, 4, 3, hidden=(8,) * 16)
    d17, keep17 = deep.t.ode.mlp_desc()
    assert d17.n_linear == 17
    assert create(d17, D, C, F, fr.data_ptr()) == E.ZK_EUNSUPPORTED and "17 linear layers" in last_error()
    del keep, keep17


# --------------------------------------------------------------------------- #
# 7. the Python layer
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
def test_leading_dimensions_and_context_forms(device):
    eng = make(device, 3, 4, 3, (32, 32), "SiLU")
    S, B, D, C = 3, 20, 3, 4
    rng = np.random.default_rng(15)
    x = torch.as_tensor(rng.standard_normal((S, B, D)), dtype=torch.float32, device=device)
    cb = torch.as_tensor(rng.standard_normal((B, C)), dtype=torch.float32, device=device)
    big = torch.full((S, B, C + 5), NAN, device=device)
    big[..., 2 : 2 + C] = torch.as_tensor(rng.standard_normal((S, B, C)), dtype=torch.float32, device=device)
    tposed = torch.as_tensor(rng.standard_normal((C, B, S)), dtype=torch.float32, device=device).permute(2, 1, 0)
    forms = {
        "rows": (cb, cb.expand(S, B, C)),
        "vector": (cb[0], cb[0].expand(S, B, C)),
        "one_row": (cb[:1], cb[:1].expand(S, B, C)),
        "padded_view": (big[..., 2 : 2 + C], big[..., 2 : 2 + C]),
        "transposed_view": (tposed, tposed),
    }
    for name, (c, rows) in forms.items():
        with torch.no_grad():
            t = eng.flow(c).transform
            z, ladj = t.call_and_ladj(x)
        ref = eng.run(x.reshape(-1, D), rows.reshape(-1, C).contiguous())
        assert z.shape == (S, B, D) and ladj.shape == (S, B), name
        assert torch.equal(z.reshape(-1, D), ref[0]) and torch.equal(ladj.reshape(-1), ref[1]), name
        assert t.stats == ref[2], name


@pytest.mark.gpu
def test_hutchinson_draw(device):
    eng = make(device, 4, 2, exact=False)
    x, c, _ = inputs(eng, 64, seed=16)
    xt = torch.as_tensor(x, dtype=torch.float32, device=device)
    ct = torch.as_tensor(c, dtype=torch.float32, device=device)
    torch.cuda.manual_seed(123)
    with torch.no_grad():
        z, ladj = eng.flow(ct).transform.call_and_ladj(xt)
    torch.cuda.manual_seed(123)
    eps = torch.randn_like(xt)
    ref = eng.run(xt, ct, R.TRACE_HUTCHINSON, eps=eps)
    assert torch.equal(z, ref[0]) and torch.equal(ladj, ref[1])
    replay_check(eng, x, c, ref, R.TRACE_HUTCHINSON, eps=cpu(eps))


@pytest.mark.gpu
def test_handle_repacked_after_updates(device):
    eng = make(device, 3, 2)
    x, c, _ = inputs(eng, 40, seed=17)
    xt = torch.as_tensor(x, dtype=torch.float32, device=device)
    ct = torch.as_tensor(c, dtype=torch.float32, device=device)

    def result(flow):
        with torch.no_grad():
            return flow(ct).transform.call_and_ladj(xt)

    def fresh():
        f = CNF(3, 2).eval()
        f.load_state_dict(eng.flow.state_dict())
        return f.to(device)

    before = result(eng.flow)
    updates = {
        "weight": lambda: eng.t.ode[2].weight.mul_(1.5),
        "freqs": lambda: eng.t.freqs.mul_(1.25),
        "load_state_dict": lambda: eng.flow.load_state_dict(make(device, 3, 2, seed=5).flow.state_dict()),
    }
    for name, update in updates.items():
        with torch.no_grad():
            update()
        now = result(eng.flow)
        assert not torch.equal(now[0], before[0]), name
        ref = result(fresh())
        assert torch.equal(now[0], ref[0]) and torch.equal(now[1], ref[1]), name
        before = now


@pytest.mark.gpu
def test_sample_fits_where_log_prob_does_not(device):
    eng = make(device, 256, 0)
    h = eng.t._cnf_handle()
    assert plan(h, 1, R.TRACE_NONE)[1][1] == 32 and plan(h, 1, R.TRACE_EXACT)[0] == E.ZK_EUNSUPPORTED
    B = 24
    torch.cuda.manual_seed(5)
    with torch.no_grad():
        s = eng.flow().sample((B,))
    torch.cuda.manual_seed(5)
    z = eng.flow().base.rsample((B,))
    out = eng.run(z, None, R.TRACE_NONE, direction=-1)
    assert torch.equal(s, out[0])
    _check_replay(eng, cpu(z), None, out[0], None, out[3], R.TRACE_NONE, -1)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="does not fit"):
        eng.flow().log_prob(s)


@pytest.mark.gpu
def test_python_refusals(device):
    eng = make(device, 3, 2)
    x = torch.zeros(5, 3, device=device)
    c = torch.zeros(5, 2, device=device)
    t = eng.flow(c).transform
    with torch.no_grad():
        with pytest.raises(TypeError, match="float32"):
            t(x.double())
        with pytest.raises(E.EngineError, match="CUDA"):
            t(x.cpu())
        with pytest.raises(TypeError, match="float32"):
            eng.flow(c.double()).transform(x)
        with pytest.raises(E.EngineError, match="CUDA"):
            eng.flow(c.cpu()).transform(x)
