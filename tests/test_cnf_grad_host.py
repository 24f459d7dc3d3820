"""CPU tests of the CNF backward: the fp64 restatement of the adaptive checkpoint adjoint
(tests/cnf_adjoint_reference.py) against the reference's gradient goldens (tests/golden/make_golden_cnf_grad.py)
and a closed form, act'' of every activation against torch's double backward (g++ harness of activations.cuh),
the Python layer's gradient rules, the backward plan's restatement and the C-ABI additions."""

import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy.linalg import expm

import cnf_adjoint_reference as A
import cnf_reference as R
from cases import load
from test_cnf_host import CASES, DEFAULT, field_of
from zuko_b200 import _engine as E
from zuko_b200.flows import CNF, FFJTransform
from zuko_b200.transforms import FreeFormJacobianTransform

ROOT = Path(__file__).resolve().parent.parent

# golden op -> (trace, input key, direction)
GOPS = {
    "lp": (R.TRACE_EXACT, "x", +1),
    "fwd": (R.TRACE_NONE, "x", +1),
    "rs": (R.TRACE_EXACT, "z", -1),
    "hut": (R.TRACE_HUTCHINSON, "x", +1),
}
# the stiff cases (weights x3): their ~30 steps of a 3x stiffer field amplify the fp64 rounding of the restatement
# and of the reference's autograd, so they are held to 1e-7 of the largest entry instead of the default cases' 1e-9
STIFF_BAR = 1e-7


def relmax(ours, ref) -> float:
    """Largest error relative to the largest entry of ref."""
    ours, ref = np.asarray(ours, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(ours - ref)) / max(np.max(np.abs(ref)), 1e-30))


def golden_grads(g: dict, op: str, tag: str) -> dict:
    p = f"g_{op}_{tag}/"
    return {k[len(p) :]: v for k, v in g.items() if k.startswith(p)}


def gap(g: dict, op: str, key: str) -> float:
    """The reference's own fp32-fp64 gap of one gradient tensor."""
    return relmax(g[f"g_{op}_32/{key}"], g[f"g_{op}_64/{key}"])


def back_plan(D: int, C: int, F: int, dims: list, trace: int):
    """numpy restatement of cnf_back_geometry: (threads, shared memory bytes), or None when refused."""
    nl = len(dims) - 1
    pads = [-(-dims[i + 1] // 8) * 8 for i in range(nl)]
    wfloats = sum(dims[i] * pads[i] + pads[i] for i in range(nl))
    S = max(D + C, *pads)
    hidden = sum(pads[:-1])
    tf = D + C + 2 * hidden + 3 * S + (3 * hidden + D if trace else 0)
    best = None
    for nt in (256, 128, 64, 32):
        s = (wfloats + 7 * 2 * 32 + nt + (nt + 1) * tf) * 4
        if s > 232448:
            continue
        res = min(233472 // (s + 1024), 2048 // nt, 32) * nt
        if best is None or res > best[0]:
            best = (res, nt, s)
    return None if best is None else best[1:]


def restated(g: dict, op: str, tag: str):
    """The restatement's gradients of a golden op at the golden's own step log of dtype `tag`."""
    trace, key, _ = GOPS["lp" if op in ("eval", "bcast") else op]
    field = field_of(g)
    inp = g[key].astype(np.float64)
    c = g.get("c")
    if op == "bcast":
        c = c[0]
    lg = g[f"log_{op}_{tag}"]
    eps = g[f"hut_eps_{tag}"].astype(np.float64) if op == "hut" else None
    if op in ("lp", "eval", "bcast"):
        y = R.replay(field, inp, c, lg, trace)[0]
        w = g["w"].astype(np.float64)
        gy, gl = -w[:, None] * y, w
    else:
        gy, gl = g["gy"].astype(np.float64), (g["gl"].astype(np.float64) if trace else None)
    out = A.adjoint(field, inp, c, lg, trace, eps, gy, gl)
    res = {"in0": out["x"]}
    if out["c"] is not None:
        res["in1"] = out["c"].sum(0) if op == "bcast" else out["c"]
    for i in range(len(out["W"])):
        res[f"ode.{2 * i}.weight"] = out["W"][i]
        res[f"ode.{2 * i}.bias"] = out["b"][i]
    return res


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("op", [*GOPS, "bcast"])
def test_restatement_reproduces_reference_fp64(name, op):
    g = load(f"cnfgrad_{name}")
    if f"log_{op}_64" not in g:
        pytest.skip("no context")
    gold = golden_grads(g, op, "64")
    ours = restated(g, op, "64")
    bar = 1e-9 if name in DEFAULT else STIFF_BAR
    assert set(ours) == set(gold)
    for k in gold:
        assert relmax(ours[k], gold[k]) <= bar, (k, relmax(ours[k], gold[k]))


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("op", list(GOPS))
def test_replay_of_fp32_steps_matches_fp32_goldens(name, op):
    """At the fp32 run's own steps the fp64 restatement lands within the reference's fp32 rounding: the basis of
    the GPU bar."""
    g = load(f"cnfgrad_{name}")
    gold = golden_grads(g, op, "32")
    ours = restated(g, op, "32")
    for k in gold:
        assert relmax(ours[k], gold[k]) <= max(20 * gap(g, op, k), 1e-4), (k, relmax(ours[k], gold[k]), gap(g, op, k))


def test_eval_mode_goldens_give_parameters_no_grad():
    g = load("cnfgrad_cnf35")
    assert set(golden_grads(g, "eval", "64")) == {"in0", "in1"}
    np.testing.assert_allclose(g["g_eval_64/in0"], g["g_lp_64/in0"], rtol=1e-12, atol=1e-12)


def test_one_layer_linear_field_against_closed_form():
    """hidden_features=[]: f = W0 [emb(t), x, c] + b0 is linear in x, so d x(1) / d x(0) = expm(A) with A = W0[:, x]
    and grad_x = expm(A)^T gy; the trace is constant, so grad_ladj adds nothing to grad_x."""
    torch.manual_seed(0)
    flow = CNF(3, 2, hidden_features=[])
    sd = {k: v.double().numpy() for k, v in flow.state_dict().items()}
    field = R.Field.from_state_dict(sd, 3, 2, "ReLU")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, generator=g, dtype=torch.float64).numpy()
    c = torch.randn(16, 2, generator=g, dtype=torch.float64).numpy()
    gy = torch.randn(16, 3, generator=g, dtype=torch.float64).numpy()
    gl = torch.randn(16, generator=g, dtype=torch.float64).numpy()
    _, _, log = R.integrate(field, x, c, 0.0, 1.0, 1e-10, 1e-10, R.TRACE_EXACT)
    out = A.adjoint(field, x, c, log, R.TRACE_EXACT, None, gy, gl)
    Amat = field.W[0][:, 6:9]
    np.testing.assert_allclose(out["x"], gy @ expm(Amat), rtol=0, atol=1e-8)
    # d ladj / d W0[i, x_i] = 1 per row (tau = tr A), so the diagonal of that block carries sum(gl) on top
    blk = out["W"][0][:, 6:9]
    gy0 = A.adjoint(field, x, c, log, R.TRACE_NONE, None, gy, None)["W"][0][:, 6:9]
    np.testing.assert_allclose(blk - gy0, np.eye(3) * gl.sum(), rtol=0, atol=1e-8)


def test_piecewise_linear_gradients_jump_under_fp32_noise():
    """With ReLU the field is piecewise linear: its Jacobian jumps where a pre-activation changes sign, so input
    noise of fp32 size (2e-6 relative) moves the fp64 gradients by far more than 1e-4 once a kink is crossed at a
    different point; with ELU they move by ~1e-6.  This is why the GPU tests hold ReLU and LeakyReLU to a looser,
    measured bar than the smooth activations."""
    moved = {}
    for act in ("ReLU", "ELU"):
        torch.manual_seed(0)
        flow = CNF(3, 2, activation=getattr(torch.nn, act))
        field = R.Field.from_state_dict({k: v.double().numpy() for k, v in flow.state_dict().items()}, 3, 2, act)
        g = torch.Generator().manual_seed(3)
        x, c = torch.randn(48, 3, generator=g).numpy(), torch.randn(48, 2, generator=g).numpy()
        gy, gl = torch.randn(48, 3, generator=g).numpy(), torch.randn(48, generator=g).numpy()
        _, _, log = R.integrate(field, x.astype(np.float64), c, 0.0, 1.0, 1e-6, 1e-5, R.TRACE_EXACT)
        a = A.adjoint(field, x, c, log, R.TRACE_EXACT, None, gy, gl)
        noise = 1 + 2e-6 * np.random.default_rng(0).standard_normal(x.shape)
        b = A.adjoint(field, x * noise, c, log, R.TRACE_EXACT, None, gy, gl)
        moved[act] = max(relmax(b["c"], a["c"]), *(relmax(u, v) for u, v in zip(b["W"] + b["b"], a["W"] + a["b"], strict=True)))
    assert moved["ReLU"] > 1e-4 and moved["ELU"] < 1e-5, moved


@pytest.fixture(scope="module")
def act_harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libact_host.so"
    src = ROOT / "tests" / "native" / "act_deriv2_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so), "-lm"], check=True)
    lib = ctypes.CDLL(str(so))
    P = ctypes.c_void_p
    lib.act_derivs.argtypes = [P, ctypes.c_int64, ctypes.c_int, P, P]
    return lib


@pytest.mark.parametrize("name,code", [("ReLU", 1), ("ELU", 2), ("Tanh", 3), ("SiLU", 4), ("GELU", 5), ("LeakyReLU", 6),
                                       ("Softplus", 7), ("Sigmoid", 8)])  # fmt: skip
def test_act_deriv2_against_torch_double_backward(act_harness, name, code):
    v = np.concatenate([np.linspace(-8, 8, 161), [0.0, -0.0, 1e-3, -1e-3, 19.999, 20.0, 20.001, 25.0, -25.0]]).astype(np.float32)
    d1, d2 = np.empty_like(v), np.empty_like(v)
    act_harness.act_derivs(v.ctypes.data, v.size, code, d1.ctypes.data, d2.ctypes.data)
    vt = torch.tensor(v, dtype=torch.float64, requires_grad=True)
    (g1,) = torch.autograd.grad(getattr(torch.nn, name)()(vt).sum(), vt, create_graph=True)
    (g2,) = torch.autograd.grad(g1.sum(), vt, allow_unused=True)
    g2 = torch.zeros_like(vt) if g2 is None else g2
    np.testing.assert_allclose(d1, g1.detach().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(d2, g2.numpy(), rtol=1e-5, atol=1e-6)


def test_adjoint_option_is_opt_in_and_carried():
    t = FFJTransform(2, 1)
    assert t.adjoint is False
    c = torch.randn(1)
    x = torch.randn(3, 2, requires_grad=True)
    with pytest.raises(NotImplementedError, match="adjoint=True"):
        t(c)(x)
    t.adjoint = True
    ft = t(c)
    assert ft.adjoint and ft.inv.adjoint and ft.inv.inv.adjoint
    assert FFJTransform(2, 1, adjoint=True)(c).adjoint
    # training mode: phi = (c, *parameters); eval mode: (c,)
    cg = torch.randn(1, requires_grad=True)
    assert len(t.train()(cg).phi) == 1 + len(list(t.parameters()))
    assert t.eval()(cg).phi == (cg,)
    # integration times that require grad are refused before anything runs
    f = FreeFormJacobianTransform(t(c).f, torch.tensor(0.0, requires_grad=True), 1.0, (), adjoint=True)
    with pytest.raises(NotImplementedError, match="times"):
        f(x)
    # no gradient needed: today's path (the CPU tensor then meets the engine's CUDA requirement)
    with torch.no_grad(), pytest.raises(E.EngineError, match="CUDA"):
        f(x)


def test_backward_plan_restatement_cases():
    # CNF(16, 8), hidden (64, 64): one 32-thread CTA per SM with a trace, 64 threads without
    assert back_plan(16, 8, 3, [30, 64, 64, 16], R.TRACE_EXACT) == (32, 145760)
    assert back_plan(16, 8, 3, [30, 64, 64, 16], R.TRACE_HUTCHINSON) == (32, 145760)
    assert back_plan(16, 8, 3, [30, 64, 64, 16], R.TRACE_NONE) == (64, 153504)
    assert back_plan(2, 1, 3, [9, 16, 16, 2], R.TRACE_EXACT)[0] == 256
    assert back_plan(16, 8, 3, [30, 512, 512, 16], R.TRACE_EXACT) is None


def test_c_abi_symbols():
    for name in ("zk_cnf_backward_workspace_bytes", "zk_cnf_backward_min_workspace_bytes", "zk_cnf_backward_plan",
                 "zk_cnf_backward"):  # fmt: skip
        assert name in E.EXPORTED_SYMBOLS
