"""CPU tests of the continuous normalizing flow (CNF): the fp64 restatement of tests/cnf_reference.py against the
reference's goldens (tests/golden/make_golden_cnf.py), constructor parity with the reference under the same
seed, the refusals, and the C-ABI additions."""

import numpy as np
import pytest
import torch

import cnf_reference as R
from cases import crc, load
from zuko_b200 import _engine as E
from zuko_b200.flows import CNF, FFJTransform
from zuko_b200.transforms import FreeFormJacobianTransform

# name -> constructor; must mirror tests/golden/make_golden_cnf.py:CASES
CASES = {
    "cnf35": lambda: CNF(3, 5),
    "cnf168": lambda: CNF(16, 8),
    "cnf5_deep": lambda: CNF(5, 0, hidden_features=[32, 32, 32]),
    "cnf43_tanh": lambda: CNF(4, 3, activation=torch.nn.Tanh),
    "cnf42_f0": lambda: CNF(4, 2, freqs=0),
    "cnf35_stiff": lambda: CNF(3, 5),
    "cnf168_stiff": lambda: CNF(16, 8),
}
DEFAULT = [k for k in CASES if not k.endswith("_stiff")]
OPS = {  # golden key -> (trace, input key, direction)
    "lp": (R.TRACE_EXACT, "x", +1),
    "fwd": (R.TRACE_NONE, "x", +1),
    "inv": (R.TRACE_NONE, "z", -1),
    "rs": (R.TRACE_EXACT, "z", -1),
    "hut": (R.TRACE_HUTCHINSON, "x", +1),
}


def field_of(g: dict) -> R.Field:
    sd = {k[3:]: v for k, v in g.items() if k.startswith("sd/")}
    return R.Field.from_state_dict(sd, int(g["D"]), int(g["C"]), str(g["act"]))


def outputs(g: dict, op: str, y, ladj, inp) -> dict:
    """The golden quantities of `op` from an integration's (y, ladj)."""
    if op == "lp":
        return {"lp": R.log_normal(y) + ladj}
    if op == "fwd":
        return {"fwd": y}
    if op == "inv":
        return {"inv": y}
    if op == "rs":
        return {"rs_x": y, "rs_lp": R.log_normal(inp) - ladj}
    return {"hut_y": y, "hut_ladj": ladj}


def rel(ours, ref) -> float:
    ours, ref = np.asarray(ours, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(ours - ref) / np.maximum(np.abs(ref), 1.0)))


@pytest.mark.parametrize("name", list(CASES))
def test_constructor_matches_reference_state_dict(name):
    g = load(f"flow_{name}")
    torch.manual_seed(0)
    sd = CASES[name]().state_dict()
    assert list(sd.keys()) == [str(k) for k in g["sd_keys"]]
    assert [crc(v) for v in sd.values()] == [int(v) for v in g["sd_crc"]]


def test_module_tree():
    flow = CNF(3, 4)
    assert isinstance(flow.transform, FFJTransform)
    assert [type(m).__name__ for m in flow.transform.ode] == ["Linear", "ELU", "Linear", "ELU", "Linear"]
    assert flow.transform.ode[0].weight.shape == (64, 13)
    assert torch.equal(flow.transform.times, torch.tensor([0.0, 1.0]))
    assert torch.equal(flow.transform.freqs, torch.arange(1, 4) * torch.pi)
    assert flow.transform.atol == 1e-6 and flow.transform.rtol == 1e-5 and flow.transform.exact


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("op", list(OPS))
def test_restatement_reproduces_reference_fp64(name, op):
    """The restatement with its own fp64 controller takes the reference's fp64 trial sequence and lands on its
    values: 1e-10, and 2e-6 on the stiff cases, whose 30 to 40 steps amplify the different summation order of
    the reference's vector-Jacobian trace (measured worst: 9.2e-7, Hutchinson ladj of cnf168_stiff)."""
    g = load(f"flow_{name}")
    trace, key, direction = OPS[op]
    inp = g[key].astype(np.float64)
    c = g.get("c")
    eps = g["hut_eps_64"] if op == "hut" else None
    t0, t1 = (0.0, 1.0) if direction > 0 else (1.0, 0.0)
    y, ladj, log = R.integrate(field_of(g), inp, c, t0, t1, float(g["atol"]), float(g["rtol"]), trace, eps)
    ref_log = g[f"log_{op}_64"]
    assert len(log) == len(ref_log)
    np.testing.assert_array_equal(np.array([r[3] for r in log], np.float64), ref_log[:, 3])
    for k, v in outputs(g, op, y, ladj, inp).items():
        assert rel(v, g[f"{k}_64"]) <= (1e-10 if name in DEFAULT else 2e-6), k


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("tag", ["32", "64"])
def test_controller_recomputes_reference_steps(name, op, tag):
    """t and dt of every trial, bit for bit, from the logged errors alone."""
    g = load(f"flow_{name}")
    log = g[f"log_{op}_{tag}"]
    t0, t1 = (0.0, 1.0) if OPS[op][2] > 0 else (1.0, 0.0)
    dtype = np.float32 if tag == "32" else np.float64
    steps = R.controller(t0, t1, log[:, 2], dtype)
    assert len(steps) == len(log)
    for (t, dt, acc), row in zip(steps, log, strict=True):
        assert (float(t), float(dt), float(acc)) == (row[0], row[1], row[3])


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("op", list(OPS))
def test_replay_of_fp32_steps_matches_fp32_goldens(name, op):
    """Replaying the reference's fp32 accepted steps in fp64 lands within 1e-5 of its fp32 values: the basis of
    the GPU tests, which compare the engine at its own step sequence."""
    g = load(f"flow_{name}")
    trace, key, _ = OPS[op]
    inp = g[key].astype(np.float64)
    eps = g["hut_eps_32"].astype(np.float64) if op == "hut" else None
    y, ladj = R.replay(field_of(g), inp, g.get("c"), g[f"log_{op}_32"], trace, eps)
    for k, v in outputs(g, op, y, ladj, inp).items():
        assert rel(g[f"{k}_32"], v) <= 1e-5, k


def test_refusals():
    with pytest.raises(NotImplementedError):
        CNF(3, 2, normalize=True)
    with pytest.raises(NotImplementedError):
        CNF(3, 2, activation=torch.nn.Hardtanh)
    with pytest.raises(NotImplementedError):
        FreeFormJacobianTransform(lambda t, x: x)


def test_gradient_refusal_rule_follows_reference_phi():
    """Training mode puts the ODE parameters in phi (flows/continuous.py:99-103); eval mode only c."""
    t = FFJTransform(2, 1)
    c = torch.randn(1)
    assert len(t(c).phi) == len(list(t.parameters()))
    assert t.eval()(c).phi == ()
    x = torch.randn(3, 2, requires_grad=True)
    with pytest.raises(NotImplementedError, match="adjoint"):
        t(c)(x)
    with pytest.raises(NotImplementedError, match="adjoint"):
        t.train()(c).call_and_ladj(torch.randn(3, 2))


def test_c_abi_symbols():
    for name in ("zk_cnf_create", "zk_cnf_destroy", "zk_cnf_workspace_bytes", "zk_cnf_plan", "zk_cnf_integrate"):
        assert name in E.EXPORTED_SYMBOLS
    assert (E.ZK_CNF_TRACE_NONE, E.ZK_CNF_TRACE_EXACT, E.ZK_CNF_TRACE_HUTCHINSON) == (0, 1, 2)
