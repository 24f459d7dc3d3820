"""GPU tests of `zuko_b200.bayesian.BayesianModel`: flows reparameterized with a posterior draw run on the
engine and differentiate through the draw to `means` / `logvars`.

The posterior draws the reference recorded (tests/golden/bayes_*.npz, make_golden_bayes.py) are injected
by the `replay` fixture, so the engine evaluates the very weights the reference evaluated in fp64.  Bars:
log-densities as everywhere (1e-5 relative, cases.assert_log_prob_parity), inverses 1e-5 * max(1, |value|),
transforms the same in fp32 mode and 5e-5 with the split-bf16 conditioner, and every mean / log-variance
gradient within ``max(5e-5, 3 * e32)`` of the fp64 one relative to its largest entry (e32: the reference's own fp32-vs-fp64 deviation, DESIGN §6b)."""

from __future__ import annotations

import numpy as np
import pytest
import torch

import zuko_b200
from zuko_b200.bayesian import BayesianModel

from cases import assert_log_prob_parity, load
from test_bayesian_host import CASES, RecordDraws, adam_curve, bayes_cases, build_bayes

pytestmark = pytest.mark.gpu
MODES = ["fp32", "auto"]
# transform(x) against the fp64 value: the split-bf16 conditioner of "auto" moves the spline outputs of nsf168_hyper by
# 1.6e-5 (measured on an H100 80GB HBM3 at 700 W); its log-densities stay inside the 1e-5 bar
YBAR = {"fp32": 1e-5, "auto": 5e-5}
SIX = [n for n in CASES if n.endswith("35")]


@pytest.fixture
def replay():
    """`replay(g)`: a context in which `torch.randn_like` returns the draws recorded in golden `g`."""

    def make(g):
        return RecordDraws([torch.from_numpy(g[f"eps/{i}"]) for i in range(int(g["n_eps"]))])

    return make


def set_mode(bflow, mode):
    for m in bflow.base.modules():
        if hasattr(m, "gemm_mode") and hasattr(m, "_linears"):
            m.gemm_mode = mode


def cpu(t):
    return t.detach().cpu().numpy().astype(np.float64)


def assert_close_pointwise(ours, ref, rtol, what):
    ours, ref = cpu(ours), np.asarray(ref, np.float64)
    err = np.abs(ours - ref) / np.maximum(np.abs(ref), 1.0)
    assert float(err.max()) <= rtol, f"{what}: max err {float(err.max()):.3e} (bar {rtol:.1e})"


def assert_posterior_grads(bflow, g, what):
    n = len(bflow.means)
    for i, p in enumerate((*bflow.means.values(), *bflow.logvars.values())):
        tag = f"mean/{i}" if i < n else f"logvar/{i - n}"
        ref = g[f"grad/{tag}"].astype(np.float64)
        bar = max(5e-5, 3.0 * float(g[f"err32/{tag}"]))
        err = float(np.abs(cpu(p.grad) - ref).max()) / max(float(np.abs(ref).max()), 1e-30)
        assert err <= bar, f"{what} {tag}: max err {err:.3e} of max|ref| (bar {bar:.1e})"


def check_against_golden(bflow, g, replay, device, what, ybar=1e-5):
    x, c, z, w = (torch.from_numpy(g[k]).to(device) for k in ("x", "c", "z", "w"))
    # a draw of its own first: the recorded one is then allocated where this one was freed, and must still be
    # packed anew rather than served from the layer-handle caches (keyed on data pointers)
    with bflow.reparameterize() as rflow:
        rflow(c).log_prob(x).sum().backward()
    bflow.zero_grad(set_to_none=True)
    with replay(g), bflow.reparameterize() as rflow:
        dist = rflow(c)
        lp = dist.log_prob(x)
        (w * lp).sum().backward()
        with torch.no_grad():
            y = dist.transform(x)
            xi = dist.transform.inv(z)
    assert_log_prob_parity(cpu(lp), g, rtol=1e-5)
    assert_close_pointwise(y, g["y"], ybar, f"{what} transform(x)")
    assert_close_pointwise(xi, g["xinv"], 1e-5, f"{what} transform.inv(z)")
    assert_posterior_grads(bflow, g, what)
    for name, p in bflow.base.named_parameters():  # the drawn ones; the others are the base's own parameters
        if name.replace(".", "-") in bflow.means:
            assert p.grad is None, name


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASES)
def test_reparameterized_flow_matches_reference(device, replay, name, mode):
    g = load(f"bayes_{name}")
    bflow = build_bayes(zuko_b200, name).to(device)
    set_mode(bflow, mode)
    check_against_golden(bflow, g, replay, device, f"{name}/{mode}", YBAR[mode])


@pytest.mark.parametrize("name", ["nsf35", "nsf168_hyper", "tutorial"])
def test_accelerated_reference_model_matches_reference(device, replay, name):
    """`accelerate()` of a BayesianModel (the engine's own stands in for the reference's, which has the same
    class name and layout) reparameterizes through the accelerated flow's source tensors."""
    g = load(f"bayes_{name}")
    src = build_bayes(zuko_b200, name).to(device)
    acc = zuko_b200.accelerate(src)
    check_against_golden(acc, g, replay, device, f"accelerated {name}", YBAR["auto"])


@pytest.mark.parametrize("name", SIX)
def test_reference_properties(device, name):
    """The reference's own test of Bayesian flows (tests/test_bayesian.py:112-221), weight sampling."""
    torch.manual_seed(0)
    bflow = BayesianModel(bayes_cases(zuko_b200)[name][1]()).to(device)
    x, c = torch.randn(256, 3, device=device), torch.randn(5, device=device)

    bflow.zero_grad(set_to_none=True)
    with bflow.reparameterize() as rflow:
        log_p1 = rflow(c).log_prob(x)
        log_p2 = rflow(c).log_prob(x)
    with bflow.reparameterize() as rflow:
        log_p3 = rflow(c).log_prob(x)
    (-log_p3.mean()).backward()
    assert log_p1.shape == (256,) and log_p1.requires_grad
    assert torch.allclose(log_p1, log_p2) and not torch.allclose(log_p1, log_p3)
    for n, p in (*bflow.means.named_parameters(), *bflow.logvars.named_parameters()):
        assert p.grad is not None, n
    for n, p in bflow.base.named_parameters():
        assert p.grad is None, n

    bflow.zero_grad(set_to_none=True)
    sflow = bflow.sample_model()
    log_p1, log_p2 = sflow(c).log_prob(x), sflow(c).log_prob(x)
    log_p3 = bflow.sample_model()(c).log_prob(x)
    assert torch.allclose(log_p1, log_p2) and not torch.allclose(log_p1, log_p3)
    (-log_p1.mean()).backward()
    assert all(p.grad is None for p in bflow.parameters())
    assert all(p.grad is not None for p in sflow.parameters())

    with bflow.reparameterize() as rflow:
        assert rflow(c).sample((32,)).shape == (32, 3)
        xr = rflow(c).rsample()
    xr.square().sum().sqrt().backward()
    for n, p in (*bflow.means.named_parameters(), *bflow.logvars.named_parameters()):
        assert p.grad is not None, n

    x, c = torch.randn(256, 3, device=device), torch.randn(256, 5, device=device)
    with bflow.reparameterize() as rflow:
        t = rflow(c).transform
        assert torch.allclose(x, t.inv(t(x)), atol=1e-4)
        with pytest.raises(NotImplementedError, match="local reparameterization trick"):
            with bflow.reparameterize(local_trick=True):
                pass


def test_backward_over_several_draws(device):
    """S = 3 draws taken one after the other, their losses summed, one backward(): each graph keeps the
    weights of its own draw, so the gradient is the sum of the three single-draw gradients."""
    torch.manual_seed(0)
    bflow = BayesianModel(zuko_b200.flows.NSF(3, 5, hidden_features=[64, 64])).to(device)
    x, c = torch.randn(128, 3, device=device), torch.randn(128, 5, device=device)
    draws = []
    for _ in range(3):
        with RecordDraws() as rec, bflow.reparameterize() as rflow:
            draws.append((rflow(c).log_prob(x).mean(), [e.clone() for e in rec.draws]))
    bflow.zero_grad(set_to_none=True)
    sum(loss for loss, _ in draws).backward()
    together = [p.grad.clone() for p in bflow.parameters() if p.grad is not None]
    separate = None
    for _, eps in draws:
        bflow.zero_grad(set_to_none=True)
        with RecordDraws(eps), bflow.reparameterize() as rflow:
            rflow(c).log_prob(x).mean().backward()
        grads = [p.grad.clone() for p in bflow.parameters() if p.grad is not None]
        separate = grads if separate is None else [a + b for a, b in zip(separate, grads)]
    assert len(together) == len(separate) == 2 * len(bflow.means)
    for a, b in zip(together, separate):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def posterior(model):
    return [*model.means.values(), *model.logvars.values()]


def _draw_case(name, device):
    """A Bayesian model and the call it is evaluated with inside `reparameterize()`."""
    x, c = torch.randn(64, 3, device=device), torch.randn(64, 5, device=device)
    if name == "cnf":
        return BayesianModel(zuko_b200.flows.CNF(3, 5)), lambda r: r(c).log_prob(x)
    if name == "mlp":
        return BayesianModel(zuko_b200.nn.MLP(3, 5, hidden_features=[64, 64])), lambda r: r(x)
    if name == "masked_mlp":
        net = zuko_b200.nn.MaskedMLP(torch.rand(5, 3) < 0.5, hidden_features=[64, 64])
        return BayesianModel(net), lambda r: r(x)
    _, _, _, D, C = bayes_cases(zuko_b200)[name]
    x, c = torch.randn(64, D, device=device), torch.randn(64, C, device=device)
    return build_bayes(zuko_b200, name), lambda r: r(c).log_prob(x)


@pytest.mark.parametrize("name", ["nsf35", "nice35", "tutorial", "cnf", "mlp", "masked_mlp"])
def test_every_draw_is_packed(device, name):
    """Draws taken without autograd are freed when their context closes, and the next draw's weights are
    allocated at the same addresses with the same version: each must still be evaluated with its own
    weights (draw A, draw B, draw A again) — by flow layers, CNF integrations and bare conditioners alike."""
    torch.manual_seed(0)
    model, call = _draw_case(name, device)
    model = model.to(device)
    out = []
    with torch.no_grad():
        for k in ("a", "b", "a"):
            torch.manual_seed(ord(k))
            with model.reparameterize() as r:
                out.append(call(r))
    assert torch.equal(out[0], out[2])
    assert not torch.allclose(out[0], out[1])


def test_cnf_training_through_draws(device):
    """A CNF trained through the adjoint under `reparameterize()`: two draws in a row, each differentiated on
    its own, give the gradients of replaying each draw alone (the second is not served the first's weights)."""
    torch.manual_seed(0)
    bflow = BayesianModel(zuko_b200.flows.CNF(3, 5, adjoint=True)).to(device)
    x, c = torch.randn(64, 3, device=device), torch.randn(64, 5, device=device)
    grads, draws = [], []
    for _ in range(2):
        bflow.zero_grad(set_to_none=True)
        with RecordDraws() as rec, bflow.reparameterize() as rflow:
            rflow(c).log_prob(x).mean().backward()
        draws.append([e.clone() for e in rec.draws])
        grads.append([p.grad.clone() for p in posterior(bflow)])
        fresh = BayesianModel(zuko_b200.flows.CNF(3, 5, adjoint=True)).to(device)
    fresh.load_state_dict(bflow.state_dict())
    fresh.zero_grad(set_to_none=True)
    with RecordDraws(draws[1]), fresh.reparameterize() as rflow:
        rflow(c).log_prob(x).mean().backward()
    for a, b in zip(grads[1], (p.grad for p in posterior(fresh))):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-7)
    assert not all(torch.allclose(a, b) for a, b in zip(grads[0], grads[1]))


def test_tutorial_adam_curve_matches_reference(device):
    """The bayesian_flows tutorial's training loop, 30 Adam steps with the reference's recorded draws: every
    loss within 1e-3 of the reference's fp32 curve."""
    g = load("bayes_tutorial_adam")
    bflow = build_bayes(zuko_b200, "tutorial").to(device)
    x, c = (torch.from_numpy(g[k]).to(device) for k in ("x", "c"))
    n = int(g["n_eps"])
    draws = [[torch.from_numpy(g[f"eps/{k}/{i}"]) for i in range(n)] for k in range(x.shape[0])]
    losses, _ = adam_curve(bflow, x, c, draws)
    ref = g["losses"]
    err = np.abs(np.array(losses) - ref) / np.maximum(np.abs(ref), 1.0)
    assert float(err.max()) <= 1e-3, (float(err.max()), int(err.argmax()))
