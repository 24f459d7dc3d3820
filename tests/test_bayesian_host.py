"""`zuko_b200.bayesian.BayesianModel` on the CPU: constructor, state-dict and draw-order parity with the
reference, recorded in tests/golden/bayes_*.npz by make_golden_bayes.py.  The cases are built here with
either package (the reference's `zuko` or `zuko_b200`) under the seeds the goldens used; the GPU tests
(test_gpu_bayesian.py) evaluate them against the reference's fp64 values."""

from __future__ import annotations

import pickle

import numpy as np
import pytest
import torch

import zuko_b200
from zuko_b200.bayesian import BayesianModel, _compile, _match

from cases import crc, load

DRAW_SEED = 1234  # torch.manual_seed before the posterior draw the goldens recorded


def bayes_cases(zuko):
    """name -> (seed, flow constructor, BayesianModel keyword arguments, features, context)."""
    F = zuko.flows
    six = {
        f"{F_.__name__.lower()}35": (0, (lambda F_=F_: F_(3, 5)), {}, 3, 5)
        for F_ in (F.NICE, F.MAF, F.NSF, F.SOSPF, F.GF, F.BPF)
    }
    return {
        **six,
        # conditioner weights only, on layers wide enough for the tensor-core GEMMs, with a posterior wide
        # enough that the draw moves the density
        "nsf168_hyper": (0, lambda: F.NSF(16, 8, transforms=2, bins=8, hidden_features=[64, 64]),
                         dict(init_logvar=-5.0, include_params=["**.hyper.*"]), 16, 8),
        # the bayesian_flows tutorial's model: the output layer's weights only
        "tutorial": (0, lambda: F.NSF(2, 1, transforms=3, hidden_features=(64, 64)),
                     dict(include_params=["**.hyper.4"], exclude_params=["**.bias"]), 2, 1),
    }  # fmt: skip


def build_bayes(zuko, name):
    seed, ctor, kwargs, _, _ = bayes_cases(zuko)[name]
    torch.manual_seed(seed)
    return zuko.bayesian.BayesianModel(ctor(), **kwargs)


def case_inputs(name, features, context, rows=64):
    """x, c, z (base-space points) and the per-row weights of the differentiated sum, seeded per case."""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(rows, features, generator=g)
    c = torch.randn(rows, context, generator=g)
    z = torch.randn(rows, features, generator=g)
    w = torch.rand(rows, generator=g)
    return x, c, z, w


ADAM_STEPS = 30


def two_moons_batches(steps=ADAM_STEPS, rows=64):
    """Seeded batches of the bayesian_flows tutorial's two-moons data: (x (steps, rows, 2), c (steps, rows, 1))."""
    g = torch.Generator().manual_seed(5)
    theta = 2 * torch.pi * torch.rand(steps, rows, generator=g)
    label = (theta > torch.pi).float()
    x = torch.stack((torch.cos(theta) + label - 1 / 2, torch.sin(theta) + label / 2 - 1 / 4), dim=-1)
    return x + 0.1 * torch.randn(x.shape, generator=g), label.unsqueeze(-1)


def adam_curve(bflow, x, c, draws=None):
    """The tutorial's training loop (Adam, lr 1e-3, loss -log_prob + 1e-6 KL) over the given batches; with
    `draws`, step k replays draws[k].  Returns the losses and the draws taken."""
    opt = torch.optim.Adam(bflow.parameters(), lr=1e-3)
    losses, taken = [], []
    for k in range(x.shape[0]):
        kl = bflow.kl_divergence()
        with RecordDraws(None if draws is None else draws[k]) as rec, bflow.reparameterize() as rflow:
            loss = -rflow(c[k]).log_prob(x[k]).mean() + 1e-6 * kl
            loss.backward()
        opt.step()
        opt.zero_grad()
        losses.append(float(loss.detach()))
        taken.append([e.detach().cpu() for e in rec.draws])
    return losses, taken


class RecordDraws:
    """Replaces ``torch.randn_like`` while active: records each draw, or replays recorded ones (checking
    that the shapes are asked for in the recorded order)."""

    def __init__(self, replay=None):
        self.replay = None if replay is None else list(replay)
        self.draws = []

    def __call__(self, t, **kwargs):
        if self.replay is None:
            out = self._orig(t, **kwargs)
        else:
            assert self.replay, "more draws than recorded"
            out = self.replay.pop(0).to(device=t.device, dtype=t.dtype)
            assert out.shape == t.shape, (out.shape, t.shape)
        self.draws.append(out)
        return out

    def __enter__(self):
        self._orig = torch.randn_like
        torch.randn_like = self
        return self

    def __exit__(self, *exc):
        torch.randn_like = self._orig
        assert exc[0] is not None or not self.replay, f"{len(self.replay)} recorded draws left unused"


CASES = list(bayes_cases(zuko_b200))


@pytest.fixture(scope="module")
def goldens():
    return {name: load(f"bayes_{name}") for name in CASES}


@pytest.mark.parametrize("name", CASES)
def test_constructor_matches_reference(goldens, name):
    """Same included parameters, keys in the same order, bit-identical means and log-variances."""
    g = goldens[name]
    bflow = build_bayes(zuko_b200, name)
    keys = [str(k) for k in g["keys"]]
    assert list(bflow.means.keys()) == keys and list(bflow.logvars.keys()) == keys
    for i, k in enumerate(keys):
        assert crc(bflow.means[k]) == int(g[f"crc/mean/{i}"]), k
        assert crc(bflow.logvars[k]) == int(g[f"crc/logvar/{i}"]), k
    sd = bflow.state_dict()
    assert list(sd) == [str(k) for k in g["sd_keys"]]


@pytest.mark.parametrize("name", CASES)
def test_draws_follow_reference_order(goldens, name):
    """Under the goldens' seed, `reparameterize()` asks for the reference's draws in the reference's order
    and gets its values bit for bit."""
    g = goldens[name]
    bflow = build_bayes(zuko_b200, name)
    torch.manual_seed(DRAW_SEED)
    with RecordDraws() as rec, bflow.reparameterize():
        pass
    n = int(g["n_eps"])
    assert len(rec.draws) == n
    for i, e in enumerate(rec.draws):
        assert np.array_equal(e.numpy(), g[f"eps/{i}"]), i


@pytest.mark.parametrize("name", ["nsf35", "tutorial"])
def test_kl_divergence_matches_reference(goldens, name):
    bflow = build_bayes(zuko_b200, name).double()
    np.testing.assert_allclose(float(bflow.kl_divergence().detach()), float(goldens[name]["kl"]), rtol=1e-12)


def test_patterns_follow_reference_rules():
    """`*` is one name component, `**` any dotted run, a prefix matches what starts with it."""
    name = "transform.transforms.0.hyper.4.weight"
    hits = {"": True, "transform": True, "**.hyper.4": True, "**.hyper.*": True, "*.transforms.0": True,
            "*.hyper": False, "**.hyper.2": False, "transform.transforms.1": False, "**.bias": False}  # fmt: skip
    for prefix, hit in hits.items():
        assert _match(_compile(prefix), name) is hit, prefix
    assert _match(_compile("**.bias"), "transform.transforms.0.hyper.4.bias")
    with pytest.raises(ValueError, match="Invalid prefix"):
        _compile("hyper[0]")


def test_sample_model_and_errors():
    bflow = build_bayes(zuko_b200, "maf35")
    copy_ = bflow.sample_model()
    assert type(copy_) is type(bflow.base) and copy_ is not bflow.base
    assert all(not torch.equal(a, b) for a, b in zip(copy_.parameters(), bflow.base.parameters()))
    with pytest.raises(RuntimeError, match="should not be called directly"):
        bflow(None)
    assert bflow.transform is bflow.base.transform  # attribute lookup falls through to the base
    assert repr(bflow) and pickle.loads(pickle.dumps(bflow)).means.keys() == bflow.means.keys()


def test_local_trick_is_refused():
    """The engine does not implement the local reparameterization trick: asking for it raises before
    any draw, for flows and bare conditioners alike.  Without an included linear layer there is
    nothing to apply it to, as in the reference."""
    for base in (zuko_b200.flows.NSF(3, 5), zuko_b200.nn.MLP(3, 5), zuko_b200.nn.MaskedMLP(torch.rand(5, 3) < 0.5)):
        bm = BayesianModel(base)
        state = torch.random.get_rng_state()
        with pytest.raises(NotImplementedError, match="local reparameterization trick"):
            with bm.reparameterize(local_trick=True):
                pass
        assert torch.equal(state, torch.random.get_rng_state())
    bm = BayesianModel(zuko_b200.flows.NSF(3, 5), exclude_params=["**.weight"])
    with bm.reparameterize(local_trick=True) as rflow:
        assert rflow is bm.base


def test_accelerate_reference_bayesian_model_shares_posterior():
    """A model named like the reference's BayesianModel becomes the engine's, over the accelerated base,
    with the very same `means` / `logvars` tensors (the reference is absent here: the engine's own
    BayesianModel, which has the reference's class name and layout, stands in for it)."""
    src = build_bayes(zuko_b200, "nsf35")
    acc = zuko_b200.accelerate(src)
    assert isinstance(acc, BayesianModel) and isinstance(acc.base, zuko_b200.AcceleratedFlow)
    assert acc.means is src.means and acc.logvars is src.logvars
    assert list(acc.state_dict()) == list(src.state_dict())
    for (ka, a), (kb, b) in zip(acc.base.named_parameters(), src.base.named_parameters()):
        assert ka == kb and a is b
    with acc.reparameterize():
        pass
    for (ka, a), (kb, b) in zip(acc.base.named_parameters(), src.base.named_parameters()):  # the draw is gone again
        assert ka == kb and a is b and a.is_leaf
