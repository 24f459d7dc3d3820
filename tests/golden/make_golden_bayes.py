"""Golden data of tests/test_bayesian_host.py and tests/test_gpu_bayesian.py: the UNMODIFIED reference's
``zuko.bayesian.BayesianModel`` around the flows of ``bayes_cases``, built under the cases' seeds.

Per case: the included keys, CRC32s of the initial means / log-variances (fp32), the state-dict keys, one posterior
draw ``eps`` recorded under ``torch.manual_seed(DRAW_SEED)`` in fp32, and — with that draw replayed in
fp64 — ``log_prob(x)`` (and the reference's fp32 value of it), ``transform(x)``, ``transform.inv(z)``, the gradients of ``sum(w * log_prob(x))``
with respect to every mean and log-variance, and the KL divergence.  ``err32/*`` is the reference's own
fp32-vs-fp64 deviation of each gradient, relative to its largest entry.  bayes_tutorial_adam.npz holds the
tutorial's training loop on the tutorial case (main_adam).  Run with the reference's source
tree as the first argument:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_bayes.py <reference source tree>
"""

from __future__ import annotations

import copy
import sys
from pathlib import Path

import numpy as np
import torch

sys.dont_write_bytecode = True
HERE = Path(__file__).resolve().parent
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))

import zuko  # noqa: E402
import zuko.bayesian  # noqa: E402,F401
from cases import crc  # noqa: E402
from test_bayesian_host import (  # noqa: E402
    DRAW_SEED,
    RecordDraws,
    adam_curve,
    bayes_cases,
    build_bayes,
    case_inputs,
    two_moons_batches,
)


def evaluate(bflow, eps, x, c, z, w):
    """One replayed draw: values and the gradients of the weighted log-density sum."""
    bflow.zero_grad(set_to_none=True)
    with RecordDraws(eps), bflow.reparameterize() as rflow:
        dist = rflow(c)
        lp = dist.log_prob(x)
        (w * lp).sum().backward()
        with torch.no_grad():
            y = dist.transform(x)
            xi = dist.transform.inv(z)
    grads = [p.grad.detach().clone() for p in (*bflow.means.values(), *bflow.logvars.values())]
    return lp.detach(), y, xi, grads


def main() -> None:
    for name, (_, _, _, features, context) in bayes_cases(zuko).items():
        bflow = build_bayes(zuko, name)
        out = {
            "keys": np.array(list(bflow.means.keys()), dtype=np.str_),
            "sd_keys": np.array(list(bflow.state_dict()), dtype=np.str_),
        }
        for i, k in enumerate(bflow.means.keys()):
            out[f"crc/mean/{i}"] = np.array(crc(bflow.means[k]), dtype=np.int64)
            out[f"crc/logvar/{i}"] = np.array(crc(bflow.logvars[k]), dtype=np.int64)
        torch.manual_seed(DRAW_SEED)
        with RecordDraws() as rec, bflow.reparameterize():
            pass
        eps = [e.detach() for e in rec.draws]
        out["n_eps"] = np.array(len(eps))
        for i, e in enumerate(eps):
            out[f"eps/{i}"] = e.numpy()
        x, c, z, w = case_inputs(name, features, context)
        out.update(x=x.numpy(), c=c.numpy(), z=z.numpy(), w=w.numpy())

        b64 = copy.deepcopy(bflow).double()
        lp, y, xi, g64 = evaluate(b64, eps, x.double(), c.double(), z.double(), w.double())
        out.update(log_prob64=lp.numpy(), y=y.numpy(), xinv=xi.numpy(), kl=b64.kl_divergence().detach().numpy())
        lp32, _, _, g32 = evaluate(bflow, eps, x, c, z, w)
        out["log_prob32"] = lp32.numpy()
        n = len(eps)
        for i, (a, b) in enumerate(zip(g64, g32)):
            tag = f"mean/{i}" if i < n else f"logvar/{i - n}"
            out[f"grad/{tag}"] = a.float().numpy()  # fp32 storage: ~1e-7 relative, far inside the bars
            out[f"err32/{tag}"] = np.array(float((a - b.double()).abs().max() / a.abs().max().clamp_min(1e-300)))
        np.savez_compressed(HERE / f"bayes_{name}.npz", **out)
        print(name, len(eps), "draws", "log_prob[:3]", lp[:3].tolist())


def main_adam() -> None:
    """bayes_tutorial_adam.npz: the tutorial model trained for ADAM_STEPS steps in fp32 on seeded two-moons
    batches: every step's draws and loss."""
    bflow = build_bayes(zuko, "tutorial")
    x, c = two_moons_batches()
    torch.manual_seed(DRAW_SEED)
    losses, draws = adam_curve(bflow, x, c)
    out = {"x": x.numpy(), "c": c.numpy(), "losses": np.array(losses), "n_eps": np.array(len(draws[0]))}
    for k, step in enumerate(draws):
        for i, e in enumerate(step):
            out[f"eps/{k}/{i}"] = e.numpy()
    np.savez_compressed(HERE / "bayes_tutorial_adam.npz", **out)
    print("adam", losses[0], losses[-1])


if __name__ == "__main__":
    main()
    main_adam()
