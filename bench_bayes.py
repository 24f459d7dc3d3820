"""Benchmark of Bayesian flow training: one JSON line per workload.

Model: the config-2 shape, NSF(16, 8, transforms=4, bins=8, hidden_features=[256] * 3).  Workloads, at 2^16 and
2^20 rows: one Adam training step (forward, backward, optimizer step) of
  - ``plain``: the flow inside ``BayesianModel.reparameterize()`` (one posterior weight draw per step), loss
    ``-log_prob(x).mean() + kl_divergence() / rows``;
  - ``no_bayes``: the same flow without ``BayesianModel``, loss ``-log_prob(x).mean()``.
The local reparameterization trick is not implemented by the engine and has no line.

Per line: step ms from CUDA events around whole steps (warm-up excluded), the number of ``zk_layer_create`` calls
per step (a posterior draw gives every conditioner new weight tensors, which the engine packs into a new layer
handle), and the card name and power limit.

    python bench_bayes.py [--steps 5] [--warmup 2]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from zuko_b200 import _engine as E  # noqa: E402
from zuko_b200.bayesian import BayesianModel  # noqa: E402
from zuko_b200.flows import NSF  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout  # fmt: skip
    name, power = (s.strip() for s in q.split(",", 1))
    return {"gpu": name, "power_limit": power}


class CountCalls:
    """Counts the calls of one engine entry point (the library object caches its functions as attributes)."""

    def __init__(self, name: str) -> None:
        self.lib, self.name, self.fn, self.n = E.lib(), name, getattr(E.lib(), name), 0

    def __call__(self, *args):  # noqa: ANN002, ANN204
        self.n += 1
        return self.fn(*args)

    def __enter__(self):  # noqa: ANN204
        setattr(self.lib, self.name, self)
        return self

    def __exit__(self, *exc) -> None:  # noqa: ANN002
        setattr(self.lib, self.name, self.fn)


def workload(variant: str, rows: int, args) -> dict:  # noqa: ANN001
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    flow = NSF(16, 8, transforms=4, bins=8, hidden_features=[256] * 3)
    model = BayesianModel(flow) if variant == "plain" else flow
    model = model.to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    g = torch.Generator(device="cpu").manual_seed(1)
    x = torch.randn(rows, 16, generator=g).to(dev)
    c = torch.randn(rows, 8, generator=g).to(dev)

    def step() -> None:
        opt.zero_grad(set_to_none=True)
        if variant == "plain":
            with model.reparameterize() as rflow:
                loss = -rflow(c).log_prob(x).mean() + model.kl_divergence() / rows
        else:
            loss = -model(c).log_prob(x).mean()
        loss.backward()
        opt.step()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with CountCalls("zk_layer_create") as creates:
        start.record()
        for _ in range(args.steps):
            step()
        end.record()
        torch.cuda.synchronize()
    return {
        "workload": f"bayes_nsf16_8_{variant}", "rows": rows, "step_ms": start.elapsed_time(end) / args.steps,
        "zk_layer_create_per_step": creates.n / args.steps, **card(),
    }  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bayes.py needs a CUDA device")
    for rows in (1 << 16, 1 << 20):
        for variant in ("plain", "no_bayes"):
            print(json.dumps(workload(variant, rows, args)), flush=True)


if __name__ == "__main__":
    main()
