"""Gaussian mixture model benchmark: GMM(16, 8, components=8), full and diagonal covariance, with the default
conditioner (64, 64) and with [256] * 3 hidden layers, at 2^16 and 2^20 rows.

Per workload one JSON line: ``log_prob`` without gradients, ``sample``, or one Adam training step
(``-log_prob(x).mean()``, backward, step).  Each gives the median ms per call over ``--steps`` calls timed with
CUDA events after ``--warmup`` calls, the rows/s, and the card name and power limit.  Fails without CUDA.

    python bench_gmm.py [--steps 20] [--warmup 5]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))

import zuko_b200 as zuko  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout  # fmt: skip
    name, power = (s.strip() for s in q.split(",", 1))
    return {"gpu": name, "power_limit": power}


def workload(cov: str, hidden: list[int] | None, op: str, rows: int, args) -> dict:  # noqa: ANN001
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    kw = {} if hidden is None else {"hidden_features": hidden}
    gmm = zuko.mixtures.GMM(16, 8, components=8, covariance_type=cov, **kw).to(dev)
    x, c = torch.randn(rows, 16, device=dev), torch.randn(rows, 8, device=dev)
    opt = torch.optim.Adam(gmm.parameters(), lr=1e-4)

    def step() -> None:
        if op == "log_prob":
            with torch.no_grad():
                gmm(c).log_prob(x)
        elif op == "sample":
            gmm(c).sample()
        else:
            loss = -gmm(c).log_prob(x).mean()
            opt.zero_grad()
            loss.backward()
            opt.step()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.steps):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        step()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    ms = sorted(times)[len(times) // 2]
    return {
        "workload": f"GMM(16, 8, K=8, {cov}, hidden={hidden or [64, 64]})",
        "op": op,
        "rows": rows,
        "ms": round(ms, 4),
        "rows_per_s": round(rows / ms * 1e3, 1),
        **card(),
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gmm.py needs a CUDA device")
    for cov in ("full", "diagonal"):
        for hidden in (None, [256] * 3):
            for op in ("log_prob", "sample", "train"):
                for rows in (1 << 16, 1 << 20):
                    print(json.dumps(workload(cov, hidden, op, rows, args)), flush=True)


if __name__ == "__main__":
    main()
