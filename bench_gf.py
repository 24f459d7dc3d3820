"""Benchmark of the Gaussianization flow (GF) on one GPU.  Prints one JSON line per workload:

* ``gf16_log_prob``: ``GF(16, 8, transforms=3, components=8, hidden_features=[256] * 3)``, ``log_prob`` of 2^20 rows
  with a context row each (the conditioner GEMMs plus one bijector kernel per element-wise layer);
* ``gf64_rsample``: ``GF(64, 0, transforms=4, components=8)``, ``rsample((2^20,))``: four bisection inverses of 25 steps
  each, the part of GF the reference is slowest at.

Each line holds samples/s from CUDA events (best and median over the timed steps), the device time of the forward
and inverse ``uni_kernel`` launches from ``torch.profiler`` (a separate profiled step after the timed ones; the trace
is written under ``--out``), the card's name and power limit, and the error against the fp64 restatement of
tests/gf_reference.py: relative error of ``log_prob`` on the first 2^16 rows, and of the sample against the fp64
bisection on the first 2^12 (the fp64 restatement of 4 x 25 bisection steps over 64 features is slow on the host).
Needs a CUDA device."""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import gf_reference as R  # noqa: E402
import zuko_b200 as zuko  # noqa: E402

CHECK_ROWS = 1 << 16
CHECK_ROWS_INVERSE = 1 << 12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()  # fmt: skip
    name, power = (s.strip() for s in q.split(",", 1))
    return {"gpu": name, "power_limit": power}


def time_steps(fn, warmup: int, steps: int) -> list[float]:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    return times


def uni_kernel_times(fn, trace: Path) -> dict:
    """Device seconds of the forward / inverse uni_kernel launches in one profiled call."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(trace))
    out = {"uni_forward_s": 0.0, "uni_inverse_s": 0.0, "uni_launches": 0}
    for e in prof.events():
        if e.device_type.name != "CUDA" or "uni_kernel<" not in e.name:
            continue
        inverse = e.name.split("uni_kernel<", 1)[1].split(",")[2].strip() == "true"
        out["uni_inverse_s" if inverse else "uni_forward_s"] += e.device_time_total / 1e6
        out["uni_launches"] += 1
    return out


def errors(ours: np.ndarray, ref: np.ndarray) -> dict:
    e = np.abs(np.asarray(ours, np.float64) - ref) / np.maximum(np.abs(ref), 1.0)
    return {"max_rel_err": float(e.max()), "median_rel_err": float(np.median(e)), "rows_checked": int(ref.shape[0])}


def reference(flow, D: int, C: int, K: int) -> R.Flow:
    return R.Flow({k: v.detach().cpu().numpy() for k, v in flow.state_dict().items()}, D, C, K)


def log_prob_workload(args, dev) -> dict:
    D, C, K, B = 16, 8, 8, 1 << args.log2_rows
    torch.manual_seed(0)
    flow = zuko.flows.GF(D, C, transforms=3, components=K, hidden_features=[256] * 3).to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, D, device=dev, generator=g)
    c = torch.randn(B, C, device=dev, generator=g)
    with torch.no_grad():
        fn = lambda: flow(c).log_prob(x)  # noqa: E731
        times = time_steps(fn, args.warmup, args.steps)
        kt = uni_kernel_times(fn, args.out / "trace_gf16_log_prob.json")
        lp = fn()[:CHECK_ROWS].cpu().numpy()
    ref = reference(flow, D, C, K).log_prob(x[:CHECK_ROWS].cpu().numpy(), c[:CHECK_ROWS].cpu().numpy())
    return {"workload": "gf16_log_prob", "rows": B, **rates(B, times), **kt, **errors(lp, ref)}


def rsample_workload(args, dev) -> dict:
    D, K, B = 64, 8, 1 << args.log2_rows
    torch.manual_seed(0)
    flow = zuko.flows.GF(D, 0, transforms=4, components=K).to(dev).eval()
    with torch.no_grad():
        fn = lambda: flow().rsample((B,))  # noqa: E731
        times = time_steps(fn, args.warmup, args.steps)
        kt = uni_kernel_times(fn, args.out / "trace_gf64_rsample.json")
        z = torch.randn(CHECK_ROWS_INVERSE, D, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
        x = flow().transform.inv(z).cpu().numpy()
    ref = reference(flow, D, 0, K).inverse(z.cpu().numpy())
    return {"workload": "gf64_rsample", "rows": B, **rates(B, times), **kt, **errors(x, ref)}


def rates(B: int, times: list[float]) -> dict:
    return {"samples_per_s_best": B / min(times), "samples_per_s_median": B / float(np.median(times)),
            "step_s_best": min(times), "step_s_median": float(np.median(times)), "steps": len(times)}  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log2-rows", type=int, default=20)
    ap.add_argument("--out", type=Path, default=None, help="directory for the profiler traces (default: a new temporary one)")
    args = ap.parse_args()
    if args.steps < 20 or args.warmup < 3:
        ap.error("use at least 3 warm-up and 20 timed steps")
    if not torch.cuda.is_available():
        raise SystemExit("bench_gf.py needs a CUDA device")
    args.out = Path(tempfile.mkdtemp(prefix="bench_gf_")) if args.out is None else args.out
    args.out.mkdir(parents=True, exist_ok=True)
    dev = torch.device("cuda:0")
    for workload in (log_prob_workload, rsample_workload):
        res = workload(args, dev)
        print(json.dumps({**res, **card()}), flush=True)


if __name__ == "__main__":
    main()
