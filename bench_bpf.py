"""Benchmark of the Bernstein polynomial flow (BPF) on one GPU.  Prints one JSON line per workload:

* ``bpf16_log_prob``: ``BPF(16, 8, hidden_features=[256] * 3)``, ``log_prob`` of 2^20 rows with a context row
  each (per layer the conditioner GEMMs and one ``uni_kernel``; BPF layers never run as the fused layer kernel);
* ``bpf64_rsample``: ``BPF(64)``, ``rsample((2^20,))``: per layer one ``ar_inverse_kernel`` that runs the
  24-step bisection of every dimension in registers, the part of BPF the reference is slowest at;
* ``bpf64_inverse_paths``: the same flow's inverse of 2^16 rows through the dimension-sequential kernel and
  through the generic sweeps (``zk_set_fused_layers(0)``: 64 passes of the conditioner and ``uni_kernel`` per layer).

Each line holds samples/s from CUDA events (best and median over the timed steps), the device time of the
``uni_kernel`` / ``ar_inverse_kernel`` launches from ``torch.profiler`` (a separate profiled call after the timed
ones; the trace is written under ``--out``), the card's name and power limit, and the error against the fp64
restatement of tests/bpf_reference.py: relative error of ``log_prob`` on the first 2^12 rows, and of the sample
against the fp64 inverse on the first 2^6 (64 passes of 24 bisection steps per layer are slow on the host).
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

import bpf_reference as R  # noqa: E402
import zuko_b200 as zuko  # noqa: E402
from zuko_b200 import _engine as E  # noqa: E402

CHECK_ROWS = 1 << 12
CHECK_ROWS_INVERSE = 1 << 6
PATH_ROWS = 1 << 16


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


def kernel_times(fn, trace: Path) -> dict:
    """Device seconds of the uni_kernel (forward / inverse) and ar_inverse_kernel launches in one profiled call."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(trace))
    out = {"uni_forward_s": 0.0, "uni_inverse_s": 0.0, "ar_inverse_s": 0.0, "uni_launches": 0, "ar_inverse_launches": 0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        if "uni_kernel<" in e.name:
            inverse = e.name.split("uni_kernel<", 1)[1].split(",")[2].strip() == "true"
            out["uni_inverse_s" if inverse else "uni_forward_s"] += e.device_time_total / 1e6
            out["uni_launches"] += 1
        elif "ar_inverse_kernel<" in e.name:
            out["ar_inverse_s"] += e.device_time_total / 1e6
            out["ar_inverse_launches"] += 1
    return out


def errors(ours: np.ndarray, ref: np.ndarray) -> dict:
    e = np.abs(np.asarray(ours, np.float64) - ref) / np.maximum(np.abs(ref), 1.0)
    return {"max_rel_err": float(e.max()), "p99_rel_err": float(np.percentile(e, 99)),
            "median_rel_err": float(np.median(e)), "rows_checked": int(ref.shape[0])}  # fmt: skip


def reference(flow, D: int, C: int) -> R.Flow:
    return R.Flow({k: v.detach().cpu().numpy() for k, v in flow.state_dict().items()}, D, C, 16)


def rates(B: int, times: list[float]) -> dict:
    return {"samples_per_s_best": B / min(times), "samples_per_s_median": B / float(np.median(times)),
            "step_s_best": min(times), "step_s_median": float(np.median(times)), "steps": len(times)}  # fmt: skip


def log_prob_workload(args, dev) -> dict:
    D, C, B = 16, 8, 1 << args.log2_rows
    torch.manual_seed(0)
    flow = zuko.flows.BPF(D, C, hidden_features=[256] * 3).to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, D, device=dev, generator=g)
    c = torch.randn(B, C, device=dev, generator=g)
    with torch.no_grad():
        fn = lambda: flow(c).log_prob(x)  # noqa: E731
        times = time_steps(fn, args.warmup, args.steps)
        kt = kernel_times(fn, args.out / "trace_bpf16_log_prob.json")
        lp = fn()[:CHECK_ROWS].cpu().numpy()
    ref = reference(flow, D, C).log_prob(x[:CHECK_ROWS].cpu().numpy(), c[:CHECK_ROWS].cpu().numpy())
    return {"workload": "bpf16_log_prob", "rows": B, **rates(B, times), **kt, **errors(lp, ref)}


def rsample_flow(dev):
    torch.manual_seed(0)
    return zuko.flows.BPF(64).to(dev).eval()


def rsample_workload(args, dev) -> dict:
    D, B = 64, 1 << args.log2_rows
    flow = rsample_flow(dev)
    with torch.no_grad():
        fn = lambda: flow().rsample((B,))  # noqa: E731
        times = time_steps(fn, args.warmup, args.steps)
        kt = kernel_times(fn, args.out / "trace_bpf64_rsample.json")
        z = torch.randn(CHECK_ROWS_INVERSE, D, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
        x = flow().transform.inv(z).cpu().numpy()
    ref = reference(flow, D, 0).inverse(z.cpu().numpy())
    seq = [E.lib().zk_layer_sequential_inverse(t._zk_layer()) for t in flow.transform.transforms]
    return {"workload": "bpf64_rsample", "rows": B, "sequential_layers": int(sum(seq)), **rates(B, times), **kt,
            **errors(x, ref)}  # fmt: skip


def inverse_paths_workload(args, dev) -> dict:
    D, B = 64, PATH_ROWS
    flow = rsample_flow(dev)
    z = torch.randn(B, D, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    out = {"workload": "bpf64_inverse_paths", "rows": B}
    with torch.no_grad():
        fn = lambda: flow().transform.inv(z)  # noqa: E731
        seq_t = time_steps(fn, args.warmup, args.steps)
        x_seq = fn()
        prev = E.lib().zk_set_fused_layers(0)
        try:
            sweep_t = time_steps(fn, 1, 3)  # 64 conditioner passes per layer: a few steps suffice
            x_sweep = fn()
        finally:
            E.lib().zk_set_fused_layers(prev)
    d = (x_seq - x_sweep).abs()
    out.update(sequential_s_median=float(np.median(seq_t)), sweeps_s_median=float(np.median(sweep_t)),
               speedup=float(np.median(sweep_t) / np.median(seq_t)), max_abs_diff=float(d.max()),
               median_abs_diff=float(d.median()))  # fmt: skip
    return out


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
        raise SystemExit("bench_bpf.py needs a CUDA device")
    args.out = Path(tempfile.mkdtemp(prefix="bench_bpf_")) if args.out is None else args.out
    args.out.mkdir(parents=True, exist_ok=True)
    dev = torch.device("cuda:0")
    for workload in (log_prob_workload, rsample_workload, inverse_paths_workload):
        res = workload(args, dev)
        print(json.dumps({**res, **card()}), flush=True)


if __name__ == "__main__":
    main()
