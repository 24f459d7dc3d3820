"""Benchmark of the continuous normalizing flow (CNF): one JSON line per workload.

Workloads: CNF(16, 8) log_prob at 2^16 rows with the exact and with the Hutchinson trace, and CNF(64) sample
at 2^16 rows, each at default initialisation and with the weights scaled x3 as a stand-in for trained
(stiffer) dynamics, which take several times more Dormand-Prince trials.

Per line: samples/s from CUDA events around the whole call (warm-up excluded), trials and accepted steps, the
kernel time of zk_cnf_integrate from torch.profiler (a separate run), the achieved fp32 FLOP/s from the MACs
counted from the shapes and the number of f evaluations (the MLP, plus the tangent products of the trace),
its share of the 67 TFLOP/s fp32 data-sheet figure of the H100 SXM, the card name and power limit, and the
error against the fp64 restatement (tests/cnf_reference.py) replaying the engine's own steps on a row subset.

    python bench_cnf.py [--rows 65536] [--steps 5] [--warmup 2] [--check-rows 64]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import cnf_reference as R  # noqa: E402
from zuko_b200 import _engine as E  # noqa: E402
from zuko_b200.flows import CNF  # noqa: E402

PEAK_FP32 = 67e12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout  # fmt: skip
    name, power = (s.strip() for s in q.split(",", 1))
    return {"gpu": name, "power_limit": power}


def macs_per_eval(dims: list[int], D: int, F: int, trace: int) -> int:
    """MACs of one f evaluation of one row: the MLP, plus the tangent products of the trace (exact: D tangents,
    the first layer a column scaling, the last layer one dot product each; Hutchinson: one full tangent)."""
    mlp = sum(a * b for a, b in zip(dims[:-1], dims[1:], strict=True))
    hidden = dims[1:-1]
    if trace == E.ZK_CNF_TRACE_NONE or not hidden:
        return mlp
    mid = sum(a * b for a, b in zip(hidden[:-1], hidden[1:], strict=True))
    if trace == E.ZK_CNF_TRACE_EXACT:
        return mlp + D * (mid + hidden[-1])
    return mlp + D * hidden[0] + mid + hidden[-1] * D + D


def call(t, x, c, trace, eps, counts, log, y, ladj, ws, times):  # noqa: ANN001, ANN201
    h = t._cnf_handle()
    B, D = x.shape
    E.check(E.lib().zk_cnf_integrate(
        h, x.data_ptr(), D, None if c is None else c.data_ptr(), 0 if c is None else c.shape[1], B, times.data_ptr(),
        t.atol, t.rtol, trace, None if eps is None else eps.data_ptr(), D, log.shape[0], y.data_ptr(), D,
        None if ladj is None else ladj.data_ptr(), counts.data_ptr(), log.data_ptr(), ws.data_ptr(), ws.numel(),
        E.stream_ptr(x.device)))  # fmt: skip


def workload(name: str, D: int, C: int, trace: int, scale: float, direction: int, args) -> dict:  # noqa: ANN001
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    flow = CNF(D, C).eval()
    with torch.no_grad():
        for p in flow.parameters():
            p.mul_(scale)
    flow = flow.to(dev)
    t = flow.transform
    g = torch.Generator(device="cpu").manual_seed(1)
    B = args.rows
    x = torch.randn(B, D, generator=g).to(dev)
    c = torch.randn(B, C, generator=g).to(dev) if C else None
    eps = torch.randn(B, D, generator=g).to(dev) if trace == E.ZK_CNF_TRACE_HUTCHINSON else None
    times = torch.tensor([0.0, 1.0] if direction > 0 else [1.0, 0.0], device=dev)
    y = torch.empty(B, D, device=dev)
    ladj = torch.empty(B, device=dev) if trace else None
    counts = torch.zeros(2, dtype=torch.int32, device=dev)
    log = torch.zeros(4096, 4, device=dev)
    ws = torch.empty(E.lib().zk_cnf_workspace_bytes(t._cnf_handle(), B, trace), dtype=torch.uint8, device=dev)
    run = lambda: call(t, x, c, trace, eps, counts, log, y, ladj, ws, times)  # noqa: E731
    for _ in range(args.warmup):
        run()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.steps):
        run()
    end.record()
    torch.cuda.synchronize()
    call_s = start.elapsed_time(end) / 1e3 / args.steps
    trials, accepted = counts.tolist()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if "cnf_dopri_kernel" in e.name]
    kernel_s = sum(e.device_time_total for e in kern) / 1e6 if kern else float("nan")
    dims = [t.ode.in_features] + [m.weight.shape[0] for m in t.ode._linears()]
    evals = 6 * trials + 1
    flops = 2.0 * macs_per_eval(dims, D, t.freqs.numel(), trace) * evals * B
    # error against the fp64 replay of the engine's own steps, on the first rows
    n = args.check_rows
    lg = log[:trials].double().cpu().numpy()
    sd = {k: v.detach().double().cpu().numpy() for k, v in flow.state_dict().items()}
    field = R.Field.from_state_dict(sd, D, C, "ELU")
    yr, lr = R.replay(field, x[:n].double().cpu().numpy(), None if c is None else c[:n].double().cpu().numpy(), lg,
                      trace, None if eps is None else eps[:n].double().cpu().numpy())  # fmt: skip
    ours = y[:n].double().cpu().numpy()
    err = float(np.max(np.abs(ours - yr) / np.maximum(np.abs(yr), 1)))
    if trace:
        l = ladj[:n].double().cpu().numpy()
        err = max(err, float(np.max(np.abs(l - lr) / np.maximum(np.abs(lr), 1))))
    return {
        "workload": name, "rows": B, "samples_per_s": B / call_s, "call_ms": call_s * 1e3, "kernel_ms": kernel_s * 1e3,
        "trials": trials, "accepted": accepted, "f_evals": evals, "fp32_tflops": flops / kernel_s / 1e12,
        "share_of_fp32_peak": flops / kernel_s / PEAK_FP32,
        "bound": "fp32 FMA issue with one shared-memory weight load per 4 FMAs (thread-per-row MLP); "
                 "grid barrier per trial",
        "max_rel_err_vs_fp64_replay": err, **card(),
    }  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--check-rows", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cnf.py needs a CUDA device")
    for scale in (1.0, 3.0):
        tag = "" if scale == 1.0 else "_x3"
        for name, D, C, trace, direction in (
            ("cnf16_8_log_prob_exact", 16, 8, E.ZK_CNF_TRACE_EXACT, +1),
            ("cnf16_8_log_prob_hutchinson", 16, 8, E.ZK_CNF_TRACE_HUTCHINSON, +1),
            ("cnf64_sample", 64, 0, E.ZK_CNF_TRACE_NONE, -1),
        ):
            print(json.dumps(workload(name + tag, D, C, trace, scale, direction, args)), flush=True)


if __name__ == "__main__":
    main()
