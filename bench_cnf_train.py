"""Benchmark of CNF training through the adaptive checkpoint adjoint: one JSON line per workload.

Workloads, at 2^16 rows: a CNF(16, 8) training step (-log_prob(x).mean(), forward and backward) with the exact and
with the Hutchinson trace, at default initialisation and with the weights scaled x3 as a stand-in for trained
(stiffer) dynamics; and a CNF(64) reverse-KL step through rsample_and_log_prob with the Hutchinson trace.

Per line: forward and backward ms from CUDA events around the public API (warm-up excluded); the replay, adjoint
and reduction kernel ms from torch.profiler (a separate run); accepted steps; the achieved fp32 FLOP/s of the
backward kernels from the MACs counted from the shapes, and its share of the 67 TFLOP/s fp32 data-sheet figure of
the H100 SXM; what bounds it; the card name and power limit; and the error of grad_x and grad_c against the fp64
restatement (tests/cnf_adjoint_reference.py) replaying the engine's own steps, on a row subset.

    python bench_cnf_train.py [--rows 65536] [--steps 3] [--warmup 1] [--check-rows 8]
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

import cnf_adjoint_reference as A  # noqa: E402
import cnf_reference as R  # noqa: E402
from zuko_b200 import _engine as E  # noqa: E402
from zuko_b200.flows import CNF  # noqa: E402

PEAK_FP32 = 67e12
KERNELS = {"replay": "cnf_replay_kernel", "adjoint": "cnf_adjoint_kernel", "reduce": ("cnf_grad_reduce_kernel", "cnf_context_sum_kernel")}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout  # fmt: skip
    name, power = (s.strip() for s in q.split(",", 1))
    return {"gpu": name, "power_limit": power}


def backward_macs(dims: list[int], D: int, F: int, trace: int, accepted: int) -> int:
    """MACs of the backward per row, as the kernels run them: per accepted step the replay's 6 evaluations of f,
    and per adjoint stage the MLP, its reverse pass and (5 stages of 6) its weight-gradient outer products, plus
    per tangent (D exact, 1 Hutchinson) the tangent program forward and reverse and its outer products."""
    L = len(dims) - 1
    mlp = sum(dims[i] * dims[i + 1] for i in range(L))
    rev = mlp - 2 * F * dims[1]
    stage = mlp + rev
    wstage = mlp + sum(dims[1:])
    if trace != E.ZK_CNF_TRACE_NONE and L > 1:
        inner = sum(dims[i] * dims[i + 1] for i in range(1, L))
        fwd = sum(dims[i] * dims[i + 1] for i in range(1, L - 1))
        K = D if trace == E.ZK_CNF_TRACE_EXACT else 1
        first = dims[1] * (1 if trace == E.ZK_CNF_TRACE_EXACT else D)
        stage += K * (fwd + inner + (first if trace == E.ZK_CNF_TRACE_HUTCHINSON else 0))
        wstage += K * (inner + first)
    return accepted * (6 * mlp + 6 * stage + 5 * wstage)


def check_rows(flow, x, c, trace, n):  # noqa: ANN001, ANN201
    """Worst error of grad_x and grad_c (per row) against the fp64 restatement at the engine's own steps, for
    <gy, y> + <gl, ladj> with seeded gy, gl, on the first n rows of one direct zk_cnf_integrate / _backward pair."""
    t = flow.transform
    dev = x.device
    B, D = x.shape
    C = 0 if c is None else c.shape[1]
    h = t._cnf_handle()
    lib = E.lib()
    g = torch.Generator(device="cpu").manual_seed(7)
    gy = torch.randn(B, D, generator=g).to(dev)
    gl = torch.randn(B, generator=g).to(dev) if trace else None
    eps = torch.randn(B, D, generator=g).to(dev) if trace == E.ZK_CNF_TRACE_HUTCHINSON else None
    times = torch.tensor([0.0, 1.0], device=dev)
    y, ladj = torch.empty(B, D, device=dev), (torch.empty(B, device=dev) if trace else None)
    counts = torch.zeros(2, dtype=torch.int32, device=dev)
    log = torch.zeros(10000, 4, device=dev)
    ws = torch.empty(lib.zk_cnf_workspace_bytes(h, B, trace), dtype=torch.uint8, device=dev)
    ptr = lambda v: None if v is None else v.data_ptr()  # noqa: E731
    E.check(lib.zk_cnf_integrate(h, x.data_ptr(), D, ptr(c), C, B, times.data_ptr(), t.atol, t.rtol, trace, ptr(eps), D,
                                 log.shape[0], y.data_ptr(), D, ptr(ladj), counts.data_ptr(), log.data_ptr(), ws.data_ptr(),
                                 ws.numel(), E.stream_ptr(dev)))  # fmt: skip
    trials, acc = counts.tolist()
    gx = torch.empty(B, D, device=dev)
    gc = torch.empty(B, C, device=dev) if C else None
    need = lib.zk_cnf_backward_workspace_bytes(h, B, trace, acc)
    bws = torch.empty(need, dtype=torch.uint8, device=dev)
    E.check(lib.zk_cnf_backward(h, x.data_ptr(), D, ptr(c), C, B, log.data_ptr(), trials, acc, trace, ptr(eps), D,
                                gy.data_ptr(), D, ptr(gl), gx.data_ptr(), D, ptr(gc), C, None,
                                bws.data_ptr(), need, E.stream_ptr(dev)))  # fmt: skip
    sd = {k: v.detach().double().cpu().numpy() for k, v in flow.state_dict().items()}
    field = R.Field.from_state_dict(sd, D, C, "ELU")
    np64 = lambda v: None if v is None else v[:n].double().cpu().numpy()  # noqa: E731
    ref = A.adjoint(field, np64(x), np64(c), log[:trials].double().cpu().numpy(), trace, np64(eps), np64(gy), np64(gl))
    err = float(np.max(np.abs(np64(gx) - ref["x"])) / np.max(np.abs(ref["x"])))
    if C:
        err = max(err, float(np.max(np.abs(np64(gc) - ref["c"])) / np.max(np.abs(ref["c"]))))
    return err


def workload(name: str, D: int, C: int, exact: bool, scale: float, reverse_kl: bool, args) -> dict:  # noqa: ANN001
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    flow = CNF(D, C, exact=exact, adjoint=True)
    with torch.no_grad():
        for p in flow.parameters():
            p.mul_(scale)
    flow = flow.to(dev).train()
    g = torch.Generator(device="cpu").manual_seed(1)
    B = args.rows
    x = torch.randn(B, D, generator=g).to(dev)
    c = torch.randn(B, C, generator=g).to(dev) if C else None
    stats = {}

    def forward():  # noqa: ANN202
        dist = flow(c)
        if reverse_kl:  # KL(q || N(0, I)) up to a constant: E_q[log q(x) + |x|^2 / 2]
            # rsample_and_log_prob spelled out (distributions.py:129-138), to read the inverse's step counts
            z = dist.base.rsample((B,))
            t = dist.transform.inv
            xs, ladj = t.call_and_ladj(z)
            lp = dist.base.log_prob(z) - ladj
            loss = (lp + 0.5 * (xs * xs).sum(-1)).mean()
        else:
            t = dist.transform
            loss = -dist.log_prob(x).mean()
        stats["t"] = t
        return loss

    for _ in range(args.warmup):
        forward().backward()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    fwd_ms = bwd_ms = 0.0
    for _ in range(args.steps):
        flow.zero_grad()
        ev[0].record()
        loss = forward()
        ev[1].record()
        loss.backward()
        ev[2].record()
        torch.cuda.synchronize()
        fwd_ms += ev[0].elapsed_time(ev[1]) / args.steps
        bwd_ms += ev[1].elapsed_time(ev[2]) / args.steps
    trials, accepted = stats["t"].stats
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        forward().backward()
        torch.cuda.synchronize()
    kern = {}
    for k, names in KERNELS.items():
        names = (names,) if isinstance(names, str) else names
        kern[k] = sum(e.device_time_total for e in prof.events() if any(s in e.name for s in names)) / 1e3
    t = flow.transform
    dims = [t.ode.in_features] + [m.weight.shape[0] for m in t.ode._linears()]
    trace = E.ZK_CNF_TRACE_EXACT if exact else E.ZK_CNF_TRACE_HUTCHINSON
    acc_prof = stats["t"].stats[1]  # the profiled step's own count (Hutchinson draws a new eps per call)
    flops = 2.0 * backward_macs(dims, D, t.freqs.numel(), trace, acc_prof) * B
    bk_s = (kern["replay"] + kern["adjoint"] + kern["reduce"]) / 1e3
    xe = x if not reverse_kl else torch.randn(B, D, generator=g).to(dev)
    err = check_rows(flow, xe, c, trace, args.check_rows)
    return {
        "workload": name, "rows": B, "forward_ms": fwd_ms, "backward_ms": bwd_ms,
        "replay_kernel_ms": kern["replay"], "adjoint_kernel_ms": kern["adjoint"], "reduction_kernel_ms": kern["reduce"],
        "trials": trials, "accepted": accepted, "backward_fp32_tflops": flops / bk_s / 1e12,
        "share_of_fp32_peak": flops / bk_s / PEAK_FP32,
        "bound": "fp32 FMA issue from shared memory at the few threads per SM that the per-row adjoint state "
                 "leaves (one 32-row CTA per SM for CNF(16, 8)'s hidden (64, 64) with a trace), plus one CTA barrier per "
                 "weight-gradient outer product",
        "grad_rel_err_vs_fp64_restatement": err, **card(),
    }  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check-rows", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cnf_train.py needs a CUDA device")
    for scale in (1.0, 3.0):
        tag = "" if scale == 1.0 else "_x3"
        for name, exact in (("cnf16_8_train_exact", True), ("cnf16_8_train_hutchinson", False)):
            print(json.dumps(workload(name + tag, 16, 8, exact, scale, False, args)), flush=True)
    print(json.dumps(workload("cnf64_reverse_kl_hutchinson", 64, 0, False, 1.0, True, args)), flush=True)


if __name__ == "__main__":
    main()
