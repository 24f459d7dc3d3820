"""Benchmark of the fused layer kernel on one GPU: one flow layer's ``zk_layer_forward`` (conditioner + bijector + ladj
in one launch) at the shapes of the benchmarked configurations.  Prints one JSON line:

* ``layers``: per shape and GEMM mode, ms per launch from CUDA events over ``--launches`` launches after warm-up
  (inputs rotate over buffers larger than the 50 MB L2), the kernel's row tile, and the rates the kernel achieves:
  issued tensor TFLOP/s (every non-zero weight tile at the width and depth the kernel multiplies it, all split-bf16
  terms, over whole row tiles) and weight-streaming GB/s (L2 -> shared memory: each row tile loads every non-zero tile,
  16 KB in bf16x3 and 8 KB in bf16x1, three quarters of that for an RQS output tile; `zk_layer_fused_stream_bytes`).  The shapes are the flagship layer (NSF(16, 8, bins=8, hidden=[256] * 3), 2^20 rows) at bf16x3 and at
  bf16x1 — half the weight bytes and a third of the MMAs, so the ratio of the two times shows which resource the
  kernel is sensitive to — and the layers of cfg3 (MAF(32, hidden=[512] * 4), 2^20 rows) and cfg5 (NSF(64, 16,
  bins=16, hidden=[512] * 3), 2^21 rows);
* the card's name and power limit, and the median SM clock over the timed regions.

Needs a CUDA device."""

from __future__ import annotations

import argparse
import ctypes
import json
import math
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from bench import ClockSampler  # noqa: E402
from bench_gf import card  # noqa: E402

import zuko_b200 as zuko  # noqa: E402
from zuko_b200 import _engine as E  # noqa: E402

NBUF = 3  # input sets per shape, each >= 50 MB at the timed batch sizes: consecutive launches miss in L2

SHAPES = [
    {"name": "flagship", "kind": "nsf", "D": 16, "C": 8, "K": 8, "H": [256] * 3, "rows": 1 << 20, "gemm_mode": "bf16x3"},
    {"name": "flagship_bf16x1", "kind": "nsf", "D": 16, "C": 8, "K": 8, "H": [256] * 3, "rows": 1 << 20, "gemm_mode": "bf16x1"},
    {"name": "cfg3_layer", "kind": "maf", "D": 32, "C": 0, "K": 0, "H": [512] * 4, "rows": 1 << 20, "gemm_mode": "bf16x3"},
    {"name": "cfg5_layer", "kind": "nsf", "D": 64, "C": 16, "K": 16, "H": [512] * 3, "rows": 1 << 21, "gemm_mode": "bf16x3"},
]  # fmt: skip


def build_layer(s, dev):
    torch.manual_seed(0)
    if s["kind"] == "maf":
        flow = zuko.flows.MAF(s["D"], s["C"], transforms=1, hidden_features=s["H"])
    else:
        flow = zuko.flows.NSF(s["D"], s["C"], transforms=1, bins=s["K"], hidden_features=s["H"])
    t = flow.transform.transforms[0]
    t.hyper.gemm_mode = s["gemm_mode"]
    return t.to(dev).eval()


def tile_rows(handle) -> int:
    lib = E.lib()
    if not hasattr(lib, "zk_layer_fused_tile_rows"):  # libraries older than the query run 64-row tiles only
        return 64
    return int(lib.zk_layer_fused_tile_rows(handle))


def stream_bytes(handle, n_tiles: int, gemm_mode: str) -> int:
    """Weight bytes brought into shared memory per row tile."""
    lib = E.lib()
    if not hasattr(lib, "zk_layer_fused_stream_bytes"):  # libraries older than the query stream whole 64 x 64 tiles
        return n_tiles * (16384 if gemm_mode == "bf16x3" else 8192)
    return int(lib.zk_layer_fused_stream_bytes(handle))


def time_layer(s, dev, args, clk_rows: list) -> dict:
    layer = build_layer(s, dev)
    B, D, C = s["rows"], s["D"], s["C"]
    g = torch.Generator(device=dev).manual_seed(1)
    xs = [torch.randn(B, D, device=dev, generator=g) for _ in range(NBUF)]
    cs = [torch.randn(B, C, device=dev, generator=g) if C else None for _ in range(NBUF)]
    fn = lambda i: layer(cs[i % NBUF]).call_and_ladj(xs[i % NBUF])  # noqa: E731
    with torch.no_grad():
        fn(0)  # packs
        handle = layer._zk_layer()
        info = (ctypes.c_double * 4)()
        kind = E.lib().zk_layer_fused_info(handle, info)
        if kind != 1:
            raise SystemExit(f"bench_fused.py: {s['name']} does not run as the fused layer kernel")
        rows = tile_rows(handle)
        for i in range(args.warmup):
            fn(i)
        torch.cuda.synchronize()
        n0 = E.lib().zk_launch_count()
        clk = ClockSampler(torch.cuda.current_device()).prepare()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with clk:
            e0.record()
            for i in range(args.launches):
                fn(i)
            e1.record()
            torch.cuda.synchronize()
        launches = E.lib().zk_launch_count() - n0
    if launches != args.launches:
        raise SystemExit(f"bench_fused.py: {s['name']}: {launches} launches for {args.launches} layer calls")
    clk_rows += [r[0] for r in clk.rows]
    ms = e0.elapsed_time(e1) / args.launches
    n_tiles, issued_macs_per_row = int(info[1]), info[2]
    row_tiles = math.ceil(B / rows)
    tile_stream = stream_bytes(handle, n_tiles, s["gemm_mode"])
    return {
        "name": s["name"], "gemm_mode": s["gemm_mode"], "rows": B, "tile_rows": rows, "weight_tiles_per_row_tile": n_tiles,
        "ms_per_launch": ms, "launches": args.launches,
        "issued_tflops": 2.0 * issued_macs_per_row * row_tiles * rows / (ms * 1e-3) / 1e12,
        "weight_stream_gbs": row_tiles * tile_stream / (ms * 1e-3) / 1e9,
    }  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if args.launches < 200 or args.warmup < 3:
        ap.error("use at least 3 warm-up and 200 timed launches")
    if not torch.cuda.is_available():
        raise SystemExit("bench_fused.py needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    clk_rows: list[float] = []
    layers = []
    for s in SHAPES:
        layers.append(time_layer(s, dev, args, clk_rows))
        torch.cuda.empty_cache()
    sm = sorted(clk_rows)
    line = {"layers": layers, **card(), "sm_mhz_median": sm[len(sm) // 2] if sm else None}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
