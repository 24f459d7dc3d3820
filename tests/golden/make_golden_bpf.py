"""Golden vectors of the Bernstein polynomial flow (BPF, zuko/flows/polynomial.py:79-117) and of its
bijector alone (BoundedBernsteinTransform, zuko/transforms.py:640-831), from the UNMODIFIED reference.
Separate from make_golden.py so that the existing files are not rewritten.  Run in the build container
only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_bpf.py
"""

from __future__ import annotations

import os
import sys
from functools import partial
from pathlib import Path

import numpy as np
import torch

sys.dont_write_bytecode = True
sys.path.insert(0, "/root/reference")
sys.path.insert(0, str(Path(__file__).resolve().parent))

import make_golden as MG  # noqa: E402  (flow_case; imports the reference)
import make_golden_grad as MGG  # noqa: E402
import make_golden_inv_grad as MIG  # noqa: E402
from zuko.flows import BPF, MAF  # noqa: E402
from zuko.transforms import BoundedBernsteinTransform  # noqa: E402

OUT = Path(__file__).resolve().parent

# name -> (constructor, batch, context, x_scale, store); mirrored by tests/test_bpf_host.py:BPF_CASES
CASES = {
    "bpf53": (lambda: BPF(5, 3, hidden_features=[32, 32]), 256, ("batch", 3), 1.0, True),
    "bpf35_row": (lambda: BPF(3, 5), 256, ("row", 5), 1.0, True),
    "bpf6_uncond": (lambda: BPF(6, 0, transforms=4, degree=7), 256, None, 1.0, True),
    "bpf53_stress": (lambda: BPF(5, 3, hidden_features=[32, 32]), 256, ("batch", 3), 3.0, True),
    "bpf16_wide": (lambda: BPF(16, 8, hidden_features=[256] * 3), 256, ("batch", 8), 1.0, False),
    "bpf42_b3": (lambda: MAF(4, 2, univariate=partial(BoundedBernsteinTransform, bound=3.0), shapes=[(9,)]),
                 256, ("batch", 2), 1.0, True),  # fmt: skip
}
GRAD_ROWS = {"bpf53": 128, "bpf35_row": 128, "bpf6_uncond": 128}
INV_GRAD_ROWS = {"bpf53": 64, "bpf35_row": 64, "bpf6_uncond": 64}


def edge_x(bound: float, eps: float) -> torch.Tensor:
    """x at +-B and its fp32 neighbours, at the x whose fp32 t = (x + B) / 2B is the last one <= eps /
    the first one >= 1 - eps (and one ulp either side), at +-7, +-1e3 and 0."""
    f32 = np.float32
    B, two_b = f32(bound), f32(2 * bound)
    out = [B, -B, np.nextafter(B, f32(np.inf)), np.nextafter(B, f32(0)), np.nextafter(-B, f32(-np.inf)),
           np.nextafter(-B, f32(0)), f32(7), f32(-7), f32(1e3), f32(-1e3), f32(0)]  # fmt: skip
    lo, hi = f32(eps), f32(1 - eps)
    x = f32(-bound + 2 * bound * eps)  # walk to the last x with t <= eps
    while (x + B) / two_b > lo:
        x = np.nextafter(x, f32(-np.inf))
    while (np.nextafter(x, f32(np.inf)) + B) / two_b <= lo:
        x = np.nextafter(x, f32(np.inf))
    out += [np.nextafter(x, f32(-np.inf)), x, np.nextafter(x, f32(np.inf))]
    x = f32(bound - 2 * bound * eps)  # the first x with t >= 1 - eps
    while (x + B) / two_b < hi:
        x = np.nextafter(x, f32(np.inf))
    while (np.nextafter(x, f32(-np.inf)) + B) / two_b >= hi:
        x = np.nextafter(x, f32(-np.inf))
    out += [np.nextafter(x, f32(-np.inf)), x, np.nextafter(x, f32(np.inf))]
    return torch.tensor(np.array(out, np.float32))


def edge_y(bound: float) -> torch.Tensor:
    """y at +-B, +-B -+ 1e-5 (inside the jump at the bounds), +-1e3 and 0."""
    B = bound
    return torch.tensor([B, -B, B - 1e-5, -B + 1e-5, B + 1e-5, -B - 1e-5, 1e3, -1e3, 0.0], dtype=torch.float32)


def unit_cases():
    """The bijector alone for degrees 0, 4, 16 and 40 with per-element parameters (degree 16 also with u
    scaled x10: tiny softmax entries, flat regions), one shared parameter row, and eps = 1e-4 with
    bound 3: forward in fp32 / fp64, fp64 autograd gradients of <gy, y> + <gl, ladj>, and the inverse on
    inputs inside and beyond [-B, B]."""
    out = {}
    N = 512
    specs = [("d0", 0, True, 1.0, 5.0, 1e-6), ("d4", 4, True, 1.0, 5.0, 1e-6), ("d16", 16, True, 1.0, 5.0, 1e-6),
             ("d16x10", 16, True, 10.0, 5.0, 1e-6), ("d40", 40, True, 1.0, 5.0, 1e-6),
             ("shared16", 16, False, 1.0, 5.0, 1e-6), ("eps4_b3", 4, True, 1.0, 3.0, 1e-4)]  # fmt: skip
    for i, (tag, degree, batched, u_scale, bound, eps) in enumerate(specs):
        P = degree + 1
        u = MG.gen(3100 + i, *((N, P) if batched else (P,))) * u_scale
        xe, ye = edge_x(bound, eps), edge_y(bound)
        x = torch.cat([MG.gen(3300 + i, N - xe.numel(), scale=2.5), xe])
        z = torch.cat([MG.gen(3400 + i, N - ye.numel(), scale=2.5), ye])

        def make(u_):
            return BoundedBernsteinTransform(u_, bound=bound, eps=eps)

        with torch.no_grad():
            y32, l32 = make(u).call_and_ladj(x)
            xi32 = make(u).inv(z)
            xi64 = make(u.double()).inv(z.double())
        u64 = u.double().requires_grad_(True)
        x64 = x.double().requires_grad_(True)
        y64, l64 = make(u64).call_and_ladj(x64)
        gy, gl = MGG.gen(3500 + i, N).double(), MGG.gen(3600 + i, N).double()
        ((gy * y64).sum() + (gl * l64).sum()).backward()
        out.update({
            f"{tag}_u": u.numpy(), f"{tag}_x": x.numpy(), f"{tag}_z": z.numpy(),
            f"{tag}_bound": np.float64(bound), f"{tag}_eps": np.float64(eps),
            f"{tag}_y32": y32.detach().numpy(), f"{tag}_ladj32": l32.detach().numpy(), f"{tag}_xinv32": xi32.detach().numpy(),
            f"{tag}_y64": y64.detach().numpy(), f"{tag}_ladj64": l64.detach().numpy(), f"{tag}_xinv64": xi64.detach().numpy(),
            f"{tag}_gy": gy.numpy(), f"{tag}_gl": gl.numpy(), f"{tag}_gx": x64.grad.numpy(), f"{tag}_gu": u64.grad.numpy(),
            f"{tag}_batched": np.bool_(batched),
        })  # fmt: skip
    np.savez_compressed(OUT / "units_bpf.npz", **out)
    print("units_bpf: done")


def main():
    torch.set_num_threads(os.cpu_count())
    unit_cases()
    for name, (build, B, ctx, x_scale, store) in CASES.items():
        MG.flow_case(name, build, B, ctx, store=store, x_scale=x_scale, inverse_rows=64)
    for name, rows in GRAD_ROWS.items():
        MGG.grad_case(name, CASES[name][0], rows)
    for name, rows in INV_GRAD_ROWS.items():
        MIG.inv_grad_case(name, CASES[name][0], rows)


if __name__ == "__main__":
    main()
