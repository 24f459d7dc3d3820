"""Golden vectors of the sum-of-squares polynomial flow (SOSPF, zuko/flows/polynomial.py:31-76) and of
its bijector alone (ShiftedSOSPTransform / SOSPolynomialTransform, flows/polynomial.py:23-28,
zuko/transforms.py:878-963), from the UNMODIFIED reference.  Separate from make_golden.py so that the
existing files are not rewritten.  Run in the build container only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_sospf.py
"""

from __future__ import annotations

import os
import sys
from pathlib import Path

import numpy as np
import torch

sys.dont_write_bytecode = True
sys.path.insert(0, "/root/reference")
sys.path.insert(0, str(Path(__file__).resolve().parent))

import make_golden as MG  # noqa: E402  (flow_case; imports the reference)
import make_golden_grad as MGG  # noqa: E402
import make_golden_inv_grad as MIG  # noqa: E402
from zuko.flows import SOSPF  # noqa: E402
from zuko.flows.polynomial import ShiftedSOSPTransform  # noqa: E402
from zuko.transforms import SOSPolynomialTransform  # noqa: E402

OUT = Path(__file__).resolve().parent

# name -> (constructor, batch, context, x_scale, store); mirrored by tests/test_sospf_host.py:SOSPF_CASES
CASES = {
    "sospf53": (lambda: SOSPF(5, 3, hidden_features=[32, 32]), 256, ("batch", 3), 1.0, True),
    "sospf35_row": (lambda: SOSPF(3, 5), 256, ("row", 5), 1.0, True),
    "sospf6_uncond": (lambda: SOSPF(6, 0, transforms=4, degree=3, polynomials=2), 256, None, 1.0, True),
    "sospf53_stress": (lambda: SOSPF(5, 3, hidden_features=[32, 32]), 256, ("batch", 3), 3.0, True),
    "sospf16_wide": (lambda: SOSPF(16, 8, hidden_features=[256] * 3), 256, ("batch", 8), 1.0, False),
}
GRAD_ROWS = {"sospf53": 128, "sospf35_row": 128, "sospf6_uncond": 128}
INV_GRAD_ROWS = {"sospf53": 64, "sospf35_row": 64}


def unit_cases():
    """The bijector alone for (K, L) in {(1, 0), (3, 4), (2, 7), (4, 15)} with per-element parameters,
    and one shared coefficient set: forward in fp32 / fp64, fp64 autograd gradients of
    <gy, y> + <gl, ladj>, and the bisection inverse on inputs inside and beyond f([-10, 10]).  The
    shifted cases carry a constant (ShiftedSOSPTransform), the others are SOSPolynomialTransform."""
    out = {}
    N = 512
    xedge = torch.tensor([0.0, 9.9, -9.9, 10.5, -10.5, 12.0, -12.0, 30.0])
    zedge = torch.tensor([0.0, 1e3, -1e3, 40.0, -40.0, 1e6, -1e6, 5.0])
    specs = [("k1l0", 1, 0, True, True), ("k3l4", 3, 4, True, True), ("k2l7", 2, 7, True, False),
             ("k4l15", 4, 15, True, True), ("shared34", 3, 4, False, False)]  # fmt: skip
    for i, (tag, K, L, batched, shifted) in enumerate(specs):
        shape = (N, K, L + 1) if batched else (K, L + 1)
        a = MG.gen(2100 + i, *shape) * 0.5
        const = MG.gen(2200 + i, N) if shifted else torch.zeros(N)
        x = torch.cat([MG.gen(2300 + i, N - xedge.numel(), scale=4.0), xedge])
        z = torch.cat([MG.gen(2400 + i, N - zedge.numel(), scale=4.0), zedge])

        def make(a_, c_):
            return ShiftedSOSPTransform(a_, c_) if shifted else SOSPolynomialTransform(a_)

        with torch.no_grad():
            y32, l32 = make(a, const).call_and_ladj(x)
            xi32 = make(a, const).inv(z)
            xi64 = make(a.double(), const.double()).inv(z.double())
        a64 = a.double().requires_grad_(True)
        c64 = const.double().requires_grad_(True)
        x64 = x.double().requires_grad_(True)
        y64, l64 = make(a64, c64).call_and_ladj(x64)
        gy, gl = MGG.gen(2500 + i, N).double(), MGG.gen(2600 + i, N).double()
        ((gy * y64).sum() + (gl * l64).sum()).backward()
        out.update({
            f"{tag}_a": a.numpy(), f"{tag}_const": const.numpy(), f"{tag}_x": x.numpy(), f"{tag}_z": z.numpy(),
            f"{tag}_y32": y32.numpy(), f"{tag}_ladj32": l32.numpy(), f"{tag}_xinv32": xi32.numpy(),
            f"{tag}_y64": y64.detach().numpy(), f"{tag}_ladj64": l64.detach().numpy(), f"{tag}_xinv64": xi64.numpy(),
            f"{tag}_gy": gy.numpy(), f"{tag}_gl": gl.numpy(), f"{tag}_gx": x64.grad.numpy(),
            f"{tag}_ga": a64.grad.numpy(), f"{tag}_gconst": c64.grad.numpy() if shifted else np.zeros(N),
            f"{tag}_shifted": np.bool_(shifted), f"{tag}_batched": np.bool_(batched),
        })  # fmt: skip
    np.savez_compressed(OUT / "units_sospf.npz", **out)
    print("units_sospf: done")


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
