"""Golden vectors of the Gaussianization flow (GF, zuko/flows/gaussianization.py:97-155) and of
GaussianizationTransform alone (zuko/transforms.py:834-875), from the UNMODIFIED reference.  Separate
from make_golden.py so that the existing files are not rewritten.  Run in the build container only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_gf.py
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
from zuko.flows import GF  # noqa: E402
from zuko.transforms import GaussianizationTransform  # noqa: E402

OUT = Path(__file__).resolve().parent

# name -> (constructor, batch, context, x_scale, store); mirrored by tests/test_gf_host.py:GF_CASES
CASES = {
    "gf53": (lambda: GF(5, 3, hidden_features=[32, 32]), 256, ("batch", 3), 1.0, True),
    "gf35_row": (lambda: GF(3, 5), 256, ("row", 5), 1.0, True),
    "gf6_uncond": (lambda: GF(6, 0, transforms=4, components=16), 256, None, 1.0, True),
    "gf53_stress": (lambda: GF(5, 3, hidden_features=[32, 32]), 256, ("batch", 3), 3.0, True),
    "gf16_wide": (lambda: GF(16, 8, components=8, hidden_features=[256] * 3), 256, ("batch", 8), 1.0, False),
}
GRAD_ROWS = {"gf53": 128, "gf35_row": 128, "gf6_uncond": 128}
INV_GRAD_ROWS = {"gf53": 64, "gf35_row": 64}


def unit_cases():
    """The bijector alone: per-element (batched) parameters for K in {1, 8, 16}, one shared parameter
    vector, and a partial with non-default bound / eps; forward in fp32 / fp64, fp64 autograd
    gradients of <gy, y> + <gl, ladj>, and the bisection inverse on inputs inside and beyond the
    range of f (about +-4.889 with the defaults)."""
    out = {}
    N = 512
    edge = torch.tensor([0.0, 4.8, 4.9, 6.0, -4.9, -6.0, -4.8, 100.0])
    specs = [("k1", 1, True, {}), ("k8", 8, True, {}), ("k16", 16, True, {}), ("shared8", 8, False, {}),
             ("partial8", 8, True, {"bound": 5.0, "eps": 1e-4})]  # fmt: skip
    for i, (tag, K, batched, kw) in enumerate(specs):
        shape = (N, K) if batched else (K,)
        shift = MG.gen(1100 + i, *shape)
        scale = MG.gen(1200 + i, *shape) * 0.5
        x = MG.gen(1300 + i, N, scale=1.5)
        z = torch.cat([MG.gen(1400 + i, N - edge.numel(), scale=1.5), edge])
        ctor = partial(GaussianizationTransform, **kw) if kw else GaussianizationTransform
        t32 = ctor(shift, scale)
        with torch.no_grad():
            y32, l32 = t32.call_and_ladj(x)
            xi32 = t32.inv(z)
        s64 = shift.double().requires_grad_(True)
        a64 = scale.double().requires_grad_(True)
        x64 = x.double().requires_grad_(True)
        t64 = ctor(s64, a64)
        y64, l64 = t64.call_and_ladj(x64)
        gy, gl = MGG.gen(1500 + i, N).double(), MGG.gen(1600 + i, N).double()
        ((gy * y64).sum() + (gl * l64).sum()).backward()
        with torch.no_grad():
            xi64 = ctor(shift.double(), scale.double()).inv(z.double())
        out.update({
            f"{tag}_shift": shift.numpy(), f"{tag}_scale": scale.numpy(), f"{tag}_x": x.numpy(), f"{tag}_z": z.numpy(),
            f"{tag}_y32": y32.detach().numpy(), f"{tag}_ladj32": l32.detach().numpy(), f"{tag}_xinv32": xi32.detach().numpy(),
            f"{tag}_y64": y64.detach().numpy(), f"{tag}_ladj64": l64.detach().numpy(), f"{tag}_xinv64": xi64.detach().numpy(),
            f"{tag}_gy": gy.numpy(), f"{tag}_gl": gl.numpy(), f"{tag}_gx": x64.grad.numpy(),
            f"{tag}_gshift": s64.grad.numpy(), f"{tag}_gscale": a64.grad.numpy(),
            f"{tag}_bound": np.float64(kw.get("bound", 10.0)), f"{tag}_eps": np.float64(kw.get("eps", 1e-6)),
        })  # fmt: skip
    np.savez_compressed(OUT / "units_gf.npz", **out)
    print("units_gf: done")


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
