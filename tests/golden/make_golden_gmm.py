"""Golden data of tests/test_gmm_host.py and tests/test_gpu_gmm.py: the UNMODIFIED reference's
``zuko.mixtures.GMM`` on the cases of tests/gmm_cases.py, built under the cases' seeds.

gmm_<case>.npz: the state-dict keys and CRC32s of the initial (fp32) tensors, x, c, w, and — with the model
and inputs in fp64 — ``log_prob(x)`` (and the reference's fp32 value of it), the conditioner output phi, the
gradients of ``sum(w * log_prob(x))`` with respect to phi, x, c and every parameter (``grad/<key>``), and
``err32/<name>``, the reference's own fp32-vs-fp64 deviation of each gradient relative to its largest entry.
A weight gradient of more than 16384 entries is stored as its two fp64 factors from the reference's backward, the
layer's output gradient ``gout/grad/<key>`` and its input ``input/grad/<key>`` (the gradient is gout^T @ input).
gmm_init.npz: the parameters after ``initialize`` (each strategy, seeded).  gmm_adam.npz: the losses of 30
Adam steps of a conditional GMM on seeded data.  Run with the reference's source tree as the first argument:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_gmm.py <reference source tree>
"""

from __future__ import annotations

import copy
import sys
from pathlib import Path

import numpy as np
import torch

sys.dont_write_bytecode = True
HERE = Path(__file__).resolve().parent
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, str(HERE.parent))

import zuko  # noqa: E402
import zuko.mixtures  # noqa: E402
from zuko.utils import unpack  # noqa: E402

from gmm_cases import GMM_CASES, INIT_CASES, adam_batches, adam_curve, adam_model, build, init_data, inputs  # noqa: E402


def crc(t: torch.Tensor) -> int:
    import zlib

    return zlib.crc32(np.ascontiguousarray(t.detach().cpu().numpy()).tobytes())


def evaluate(gmm, x, c, w):  # noqa: ANN001
    """log_prob, phi, the gradients of sum(w * log_prob) (phi, x, c, parameters) and, per conditioner layer, its
    input and the gradient of its output (``factors``)."""
    gmm.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_()
    c = None if c is None else c.clone().requires_grad_()
    factors, hooks = {}, []
    if c is not None:
        for i, m in enumerate(gmm.hyper):
            if getattr(m, "weight", None) is not None and m.weight.dim() == 2:

                def keep(mod, inputs, out, key=f"hyper.{i}.weight"):  # noqa: ANN001, ANN202
                    out.retain_grad()
                    factors[key] = (inputs[0].detach(), out)

                hooks.append(m.register_forward_hook(keep))
    lp = gmm(c).log_prob(x)
    for h in hooks:
        h.remove()
    (w * lp).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in gmm.named_parameters()}
    factors = {k: (out.grad.detach(), a) for k, (a, out) in factors.items()}
    # the same density from the conditioner's output, through the reference's own mixture code
    if c is None:
        phi = torch.cat([p.detach().reshape(-1) for p in gmm.phi]).requires_grad_()
        parts = unpack(phi, gmm.shapes)
    else:
        phi = gmm.hyper(c.detach()).detach().requires_grad_()
        parts = unpack(phi, gmm.shapes)
    forward = gmm._forward_full if gmm.covariance_type == "full" else gmm._forward_diagonal
    lp2 = forward(*parts).log_prob(x.detach())
    (w * lp2).sum().backward()
    return lp.detach(), phi.detach(), phi.grad.detach(), x.grad.detach(), None if c is None else c.grad.detach(), grads, factors


def main() -> None:
    for name in GMM_CASES:
        gmm = build(zuko, name)
        x, c, w = inputs(name)
        out = {"keys": np.array(list(gmm.state_dict().keys())), "crc": np.array([crc(t) for t in gmm.state_dict().values()], np.int64)}
        out["x"], out["w"] = x.numpy(), w.numpy()
        if c is not None:
            out["c"] = c.numpy()
        lp32, _, _, gx32, gc32, g32, _ = evaluate(gmm, x, c, w)
        g64 = copy.deepcopy(gmm).double()
        lp, phi, gphi, gx, gc, grads, factors = evaluate(g64, x.double(), None if c is None else c.double(), w.double())
        out["lp"], out["lp32"], out["phi"], out["gphi"], out["gx"] = lp.numpy(), lp32.numpy(), phi.numpy(), gphi.numpy(), gx.numpy()
        pairs = [("gx", gx32, gx)] + [(f"grad/{k}", g32[k], grads[k]) for k in grads]
        if gc is not None:
            out["gc"] = gc.numpy()
            pairs.append(("gc", gc32, gc))
        for key, a32, a64 in pairs:
            if a64.numel() <= 16384:
                out[key] = a64.numpy()
            else:  # a wide layer's weight gradient as its two fp64 factors: grad = gout^T @ input (size)
                gout, inp = factors[key.removeprefix("grad/")]
                assert torch.allclose(gout.T @ inp, a64, rtol=1e-12, atol=1e-12 * a64.abs().max().item())
                out[f"gout/{key}"], out[f"input/{key}"] = gout.numpy(), inp.numpy()
            out[f"err32/{key}"] = np.array((a32.double() - a64).abs().max().item() / max(a64.abs().max().item(), 1e-300))
        np.savez_compressed(HERE / f"gmm_{name}.npz", **out)
        print(name, "lp", lp[:3].numpy(), "err32 gx", out["err32/gx"])

    init = {}
    for name, (_, _, _, strategy) in INIT_CASES.items():
        gmm = build(zuko, name)
        torch.manual_seed(11)
        gmm.initialize(init_data(), strategy)
        for k, t in gmm.state_dict().items():
            init[f"{name}/{k}"] = t.numpy()
    np.savez_compressed(HERE / "gmm_init.npz", **init)

    gmm = adam_model(zuko)
    np.savez_compressed(HERE / "gmm_adam.npz", losses=np.array(adam_curve(gmm, adam_batches())))


if __name__ == "__main__":
    main()
