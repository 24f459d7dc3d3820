"""Golden vectors of the continuous normalizing flow (CNF, zuko/flows/continuous.py) from the UNMODIFIED
reference, in fp32 and fp64, with the reference's per-trial step log (t, dt, error, accepted), recorded by
wrapping zuko.utils.dopri45 inside this script only.  Run in the build container only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_cnf.py

Per case and dtype: log_prob(x) (exact trace), transform(x), transform.inv(z), rsample_and_log_prob's two
outputs for a given z (x = inv(z), base.log_prob(z) - inv.call_and_ladj(z)[1]), and one Hutchinson
call_and_ladj(x) with its eps, each with its step log.
"""

from __future__ import annotations

import sys
import zlib
from pathlib import Path

import numpy as np
import torch

sys.dont_write_bytecode = True
sys.path.insert(0, "/root/reference")

import zuko.utils as U  # noqa: E402
from zuko.flows import CNF  # noqa: E402

OUT = Path(__file__).resolve().parent

# name -> (constructor, batch, weight scale); mirrored by tests/test_cnf_host.py:CASES
CASES = {
    "cnf35": (lambda: CNF(3, 5), 256, 1.0),
    "cnf168": (lambda: CNF(16, 8), 256, 1.0),
    "cnf5_deep": (lambda: CNF(5, 0, hidden_features=[32, 32, 32]), 256, 1.0),
    "cnf43_tanh": (lambda: CNF(4, 3, activation=torch.nn.Tanh), 256, 1.0),
    "cnf42_f0": (lambda: CNF(4, 2, freqs=0), 256, 1.0),
    "cnf35_stiff": (lambda: CNF(3, 5), 256, 3.0),
    "cnf168_stiff": (lambda: CNF(16, 8), 256, 3.0),
}

_dopri = U.dopri45
LOG: list = []
TOL: list = []  # (atol, rtol) of the integration being recorded


def _logged(f, x, t, dt, error=False):  # noqa: ANN001, ANN202
    out = _dopri(f, x, t, dt, error)
    if error:
        y, err = out
        atol, rtol = TOL[0]
        tol = atol + rtol * torch.max(abs(x), abs(y))
        e = torch.max(err / tol).clip(min=1e-9).item()  # the reference's own expression, utils.py:541-543
        LOG.append((float(t), float(dt), e, float(e < 1.0)))
    return out


U.dopri45 = _logged


def crc(t: torch.Tensor) -> int:
    return zlib.crc32(np.ascontiguousarray(t.detach().cpu().numpy()).tobytes())


def run(fn):  # noqa: ANN001, ANN202
    LOG.clear()
    with torch.no_grad():
        out = fn()
    return out, np.array(LOG, np.float64).reshape(-1, 4)


def case(name: str) -> dict:
    ctor, B, scale = CASES[name]
    torch.manual_seed(0)
    flow = ctor().eval()
    out = {"sd_keys": np.array(list(flow.state_dict().keys())), "sd_crc": np.array([crc(v) for v in flow.state_dict().values()], np.uint32)}
    with torch.no_grad():
        for p in flow.parameters():
            p.mul_(scale)
    for k, v in flow.state_dict().items():
        out[f"sd/{k}"] = v.numpy()
    t = flow.transform
    D, C = t.ode[-1].weight.shape[0], t.ode[0].weight.shape[1] - t.ode[-1].weight.shape[0] - 2 * t.freqs.numel()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, D, generator=g)
    z = torch.randn(B, D, generator=g)
    c = torch.randn(B, C, generator=g) if C else None
    out.update(x=x.numpy(), z=z.numpy(), D=D, C=C, atol=t.atol, rtol=t.rtol)
    if c is not None:
        out["c"] = c.numpy()
    out["act"] = np.array(type(t.ode[1]).__name__ if len(t.ode) > 1 else "ReLU")
    TOL[:] = [(t.atol, t.rtol)]
    for tag, dtype in (("32", torch.float32), ("64", torch.float64)):
        f = flow.to(dtype)
        xd, zd = x.to(dtype), z.to(dtype)
        cd = None if c is None else c.to(dtype)
        lp, out[f"log_lp_{tag}"] = run(lambda: f(cd).log_prob(xd))
        out[f"lp_{tag}"] = lp.numpy()
        y, out[f"log_fwd_{tag}"] = run(lambda: f(cd).transform(xd))
        out[f"fwd_{tag}"] = y.numpy()
        xi, out[f"log_inv_{tag}"] = run(lambda: f(cd).transform.inv(zd))
        out[f"inv_{tag}"] = xi.numpy()
        dist = f(cd)
        (xs, ladj), out[f"log_rs_{tag}"] = run(lambda: dist.transform.inv.call_and_ladj(zd))
        out[f"rs_x_{tag}"] = xs.numpy()
        out[f"rs_lp_{tag}"] = (dist.base.log_prob(zd) - ladj).numpy()
        f.transform.exact = False
        torch.manual_seed(123)
        eps = torch.randn_like(xd)
        torch.manual_seed(123)
        (yh, lh), out[f"log_hut_{tag}"] = run(lambda: f(cd).transform.call_and_ladj(xd))
        f.transform.exact = True
        out[f"hut_eps_{tag}"] = eps.numpy()
        out[f"hut_y_{tag}"] = yh.numpy()
        out[f"hut_ladj_{tag}"] = lh.numpy()
    # the reference's own fp32-fp64 gap per output (relative, max(1, |v|) floor)
    for k in ("lp", "fwd", "inv", "rs_x", "rs_lp"):
        a, b = out[f"{k}_32"].astype(np.float64), out[f"{k}_64"]
        out[f"gap_{k}"] = float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1.0)))
    return out


def main() -> None:
    torch.set_num_threads(8)
    for name in CASES:
        out = case(name)
        np.savez_compressed(OUT / f"flow_{name}.npz", **out)
        print(name, {k: len(v) for k, v in out.items() if k.startswith("log_")}, f"gap_lp {out['gap_lp']:.2e}", flush=True)


if __name__ == "__main__":
    main()
