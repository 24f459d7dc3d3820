"""Gradient goldens of the continuous normalizing flow (CNF) from the UNMODIFIED reference's adaptive checkpoint
adjoint (zuko/utils.py:556-593), in fp32 and fp64, each with the forward's per-trial step log (t, dt, error,
accepted), recorded by wrapping zuko.utils.dopri45 inside this script only.  Run in the build container only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_cnf_grad.py

Per case of make_golden_cnf.py (same flows, weights and inputs) and dtype, in training mode:
  lp:  sum_i w_i log_prob(x)_i for seeded weights w;
  fwd: <gy, transform(x)>;
  rs:  <gy, x> + <gl, ladj> of inv.call_and_ladj(z) (the direction of rsample_and_log_prob);
  hut: <gy, y> + <gl, ladj> of a Hutchinson call_and_ladj(x), with its eps;
each with the gradients of x (or z), c and every weight and bias.  Then, in eval mode, lp's gradients of x and c
(asserting that the parameters get no .grad), a broadcast context c of shape (C,), and the loss curve of 20 Adam
steps of a small CNF on a seeded dataset.
"""

from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

sys.dont_write_bytecode = True
sys.path.insert(0, "/root/reference")

import zuko.utils as U  # noqa: E402
from zuko.flows import CNF  # noqa: E402

OUT = Path(__file__).resolve().parent

# mirrors make_golden_cnf.py:CASES
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
TOL: list = []
RECORD = [True]


def _logged(f, x, t, dt, error=False):  # noqa: ANN001, ANN202
    out = _dopri(f, x, t, dt, error)
    if error and RECORD[0]:
        y, err = out
        atol, rtol = TOL[0]
        tol = atol + rtol * torch.max(abs(x), abs(y))
        e = torch.max(err / tol).clip(min=1e-9).item()
        LOG.append((float(t), float(dt), e, float(e < 1.0)))
    return out


U.dopri45 = _logged


def grads(flow, loss_fn, *inputs):  # noqa: ANN001, ANN202
    """Runs loss_fn (forward logged, backward not), returns (forward log, {name: grad})."""
    for p in flow.parameters():
        p.grad = None
    LOG.clear()
    RECORD[0] = True
    loss = loss_fn()
    log = np.array(LOG, np.float64).reshape(-1, 4)
    RECORD[0] = False
    loss.backward()
    out = {}
    for i, t in enumerate(inputs):
        if t is not None:
            out[f"in{i}"] = t.grad.numpy().copy()
    for k, p in flow.transform.named_parameters():
        if p.grad is not None:
            out[k] = p.grad.numpy().copy()
    return log, out


def case(name: str) -> dict:
    ctor, B, scale = CASES[name]
    torch.manual_seed(0)
    flow = ctor()
    with torch.no_grad():
        for p in flow.parameters():
            p.mul_(scale)
    out = {f"sd/{k}": v.numpy() for k, v in flow.state_dict().items()}
    t = flow.transform
    D, C = t.ode[-1].weight.shape[0], t.ode[0].weight.shape[1] - t.ode[-1].weight.shape[0] - 2 * t.freqs.numel()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, D, generator=g)
    z = torch.randn(B, D, generator=g)
    c = torch.randn(B, C, generator=g) if C else None
    g2 = torch.Generator().manual_seed(2)
    w = torch.randn(B, generator=g2)
    gy = torch.randn(B, D, generator=g2)
    gl = torch.randn(B, generator=g2)
    out.update(x=x.numpy(), z=z.numpy(), w=w.numpy(), gy=gy.numpy(), gl=gl.numpy(), D=D, C=C, atol=t.atol, rtol=t.rtol)
    if c is not None:
        out["c"] = c.numpy()
    out["act"] = np.array(type(t.ode[1]).__name__ if len(t.ode) > 1 else "ReLU")
    TOL[:] = [(t.atol, t.rtol)]
    for tag, dtype in (("32", torch.float32), ("64", torch.float64)):
        f = flow.to(dtype).train()

        def leaf(v):  # noqa: ANN001, ANN202
            return None if v is None else v.to(dtype).clone().requires_grad_()

        ops = {}
        xd, cd = leaf(x), leaf(c)
        ops["lp"] = grads(f, lambda: (f(cd).log_prob(xd) * w.to(dtype)).sum(), xd, cd)
        xd, cd = leaf(x), leaf(c)
        ops["fwd"] = grads(f, lambda: (f(cd).transform(xd) * gy.to(dtype)).sum(), xd, cd)
        zd, cd = leaf(z), leaf(c)

        def rs():  # noqa: ANN202
            xs, ladj = f(cd).transform.inv.call_and_ladj(zd)
            return (xs * gy.to(dtype)).sum() + (ladj * gl.to(dtype)).sum()

        ops["rs"] = grads(f, rs, zd, cd)
        xd, cd = leaf(x), leaf(c)
        f.transform.exact = False
        torch.manual_seed(123)
        eps = torch.randn(B, D, dtype=dtype)
        torch.manual_seed(123)

        def hut():  # noqa: ANN202
            y, ladj = f(cd).transform.call_and_ladj(xd)
            return (y * gy.to(dtype)).sum() + (ladj * gl.to(dtype)).sum()

        ops["hut"] = grads(f, hut, xd, cd)
        f.transform.exact = True
        out[f"hut_eps_{tag}"] = eps.numpy()
        f.eval()
        xd, cd = leaf(x), leaf(c)
        ops["eval"] = grads(f, lambda: (f(cd).log_prob(xd) * w.to(dtype)).sum(), xd, cd)
        assert all(p.grad is None for p in f.parameters()), "eval mode: the ODE parameters must get no .grad"
        if c is not None:
            f.train()
            xd, cb = leaf(x), leaf(c[0])
            ops["bcast"] = grads(f, lambda: (f(cb).log_prob(xd) * w.to(dtype)).sum(), xd, cb)
        for op, (log, gr) in ops.items():
            out[f"log_{op}_{tag}"] = log
            for k, v in gr.items():
                out[f"g_{op}_{tag}/{k}"] = v
    return out


def adam_curve() -> dict:
    """20 Adam steps (lr 1e-2) of CNF(2, 1, hidden_features=[16, 16]) on 256 seeded rows, fp32."""
    torch.manual_seed(0)
    flow = CNF(2, 1, hidden_features=[16, 16])
    g = torch.Generator().manual_seed(5)
    c = torch.randn(256, 1, generator=g)
    x = torch.randn(256, 2, generator=g) * 0.5 + c
    out = {f"adam_sd/{k}": v.numpy().copy() for k, v in flow.state_dict().items()}
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    losses, steps = [], []
    RECORD[0] = True
    for _ in range(20):
        LOG.clear()
        loss = -flow(c).log_prob(x).mean()
        steps.append(int(np.array(LOG).reshape(-1, 4)[:, 3].sum()))
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    out.update(adam_x=x.numpy(), adam_c=c.numpy(), adam_loss=np.array(losses), adam_accepted=np.array(steps))
    return out


def main() -> None:
    torch.set_num_threads(8)
    TOL[:] = [(1e-6, 1e-5)]
    np.savez_compressed(OUT / "cnfgrad_adam.npz", **adam_curve())
    for name in CASES:
        out = case(name)
        np.savez_compressed(OUT / f"cnfgrad_{name}.npz", **out)
        print(name, {k: len(v) for k, v in out.items() if k.startswith("log_")}, flush=True)


if __name__ == "__main__":
    main()
