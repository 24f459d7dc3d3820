"""fp64 restatement of the CNF backward (AdaptiveCheckpointAdjoint.backward, zuko/utils.py:556-593, on the packed
state (x, L) of call_and_ladj, transforms.py:1147-1179) at a given step log.

The states after each accepted step are replayed in fp64 (cnf_reference.dopri).  From each (t + dt, x_k) one
6-stage Dormand-Prince step of -dt is taken on (a, g_phi) with
    da/dt = -(a^T df/dx + a_L 1e-2 dtau/dx),   dg_phi/dt = -(a^T df/dphi + a_L 1e-2 dtau/dphi),
a_L = grad_ladj / 1e-2.  The vector-Jacobian products, second-order terms of the trace included, come from torch
autograd in float64 on the CPU (double backward through the trace), so this shares no code with the engine's
hand-written reverse mode."""

from __future__ import annotations

import numpy as np
import torch

import cnf_reference as R

_ACTS = {
    "ReLU": torch.nn.ReLU(),
    "ELU": torch.nn.ELU(),
    "Tanh": torch.nn.Tanh(),
    "SiLU": torch.nn.SiLU(),
    "GELU": torch.nn.GELU(),
    "LeakyReLU": torch.nn.LeakyReLU(),
    "Softplus": torch.nn.Softplus(),
    "Sigmoid": torch.nn.Sigmoid(),
}


def _f(field: R.Field, W, b, t: float, x, c):
    """f(t, x, c) of the field with torch weights W, b (rows of x, c)."""
    ft = torch.as_tensor(field.freqs * t, dtype=torch.float64)
    emb = torch.cat([ft.cos(), ft.sin()]).expand(x.shape[0], -1)
    h = torch.cat([emb, x] + ([c] if field.C else []), dim=1)
    n = len(W)
    for i in range(n):
        h = h @ W[i].T + b[i]
        if i < n - 1:
            h = _ACTS[field.act](h)
    return h


def _tau(f, x, trace: int, eps):
    """tau(x) per row with its graph: tr(df/dx) or eps^T (df/dx) eps."""
    if trace == R.TRACE_EXACT:
        return sum(torch.autograd.grad(f[:, i].sum(), x, create_graph=True)[0][:, i] for i in range(x.shape[1]))
    return (torch.autograd.grad(f, x, eps, create_graph=True)[0] * eps).sum(dim=1)


def adjoint(field: R.Field, x, c, step_log, trace: int, eps=None, gy=None, gl=None):
    """Gradients of <gy, y> + <gl, ladj> for the integration of x (B, D) along the accepted steps of step_log
    (rows (t, dt, error, accepted)): dict with "x" (B, D), "c" (B, C) per row or None, "W" / "b" lists."""
    x = np.asarray(x, np.float64)
    B, D = x.shape
    states = [x]
    L = np.zeros(B) if trace else None
    steps = [(float(t), float(dt)) for t, dt, _, acc in step_log if acc]
    for t, dt in steps:
        nxt, _, _ = R.dopri(field, states[-1], L, t, dt, c, trace, eps)
        states.append(nxt[:, :D])
        L = nxt[:, -1] if trace else None
    W = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in field.W]
    bb = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in field.b]
    ct = None
    if field.C:
        ct = torch.tensor(np.broadcast_to(np.asarray(c, np.float64), (B, field.C)).copy(), requires_grad=True)
    et = None if eps is None else torch.tensor(np.asarray(eps, np.float64))
    a = np.zeros((B, D)) if gy is None else np.asarray(gy, np.float64).copy()
    alpha = None
    if trace:
        alpha = torch.tensor(np.asarray(gl, np.float64) / R.TRACE_SCALE * R.TRACE_SCALE)
    params = W + bb + ([ct] if ct is not None else [])
    gphi = [np.zeros(p.shape) for p in params]
    b6 = R.A[6]
    for k in range(len(steps), 0, -1):
        t, dt = steps[k - 1]
        tp, h = t + dt, -dt
        xk = states[k]
        kx, ka = [], []
        for s in range(6):
            xs = xk + sum(R.A[s][m] * h * kx[m] for m in range(s)) if s else xk
            as_ = a + sum(R.A[s][m] * h * ka[m] for m in range(s)) if s else a
            xt = torch.tensor(xs, requires_grad=True)
            f = _f(field, W, bb, tp + R.C[s] * h, xt, ct)
            phi_ = (f * torch.tensor(as_)).sum()
            if trace:
                phi_ = phi_ + (alpha * _tau(f, xt, trace, et)).sum()
            g = torch.autograd.grad(phi_, [xt, *params], allow_unused=True)
            kx.append(f.detach().numpy())
            ka.append(-g[0].numpy())
            if b6[s] != 0:
                for i, gi in enumerate(g[1:]):
                    if gi is not None:
                        gphi[i] += dt * b6[s] * gi.numpy()
        a = a + sum(b6[m] * h * ka[m] for m in range(6))
    n = len(W)
    return {"x": a, "W": gphi[:n], "b": gphi[n : 2 * n], "c": gphi[2 * n] if ct is not None else None}
