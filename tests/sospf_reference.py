"""fp64 restatement of the sum-of-squares polynomial bijector and flow (zuko/transforms.py:878-963,
zuko/utils.py:159-183, 246-363, zuko/flows/polynomial.py:23-76) in numpy, for the SOSPF tests.

The flow is evaluated from a state dict with the key layout of ``SOSPF``: ``transforms.{2i}`` masked
autoregressive layers (``order`` buffer, ``hyper.{j}.weight / bias / mask`` with ReLU between the linear
layers), ``transforms.{2i+1}`` soft clips with bound 11, and a ``DiagNormal`` base."""

from __future__ import annotations

import math

import numpy as np


def steps(bound: float = 10.0, eps: float = 1e-6) -> int:
    return math.ceil(math.log2(2 * bound / eps))


def nodes(n: int):
    """Gauss-Legendre nodes and weights on [0, 1] (GaussLegendre.nodes, utils.py:323-340)."""
    t, w = np.polynomial.legendre.leggauss(n)
    return (t + 1) / 2, w / 2


def g(x, a, slope=1e-3, bound=10.0):
    """(1/K) sum_k (1 + sum_j a_kj (x / B)^j)^2 + slope; a (..., K, L+1) broadcast with x (...)."""
    x = np.asarray(x, np.float64)
    a = np.asarray(a, np.float64)
    v = (x / bound)[..., None] ** np.arange(a.shape[-1])  # (..., L+1)
    p = 1 + np.einsum("...kj,...j->...k", a, v)
    return np.mean(p**2, -1) + slope


def f(x, a, slope=1e-3, bound=10.0):
    """x sum_i w_i g(t_i x), the quadrature of SOSPolynomialTransform.f with n = L + 1 nodes."""
    x = np.asarray(x, np.float64)
    t, w = nodes(np.shape(a)[-1])
    return x * sum(w[i] * g(t[i] * x, a, slope, bound) for i in range(len(t)))


def forward(x, a, constant, slope=1e-3, bound=10.0):
    """y, ladj of ShiftedSOSPTransform(a, constant)."""
    return f(x, a, slope, bound) + np.asarray(constant, np.float64), np.log(g(x, a, slope, bound))


def inverse(y, a, constant, slope=1e-3, bound=10.0, eps=1e-6):
    """The reference's bisection (utils.py:159-183) on y - constant, in fp64."""
    y = np.asarray(y, np.float64) - np.asarray(constant, np.float64)
    lo = np.full_like(y, -bound)
    hi = np.full_like(y, bound)
    for _ in range(steps(bound, eps)):
        m = (lo + hi) / 2
        below = f(m, a, slope, bound) < y
        lo = np.where(below, m, lo)
        hi = np.where(below, hi, m)
    return (lo + hi) / 2


def grad(x, a, constant, gy, gl, slope=1e-3, bound=10.0):
    """(gx, ga, gconst) of <gy, y> + <gl, ladj>, per element (no reduction over broadcast parameters)."""
    x = np.asarray(x, np.float64)
    a = np.broadcast_to(np.asarray(a, np.float64), x.shape + np.shape(a)[-2:])
    K, n = a.shape[-2:]
    gy, gl = np.asarray(gy, np.float64), np.asarray(gl, np.float64)
    j = np.arange(n)
    t, w = nodes(n)

    def p_and_pow(u):
        v = (u / bound)[..., None] ** j
        return 1 + np.einsum("...kj,...j->...k", a, v), v

    gv = g(x, a, slope, bound)
    px, vx = p_and_pow(x)
    dv = np.where(j > 0, j * (x / bound)[..., None] ** np.maximum(j - 1, 0), 0.0) / bound  # d v^j / dx
    dg = (2 / K) * np.sum(px * np.einsum("...kj,...j->...k", a, dv), -1)
    gx = gy * gv + gl * dg / gv
    ga = (gl / gv)[..., None, None] * (2 / K) * px[..., :, None] * vx[..., None, :]
    for i in range(n):
        pi, vi = p_and_pow(t[i] * x)
        ga = ga + (gy * x * w[i])[..., None, None] * (2 / K) * pi[..., :, None] * vi[..., None, :]
    return gx, ga, gy.copy()


class Flow:
    """An SOSPF from its state dict (numpy arrays)."""

    def __init__(self, sd: dict, features: int, context: int, polynomials: int, degree: int, slope: float = 1e-3) -> None:
        self.D, self.C, self.K, self.L, self.slope = features, context, polynomials, degree, slope
        n = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transform.transforms."))
        self.layers = []
        for i in range(n):
            pre = f"transform.transforms.{i}."
            if i % 2:
                self.layers.append(("clip", None))
                continue
            lin = sorted({int(k[len(pre) + 6 :].split(".")[0]) for k in sd if k.startswith(pre + "hyper.")})
            Ws = [np.asarray(sd[f"{pre}hyper.{j}.weight"], np.float64) * np.asarray(sd[f"{pre}hyper.{j}.mask"], np.float64) for j in lin]
            bs = [np.asarray(sd[f"{pre}hyper.{j}.bias"], np.float64) for j in lin]
            self.layers.append(("maf", (Ws, bs, int(np.max(sd[pre + "order"])) + 1)))
        self.loc = np.asarray(sd["base.loc"], np.float64)
        self.scale = np.asarray(sd["base.scale"], np.float64)

    def _params(self, p, x, c):
        Ws, bs, _ = p
        B = x.shape[0]
        h = x if not self.C else np.concatenate([x, np.broadcast_to(np.asarray(c, np.float64), (B, self.C))], -1)
        for j, (W, b) in enumerate(zip(Ws, bs)):
            h = h @ W.T + b
            if j < len(Ws) - 1:
                h = np.maximum(h, 0.0)
        P = self.K * (self.L + 1) + 1
        h = h.reshape(B, self.D, P)
        return h[..., :-1].reshape(B, self.D, self.K, self.L + 1), h[..., -1]

    def call_and_ladj(self, x, c=None):
        z = np.asarray(x, np.float64)
        ladj = np.zeros(z.shape[0])
        for kind, p in self.layers:
            if kind == "clip":
                ladj += (-2 * np.log1p(np.abs(z / 11.0))).sum(-1)
                z = z / (1 + np.abs(z / 11.0))
                continue
            a, const = self._params(p, z, c)
            z, l = forward(z, a, const, self.slope)
            ladj += l.sum(-1)
        return z, ladj

    def log_prob(self, x, c=None):
        z, ladj = self.call_and_ladj(x, c)
        u = (z - self.loc) / self.scale
        return ladj + (-0.5 * u**2 - np.log(self.scale) - 0.5 * math.log(2 * math.pi)).sum(-1)

    def inverse(self, z, c=None):
        """The reference's inverse: per autoregressive layer, `passes` fixed-point sweeps from x = 0
        (transforms.py:994-1000), each a bisection per element."""
        y = np.asarray(z, np.float64)
        for kind, p in reversed(self.layers):
            if kind == "clip":
                y = y / (1 - np.abs(y / 11.0))
                continue
            x = np.zeros_like(y)
            for _ in range(p[2]):
                a, const = self._params(p, x, c)
                x = inverse(y, a, const, self.slope)
            y = x
        return y
