"""fp64 restatement of the Gaussianization bijector and flow (zuko/transforms.py:834-875,
zuko/utils.py:159-183, zuko/flows/gaussianization.py:97-155) in numpy / scipy, for the GF tests.

The flow is evaluated from a state dict with the key layout of ``GF``: ``transforms.{2i}`` element-wise
layers (``hyper.*`` MLP with ReLU, or ``phi.{0,1}`` tables), ``transforms.{2i+1}.A`` rotation generators
and a ``DiagNormal`` base."""

from __future__ import annotations

import math

import numpy as np
from scipy.linalg import expm
from scipy.special import erf, erfinv, logsumexp

C = 1.0 - 1e-6


def steps(bound: float, eps: float) -> int:
    return math.ceil(math.log2(2 * bound / eps))


def forward(x, shift, scale):
    """y, ladj of GaussianizationTransform(shift, scale) at x; shift / scale (..., K) broadcast with x (...)."""
    x = np.asarray(x, np.float64)[..., None]
    shift, scale = np.asarray(shift, np.float64), np.asarray(scale, np.float64)
    K = shift.shape[-1]
    u = x * np.exp(scale) + shift
    y = math.sqrt(2) * erfinv(np.mean(erf(u / math.sqrt(2)), -1) * C)
    ladj = 0.5 * y**2 + math.log(C / K) + logsumexp(scale - 0.5 * u**2, axis=-1)
    return y, ladj


def grad(x, shift, scale, gy, gl):
    """(gx, gshift, gscale) of <gy, y> + <gl, ladj>, per element (no reduction over broadcast parameters)."""
    x = np.asarray(x, np.float64)
    y, _ = forward(x, shift, scale)
    s = np.exp(np.asarray(scale, np.float64))
    u = x[..., None] * s + shift
    t = scale - 0.5 * u**2
    L = logsumexp(t, axis=-1, keepdims=True)
    w = np.exp(t - L)
    K = s.shape[-1]
    e = np.exp(0.5 * y[..., None] ** 2 + math.log(C / K) - 0.5 * u**2)  # dy/dshift_k
    G = (gy + gl * y)[..., None]
    gl_ = np.asarray(gl, np.float64)[..., None]
    gx = (G[..., 0] * (e * s).sum(-1)) - gl * (w * u * s).sum(-1)
    gshift = G * e - gl_ * w * u
    gscale = G * e * s * x[..., None] + gl_ * w * (1.0 - u * s * x[..., None])
    return gx, gshift, gscale


def inverse(y, shift, scale, bound: float = 10.0, eps: float = 1e-6):
    """The reference's bisection (utils.py:159-183), in fp64."""
    y = np.asarray(y, np.float64)
    a = np.full_like(y, -bound)
    b = np.full_like(y, bound)
    for _ in range(steps(bound, eps)):
        m = (a + b) / 2
        below = forward(m, shift, scale)[0] < y
        a = np.where(below, m, a)
        b = np.where(below, b, m)
    return (a + b) / 2


class Flow:
    """A GF from its state dict (numpy arrays)."""

    def __init__(self, sd: dict, features: int, context: int, components: int) -> None:
        self.D, self.C, self.K = features, context, components
        n = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transform.transforms."))
        self.layers = []
        for i in range(n):
            pre = f"transform.transforms.{i}."
            if i % 2:
                A = np.asarray(sd[pre + "A"], np.float64)
                self.layers.append(("rot", expm(A - A.T)))
            elif context:
                lin = sorted({int(k[len(pre) + 6 :].split(".")[0]) for k in sd if k.startswith(pre + "hyper.")})
                Ws = [np.asarray(sd[f"{pre}hyper.{j}.weight"], np.float64) for j in lin]
                bs = [np.asarray(sd[f"{pre}hyper.{j}.bias"], np.float64) for j in lin]
                self.layers.append(("mlp", (Ws, bs)))
            else:
                self.layers.append(("phi", (np.asarray(sd[pre + "phi.0"], np.float64), np.asarray(sd[pre + "phi.1"], np.float64))))
        self.loc = np.asarray(sd["base.loc"], np.float64)
        self.scale = np.asarray(sd["base.scale"], np.float64)

    def _params(self, kind, p, c, B):
        if kind == "phi":
            return p
        Ws, bs = p
        h = np.broadcast_to(np.asarray(c, np.float64), (B, self.C))
        for j, (W, b) in enumerate(zip(Ws, bs)):
            h = h @ W.T + b
            if j < len(Ws) - 1:
                h = np.maximum(h, 0.0)
        h = h.reshape(B, self.D, 2 * self.K)
        return h[..., : self.K], h[..., self.K :]

    def call_and_ladj(self, x, c=None):
        z = np.asarray(x, np.float64)
        B = z.shape[0]
        ladj = np.zeros(B)
        for kind, p in self.layers:
            if kind == "rot":
                z = z @ p.T
                continue
            shift, scale = self._params(kind, p, c, B)
            z, l = forward(z, shift, scale)
            ladj += l.sum(-1)
        return z, ladj

    def log_prob(self, x, c=None):
        z, ladj = self.call_and_ladj(x, c)
        u = (z - self.loc) / self.scale
        return ladj + (-0.5 * u**2 - np.log(self.scale) - 0.5 * math.log(2 * math.pi)).sum(-1)

    def inverse(self, z, c=None, bound: float = 10.0, eps: float = 1e-6):
        x = np.asarray(z, np.float64)
        B = x.shape[0]
        for kind, p in reversed(self.layers):
            if kind == "rot":
                x = x @ p
                continue
            shift, scale = self._params(kind, p, c, B)
            x = inverse(x, shift, scale, bound, eps)
        return x
