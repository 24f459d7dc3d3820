"""fp64 restatement of the bounded Bernstein bijector and the Bernstein polynomial flow
(zuko/transforms.py:640-831, zuko/utils.py:159-209, zuko/flows/polynomial.py:79-117) in numpy, for the
BPF tests.

The bijector is evaluated by de Casteljau's algorithm on the coefficients theta (O(M^2), every step a
convex combination), the accuracy yardstick of the kernels' O(M) ratio recurrence.  The flow is
evaluated from a state dict with the key layout of ``MAF``: ``transform.transforms.{i}`` masked
autoregressive layers (``order`` buffer, ``hyper.{j}.weight / bias / mask`` with ReLU between the linear
layers) and a ``DiagNormal`` base."""

from __future__ import annotations

import math

import numpy as np


def steps(bound: float = 5.0, eps: float = 1e-6) -> int:
    return math.ceil(math.log2(2 * bound / eps))


def softmax(u):
    u = np.asarray(u, np.float64)
    e = np.exp(u - u.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def theta(u, bound=5.0):
    """The M + 1 rising coefficients of BoundedBernsteinTransform._constrain_theta: M = P + 4, or 3 when
    P = 1 (``ones_like(diffs[..., :2])`` then has one entry)."""
    u = np.asarray(u, np.float64)
    P = u.shape[-1]
    db = 2 * bound / (P + 4)
    ones = np.ones(u.shape[:-1] + (min(P, 2),))
    diffs = np.concatenate([-bound * ones[..., :1], db * ones, softmax(u) * (2 * bound - 4 * db), db * ones], -1)
    return np.cumsum(diffs, -1)


def casteljau(c, t):
    """sum_i c_i b_{i,n}(t) for coefficients c (..., n + 1) and t (...)."""
    c = np.array(c, np.float64)
    t = np.asarray(t, np.float64)[..., None]
    while c.shape[-1] > 1:
        c = (1 - t) * c[..., :-1] + t * c[..., 1:]
    return c[..., 0]


def forward(x, u, bound=5.0, eps=1e-6):
    """y, ladj of BoundedBernsteinTransform(u, bound, eps); u broadcasts with x (..., P)."""
    x = np.asarray(x, np.float64)
    th = theta(u, bound)
    th = np.broadcast_to(th, x.shape + th.shape[-1:])
    M = th.shape[-1] - 1
    t = (x + bound) / (2 * bound)
    lo, hi = t <= eps, t >= 1 - eps
    ts = np.where(lo | hi, 0.5, t)
    y = casteljau(th, ts)
    dy = M * casteljau(np.diff(th, axis=-1), ts) / (2 * bound)
    y = np.where(lo, 2 * bound * (t - eps) - bound, y)
    y = np.where(hi, 2 * bound * (t - 1 + eps) + bound, y)
    dy = np.where(lo | hi, 1.0, dy)
    return y, np.log(dy)


def inverse(y, u, bound=5.0, eps=1e-6):
    """The reference's inverse: the linear branches beyond [-B, B], else bisection of the full f."""
    y = np.asarray(y, np.float64)
    lo = np.full_like(y, -bound)
    hi = np.full_like(y, bound)
    for _ in range(steps(bound, eps)):
        m = (lo + hi) / 2
        below = forward(m, u, bound, eps)[0] < y
        lo = np.where(below, m, lo)
        hi = np.where(below, hi, m)
    x = (lo + hi) / 2
    x0 = ((y + bound) / (2 * bound) + eps) * 2 * bound - bound
    x1 = ((y - bound) / (2 * bound) - eps + 1) * 2 * bound - bound
    return np.where(y <= -bound, x0, np.where(y >= bound, x1, x))


def grad(x, u, gy, gl, bound=5.0, eps=1e-6):
    """(gx, gu) of <gy, y> + <gl, ladj>, per element (no reduction over broadcast parameters)."""
    x = np.asarray(x, np.float64)
    u = np.broadcast_to(np.asarray(u, np.float64), x.shape + np.shape(u)[-1:])
    gy, gl = np.asarray(gy, np.float64), np.asarray(gl, np.float64)
    P = u.shape[-1]
    e = min(P, 2)
    M = P + 2 * e
    t = (x + bound) / (2 * bound)
    inside = (t > eps) & (t < 1 - eps)
    ts = np.where(inside, t, 0.5)
    th = theta(u, bound)
    d = np.diff(th, axis=-1)  # Delta_1 .. Delta_M
    k = np.arange(M + 1)
    comb = np.array([math.comb(M, i) for i in k], np.float64)
    b = comb * ts[..., None] ** k * (1 - ts[..., None]) ** (M - k)  # b_{i,M}
    k1 = np.arange(M)
    b1 = np.array([math.comb(M - 1, i) for i in k1]) * ts[..., None] ** k1 * (1 - ts[..., None]) ** (M - 1 - k1)
    fp = M / (2 * bound) * (d * b1).sum(-1)
    fpp = M * (M - 1) / (2 * bound) ** 2 * casteljau(np.diff(d, axis=-1), ts)
    gx = np.where(inside, gy * fp + gl * fpp / fp, gy)
    S = np.cumsum(b[..., ::-1], -1)[..., ::-1][..., 1:]  # S_j = sum_{i >= j} b_{i,M}, j = 1 .. M
    gd = gy[..., None] * S + (gl / fp)[..., None] * (M / (2 * bound)) * b1
    w = softmax(u)
    dw = 2 * bound - 4 * 2 * bound / (P + 4)
    gw = dw * gd[..., e : M - e]
    gu = w * (gw - (w * gw).sum(-1, keepdims=True))
    return gx, np.where(inside[..., None], gu, 0.0)


class Flow:
    """A MAF with BoundedBernsteinTransform(bound) from its state dict (numpy arrays)."""

    def __init__(self, sd: dict, features: int, context: int, degree: int, bound: float = 5.0) -> None:
        self.D, self.C, self.P, self.bound = features, context, degree + 1, bound
        n = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transform.transforms."))
        self.layers = []
        for i in range(n):
            pre = f"transform.transforms.{i}."
            lin = sorted({int(k[len(pre) + 6 :].split(".")[0]) for k in sd if k.startswith(pre + "hyper.")})
            Ws = [np.asarray(sd[f"{pre}hyper.{j}.weight"], np.float64) * np.asarray(sd[f"{pre}hyper.{j}.mask"], np.float64) for j in lin]
            bs = [np.asarray(sd[f"{pre}hyper.{j}.bias"], np.float64) for j in lin]
            self.layers.append((Ws, bs, int(np.max(sd[pre + "order"])) + 1))
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
        return h.reshape(B, self.D, self.P)

    def call_and_ladj(self, x, c=None):
        z = np.asarray(x, np.float64)
        ladj = np.zeros(z.shape[0])
        for p in self.layers:
            z, l = forward(z, self._params(p, z, c), self.bound)
            ladj += l.sum(-1)
        return z, ladj

    def log_prob(self, x, c=None):
        z, ladj = self.call_and_ladj(x, c)
        u = (z - self.loc) / self.scale
        return ladj + (-0.5 * u**2 - np.log(self.scale) - 0.5 * math.log(2 * math.pi)).sum(-1)

    def inverse(self, z, c=None):
        """The reference's inverse: per layer, `passes` fixed-point sweeps from x = 0
        (transforms.py:994-1000), each a bisection per element."""
        y = np.asarray(z, np.float64)
        for p in reversed(self.layers):
            x = np.zeros_like(y)
            for _ in range(p[2]):
                x = inverse(y, self._params(p, x, c), self.bound)
            y = x
        return y
