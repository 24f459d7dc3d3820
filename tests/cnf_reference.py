"""fp64 numpy restatement of the continuous normalizing flow (zuko/flows/continuous.py, transforms.py:1095-1179,
utils.py:443-554): the vector field's MLP, the forward-mode trace, one Dormand-Prince step, and the batch-shared
step controller.  `integrate` runs its own controller; `replay` integrates a given sequence of accepted steps,
which is how the engine's fp32 results are compared: at the engine's own step sequence, not at an
independently controlled one (a different accept / reject decision moves the result by far more than fp32
rounding does)."""

from __future__ import annotations

import math

import numpy as np
from scipy.special import erf

TRACE_NONE, TRACE_EXACT, TRACE_HUTCHINSON = 0, 1, 2
TRACE_SCALE = 1e-2

A = [
    [],
    [1 / 5],
    [3 / 40, 9 / 40],
    [44 / 45, -56 / 15, 32 / 9],
    [19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729],
    [9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656],
    [35 / 384, 0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84],
]
E7 = [5179 / 57600, 0, 7571 / 16695, 393 / 640, -92097 / 339200, 187 / 2100, 1 / 40]
C = [0, 1 / 5, 3 / 10, 4 / 5, 8 / 9, 1, 1]


def _act(name: str, v: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """(act(v), act'(v)) in fp64."""
    if name == "ReLU":
        return np.maximum(v, 0), (v > 0).astype(v.dtype)
    if name == "ELU":
        return np.where(v > 0, v, np.expm1(np.minimum(v, 0))), np.where(v > 0, 1.0, np.exp(np.minimum(v, 0)))
    if name == "Tanh":
        t = np.tanh(v)
        return t, 1 - t * t
    if name == "SiLU":
        s = 1 / (1 + np.exp(-v))
        return v * s, s * (1 + v * (1 - s))
    if name == "GELU":
        return 0.5 * v * (1 + erf(v / math.sqrt(2))), 0.5 * (1 + erf(v / math.sqrt(2))) + v * np.exp(-0.5 * v * v) / math.sqrt(2 * math.pi)
    if name == "LeakyReLU":
        return np.where(v > 0, v, 0.01 * v), np.where(v > 0, 1.0, 0.01)
    if name == "Softplus":
        return np.where(v > 20, v, np.log1p(np.exp(np.minimum(v, 20)))), np.where(v > 20, 1.0, 1 / (1 + np.exp(-v)))
    if name == "Sigmoid":
        s = 1 / (1 + np.exp(-v))
        return s, s * (1 - s)
    raise ValueError(name)


class Field:
    """f(t, x, c) = ode(cat(cos(freqs t), sin(freqs t), x, c)) and its trace (flows/continuous.py:88-97)."""

    def __init__(self, weights, biases, freqs, D: int, C: int, act: str) -> None:
        self.W = [np.asarray(w, np.float64) for w in weights]
        self.b = [np.asarray(b, np.float64) for b in biases]
        self.freqs = np.asarray(freqs, np.float64)
        self.D, self.C, self.act = D, C, act

    @classmethod
    def from_state_dict(cls, sd: dict, D: int, C: int, act: str) -> Field:
        n = len([k for k in sd if k.startswith("transform.ode.") and k.endswith(".weight")])
        W = [sd[f"transform.ode.{2 * i}.weight"] for i in range(n)]
        b = [sd[f"transform.ode.{2 * i}.bias"] for i in range(n)]
        return cls(W, b, sd["transform.freqs"], D, C, act)

    def __call__(self, t: float, x: np.ndarray, c: np.ndarray | None, trace: int, eps: np.ndarray | None):
        B, D = x.shape
        ft = self.freqs * t
        emb = np.broadcast_to(np.concatenate([np.cos(ft), np.sin(ft)]), (B, 2 * len(self.freqs)))
        h = np.concatenate([emb, x] + ([np.broadcast_to(c, (B, self.C))] if self.C else []), axis=1)
        F2 = 2 * len(self.freqs)
        derivs = []
        n = len(self.W)
        for i, (W, b) in enumerate(zip(self.W, self.b, strict=True)):
            pre = h @ W.T + b
            if i < n - 1:
                h, d = _act(self.act, pre)
                derivs.append(d)
            else:
                h = pre
        if trace == TRACE_NONE:
            return h, None
        # forward-mode tangents through the MLP
        if trace == TRACE_EXACT:
            T = np.broadcast_to(self.W[0][:, F2 : F2 + D], (B, *self.W[0][:, F2 : F2 + D].shape)).copy()  # (B, H, D)
        else:
            T = (eps @ self.W[0][:, F2 : F2 + D].T)[:, :, None]  # (B, H, 1)
        for i in range(1, n):
            T = T * derivs[i - 1][:, :, None]
            T = np.einsum("oh,bhk->bok", self.W[i], T)
        if trace == TRACE_EXACT:
            tr = np.einsum("bii->b", T)
        else:
            tr = np.einsum("bi,bi->b", T[:, :, 0], eps)
        return h, tr


def dopri(field: Field, x: np.ndarray, L: np.ndarray | None, t: float, dt: float, c, trace: int, eps):
    """One Dormand-Prince step (utils.py:443-497) on the packed state (x, L): (x_next, L_next, |x_next - x_star|)."""
    ks = []
    S = x if L is None else np.concatenate([x, L[:, None]], axis=1)
    D = x.shape[1]
    for s in range(7):
        if s < 6:
            xs = S + sum(a * k for a, k in zip(A[s], ks, strict=False)) if s else S
        else:
            xs = nxt
        f, tr = field(t + C[s] * dt, xs[:, :D], c, trace, eps)
        fk = f if L is None else np.concatenate([f, (tr * TRACE_SCALE)[:, None]], axis=1)
        ks.append(dt * fk)
        if s == 5:
            nxt = S + sum(a * k for a, k in zip(A[6], ks, strict=True))
    star = S + sum(e * k for e, k in zip(E7, ks, strict=True))
    err = np.abs(nxt - star)
    return nxt, err, S


def controller_factor(error: float) -> float:
    return min(10.0, max(0.1, 0.9 / error ** (1 / 5)))


def controller(t0, t1, errors, dtype=np.float32):
    """The step controller of utils.py:532-552 driven by a given sequence of per-trial errors (already clipped
    at 1e-9, as logged): [(t, dt, accepted)] per trial, with t and dt in `dtype` (fp32 for the engine and for
    the reference's fp32 runs)."""
    f = dtype
    t0, t1 = f(t0), f(t1)
    t, dt = t0, f(t1 - t0)
    sign = f(np.sign(dt))
    out = []
    it = iter(errors)
    while sign * (t1 - t) > 0:
        dt = f(sign * min(abs(dt), abs(f(t1 - t))))
        while True:
            e = next(it, None)
            if e is None:
                return out
            acc = bool(e < 1.0)
            out.append((t, dt, acc))
            if acc:
                t = f(t + dt)
            dt = f(dt * f(controller_factor(float(e))))
            if acc:
                break
    return out


def error_ratio(err: np.ndarray, S: np.ndarray, nxt: np.ndarray, atol: float, rtol: float) -> float:
    tol = atol + rtol * np.maximum(np.abs(S), np.abs(nxt))
    return max(float(np.max(err / tol)), 1e-9)


def integrate(field: Field, x, c, t0: float, t1: float, atol: float, rtol: float, trace: int, eps=None, max_trials=10000):
    """The reference's own fp64 integration: (y, ladj or None, log [(t, dt, error, accepted)])."""
    x = np.asarray(x, np.float64)
    L = np.zeros(x.shape[0]) if trace else None
    t, dt = t0, t1 - t0
    sign = np.sign(dt)
    log = []
    while sign * (t1 - t) > 0:
        dt = sign * min(abs(dt), abs(t1 - t))
        while True:
            if len(log) >= max_trials:
                raise RuntimeError("max_trials")
            nxt, err, S = dopri(field, x, L, t, dt, c, trace, eps)
            e = error_ratio(err, S, nxt, atol, rtol)
            acc = e < 1.0
            log.append((t, dt, e, acc))
            if acc:
                x, L = nxt[:, : x.shape[1]], (nxt[:, -1] if trace else None)
                t = t + dt
            dt = dt * controller_factor(e)
            if acc:
                break
    return x, (None if L is None else L / TRACE_SCALE), log


def replay(field: Field, x, c, step_log, trace: int, eps=None):
    """Integrates the accepted steps of `step_log` (rows (t, dt, error, accepted)) in fp64: (y, ladj or None)."""
    x = np.asarray(x, np.float64)
    L = np.zeros(x.shape[0]) if trace else None
    for t, dt, _, acc in step_log:
        if not acc:
            continue
        nxt, _, _ = dopri(field, x, L, float(t), float(dt), c, trace, eps)
        x, L = nxt[:, : x.shape[1]], (nxt[:, -1] if trace else None)
    return x, (None if L is None else L / TRACE_SCALE)


def replay_errors(field: Field, x, c, step_log, trace: int, atol: float, rtol: float, eps=None):
    """The restatement's error ratio at every logged trial, the state advanced by the logged accepted steps."""
    x = np.asarray(x, np.float64)
    L = np.zeros(x.shape[0]) if trace else None
    out = []
    for t, dt, _, acc in step_log:
        nxt, err, S = dopri(field, x, L, float(t), float(dt), c, trace, eps)
        out.append(error_ratio(err, S, nxt, atol, rtol))
        if acc:
            x, L = nxt[:, : x.shape[1]], (nxt[:, -1] if trace else None)
    return np.array(out)


def log_normal(z: np.ndarray) -> np.ndarray:
    return -0.5 * np.sum(z * z, axis=1) - 0.5 * z.shape[1] * math.log(2 * math.pi)
