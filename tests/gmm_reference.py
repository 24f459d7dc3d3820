"""fp64 numpy restatement of the Gaussian mixture model's log-density, its closed-form gradients and
sampling from given (u, z) — written from the model's definition (zuko/mixtures.py:25-99,
zuko/distributions.py:216-290), sharing no code with the kernels (zuko_b200/csrc/gmm_math.cuh).

phi rows hold logits (K) | loc (K, D) | diag (L, Dd) | tril (L, D (D - 1) / 2) (full covariance only),
L = 1 if tied else K, Dd = 1 for a spherical covariance."""

from __future__ import annotations

import numpy as np

COV = {"full": 0, "diagonal": 1, "spherical": 2}


def shapes(D: int, K: int, cov: str, tied: bool) -> list[tuple[int, ...]]:
    L = 1 if tied else K
    extra = {"full": [(L, D), (L, D * (D - 1) // 2)], "diagonal": [(L, D)], "spherical": [(L, 1)]}[cov]
    return [(K,), (K, D), *extra]


def total(D: int, K: int, cov: str, tied: bool) -> int:
    return sum(int(np.prod(s)) for s in shapes(D, K, cov, tied))


def unpack(phi: np.ndarray, D: int, K: int, cov: str, tied: bool) -> list[np.ndarray]:
    out, at = [], 0
    for s in shapes(D, K, cov, tied):
        n = int(np.prod(s))
        out.append(phi[..., at : at + n].reshape(*phi.shape[:-1], *s))
        at += n
    return out


def scale_tril(phi: np.ndarray, D: int, K: int, cov: str, tied: bool, eps: float) -> tuple[np.ndarray, np.ndarray]:
    """(loc (..., K, D), L (..., K, D, D)) of every component."""
    parts = unpack(phi, D, K, cov, tied)
    loc, diag = parts[1], parts[2]
    lead = phi.shape[:-1]
    s = np.exp(diag) + eps  # (..., L, Dd)
    s = np.broadcast_to(s, (*lead, K, D))
    L = np.zeros((*lead, K, D, D))
    idx = np.arange(D)
    L[..., idx, idx] = s
    if cov == "full":
        r, c = np.tril_indices(D, -1)
        L[..., r, c] = np.broadcast_to(parts[3], (*lead, K, r.size))
    return loc, L


def log_prob(x: np.ndarray, phi: np.ndarray, D: int, K: int, cov: str, tied: bool, eps: float) -> np.ndarray:
    """log p(x) for rows x (B, D) and phi (B, P) or one row (P,)."""
    phi = np.broadcast_to(phi, (x.shape[0], phi.shape[-1]))
    logits = unpack(phi, D, K, cov, tied)[0]
    loc, L = scale_tril(phi, D, K, cov, tied, eps)
    e = x[:, None, :] - loc
    v = np.linalg.solve(L, e[..., None])[..., 0]  # (B, K, D)
    logdet = np.log(np.diagonal(L, axis1=-2, axis2=-1)).sum(-1)
    lp = -0.5 * (D * np.log(2 * np.pi) + (v**2).sum(-1)) - logdet
    logw = logits - _lse(logits)[:, None]
    return _lse(logw + lp)


def grads(x: np.ndarray, phi: np.ndarray, g: np.ndarray, D: int, K: int, cov: str, tied: bool, eps: float):
    """(d/dx (B, D), d/dphi per row (B, P)) of sum(g * log_prob(x))."""
    B = x.shape[0]
    phi = np.ascontiguousarray(np.broadcast_to(phi, (B, phi.shape[-1])))
    parts = unpack(phi, D, K, cov, tied)
    logits, diag = parts[0], parts[2]
    loc, L = scale_tril(phi, D, K, cov, tied, eps)
    e = x[:, None, :] - loc
    v = np.linalg.solve(L, e[..., None])[..., 0]
    w = np.linalg.solve(np.swapaxes(L, -1, -2), v[..., None])[..., 0]  # L^-T v
    logdet = np.log(np.diagonal(L, axis1=-2, axis2=-1)).sum(-1)
    t = logits - _lse(logits)[:, None] - 0.5 * (D * np.log(2 * np.pi) + (v**2).sum(-1)) - logdet
    out = _lse(t)
    r = g[:, None] * np.exp(t - out[:, None])  # (B, K)
    soft = np.exp(logits - _lse(logits)[:, None])
    gx = -(r[..., None] * w).sum(1)
    g_logits = r - g[:, None] * soft
    g_loc = r[..., None] * w
    gL = r[..., None, None] * (w[..., :, None] * v[..., None, :])  # (B, K, D, D)
    idx = np.arange(D)
    gL[..., idx, idx] -= r[..., None] / L[..., idx, idx]
    gs = gL[..., idx, idx]  # d/d L_ii
    s_raw = np.exp(np.broadcast_to(diag, (B, diag.shape[1], diag.shape[2])))
    if cov == "spherical":
        gdiag = gs.sum(-1, keepdims=True) * np.exp(np.broadcast_to(diag, (B, diag.shape[1], 1)))
    else:
        gdiag = gs * s_raw
    if tied:
        gdiag = gdiag.sum(1, keepdims=True)
    pieces = [g_logits, g_loc.reshape(B, -1), gdiag.reshape(B, -1)]
    if cov == "full":
        rr, cc = np.tril_indices(D, -1)
        gt = gL[..., rr, cc]
        if tied:
            gt = gt.sum(1, keepdims=True)
        pieces.append(gt.reshape(B, -1))
    return gx, np.concatenate(pieces, axis=-1)


def sample(phi: np.ndarray, u: np.ndarray, z: np.ndarray, D: int, K: int, cov: str, tied: bool, eps: float):
    """(x (B, D), component (B,), distance of u to the nearest inner CDF boundary (B,))."""
    B = u.shape[0]
    phi = np.broadcast_to(phi, (B, phi.shape[-1]))
    logits = unpack(phi, D, K, cov, tied)[0]
    p = np.exp(logits - _lse(logits)[:, None])
    cdf = np.cumsum(p, axis=-1)[:, :-1]
    k = (u[:, None] >= cdf).sum(-1)
    margin = np.abs(u[:, None] - cdf).min(-1) if K > 1 else np.full(B, np.inf)
    loc, L = scale_tril(phi, D, K, cov, tied, eps)
    rows = np.arange(B)
    x = loc[rows, k] + np.einsum("bij,bj->bi", L[rows, k], z)
    return x, k, margin


def _lse(a: np.ndarray) -> np.ndarray:
    m = a.max(-1)
    return m + np.log(np.exp(a - m[..., None]).sum(-1))
