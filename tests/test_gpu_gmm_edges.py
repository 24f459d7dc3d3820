"""GPU tests of the Gaussian mixture model (gmm.cu, gmm_math.cuh, mixtures.py) at its edges against fp64: the
restatement tests/gmm_reference.py composed with the fp64 conditioner (oracle.Conditioner.trace) and its reverse
mode (oracle_grad.conditioner_backward).

* `CASES` reaches the 6 instantiations (covariance x tied) of the log-density, backward and sampling kernels, both
  thread plans (128 threads while 2D + K <= 96, 64 above; the boundary pairs (32, 32), (40, 16) | (33, 31),
  (40, 17); D = 64, K = 32; D = 1, K = 1), the three sources of phi (the unconditional table, per-row context,
  a broadcast context with ldc = 0), batches of 1, T - 1, T, T + 1, 2T + 1 and thousands rows, and one, two or
  many row chunks (the last of one row) on every path; tests/test_gmm_edges_host.py checks that it does.
* Every case runs with padded strides whose pads hold NaN canaries, pre-filled gradient buffers (the backward
  ACCUMULATES grad_c and the parameter gradients), twice with one workspace (bit-identical), and samples against
  the restatement with the rows at a CDF boundary checked rather than dropped.
* Conditioners: fp32 handles, and a ReLU handle packed for the tensor cores ([256] * 2 hidden) with
  zk_set_tc_backward(1) and (0).  The broadcast path runs its conditioner in fp32 under either setting.

Bars (max|ours - ref| over max|ref| per tensor; log_prob: |ours - ref| / max(|ref|, 1)): log_prob 2e-5 for
D <= 16, 1e-4 above; gradients 5e-5 for D <= 16, 1e-4 above and at ill-conditioned scales.  Rows with a hidden
pre-activation within rounding of a ReLU kink get zero upstream weight on a tensor-core handle (cases.py)."""

from __future__ import annotations

import ctypes
from typing import NamedTuple

import gmm_reference as R
import numpy as np
import pytest
import torch

import zuko_b200 as zuko
from oracle import oracle as O
from oracle import oracle_grad as OG
from zuko_b200 import _engine as E

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EPS = 1e-6
NAN = float("nan")
CTX = 5  # context features of the conditional cases
PAD = 3  # odd pad of every padded row stride
HIDDEN = {"fp32": [32, 32], "tc": [256, 256]}
GEMM = {"fp32": "fp32", "tc": "bf16x3"}
SMEM_CAP = 48 * 1024


class Case(NamedTuple):
    cov: str
    tied: bool
    D: int
    K: int
    src: str  # "table" (unconditional), "rows" (per-row context), "bcast" (one context row, ldc = 0)
    B: int | None  # None: derived from the chunk plan
    chunks: object = 1  # 1, 2, "many" (the last chunk holds one row) or "min" (zk_gmm_min_workspace_bytes)
    hyper: str = "fp32"  # conditioner: "fp32" handle or "tc" (packed for the tensor cores)

    @property
    def id(self) -> str:
        return (f"{self.cov}-{'tied' if self.tied else 'untied'}-D{self.D}K{self.K}-{self.src}-B{self.B}-c{self.chunks}"
                + ("" if self.src == "table" else f"-{self.hyper}"))  # fmt: skip


def threads(D: int, K: int) -> int:
    T = 128
    while T > 32 and T * (2 * D + K) * 4 > SMEM_CAP:
        T //= 2
    return T


CASES = [
    # 128 threads: 1, T - 1, T, T + 1, 2T + 1, thousands
    Case("full", False, 3, 2, "rows", 1),
    Case("diagonal", True, 4, 3, "rows", 127),
    Case("spherical", False, 5, 4, "bcast", 128),
    Case("full", True, 3, 3, "table", 129),
    Case("diagonal", False, 6, 5, "rows", 257, 1, "tc"),
    Case("spherical", True, 3, 2, "rows", 3001),
    Case("diagonal", False, 4, 2, "table", 4099),
    Case("full", False, 3, 4, "bcast", 2053, 1, "tc"),
    # the plan's boundary: 2D + K = 96 keeps 128 threads, 97 runs 64
    Case("full", False, 32, 32, "rows", 129),
    Case("diagonal", True, 40, 16, "bcast", 257),
    Case("full", True, 33, 31, "rows", 63, 1, "tc"),
    Case("spherical", False, 40, 17, "table", 64),
    Case("diagonal", False, 33, 31, "bcast", 65, 1, "tc"),
    Case("full", False, 40, 17, "rows", 129),
    Case("spherical", True, 33, 31, "table", 2001),
    Case("diagonal", True, 40, 17, "rows", 1),
    # the largest covered shape and the smallest
    Case("full", True, 64, 32, "rows", 65),
    Case("full", False, 64, 32, "table", 64),
    Case("spherical", False, 64, 32, "bcast", 63),
    Case("full", False, 1, 1, "rows", 128),
    Case("spherical", True, 1, 1, "table", 1),
    Case("full", True, 1, 1, "bcast", 127, 1, "tc"),
    # row chunks on every path (fp32 handles: the chunk plan is restated exactly)
    Case("full", False, 5, 3, "rows", None, 2),
    Case("diagonal", False, 5, 3, "rows", None, "many"),
    Case("spherical", True, 4, 3, "bcast", None, 2),
    Case("full", True, 4, 3, "bcast", None, "many"),
    Case("diagonal", True, 4, 4, "table", None, 2),
    Case("full", False, 3, 4, "table", None, "many"),
    Case("full", True, 40, 17, "rows", None, "many"),
    Case("diagonal", False, 6, 5, "rows", 400, "min", "tc"),
    Case("full", True, 6, 5, "bcast", 400, "min", "tc"),
]


# --------------------------------------------------------------------------- #
# models, the fp64 oracle and the engine calls
# --------------------------------------------------------------------------- #


def make_gmm(cov, tied, D, K, src, hyper="fp32", seed=0):
    """A GMM on the device whose covariance outputs are scaled by 0.1 (well-conditioned scale matrices at D = 64)."""
    torch.manual_seed(seed)
    C = 0 if src == "table" else CTX
    kw = {} if C == 0 else dict(hidden_features=HIDDEN[hyper])
    gmm = zuko.mixtures.GMM(D, C, components=K, covariance_type=cov, tied=tied, **kw)
    at = K + K * D
    with torch.no_grad():
        if C:
            gmm.hyper[-1].weight[at:] *= 0.1
            gmm.hyper[-1].bias[at:] *= 0.1
            gmm.hyper.gemm_mode = GEMM[hyper]
        else:
            for p in gmm.phi[2:]:
                p.mul_(0.1)
    return gmm.to(DEV)


def cpu64(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().double().numpy()


def table_of(gmm) -> torch.Tensor | None:
    return None if hasattr(gmm, "hyper") else torch.cat([p.detach().reshape(-1) for p in gmm.params()]).contiguous()


def block_rows(D: int, K: int) -> int:
    """Rows per block of the oracle: R.grads holds (rows, K, D, D) fp64 matrices; about 64 MB each."""
    return max(1, (64 << 20) // (K * D * D * 8 * 4))


class Ref(NamedTuple):
    lp: np.ndarray
    gx: np.ndarray
    gc: np.ndarray | None  # (B, C) rows, (C,) for a broadcast context
    params: list  # fp64 gradient of every tensor of gmm.params()
    phi: np.ndarray  # (B, P) or (P,)


def oracle(gmm, x: np.ndarray, c: np.ndarray | None, g: np.ndarray) -> Ref:
    """fp64 log_prob and gradients of sum(g * log_prob) for x (B, D) and c (B, C), (C,) or None."""
    D, K, cov, tied = gmm.features, gmm.components, gmm.covariance_type, gmm.tied
    B = x.shape[0]
    cond = None
    if c is None:
        phi = cpu64(table_of(gmm))
    else:
        cond = O.conditioner_from_module(gmm.hyper)
        phi = cond.trace(np.atleast_2d(c))[0][-1]
        if c.ndim == 1:
            phi = phi[0]
    shared = phi.ndim == 1
    lp, gx = np.empty(B), np.empty((B, D))
    gphi = np.zeros(phi.shape[-1]) if shared else np.empty((B, phi.shape[-1]))
    n = block_rows(D, K)
    for r0 in range(0, B, n):
        s = slice(r0, min(B, r0 + n))
        p = phi if shared else phi[s]
        lp[s] = R.log_prob(x[s], p, D, K, cov, tied, EPS)
        gx[s], gp = R.grads(x[s], p, g[s], D, K, cov, tied, EPS)
        if shared:
            gphi += gp.sum(0)
        else:
            gphi[s] = gp
    if cond is None:
        sizes = [p.numel() for p in gmm.params()]
        return Ref(lp, gx, None, np.split(gphi, np.cumsum(sizes)[:-1]), phi)
    gc, cg = OG.conditioner_backward(cond, np.atleast_2d(c), np.atleast_2d(gphi))
    params = [t for w, b in zip(cg.weights, cg.biases, strict=True) for t in (w, b) if b is not None]
    return Ref(lp, gx, gc[0] if c.ndim == 1 else gc, params, phi)


def kink_rows(gmm, c: np.ndarray | None, B: int, tau: float = 1e-5) -> np.ndarray:
    """Rows with a hidden pre-activation within tau (sum |a w| + |b|) of zero (cases.relu_kink_rows): there the
    split-bf16 recompute of a tensor-core handle may take the other side of the ReLU."""
    bad = np.zeros(B, dtype=bool)
    if c is None or c.ndim == 1:
        return bad
    cond = O.conditioner_from_module(gmm.hyper)
    a, outs = cond.trace(c)
    for i in range(len(cond.weights) - 1):
        mag = np.abs(a[i]) @ np.abs(cond.weights[i]).T + np.abs(cond.biases[i])
        bad |= (np.abs(outs[i]) < tau * mag).any(-1)
    return bad


def padded(a: np.ndarray, ld: int) -> torch.Tensor:
    """(B, ld) device rows holding a (B, n) with NaN canaries in the pad."""
    out = torch.full((a.shape[0], ld), NAN, device=DEV)
    out[:, : a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)
    return out


def pads_intact(t: torch.Tensor, n: int) -> bool:
    return bool(torch.isnan(t[:, n:]).all())


def ptr(t: torch.Tensor | None):
    return None if t is None else t.data_ptr()


def workspace(nbytes: int) -> torch.Tensor:
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=DEV)


class Grads:
    """Parameter gradient buffers of a GMM, pre-filled, and the zk_layer_grads that points at them."""

    def __init__(self, gmm, fill: list, bias: bool = True):
        self.bufs = [torch.from_numpy(np.asarray(f, np.float32)).to(DEV).reshape(p.shape) for f, p in zip(fill, gmm.params(), strict=True)]
        if hasattr(gmm, "hyper"):
            weights, biases = gmm._split(self.bufs)
            self.W = (ctypes.c_void_p * len(weights))(*[w.data_ptr() for w in weights])
            self.Bv = (ctypes.c_void_p * len(biases))(*[b.data_ptr() for b in biases])
            bp = ctypes.cast(self.Bv, ctypes.POINTER(ctypes.c_void_p)) if bias else None
            self.s = E.LayerGrads(ctypes.cast(self.W, ctypes.POINTER(ctypes.c_void_p)), bp, None, None)
        else:
            self.flat = torch.cat([b.reshape(-1) for b in self.bufs]).contiguous()
            self.s = E.LayerGrads(None, None, self.flat.data_ptr(), None)

    def values(self) -> list[np.ndarray]:
        torch.cuda.synchronize()
        if hasattr(self, "flat"):
            sizes = [b.numel() for b in self.bufs]
            return [a.reshape(-1) for a in np.split(cpu64(self.flat), np.cumsum(sizes)[:-1])]
        return [cpu64(b).reshape(-1) for b in self.bufs]


def log_prob_call(gmm, x, ldx, c, ldc, B, ws) -> tuple[int, torch.Tensor]:
    h = gmm.handle(gmm.params())
    t = table_of(gmm)
    out = torch.full((max(B, 1),), 7.0, device=DEV)
    st = E.lib().zk_gmm_log_prob(h, ptr(x), ldx, ptr(c), ldc, ptr(t), B, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                 E.stream_ptr(DEV))  # fmt: skip
    return st, out


def sample_call(gmm, c, ldc, u, z, ldz, B, ldxs, ws) -> tuple[int, torch.Tensor]:
    h = gmm.handle(gmm.params())
    t = table_of(gmm)
    xs = torch.full((max(B, 1), ldxs), NAN, device=DEV)
    st = E.lib().zk_gmm_sample(h, ptr(c), ldc, ptr(t), ptr(u), ptr(z), ldz, B, xs.data_ptr(), ldxs, ws.data_ptr(),
                               ws.numel(), E.stream_ptr(DEV))  # fmt: skip
    return st, xs


def backward_call(gmm, x, ldx, c, ldc, B, g, gx, ldgx, gc, ldgc, grads, ws) -> int:
    h = gmm.handle(gmm.params())
    t = table_of(gmm)
    return E.lib().zk_gmm_backward(h, ptr(x), ldx, ptr(c), ldc, ptr(t), B, ptr(g), ptr(gx), ldgx, ptr(gc), ldgc,
                                   None if grads is None else ctypes.byref(grads.s), ws.data_ptr(), ws.numel(),
                                   E.stream_ptr(DEV))  # fmt: skip


# --------------------------------------------------------------------------- #
# the chunk plan, restated for fp32 conditioners and the unconditional table
# --------------------------------------------------------------------------- #


def a256(n: int) -> int:
    return (n + 255) // 256 * 256


class ChunkPlan:
    """Row chunks of zk_gmm_backward per path.  Unconditional: zk_gmm_chunk_rows is the path's own.  An fp32
    conditioner (dims d_0..d_n, ReLU hidden layers): the per-row path needs
        A(n) + S,  A(n) = sum_i a256(4 n d_i) + 2 a256(4 n max hidden) + a256(4 n d_0) + a256(4 n P)
    (activations, two gradient buffers, the input gradient, the phi gradient rows) and the broadcast path
        A(1) + S + a256(256 P) + a256(4 n P)
    (the conditioner over one row, its column-sum scratch, the per-sample gradient rows); S, the conditioner's
    fixed scratch, is read off zk_gmm_backward_workspace_bytes at large n, where the per-row path is the larger,
    and the whole restatement is checked against zk_gmm_backward_workspace_bytes and zk_gmm_chunk_rows."""

    def __init__(self, gmm):
        self.gmm, self.h = gmm, gmm.handle(gmm.params())
        self.P = gmm.total
        if hasattr(gmm, "hyper"):
            self.dims = [gmm.hyper._linears()[0].in_features] + [m.out_features for m in gmm.hyper._linears()]
            self.S = E.lib().zk_gmm_backward_workspace_bytes(self.h, 1 << 16) - self.A(1 << 16)
            assert self.S == E.lib().zk_gmm_backward_workspace_bytes(self.h, 1 << 17) - self.A(1 << 17)
            for n in (1, 2, 3, 64, 1000):
                assert E.lib().zk_gmm_backward_workspace_bytes(self.h, n) == max(self.need("rows", n), self.need("bcast", n))

    def A(self, n: int) -> int:
        d = self.dims
        return sum(a256(4 * n * k) for k in d) + 2 * a256(4 * n * max(d[1:-1])) + a256(4 * n * d[0]) + a256(4 * n * self.P)

    def need(self, path: str, n: int) -> int:
        if path == "rows":
            return self.A(n) + self.S
        return self.A(1) + self.S + a256(256 * self.P) + a256(4 * n * self.P)

    def rows(self, path: str, B: int, ws: int) -> int:
        if path == "table":
            return E.lib().zk_gmm_chunk_rows(self.h, B, 1, ws)
        lo, hi = 0, B
        while lo < hi:
            mid = (lo + hi + 1) // 2
            if self.need(path, mid) <= ws:
                lo = mid
            else:
                hi = mid - 1
        return lo

    def workspace_for(self, path: str, chunks: object, B0: int = 40) -> tuple[int, int, int]:
        """(B, workspace bytes, rows per chunk) with two chunks, or many whose last holds one row; the workspace
        is at least zk_gmm_min_workspace_bytes."""
        lowest = E.lib().zk_gmm_min_workspace_bytes(self.h)
        for n in range(B0, 4 * B0):
            ws = max(lowest, E.lib().zk_gmm_backward_workspace_bytes(self.h, n) if path == "table" else self.need(path, n))
            r = self.rows(path, 1 << 20, ws)
            B = r + r // 2 + 1 if chunks == 2 else 3 * r + 1
            if path != "table":
                assert E.lib().zk_gmm_chunk_rows(self.h, B, 1, ws) == min(self.rows("rows", B, ws), self.rows("bcast", B, ws))
            if self.rows(path, B, ws) == r and r >= 2:
                return B, ws, r
        raise AssertionError(f"no workspace gives {chunks} chunks on the {path} path")


# --------------------------------------------------------------------------- #
# checks
# --------------------------------------------------------------------------- #


def bars(D: int, ill: bool = False) -> tuple[float, float]:
    """(log_prob, gradient) bars."""
    return (2e-5 if D <= 16 else 1e-4), (1e-4 if D > 16 or ill else 5e-5)


def check_lp(ours: np.ndarray, ref: np.ndarray, bar: float, what: str) -> float:
    err = float(np.max(np.abs(ours - ref) / np.maximum(np.abs(ref), 1.0))) if ref.size else 0.0
    assert np.isfinite(ours).all() and err <= bar, f"{what} log_prob: {err:.3e} > {bar:.0e}"
    return err


def check_grad(ours: np.ndarray, ref: np.ndarray, bar: float, what: str) -> float:
    ours, ref = np.asarray(ours, np.float64).reshape(-1), np.asarray(ref, np.float64).reshape(-1)
    scale = max(float(np.abs(ref).max()), 1e-30)
    err = float(np.abs(ours - ref).max()) / scale
    assert np.isfinite(ours).all() and err <= bar, f"{what}: max err {err:.3e} of max|ref| {scale:.3e} (bar {bar:.0e})"
    return err


def check_rows(B: int, T: int, seed: int = 0) -> np.ndarray:
    """Every row of a batch up to 4096; above, the first and last CTA, every row within 2 of a CTA edge and 512
    random rows."""
    if B <= 4096:
        return np.arange(B)
    edges = np.arange(0, B + T, T)
    near = (edges[:, None] + np.arange(-2, 3)[None]).reshape(-1)
    pick = np.concatenate([np.arange(T), np.arange(B - T, B), near, np.random.default_rng(seed).integers(0, B, 512)])
    return np.unique(pick[(pick >= 0) & (pick < B)])


def check_samples(phi: np.ndarray, u: np.ndarray, z: np.ndarray, xs: np.ndarray, D, K, cov, tied, what: str) -> None:
    """xs against R.sample.  A row whose u lies within 1e-6 of a CDF boundary is checked, not dropped: its
    component is one of the two beside the boundary, has positive weight, and x = mu_k + L_k z for it.  The band
    is 1e-4 wide: a conditioner's fp32 or split-bf16 rows move the boundaries by up to a few 1e-5."""
    ref, k, margin = R.sample(phi, u, z, D, K, cov, tied, EPS)
    tol = 1e-4 * np.maximum(1.0, np.abs(ref))
    near = margin <= 1e-4
    assert np.all(np.abs(xs[~near] - ref[~near]) <= tol[~near]), f"{what}: samples off the restatement"
    if not near.any():
        return
    rows = np.nonzero(near)[0]
    ph = phi if phi.ndim == 1 else phi[rows]
    ph = np.broadcast_to(ph, (rows.size, phi.shape[-1]))
    logits = R.unpack(ph, D, K, cov, tied)[0]
    p = np.exp(logits - logits.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    cdf = np.cumsum(p, -1)[:, :-1]
    j = np.abs(u[rows, None] - cdf).argmin(-1)  # the boundary between components j and j + 1
    loc, L = R.scale_tril(ph, D, K, cov, tied, EPS)
    for i, b in enumerate(rows):
        hits = [kk for kk in (j[i], j[i] + 1) if np.all(np.abs(xs[b] - (loc[i, kk] + L[i, kk] @ z[b])) <= tol[b])]
        assert hits and all(p[i, kk] > 0 for kk in hits), f"{what}: row {b} at a CDF boundary drew off its neighbours"


class TcBackward:
    """zk_set_tc_backward(on) for a with-block, restored on exit."""

    def __init__(self, on: int):
        self.on = on

    def __enter__(self):
        self.prev = E.lib().zk_set_tc_backward(self.on)

    def __exit__(self, *exc):
        E.lib().zk_set_tc_backward(self.prev)


# --------------------------------------------------------------------------- #
# the case table
# --------------------------------------------------------------------------- #

ERRORS: dict = {}  # measured maxima per path, printed at the end of each case (pytest -s)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_case_against_fp64(case):
    cov, tied, D, K, src = case.cov, case.tied, case.D, case.K, case.src
    gmm = make_gmm(cov, tied, D, K, src, case.hyper, seed=CASES.index(case))
    h = gmm.handle(gmm.params())
    T = threads(D, K)
    # workspace and batch
    if case.chunks in (2, "many"):
        path = {"rows": "rows", "bcast": "bcast", "table": "table"}[src]
        B, ws_b, r = ChunkPlan(gmm).workspace_for(path, case.chunks)
        assert -(-B // r) == 2 if case.chunks == 2 else (B % r == 1 and B // r >= 3)
        ws_f = None
        if src == "rows":  # the per-row forward: zk_gmm_chunk_rows is its own (the broadcast one needs one row)
            for n in range(1, B):
                ws_f = E.lib().zk_gmm_workspace_bytes(h, n)
                rf = E.lib().zk_gmm_chunk_rows(h, B, 0, ws_f)
                if (-(-B // rf) == 2) if case.chunks == 2 else (B % rf == 1 and B // rf >= 3):
                    break
            else:
                raise AssertionError("no forward workspace for the chunk count")
        ws_f = ws_f or ws_b
    elif case.chunks == "min":
        B = case.B
        ws_f = ws_b = E.lib().zk_gmm_min_workspace_bytes(h)
        assert E.lib().zk_gmm_chunk_rows(h, B, 1, ws_b) < B
    else:
        B = case.B
        ws_f = ws_b = max(E.lib().zk_gmm_workspace_bytes(h, B), E.lib().zk_gmm_backward_workspace_bytes(h, B))
        assert E.lib().zk_gmm_chunk_rows(h, B, 0, ws_f) == B and E.lib().zk_gmm_chunk_rows(h, B, 1, ws_b) == B
    # data
    gen = torch.Generator().manual_seed(1000 + B)
    x = torch.randn(B, D, generator=gen).numpy().astype(np.float64)
    c = None
    if src == "rows":
        c = torch.randn(B, CTX, generator=gen).double().numpy()
    elif src == "bcast":
        c = torch.randn(CTX, generator=gen).double().numpy()
    g = (torch.rand(B, generator=gen) + 0.5).double().numpy()
    if case.hyper == "tc":
        g[kink_rows(gmm, c, B)] = 0.0
    g = g.astype(np.float32).astype(np.float64)
    ref = oracle(gmm, x, c, g)
    lp_bar, g_bar = bars(D)
    ldx = D + PAD
    xd = padded(x, ldx)
    cd, ldc = None, 0
    if src == "rows":
        cd, ldc = padded(c, CTX + PAD), CTX + PAD
    elif src == "bcast":
        cd = torch.from_numpy(c.astype(np.float32)).to(DEV)
    gd = torch.from_numpy(g.astype(np.float32)).to(DEV)
    rows = check_rows(B, T)
    errs = ERRORS.setdefault(f"{src}/{case.hyper if src != 'table' else 'table'}/D{'<=16' if D <= 16 else '>16'}", {})

    def upd(k, v):
        errs[k] = max(errs.get(k, 0.0), v)

    # log_prob
    st, lp = log_prob_call(gmm, xd, ldx, cd, ldc, B, workspace(ws_f))
    E.check(st)
    assert pads_intact(xd, D) and (cd is None or ldc == 0 or pads_intact(cd, CTX))
    upd("log_prob", check_lp(cpu64(lp)[rows], ref.lp[rows], lp_bar, case.id))

    # backward, twice with one workspace, into pre-filled buffers
    rng = np.random.default_rng(B)
    fill = [0.5 * max(np.abs(r).max(), 1e-3) * rng.uniform(-1, 1, r.size) for r in ref.params]
    fill = [f.astype(np.float32).astype(np.float64) for f in fill]
    gc_fill = None
    if c is not None:
        gc_fill = (0.5 * max(np.abs(ref.gc).max(), 1e-3) * rng.uniform(-1, 1, ref.gc.shape)).astype(np.float32).astype(np.float64)
    ws = workspace(ws_b)
    modes = (1, 0) if case.hyper == "tc" else (1,)
    results = {}
    for mode in modes:
        with TcBackward(mode):
            runs = []
            for _ in range(2):
                gx = torch.full((B, D + PAD), NAN, device=DEV)
                gc = None
                if c is not None:
                    gc = padded(np.atleast_2d(gc_fill), CTX + PAD) if src == "rows" else torch.from_numpy(gc_fill.astype(np.float32)).to(DEV)
                grads = Grads(gmm, fill)
                E.check(backward_call(gmm, xd, ldx, cd, ldc, B, gd, gx, D + PAD, gc, CTX + PAD, grads, ws))
                runs.append((gx, gc, grads.values()))
            (gx, gc, gv), (gx2, gc2, gv2) = runs
            assert torch.equal(gx[:, :D], gx2[:, :D]) and (gc is None or torch.equal(gc[..., :CTX], gc2[..., :CTX]))
            assert all(np.array_equal(a, b) for a, b in zip(gv, gv2, strict=True)), f"{case.id}: two runs differ"
            assert pads_intact(gx, D), f"{case.id}: grad_x pad overwritten"
            assert not (src == "rows" and not pads_intact(gc, CTX)), f"{case.id}: grad_c pad overwritten"
            w = "" if mode else " tc off"
            upd("grad_x", check_grad(cpu64(gx[:, :D])[rows], ref.gx[rows], g_bar, f"{case.id}{w} grad_x"))
            if gc is not None:
                got = cpu64(gc[:, :CTX] if src == "rows" else gc)
                upd("grad_c", check_grad(got - gc_fill, ref.gc, g_bar, f"{case.id}{w} grad_c (accumulated)"))
            for i, (got, f, r) in enumerate(zip(gv, fill, ref.params, strict=True)):
                upd("params", check_grad(got - f, r, g_bar, f"{case.id}{w} parameter {i} (accumulated)"))
            results[mode] = [cpu64(gx[:, :D])] + ([] if gc is None else [cpu64(gc)]) + gv
    if src == "bcast" and case.hyper == "tc":  # the broadcast conditioner runs fp32 under either setting
        assert all(np.array_equal(a, b) for a, b in zip(results[1], results[0], strict=True))

    # sampling, with rows placed on the fp64 CDF boundaries
    u = torch.rand(B, generator=gen).double().numpy()
    z = torch.randn(B, D, generator=gen).double().numpy()
    if K > 1:
        ph = np.broadcast_to(ref.phi, (B, ref.phi.shape[-1]))
        logits = ph[:, :K]
        p = np.exp(logits - logits.max(-1, keepdims=True))
        cdf = np.cumsum(p / p.sum(-1, keepdims=True), -1)
        first = np.arange(min(B, 4 * (K - 1)))
        u[first] = cdf[first, first % (K - 1)]
    u = u.astype(np.float32).astype(np.float64)
    u[u >= 1] = np.nextafter(np.float32(1), np.float32(0))
    z = z.astype(np.float32).astype(np.float64)
    zd = padded(z, D + PAD)
    st, xs = sample_call(gmm, cd, ldc, torch.from_numpy(u.astype(np.float32)).to(DEV), zd, D + PAD, B, D + PAD, workspace(ws_f))
    E.check(st)
    assert pads_intact(xs, D) and pads_intact(zd, D), f"{case.id}: sample pads overwritten"
    phi_rows = ref.phi if ref.phi.ndim == 1 else ref.phi[rows]
    check_samples(phi_rows, u[rows], z[rows], cpu64(xs[:, :D])[rows], D, K, cov, tied, case.id)
    print(f"{case.id}: {errs}")


# --------------------------------------------------------------------------- #
# nullable outputs, empty batches and the workspace API
# --------------------------------------------------------------------------- #


@pytest.mark.parametrize("src", ["rows", "bcast", "table"])
def test_nullable_outputs(src):
    """grad_x = NULL, grad_c = NULL, grads = NULL and grad_bias = NULL beside grad_weight: what is computed still
    matches fp64, and what is not asked for is not touched."""
    D, K, B = 5, 3, 300
    gmm = make_gmm("full", True, D, K, src, seed=3)
    h = gmm.handle(gmm.params())
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(B, D, generator=gen).double().numpy()
    c = None if src == "table" else (torch.randn(B, CTX, generator=gen) if src == "rows" else torch.randn(CTX, generator=gen)).double().numpy()
    g = np.ones(B)
    ref = oracle(gmm, x, c, g)
    xd = padded(x, D)
    cd = None if c is None else torch.from_numpy(c.astype(np.float32)).to(DEV)
    ldc = CTX if src == "rows" else 0
    ws = workspace(E.lib().zk_gmm_backward_workspace_bytes(h, B))
    gd = torch.ones(B, device=DEV)
    zeros = [np.zeros(p.numel()) for p in gmm.params()]
    _, bar = bars(D)
    # grad_x = NULL
    gc = None if c is None else torch.zeros_like(cd)
    grads = Grads(gmm, zeros)
    E.check(backward_call(gmm, xd, D, cd, ldc, B, gd, None, D, gc, CTX, grads, ws))
    for i, (got, r) in enumerate(zip(grads.values(), ref.params, strict=True)):
        check_grad(got, r, bar, f"{src} gx=NULL parameter {i}")
    if gc is not None:
        check_grad(cpu64(gc), ref.gc, bar, f"{src} gx=NULL grad_c")
    # grad_c = NULL and grads = NULL: grad_x alone
    gx = torch.full((B, D), NAN, device=DEV)
    E.check(backward_call(gmm, xd, D, cd, ldc, B, gd, gx, D, None, CTX, None, ws))
    check_grad(cpu64(gx), ref.gx, bar, f"{src} gc=grads=NULL grad_x")
    if src != "table":
        # grad_bias = NULL beside grad_weight: the biases' buffers stay as they were
        grads = Grads(gmm, [np.full(p.numel(), 3.0) for p in gmm.params()], bias=False)
        E.check(backward_call(gmm, xd, D, cd, ldc, B, gd, gx, D, None, CTX, grads, ws))
        v = grads.values()
        for i, (got, r) in enumerate(zip(v, ref.params, strict=True)):
            if gmm.params()[i].dim() == 1:  # a bias
                assert np.all(got == 3.0), f"{src}: bias gradient {i} written with grad_bias = NULL"
            else:
                check_grad(got - 3.0, r, bar, f"{src} grad_bias=NULL weight {i}")


@pytest.mark.parametrize("src", ["rows", "bcast", "table"])
def test_empty_batch_touches_nothing(src):
    D, K = 4, 3
    gmm = make_gmm("diagonal", False, D, K, src, seed=4)
    h = gmm.handle(gmm.params())
    ws = workspace(E.lib().zk_gmm_min_workspace_bytes(h))
    x = torch.zeros(1, D, device=DEV)
    c = None if src == "table" else torch.zeros(1, CTX, device=DEV)
    ldc = CTX if src == "rows" else 0
    st, lp = log_prob_call(gmm, x, D, c, ldc, 0, ws)
    assert st == E.ZK_OK and lp.item() == 7.0
    u, z = torch.zeros(1, device=DEV), torch.zeros(1, D, device=DEV)
    st, xs = sample_call(gmm, c, ldc, u, z, D, 0, D, ws)
    assert st == E.ZK_OK and torch.isnan(xs).all()
    gx = torch.full((1, D), 5.0, device=DEV)
    gc = None if c is None else torch.full((1, CTX), 6.0, device=DEV)
    grads = Grads(gmm, [np.full(p.numel(), 2.0) for p in gmm.params()])
    st = backward_call(gmm, x, D, c, ldc, 0, torch.ones(1, device=DEV), gx, D, gc, CTX, grads, ws)
    assert st == E.ZK_OK
    torch.cuda.synchronize()
    assert (gx == 5.0).all() and (gc is None or (gc == 6.0).all())
    assert all(np.all(v == 2.0) for v in grads.values())


@pytest.mark.parametrize("src,hyper", [("rows", "fp32"), ("rows", "tc"), ("table", "fp32")])
def test_workspace_api(src, hyper):
    """Host-side: a full workspace is one chunk, the minimum at least one row, and one byte below the minimum
    is refused before anything runs (the outputs stay untouched)."""
    D, K = 6, 4
    gmm = make_gmm("full", False, D, K, src, hyper, seed=5)
    h = gmm.handle(gmm.params())
    for B in (1, 127, 1000, 100_003):
        assert E.lib().zk_gmm_chunk_rows(h, B, 0, E.lib().zk_gmm_workspace_bytes(h, B)) == B
        assert E.lib().zk_gmm_chunk_rows(h, B, 1, E.lib().zk_gmm_backward_workspace_bytes(h, B)) == B
        lo = E.lib().zk_gmm_min_workspace_bytes(h)
        assert E.lib().zk_gmm_chunk_rows(h, B, 0, lo) >= 1 and E.lib().zk_gmm_chunk_rows(h, B, 1, lo) >= 1
    B = 64
    lo = E.lib().zk_gmm_min_workspace_bytes(h)
    ws = workspace(lo - 1)
    x = torch.zeros(B, D, device=DEV)
    assert ws.numel() == lo - 1
    # the call whose one-row need is the minimum: the broadcast backward for a conditioner, the table's backward
    c = None if src == "table" else torch.zeros(CTX, device=DEV)
    gx = torch.full((B, D), 5.0, device=DEV)
    gc = None if c is None else torch.full((CTX,), 6.0, device=DEV)
    grads = Grads(gmm, [np.full(p.numel(), 2.0) for p in gmm.params()])
    if hyper == "fp32":
        if src == "rows":
            assert ChunkPlan(gmm).need("bcast", 1) == lo
        st = backward_call(gmm, x, D, c, 0, B, torch.ones(B, device=DEV), gx, D, gc, CTX, grads, ws)
        assert st == E.ZK_EINVAL
        torch.cuda.synchronize()
        assert (gx == 5.0).all() and (gc is None or (gc == 6.0).all())
        assert all(np.all(v == 2.0) for v in grads.values())
    if src == "rows":  # the forward's one-row need is zk_gmm_workspace_bytes(h, 1) on either path
        ws = workspace(E.lib().zk_gmm_workspace_bytes(h, 1) - 1)
        for cc, ldc in ((torch.zeros(B, CTX, device=DEV), CTX), (torch.zeros(CTX, device=DEV), 0)):
            st, lp = log_prob_call(gmm, x, D, cc, ldc, B, ws)
            assert st == E.ZK_EINVAL and (lp == 7.0).all()
            st, xs = sample_call(gmm, cc, ldc, torch.zeros(B, device=DEV), x, D, B, D, ws)
            assert st == E.ZK_EINVAL and torch.isnan(xs).all()


# --------------------------------------------------------------------------- #
# component selection and numerics
# --------------------------------------------------------------------------- #


@pytest.mark.parametrize("K", range(2, 33))
def test_component_selection_edges(K):
    """u at 0, 2^-24, 1/2, the fp32 running sums and 1 - j 2^-24 (j = 1..64); a component of zero weight
    (logit -200 or -1e4) last, first or in the middle, or one at +80 dominating the rest.  D = 1, means 10 k and
    z = 0, so each draw names its component (test_gmm_host.check_selection)."""
    from test_gmm_host import check_selection, selection_uniforms

    gmm = make_gmm("diagonal", False, 1, K, "table", seed=6)
    h = gmm.handle(gmm.params())
    ws = workspace(E.lib().zk_gmm_min_workspace_bytes(h))
    setups = [(v, at) for v in (-200.0, -1e4, 80.0) for at in sorted({0, K // 2, K - 1})]
    for value, at in setups:
        logits = np.zeros(K, np.float32)
        logits[at] = value
        u = selection_uniforms(logits)
        phi = torch.from_numpy(np.concatenate([logits, 10.0 * np.arange(K), np.zeros(K)]).astype(np.float32)).to(DEV)
        ud = torch.from_numpy(u).to(DEV)
        x = torch.empty(u.size, 1, device=DEV)
        z = torch.zeros(u.size, 1, device=DEV)
        E.check(E.lib().zk_gmm_sample(h, None, 0, phi.data_ptr(), ud.data_ptr(), z.data_ptr(), 1,
                                      u.size, x.data_ptr(), 1, ws.data_ptr(), ws.numel(), E.stream_ptr(DEV)))  # fmt: skip
        xs = x.cpu().numpy()[:, 0]
        k = np.rint(xs / 10).astype(int)
        assert np.array_equal(xs, 10.0 * k) and ((k >= 0) & (k < K)).all()
        # a dominating component leaves the others weights of 1e-35, which the inverse CDF still draws for u in
        # their intervals; a dead one (weight 0 in fp32) is never drawn
        check_selection(logits, u, k, f"K={K} logit {value} at {at}", floor=1e-30 if value < 0 else 0.0)


@pytest.mark.parametrize("kind", ["far", "logits", "floor", "tied32"])
@pytest.mark.parametrize("cov", ["full", "diagonal", "spherical"])
def test_extreme_parameters(kind, cov):
    """far: x about 10^3 scale lengths from every mean (every t_k far below zero); logits spread +-40 over
    components 20 scale lengths apart; floor:
    diag = -20, so L_ii = exp(-20) + eps is about eps, and x within a few eps of a mean; tied32: K = 32 tied, the
    covariance gradient a sum over 32 comparable components.  Unconditional tables, D = 8."""
    D, K = 8, (32 if kind == "tied32" else 4)
    tied = kind == "tied32"
    gmm = make_gmm(cov, tied, D, K, "table", seed=7)
    gen = torch.Generator().manual_seed(7)
    B = 257
    with torch.no_grad():
        logits, loc, diag = gmm.phi[0], gmm.phi[1], gmm.phi[2]
        if kind == "logits":  # means far apart: each x's responsibilities are one-hot, not the prior's
            logits.copy_(torch.linspace(-40, 40, K))
            loc.mul_(20)
        if kind == "tied32":
            loc.mul_(0.05)
        if kind == "floor":
            diag.fill_(-20.0)
            if cov == "full":
                gmm.phi[3].mul_(1e-6)
    phi = cpu64(table_of(gmm))
    loc_ = phi[K : K + K * D].reshape(K, D)
    comp = torch.randint(0, K, (B,), generator=gen).numpy()
    zz = torch.randn(B, D, generator=gen).double().numpy()
    if kind == "far":
        x = loc_[comp] + 1e3 * zz / np.linalg.norm(zz, axis=-1, keepdims=True)
    elif kind == "floor":
        x = loc_[comp] + 2e-6 * zz
    else:
        x = loc_[comp] + zz
    x = x.astype(np.float32).astype(np.float64)
    g = np.ones(B)
    ref = oracle(gmm, x, None, g)
    assert np.isfinite(ref.lp).all()
    lp_bar, g_bar = bars(D, ill=kind in ("floor", "far"))
    ws = workspace(E.lib().zk_gmm_backward_workspace_bytes(gmm.handle(gmm.params()), B))
    xd = padded(x, D)
    st, lp = log_prob_call(gmm, xd, D, None, 0, B, ws)
    E.check(st)
    check_lp(cpu64(lp), ref.lp, lp_bar, f"{kind} {cov}")
    gx = torch.empty(B, D, device=DEV)
    grads = Grads(gmm, [np.zeros(p.numel()) for p in gmm.params()])
    E.check(backward_call(gmm, xd, D, None, 0, B, torch.ones(B, device=DEV), gx, D, None, 0, grads, ws))
    check_grad(cpu64(gx), ref.gx, g_bar, f"{kind} {cov} grad_x")
    for i, (got, r) in enumerate(zip(grads.values(), ref.params, strict=True)):
        if np.abs(r).max() > 0:
            check_grad(got, r, g_bar, f"{kind} {cov} parameter {i}")


# --------------------------------------------------------------------------- #
# the Python layer
# --------------------------------------------------------------------------- #


def reduce_to(a: np.ndarray, shape: tuple) -> np.ndarray:
    """A gradient over the broadcast shape summed back to an operand's shape."""
    a = a.sum(axis=tuple(range(a.ndim - len(shape)))) if a.ndim > len(shape) else a
    axes = tuple(i for i, s in enumerate(shape) if s == 1 and a.shape[i] != 1)
    return a.sum(axis=axes, keepdims=True) if axes else a


@pytest.mark.parametrize("shapes", [((6, 4), (4,)), ((), (9,)), ((11,), (1,))], ids=["x-N4-c-4", "x-D-c-B", "x-N-c-1"])
@pytest.mark.parametrize("want", ["all", "x", "c", "frozen"])
def test_mixture_broadcasting_and_gradients(shapes, want):
    """Mixture.log_prob over x (*xb, D) and c (*cb, C) broadcast against each other, with gradients asked for
    everything, for x alone, for c alone, or for x and c with frozen parameters; against the fp64 oracle on the
    broadcast rows, the x and c gradients reduced to their own shapes."""
    xb, cb = shapes
    D, K = 3, 4
    gmm = make_gmm("full", False, D, K, "rows", seed=8)
    gen = torch.Generator().manual_seed(8)
    x = torch.randn(*xb, D, generator=gen)
    c = torch.randn(*cb, CTX, generator=gen)
    lead = torch.broadcast_shapes(xb, cb)
    g = torch.rand(lead, generator=gen) + 0.5
    xr = x.expand(*lead, D).reshape(-1, D).double().numpy()
    cr = c.expand(*lead, CTX).reshape(-1, CTX).double().numpy()
    ref = oracle(gmm, xr, cr, g.reshape(-1).double().numpy())
    for p in gmm.parameters():
        p.requires_grad_(want == "all")
    xd = x.to(DEV).requires_grad_(want in ("all", "x", "frozen"))
    cd = c.to(DEV).requires_grad_(want in ("all", "c", "frozen"))
    lp = gmm(cd).log_prob(xd)
    assert lp.shape == lead
    check_lp(cpu64(lp).reshape(-1), ref.lp, 2e-5, f"{shapes}")
    (g.to(DEV) * lp).sum().backward()
    for t, r, n in ((xd, ref.gx.reshape(*lead, D), "x"), (cd, ref.gc.reshape(*lead, CTX), "c")):
        if t.requires_grad:
            check_grad(cpu64(t.grad), reduce_to(r, tuple(t.shape)), 5e-5, f"{shapes} {want} grad {n}")
        else:
            assert t.grad is None
    for (n, p), r in zip(gmm.named_parameters(), ref.params, strict=True):
        if want == "all":
            check_grad(cpu64(p.grad), r, 5e-5, f"{shapes} {n}")
        else:
            assert p.grad is None, n


def test_mixture_sample_with_batched_context():
    """Mixture.sample((3,)) over c (4, C): u = rand(12), z = randn(12, D) drawn on the device in that order, then
    one zk_gmm_sample call; against R.sample on the conditioner's fp64 rows."""
    D, K = 5, 6
    gmm = make_gmm("full", True, D, K, "rows", seed=9)
    c = torch.randn(4, CTX, generator=torch.Generator().manual_seed(9)).to(DEV)
    torch.manual_seed(21)
    xs = gmm(c).sample((3,))
    assert xs.shape == (3, 4, D)
    torch.manual_seed(21)
    u = torch.rand(12, device=DEV)
    z = torch.randn(12, D, device=DEV)
    cond = O.conditioner_from_module(gmm.hyper)
    phi = cond.trace(cpu64(c.expand(3, 4, CTX).reshape(-1, CTX)))[0][-1]
    check_samples(phi, cpu64(u), cpu64(z), cpu64(xs).reshape(-1, D), D, K, "full", True, "Mixture.sample")
