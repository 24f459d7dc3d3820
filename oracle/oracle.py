"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes/numpy front-end of the plain-C CPU restatement in ``zuko_oracle.c`` plus
the layer/flow composition logic of the reference, restated with numpy.

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may import this module.  The product
(``zuko_b200``) never does: it fails loudly when its CUDA library is missing.

Parity status: PINNED.  ``tests/test_oracle.py`` checks this module against the
golden vectors in ``tests/golden/`` which were produced by the unmodified Python
reference (``tests/golden/make_golden.py`` imports /root/reference).

Reference citations are file:line in probabilists/zuko @ 1063ae4.
"""

from __future__ import annotations

import ctypes
import os
import subprocess
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "libzuko_oracle.so"
_lib = None


def build(force: bool = False) -> Path:
    """Compiles the C restatement (gcc, OpenMP when available)."""
    src = _HERE / "zuko_oracle.c"
    hdr = _HERE / "zuko_oracle_impl.h"
    if (
        not force
        and _LIB_PATH.exists()
        and _LIB_PATH.stat().st_mtime >= max(src.stat().st_mtime, hdr.stat().st_mtime)
    ):
        return _LIB_PATH
    cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
    base = [cc, "-O3", "-fPIC", "-shared", str(src), "-o", str(_LIB_PATH), "-lm"]
    # AVX2 + FMA (every x86 host of an H100 has them) and OpenMP when the toolchain allows;
    # no -ffast-math: the fp32 variant must round like the reference's eager ops.
    for extra in (["-mavx2", "-mfma", "-fopenmp"], ["-fopenmp"], []):
        try:
            subprocess.run(base[:2] + extra + base[2:], check=True, capture_output=True)
            break
        except subprocess.CalledProcessError:
            if not extra:
                raise
    return _LIB_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(str(_LIB_PATH))
    return _lib


def set_threads(n: int) -> int:
    """Sets the OpenMP thread count of the C restatement; returns the count in effect."""
    lib().zo_set_threads(int(n))
    return int(lib().zo_get_threads())


_i64 = ctypes.c_int64
_int = ctypes.c_int


def _sfx(dtype) -> str:
    dtype = np.dtype(dtype)
    if dtype == np.float32:
        return "_f32"
    if dtype == np.float64:
        return "_f64"
    raise TypeError(f"oracle supports float32/float64, got {dtype}")


def _real(dtype):
    return ctypes.c_float if np.dtype(dtype) == np.float32 else ctypes.c_double


def _p(a: np.ndarray | None):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _c(a, dtype) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=dtype)


# --------------------------------------------------------------------------- #
# element-level functions (thin wrappers over the C restatement)
# --------------------------------------------------------------------------- #


def linear(x, c, W, mask, b, relu: bool, dtype=np.float64) -> np.ndarray:
    """``relu?(cat(x, c) @ (mask * W).T + b)`` — zuko/nn.py:217-218,
    flows/autoregressive.py:209.  ``c`` may be None, (C,) (broadcast) or (B, C)."""
    x = _c(x, dtype)
    B, dx = x.shape
    W = _c(W, dtype)
    out = W.shape[0]
    if c is None:
        cc, ldc, dc = None, 0, 0
    else:
        cc = _c(c, dtype)
        dc = cc.shape[-1]
        ldc = 0 if cc.ndim == 1 else dc
    assert W.shape[1] == dx + dc, (W.shape, dx, dc)
    m = None if mask is None else _c(mask, np.uint8)
    bb = None if b is None else _c(b, dtype)
    y = np.empty((B, out), dtype=dtype)
    getattr(lib(), "zo_linear" + _sfx(dtype))(
        _p(x), _i64(dx), _int(dx), _p(cc), _i64(ldc), _int(dc), _i64(B), _p(W), _p(m), _p(bb),
        _int(out), _int(int(relu)), _p(y), _i64(out),
    )  # fmt: skip
    return y


def _check_bins(bins: int) -> None:
    # the C restatement keeps each spline's knots in fixed stack arrays
    if not 1 <= bins <= lib().zo_max_bins():
        raise ValueError(f"oracle: bins={bins} outside [1, {lib().zo_max_bins()}]")


def _phi_args(phi, B, D, P, dtype):
    phi = _c(phi, dtype)
    if phi.size == D * P:  # shared per-dimension table (gaussianization.py:74-77)
        return phi, 0
    assert phi.size == B * D * P, (phi.shape, B, D, P)
    return phi, D * P


def rqs_forward(x, phi, bins: int, bound=5.0, slope=1e-3, dtype=np.float64):
    """MonotonicRQSTransform(*unpack(phi)).call_and_ladj(x) — transforms.py:469-567.
    Returns (y, ladj) both (B, D); ladj is per element (not summed)."""
    _check_bins(bins)
    x = _c(x, dtype)
    B, D = x.shape
    P = 3 * bins - 1
    phi, ld = _phi_args(phi, B, D, P, dtype)
    y = np.empty_like(x)
    ladj = np.empty_like(x)
    R = _real(dtype)
    getattr(lib(), "zo_rqs_forward" + _sfx(dtype))(
        _p(x), _i64(D), _p(phi), _i64(ld), _i64(B), _int(D), _int(bins), R(bound), R(slope),
        _p(y), _i64(D), _p(ladj), _i64(D),
    )  # fmt: skip
    return y, ladj


def rqs_inverse(y, phi, bins: int, bound=5.0, slope=1e-3, dtype=np.float64):
    """MonotonicRQSTransform(*unpack(phi))._inverse(y) — transforms.py:534-548."""
    _check_bins(bins)
    y = _c(y, dtype)
    B, D = y.shape
    P = 3 * bins - 1
    phi, ld = _phi_args(phi, B, D, P, dtype)
    x = np.empty_like(y)
    R = _real(dtype)
    getattr(lib(), "zo_rqs_inverse" + _sfx(dtype))(
        _p(y), _i64(D), _p(phi), _i64(ld), _i64(B), _int(D), _int(bins), R(bound), R(slope),
        _p(x), _i64(D),
    )  # fmt: skip
    return x


def rqs_knots(phi, bins: int, bound=5.0, slope=1e-3, dtype=np.float64):
    """(horizontal, vertical, derivatives) of transforms.py:488-490 for phi (..., 3K-1)."""
    _check_bins(bins)
    phi = _c(phi, dtype)
    lead = phi.shape[:-1]
    n = int(np.prod(lead)) if lead else 1
    X = np.empty((n, bins + 1), dtype=dtype)
    Y = np.empty_like(X)
    Dv = np.empty_like(X)
    R = _real(dtype)
    getattr(lib(), "zo_rqs_knots" + _sfx(dtype))(
        _p(phi), _i64(n), _int(bins), R(bound), R(slope), _p(X), _p(Y), _p(Dv)
    )
    shp = (*lead, bins + 1)
    return X.reshape(shp), Y.reshape(shp), Dv.reshape(shp)


def affine_forward(x, phi, slope=1e-3, dtype=np.float64):
    """MonotonicAffineTransform(shift, scale).call_and_ladj — transforms.py:426-446."""
    x = _c(x, dtype)
    B, D = x.shape
    phi, ld = _phi_args(phi, B, D, 2, dtype)
    y = np.empty_like(x)
    ladj = np.empty_like(x)
    R = _real(dtype)
    getattr(lib(), "zo_affine_forward" + _sfx(dtype))(
        _p(x), _i64(D), _p(phi), _i64(ld), _i64(B), _int(D), R(slope), _p(y), _i64(D), _p(ladj),
        _i64(D),
    )  # fmt: skip
    return y, ladj


def affine_inverse(y, phi, slope=1e-3, dtype=np.float64):
    y = _c(y, dtype)
    B, D = y.shape
    phi, ld = _phi_args(phi, B, D, 2, dtype)
    x = np.empty_like(y)
    R = _real(dtype)
    getattr(lib(), "zo_affine_inverse" + _sfx(dtype))(
        _p(y), _i64(D), _p(phi), _i64(ld), _i64(B), _int(D), R(slope), _p(x), _i64(D)
    )
    return x


def softclip_forward(x, bound=1.0, dtype=np.float64):
    """SoftclipTransform — transforms.py:299-316. Returns (y, ladj) per element."""
    x = _c(x, dtype)
    y = np.empty_like(x)
    ladj = np.empty_like(x)
    getattr(lib(), "zo_softclip_forward" + _sfx(dtype))(
        _p(x), _i64(x.size), _real(dtype)(bound), _p(y), _p(ladj)
    )
    return y, ladj


def softclip_inverse(y, bound=1.0, dtype=np.float64):
    y = _c(y, dtype)
    x = np.empty_like(y)
    getattr(lib(), "zo_softclip_inverse" + _sfx(dtype))(
        _p(y), _i64(y.size), _real(dtype)(bound), _p(x)
    )
    return x


def rotate(x, R, transpose: bool = False, dtype=np.float64):
    """RotationTransform._call / _inverse with a prebuilt R — transforms.py:1235-1244."""
    x = _c(x, dtype)
    B, D = x.shape
    Rm = _c(R, dtype)
    y = np.empty_like(x)
    getattr(lib(), "zo_rotate" + _sfx(dtype))(
        _p(x), _i64(D), _p(Rm), _i64(B), _int(D), _int(int(transpose)), _p(y), _i64(D)
    )
    return y


def circular_shift(x, bound=1.0, dtype=np.float64):
    """CircularShiftTransform — transforms.py:344-348: remainder(x, 2B) - B (numpy's remainder has
    torch.remainder's sign convention)."""
    x = _c(x, dtype)
    two_b = np.asarray(2 * bound, dtype=dtype)
    return (np.remainder(x, two_b) - np.asarray(bound, dtype=dtype)).astype(dtype)


def box_uniform_log_prob(z, lower, upper, ladj=None, dtype=np.float64):
    """BoxUniform(lower, upper).log_prob(z) + ladj — distributions.py:366-396,
    torch/distributions/uniform.py: log(lower <= z) + log(z < upper) - log(upper - lower)."""
    z = _c(z, dtype)
    lo, hi = _c(lower, dtype), _c(upper, dtype)
    inside = ((lo <= z) & (z < hi)).all(-1)
    out = np.full(z.shape[0], -np.inf, dtype=dtype)
    const = -np.log(hi - lo).sum()
    out[inside] = const + (0.0 if ladj is None else np.asarray(ladj, dtype)[inside])
    return out


def permute(x, order, inverse: bool = False):
    """PermutationTransform — transforms.py:1207-1211 (bit-exact gather)."""
    order = np.asarray(order, dtype=np.int64)
    if inverse:
        order = np.argsort(order, kind="stable")
    return np.ascontiguousarray(np.asarray(x)[..., order])


def diag_normal_log_prob(z, loc, scale, ladj=None, dtype=np.float64):
    """DiagNormal(loc, scale).log_prob(z) + ladj — distributions.py:115-119,337-363;
    torch/distributions/normal.py:87-102."""
    z = _c(z, dtype)
    B, D = z.shape
    out = np.empty((B,), dtype=dtype)
    la = None if ladj is None else _c(ladj, dtype)
    getattr(lib(), "zo_diag_normal_log_prob" + _sfx(dtype))(
        _p(z), _i64(D), _p(_c(loc, dtype)), _p(_c(scale, dtype)), _i64(B), _int(D), _p(la), _p(out)
    )
    return out


# --------------------------------------------------------------------------- #
# layer / flow composition (numpy restatement of the lazy + transform layers)
# --------------------------------------------------------------------------- #


def _sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


def _erf(v):
    from scipy.special import erf

    return erf(v)


# torch defaults of the activation modules the reference may put between the linear layers
# (zuko/nn.py:160-192, 258-318: `activation()`); name -> (f, df/dv at the pre-activation v)
ACTIVATIONS = {
    "ReLU": (lambda v: np.maximum(v, 0), lambda v: (v > 0).astype(v.dtype)),
    "ELU": (lambda v: np.where(v > 0, v, np.expm1(np.minimum(v, 0))), lambda v: np.where(v > 0, 1.0, np.exp(np.minimum(v, 0))).astype(v.dtype)),
    "Tanh": (np.tanh, lambda v: 1 - np.tanh(v) ** 2),
    "SiLU": (lambda v: v * _sigmoid(v), lambda v: _sigmoid(v) * (1 + v * (1 - _sigmoid(v)))),
    "GELU": (lambda v: (0.5 * v * (1 + _erf(v / np.sqrt(2.0)))).astype(v.dtype),
             lambda v: (0.5 * (1 + _erf(v / np.sqrt(2.0))) + v * np.exp(-0.5 * v * v) / np.sqrt(2 * np.pi)).astype(v.dtype)),
    "LeakyReLU": (lambda v: np.where(v > 0, v, 0.01 * v).astype(v.dtype), lambda v: np.where(v > 0, 1.0, 0.01).astype(v.dtype)),
    "Softplus": (lambda v: np.where(v > 20, v, np.log1p(np.exp(np.minimum(v, 20)))).astype(v.dtype),
                 lambda v: np.where(v > 20, 1.0, _sigmoid(np.minimum(v, 20))).astype(v.dtype)),
    "Sigmoid": (_sigmoid, lambda v: _sigmoid(v) * (1 - _sigmoid(v))),
}  # fmt: skip


@dataclass
class Conditioner:
    """Weights of a MaskedMLP (nn.py:221-318) or MLP (nn.py:122-192), as numpy.
    ``masks[i]`` is None for dense layers; ``activation`` names the module between the layers.
    ``layer_act`` / ``layer_res`` (residual conditioners, nn.py:195-199, 297-309) give, per linear
    layer, the activation applied to its output (None = none) and whether the input of the
    previous linear layer is added to its output (second layer of a ``Residual`` block)."""

    weights: list
    biases: list
    masks: list
    activation: str = "ReLU"
    layer_act: list | None = None
    layer_res: list | None = None

    def flags(self):
        n = len(self.weights)
        if self.layer_act is None:
            return [self.activation] * (n - 1) + [None], [False] * n
        return list(self.layer_act), list(self.layer_res)

    def trace(self, inp):
        """fp64 numpy evaluation keeping everything: (inputs a[0..n], linear outputs o[0..n-1])."""
        acts, res = self.flags()
        a = [np.asarray(inp, np.float64)]
        outs = []
        for i, (W, b, m) in enumerate(zip(self.weights, self.biases, self.masks, strict=True)):
            Wm = W * (1.0 if m is None else m)
            o = a[i] @ Wm.T
            if b is not None:
                o = o + b
            if res[i]:
                o = o + a[i - 1]
            outs.append(o)
            a.append(ACTIVATIONS[acts[i]][0](o) if acts[i] else o)
        return a, outs

    def __call__(self, x, c, dtype) -> np.ndarray:
        acts, res = self.flags()
        h = None
        prev_in = None
        for i, (W, b, m) in enumerate(zip(self.weights, self.biases, self.masks, strict=True)):
            relu = acts[i] == "ReLU"
            cur_in = h
            if i == 0:
                h = linear(x, c, W, m, b, relu=relu, dtype=dtype)
            else:
                h = linear(h, None, W, m, b, relu=relu, dtype=dtype)
            if acts[i] and not relu:
                h = np.ascontiguousarray(ACTIVATIONS[acts[i]][0](h), dtype=dtype)
            if res[i]:  # x + block(x): the block's input is the input of the previous linear layer
                h = np.ascontiguousarray(h + prev_in, dtype=dtype)
            prev_in = cur_in
        return h


@dataclass
class Layer:
    """One element of the ComposedTransform (transforms.py:59-160).

    kind: 'autoregressive' (flows/autoregressive.py:24-218 + transforms.py:966-1007),
          'coupling' (flows/coupling.py:25-139 + transforms.py:1010-1073),
          'elementwise' (flows/gaussianization.py:28-94),
          'softclip', 'permutation', 'rotation' (transforms.py:286-316,1182-1244).
    """

    kind: str
    features: int = 0
    context: int = 0
    univariate: str = "affine"  # 'affine' | 'rqs' | 'crqs' (circular shift by `bound`, then RQS over [-bound, bound])
    bins: int = 0
    bound: float = 5.0
    slope: float = 1e-3
    passes: int = 0
    hyper: Conditioner | None = None
    phi: np.ndarray | None = None  # shared (D, P) table for elementwise without context
    mask: np.ndarray | None = None  # coupling mask (bool, D); True = constant split
    order: np.ndarray | None = None  # permutation order
    R: np.ndarray | None = None  # rotation matrix
    extra: dict = field(default_factory=dict)

    # -- univariate dispatch --------------------------------------------------
    def _uni_fwd(self, x, phi, dtype):
        if self.univariate == "rqs":
            return rqs_forward(x, phi, self.bins, self.bound, self.slope, dtype)
        if self.univariate == "crqs":
            # CircularRQSTransform — flows/spline.py:65-72: CircularShiftTransform(bound) (transforms.py:
            # 344-345, ladj 0) followed by MonotonicRQSTransform(bound=bound)
            return rqs_forward(circular_shift(x, self.bound, dtype), phi, self.bins, self.bound, self.slope, dtype)
        return affine_forward(x, phi, self.slope, dtype)

    def _uni_inv(self, y, phi, dtype):
        if self.univariate == "rqs":
            return rqs_inverse(y, phi, self.bins, self.bound, self.slope, dtype)
        if self.univariate == "crqs":  # ComposedTransform.inv: RQS^-1 then the shift (its own inverse)
            return circular_shift(rqs_inverse(y, phi, self.bins, self.bound, self.slope, dtype), self.bound, dtype)
        return affine_inverse(y, phi, self.slope, dtype)

    # -- forward: returns (y, ladj summed over the event dim) -----------------
    def forward(self, x, c, dtype=np.float64):
        x = _c(x, dtype)
        if self.kind == "autoregressive":
            # transforms.py:1005-1007: meta(x).call_and_ladj(x); autoregressive.py:207-215
            phi = self.hyper(x, c, dtype)
            y, ladj = self._uni_fwd(x, phi, dtype)
            return y, ladj.sum(-1)  # transforms.py:210-214
        if self.kind == "coupling":
            # transforms.py:1067-1072
            idx_a = np.nonzero(self.mask)[0]
            idx_b = np.nonzero(~self.mask)[0]
            x_a, x_b = _c(x[:, idx_a], dtype), _c(x[:, idx_b], dtype)
            phi = self.hyper(x_a, c, dtype)
            y_b, ladj = self._uni_fwd(x_b, phi, dtype)
            y = np.empty_like(x)
            y[:, idx_a] = x_a
            y[:, idx_b] = y_b
            return y, ladj.sum(-1)
        if self.kind == "elementwise":
            phi = self.phi if self.hyper is None else self._ctx_phi(x, c, dtype)
            y, ladj = self._uni_fwd(x, phi, dtype)
            return y, ladj.sum(-1)
        if self.kind == "softclip":
            y, ladj = softclip_forward(x, self.bound, dtype)
            return y, ladj.sum(-1)  # event_dim 0 -> summed by transforms.py:147
        if self.kind == "permutation":
            return permute(x, self.order), np.zeros(x.shape[0], dtype=dtype)
        if self.kind == "rotation":
            return rotate(x, self.R, False, dtype), np.zeros(x.shape[0], dtype=dtype)
        raise ValueError(self.kind)

    def _ctx_phi(self, x, c, dtype):
        # gaussianization.py:89-92: phi = hyper(c); broadcast over the batch
        cc = np.asarray(c, dtype=dtype)
        if cc.ndim == 1:
            cc = np.broadcast_to(cc, (x.shape[0], cc.shape[0]))
        return self.hyper(_c(cc, dtype), None, dtype)

    # -- inverse: returns x ----------------------------------------------------
    def inverse(self, y, c, dtype=np.float64):
        y = _c(y, dtype)
        if self.kind == "autoregressive":
            # transforms.py:994-1000: x = 0; repeat passes: x = meta(x).inv(y)
            x = np.zeros_like(y)
            for _ in range(self.passes):
                phi = self.hyper(x, c, dtype)
                x = self._uni_inv(y, phi, dtype)
            return x
        if self.kind == "coupling":
            # transforms.py:1054-1058
            idx_a = np.nonzero(self.mask)[0]
            idx_b = np.nonzero(~self.mask)[0]
            y_a, y_b = _c(y[:, idx_a], dtype), _c(y[:, idx_b], dtype)
            phi = self.hyper(y_a, c, dtype)
            x_b = self._uni_inv(y_b, phi, dtype)
            x = np.empty_like(y)
            x[:, idx_a] = y_a
            x[:, idx_b] = x_b
            return x
        if self.kind == "elementwise":
            phi = self.phi if self.hyper is None else self._ctx_phi(y, c, dtype)
            return self._uni_inv(y, phi, dtype)
        if self.kind == "softclip":
            return softclip_inverse(y, self.bound, dtype)
        if self.kind == "permutation":
            return permute(y, self.order, inverse=True)
        if self.kind == "rotation":
            return rotate(y, self.R, True, dtype)
        raise ValueError(self.kind)


@dataclass
class FlowSpec:
    """Flow(transforms, DiagNormal(loc, scale)) — lazy.py:131-172."""

    layers: list
    loc: np.ndarray  # DiagNormal loc, or BoxUniform lower when base == "uniform"
    scale: np.ndarray  # DiagNormal scale, or BoxUniform upper
    base: str = "normal"  # 'normal' | 'uniform'

    def _base_log_prob(self, z, ladj, dtype):
        if self.base == "uniform":
            return box_uniform_log_prob(z, self.loc, self.scale, ladj, dtype)
        return diag_normal_log_prob(z, self.loc, self.scale, ladj, dtype)

    def forward(self, x, c=None, dtype=np.float64):
        """ComposedTransform.call_and_ladj — transforms.py:141-150."""
        x = _c(x, dtype)
        acc = np.zeros(x.shape[0], dtype=dtype)
        for layer in self.layers:
            x, ladj = layer.forward(x, c, dtype)
            acc = acc + ladj
        return x, acc

    def inverse(self, z, c=None, dtype=np.float64):
        """ComposedTransform.inv(z) — transforms.py:121-136."""
        z = _c(z, dtype)
        for layer in reversed(self.layers):
            z = layer.inverse(z, c, dtype)
        return z

    def log_prob(self, x, c=None, dtype=np.float64):
        """NormalizingFlow.log_prob — distributions.py:115-119."""
        z, ladj = self.forward(x, c, dtype)
        return self._base_log_prob(z, ladj, dtype)

    def inverse_and_log_prob(self, z, c=None, dtype=np.float64):
        """NormalizingFlow.rsample_and_log_prob for a GIVEN z — distributions.py:129-138:
        x = transform.inv(z); log p = base.log_prob(z) - ladj_inv, where ladj_inv =
        -ladj_fwd(x) (torch/distributions/transforms.py:277-280)."""
        z = _c(z, dtype)
        x = self.inverse(z, c, dtype)
        _, ladj = self.forward(x, c, dtype)
        return x, self._base_log_prob(z, ladj, dtype)


# --------------------------------------------------------------------------- #
# duck-typed extraction of a FlowSpec from a module tree that follows the
# reference's attribute layout (works for the reference and for zuko_b200's
# host-side mirror alike; imports neither).
# --------------------------------------------------------------------------- #


def _np(t):
    return t.detach().cpu().numpy()


def conditioner_from_module(hyper) -> Conditioner:
    Ws, bs, ms = [], [], []
    layer_act, layer_res = [], []
    act = "ReLU"
    residual = False

    def add(lin, a, r):
        Ws.append(_np(lin.weight).astype(np.float64))
        bs.append(None if lin.bias is None else _np(lin.bias).astype(np.float64))
        ms.append(_np(lin.mask).astype(bool) if hasattr(lin, "mask") else None)
        layer_act.append(a)
        layer_res.append(r)

    mods = list(hyper)
    for j, m in enumerate(mods):
        name = type(m).__name__
        if name == "Residual":  # nn.py:195-199: x + (Linear, activation, Linear)(x)
            inner = list(m)
            assert len(inner) == 3 and hasattr(inner[0], "weight") and hasattr(inner[2], "weight"), inner
            a = type(inner[1]).__name__
            if a not in ACTIVATIONS:
                raise NotImplementedError(f"oracle: activation {a}")
            act = a
            residual = True
            add(inner[0], a, False)
            add(inner[2], None, True)
        elif hasattr(m, "weight"):
            nxt = mods[j + 1] if j + 1 < len(mods) else None
            a = None
            if nxt is not None and not hasattr(nxt, "weight") and type(nxt).__name__ != "Residual":
                a = type(nxt).__name__
                if a not in ACTIVATIONS:
                    raise NotImplementedError(f"oracle: activation {a}")
                act = a
            add(m, a, False)
    if residual:
        return Conditioner(Ws, bs, ms, act, layer_act, layer_res)
    return Conditioner(Ws, bs, ms, act)


def _univariate_info(t):
    """(name, bins, slope) from the module's univariate/shapes hooks
    (flows/autoregressive.py:95-104, flows/spline.py:53-61)."""
    shapes = [tuple(s) for s in t.shapes]
    uni = t.univariate
    kw = getattr(uni, "keywords", {}) or {}
    slope = float(kw.get("slope", 1e-3))
    fname = getattr(getattr(uni, "func", uni), "__name__", "")
    if len(shapes) == 3 and fname == "CircularRQSTransform":
        return "crqs", int(shapes[0][0]), slope
    if len(shapes) == 3:
        return "rqs", int(shapes[0][0]), slope
    if shapes == [(), ()]:
        return "affine", 0, slope
    raise NotImplementedError(f"oracle: univariate with shapes {shapes}")


def layer_from_module(t) -> Layer:
    name = type(t).__name__
    if name == "MaskedAutoregressiveTransform":
        uni, bins, slope = _univariate_info(t)
        in_f = t.hyper[0].weight.shape[1]
        D = t.hyper[-1].weight.shape[0] // t.total
        return Layer("autoregressive", features=D, context=in_f - D, univariate=uni, bins=bins,
                     slope=slope, passes=int(t.passes), hyper=conditioner_from_module(t.hyper),
                     bound=float(np.pi) if uni == "crqs" else 5.0)  # fmt: skip
    if name == "GeneralCouplingTransform":
        uni, bins, slope = _univariate_info(t)
        mask = _np(t.mask).astype(bool)
        D = mask.shape[0]
        in_f = t.hyper[0].weight.shape[1]
        return Layer("coupling", features=D, context=in_f - int(mask.sum()), univariate=uni,
                     bins=bins, slope=slope, mask=mask, hyper=conditioner_from_module(t.hyper))  # fmt: skip
    if name == "ElementWiseTransform":
        uni, bins, slope = _univariate_info(t)
        if hasattr(t, "hyper"):
            D = t.hyper[-1].weight.shape[0] // t.total
            return Layer("elementwise", features=D, context=t.hyper[0].weight.shape[1],
                         univariate=uni, bins=bins, slope=slope,
                         hyper=conditioner_from_module(t.hyper))  # fmt: skip
        parts = [_np(p).astype(np.float64) for p in t.phi]
        D = parts[0].shape[0]
        phi = np.concatenate([p.reshape(D, -1) for p in parts], axis=-1)
        return Layer("elementwise", features=D, univariate=uni, bins=bins, slope=slope, phi=phi)
    if name == "UnconditionalTransform":
        fname = getattr(t.f, "__name__", type(t.f).__name__)
        if fname == "SoftclipTransform":
            kw = t.kwargs
            bound = float(kw.get("bound", t.args[0] if t.args else 1.0))
            return Layer("softclip", bound=bound)
        if fname == "PermutationTransform":
            order = t.kwargs.get("order", t.args[0] if t.args else None)
            return Layer("permutation", order=_np(order).astype(np.int64))
        if fname == "RotationTransform":
            A = t.kwargs.get("A", t.args[0] if t.args else None)
            A = _np(A).astype(np.float64)
            from scipy.linalg import expm  # transforms.py:1235: matrix_exp(A - A^T)

            return Layer("rotation", R=expm(A - A.T))
        raise NotImplementedError(f"oracle: unconditional transform {fname}")
    raise NotImplementedError(f"oracle: layer {name}")


def flowspec_from_module(flow) -> FlowSpec:
    """Builds the numpy FlowSpec from a Flow module (lazy.py:131-172)."""
    tr = flow.transform
    layers = [layer_from_module(t) for t in (tr.transforms if hasattr(tr, "transforms") else [tr])]
    base = flow.base
    kw, args = base.kwargs, list(base.args)
    if getattr(base.f, "__name__", "") == "BoxUniform":  # flows/spline.py:111-116
        lower = _np(kw["lower"] if "lower" in kw else args[0]).astype(np.float64)
        upper = _np(kw["upper"] if "upper" in kw else args[-1]).astype(np.float64)
        return FlowSpec(layers, lower, upper, base="uniform")
    loc = _np(kw["loc"] if "loc" in kw else args[0]).astype(np.float64)
    scale = _np(kw["scale"] if "scale" in kw else args[-1]).astype(np.float64)
    return FlowSpec(layers, loc, scale)
