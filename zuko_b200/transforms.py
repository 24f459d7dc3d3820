"""Engine-backed transformations of the flow hot path.

Host-side mirror of the ``Transform`` protocol the reference's hot path uses
(zuko/transforms.py): ``__call__``, ``.inv``, ``log_abs_det_jacobian(x, y)`` and Zuko's
``call_and_ladj(x) -> (y, ladj)`` (transforms.py:46-56).  Every method forwards to the
C ABI of the H100 engine; no torch arithmetic runs here.

* univariate bijectors built from explicit parameters:
  ``MonotonicRQSTransform`` (transforms.py:449-567), ``MonotonicAffineTransform``
  (:412-446), ``GaussianizationTransform`` (:834-875), ``SOSPolynomialTransform`` (:931-963,
  with ``ShiftedSOSPTransform`` of zuko/flows/polynomial.py:23-28), ``BoundedBernsteinTransform``
  (:640-831), ``SoftclipTransform`` (:286-316);
* linear maps: ``PermutationTransform`` (:1182-1214), ``RotationTransform`` (:1217-1244);
* packed conditional layers produced by the lazy modules in ``zuko_b200.flows``:
  ``AutoregressiveTransform`` (:966-1007), ``CouplingTransform`` (:1010-1073),
  ``DependentTransform`` (:163-220, the element-wise case);
* ``FreeFormJacobianTransform`` (:1095-1179), the continuous flow built by ``zuko_b200.flows.FFJTransform``;
* ``ComposedTransform`` (:59-160), which hands a whole stack of packed layers to one
  flow-level engine call when it can.
"""

from __future__ import annotations

__all__ = [
    "BoundedBernsteinTransform",
    "AutoregressiveTransform",
    "CircularRQSTransform",
    "CircularShiftTransform",
    "ComposedTransform",
    "CouplingTransform",
    "DependentTransform",
    "FreeFormJacobianTransform",
    "GaussianizationTransform",
    "MonotonicAffineTransform",
    "MonotonicRQSTransform",
    "PermutationTransform",
    "RotationTransform",
    "SOSPolynomialTransform",
    "ShiftedSOSPTransform",
    "SoftclipTransform",
]

import ctypes
import math
from collections.abc import Sequence
from textwrap import indent

import torch
from torch import LongTensor, Size, Tensor
from torch.distributions import Transform, constraints
from torch.distributions.utils import _sum_rightmost

from . import _engine as E
from . import _ops


def _call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:  # noqa: ANN001
    y = self.__call__(x)
    return y, self.log_abs_det_jacobian(x, y)


# same extension of the torch protocol as zuko/transforms.py:46-56
Transform.call_and_ladj = _call_and_ladj


class _InverseOf(Transform):
    """``t.inv`` for engine transforms: swaps the two directions and negates the ladj
    (torch/distributions/transforms.py:217-283)."""

    def __init__(self, t: Transform) -> None:
        super().__init__()
        self._t = t

    domain = property(lambda self: self._t.codomain)
    codomain = property(lambda self: self._t.domain)
    bijective = True

    @property
    def inv(self) -> Transform:
        return self._t

    def __repr__(self) -> str:
        return f"Inverse({self._t})"

    def __call__(self, y: Tensor) -> Tensor:
        return self._t._inverse(y)

    def _inverse(self, x: Tensor) -> Tensor:
        return self._t(x)

    def log_abs_det_jacobian(self, y: Tensor, x: Tensor) -> Tensor:
        return -self._t.log_abs_det_jacobian(x, y)

    def call_and_ladj(self, y: Tensor) -> tuple[Tensor, Tensor]:
        x = self._t._inverse(y)
        return x, -self._t.log_abs_det_jacobian(x, y)

    def forward_shape(self, shape: Size) -> Size:
        return self._t.inverse_shape(shape)

    def inverse_shape(self, shape: Size) -> Size:
        return self._t.forward_shape(shape)


class EngineTransform(Transform):
    """Base class: subclasses implement ``call_and_ladj`` and ``_inverse``."""

    bijective = True
    sign = +1

    def __init__(self) -> None:
        super().__init__(cache_size=0)

    @property
    def inv(self) -> Transform:
        return _InverseOf(self)

    def __call__(self, x: Tensor) -> Tensor:
        return self._call(x)

    def _call(self, x: Tensor) -> Tensor:
        return self.call_and_ladj(x)[0]

    def log_abs_det_jacobian(self, x: Tensor, y: Tensor) -> Tensor:
        return self.call_and_ladj(x)[1]

    def __eq__(self, other: object) -> bool:
        return self is other

    __hash__ = object.__hash__


# --------------------------------------------------------------------------- #
# univariate bijectors with explicit parameters
# --------------------------------------------------------------------------- #


def _elementwise(phi: Tensor, x: Tensor, P: int):
    """Maps an element-wise call (x of any shape, params with broadcastable batch shape)
    onto the engine's (B, D=1) layout.  Returns (x2 (N,1), phi2, phi_ld, shape)."""
    E.require_cuda(x, "input")
    E.require_cuda(phi, "parameters")
    batch = phi.shape[:-1]
    shape = torch.broadcast_shapes(x.shape, batch)
    x2 = x.expand(shape).reshape(-1, 1).contiguous()
    if len(batch) == 0 or math.prod(batch) == 1:
        return x2, phi.reshape(1, P).contiguous(), 0, shape
    phi2 = phi.expand(*shape, P).reshape(-1, P).contiguous()
    return x2, phi2, P, shape


def _uni_forward(kind: int, K: int, bound: float, slope: float, x2: Tensor, phi: Tensor | None, ld: int):
    """(y, ladj) of a univariate bijector on the (N, 1) layout; kind 0 = softclip."""
    x2 = x2.detach()
    y = torch.empty_like(x2)
    ladj = torch.empty(x2.shape[0], device=x2.device, dtype=torch.float32)
    L, st, N = E.lib(), E.stream_ptr(x2.device), x2.shape[0]
    with torch.cuda.device(x2.device):
        if kind == E.ZK_UNI_RQS:
            E.check(L.zk_rqs_forward(x2.data_ptr(), 1, phi.detach().data_ptr(), ld, N, 1, K, bound, slope, y.data_ptr(), 1, ladj.data_ptr(), 0, st))
        elif kind == E.ZK_UNI_GAUSS:
            E.check(L.zk_gaussianization_forward(x2.data_ptr(), 1, phi.detach().data_ptr(), ld, N, 1, K, y.data_ptr(), 1, ladj.data_ptr(), 0, st))
        elif kind == E.ZK_UNI_SOSP:
            (K, deg) = K
            E.check(L.zk_sosp_forward(x2.data_ptr(), 1, phi.detach().data_ptr(), ld, N, 1, K, deg, bound, slope, y.data_ptr(), 1, ladj.data_ptr(), 0, st))
        elif kind == E.ZK_UNI_BERNSTEIN:
            (deg, eps) = K
            E.check(L.zk_bernstein_forward(x2.data_ptr(), 1, phi.detach().data_ptr(), ld, N, 1, deg, bound, eps, y.data_ptr(), 1, ladj.data_ptr(), 0, st))
        elif kind == E.ZK_UNI_AFFINE:
            E.check(L.zk_affine_forward(x2.data_ptr(), 1, phi.detach().data_ptr(), ld, N, 1, slope, y.data_ptr(), 1, ladj.data_ptr(), 0, st))
        else:
            E.check(L.zk_softclip_forward(x2.data_ptr(), 1, N, 1, bound, y.data_ptr(), 1, ladj.data_ptr(), 0, st))
    return y, ladj


class _UniFunction(torch.autograd.Function):
    """Autograd seam of the explicit-parameter bijectors: backward = ``zk_rqs_backward`` /
    ``zk_affine_backward`` / ``zk_gaussianization_backward`` / ``zk_sosp_backward`` / ``zk_softclip_backward``
    / ``zk_bernstein_backward`` (reverse mode of transforms.py:469-567, 426-446, 834-875, 878-963, 299-316,
    640-831).  ``K`` is the pair ``(polynomials, degree)`` for the sum-of-squares polynomial bijector and
    ``(degree, eps)`` for the bounded Bernstein bijector."""

    @staticmethod
    def forward(ctx, kind, K, bound, slope, ld, x2, phi):  # noqa: ANN001
        ctx.cfg = (kind, K, bound, slope, ld)
        ctx.has_phi = phi is not None
        ctx.save_for_backward(*([x2, phi] if phi is not None else [x2]))
        return _uni_forward(kind, K, bound, slope, x2, phi, ld)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy, gl):  # noqa: ANN001
        kind, K, bound, slope, ld = ctx.cfg
        x2 = ctx.saved_tensors[0]
        phi = ctx.saved_tensors[1] if ctx.has_phi else None
        need_x, need_phi = ctx.needs_input_grad[5], ctx.has_phi and ctx.needs_input_grad[6]
        gy, gl = gy.to(torch.float32).contiguous(), gl.to(torch.float32).contiguous()
        N = x2.shape[0]
        gx = torch.empty_like(x2) if need_x else None
        gphi = None
        L, st = E.lib(), E.stream_ptr(x2.device)
        with torch.cuda.device(x2.device):
            if kind == 0:
                if need_x:
                    E.check(L.zk_softclip_backward(x2.data_ptr(), 1, N, 1, bound, gy.data_ptr(), 1, gl.data_ptr(), gx.data_ptr(), 1, st))
                return None, None, None, None, None, gx, None
            P = phi.shape[-1]
            if need_phi:
                gphi = torch.zeros_like(phi)  # (N, P) per-sample, or the (1, P) table (accumulated into)
            need = L.zk_univariate_backward_workspace_bytes(N, 1, P, ld) if need_phi else 0
            ws = E.Workspace.get(x2.device, need, min(need, 64 << 20)) if need else None
            args = (gy.data_ptr(), 1, gl.data_ptr(), None if gx is None else gx.data_ptr(), 1,
                    None if gphi is None else gphi.data_ptr(), None if ws is None else ws.data_ptr(),
                    0 if ws is None else ws.numel(), st)  # fmt: skip
            if kind == E.ZK_UNI_RQS:
                E.check(L.zk_rqs_backward(x2.data_ptr(), 1, phi.data_ptr(), ld, N, 1, K, bound, slope, *args))
            elif kind == E.ZK_UNI_GAUSS:
                E.check(L.zk_gaussianization_backward(x2.data_ptr(), 1, phi.data_ptr(), ld, N, 1, K, *args))
            elif kind == E.ZK_UNI_SOSP:
                E.check(L.zk_sosp_backward(x2.data_ptr(), 1, phi.data_ptr(), ld, N, 1, *K, bound, slope, *args))
            elif kind == E.ZK_UNI_BERNSTEIN:
                E.check(L.zk_bernstein_backward(x2.data_ptr(), 1, phi.data_ptr(), ld, N, 1, K[0], bound, K[1], *args))
            else:
                E.check(L.zk_affine_backward(x2.data_ptr(), 1, phi.data_ptr(), ld, N, 1, slope, *args))
        return None, None, None, None, None, gx, gphi


def _uni_call(kind: int, K: int, bound: float, slope: float, x2: Tensor, phi: Tensor | None, ld: int):
    if torch.is_grad_enabled() and (x2.requires_grad or (phi is not None and phi.requires_grad)):
        return _UniFunction.apply(kind, K, bound, slope, ld, x2, phi)
    return _uni_forward(kind, K, bound, slope, x2, phi, ld)


_warned_inverse = False


def _no_grad_inverse(*tensors: Tensor) -> None:
    """The inverse direction has no backward pass yet: results are detached (warned once)."""
    global _warned_inverse
    if not _warned_inverse and torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        _warned_inverse = True
        import warnings

        warnings.warn("zuko_b200: the inverse of a bijector is not differentiable in this version; the result is detached.", stacklevel=3)


class MonotonicRQSTransform(EngineTransform):
    """Monotonic rational-quadratic spline with unconstrained parameters
    ``widths (*, K)``, ``heights (*, K)``, ``derivatives (*, K-1)`` — the constructor of
    zuko/transforms.py:469-490; evaluated by ``zk_rqs_forward`` / ``zk_rqs_inverse``."""

    domain = constraints.real
    codomain = constraints.real

    def __init__(self, widths: Tensor, heights: Tensor, derivatives: Tensor, bound: float = 5.0, slope: float = 1e-3) -> None:
        super().__init__()
        batch = torch.broadcast_shapes(widths.shape[:-1], heights.shape[:-1], derivatives.shape[:-1])
        parts = [t.expand(*batch, t.shape[-1]) for t in (widths, heights, derivatives)]
        self.phi = torch.cat(parts, dim=-1)  # (*, 3K-1): layout of flows/spline.py:57
        self.bins = widths.shape[-1]
        self.bound, self.slope = float(bound), float(slope)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(bins={self.bins})"

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        P = 3 * self.bins - 1
        x2, phi, ld, shape = _elementwise(self.phi, x, P)
        y, ladj = _uni_call(E.ZK_UNI_RQS, self.bins, self.bound, self.slope, x2, phi, ld)
        return y.reshape(shape), ladj.reshape(shape)

    def _inverse(self, y: Tensor) -> Tensor:
        P = 3 * self.bins - 1
        _no_grad_inverse(y, self.phi)
        y2, phi, ld, shape = _elementwise(self.phi.detach(), y.detach(), P)
        x = torch.empty_like(y2)
        with torch.cuda.device(y2.device):
            E.check(E.lib().zk_rqs_inverse(y2.data_ptr(), 1, phi.data_ptr(), ld, y2.shape[0], 1, self.bins,
                                           self.bound, self.slope, x.data_ptr(), 1, E.stream_ptr(y2.device)))  # fmt: skip
        return x.reshape(shape)


class MonotonicAffineTransform(EngineTransform):
    """``f(x) = exp(a) x + b`` with soft-clipped log-scale (zuko/transforms.py:426-446)."""

    domain = constraints.real
    codomain = constraints.real

    def __init__(self, shift: Tensor, scale: Tensor, slope: float = 1e-3) -> None:
        super().__init__()
        shift, scale = torch.broadcast_tensors(shift, scale)
        self.phi = torch.stack((shift, scale), dim=-1)  # (*, 2): (shift, unconstrained log-scale)
        self.slope = float(slope)

    def __repr__(self) -> str:
        return f"{type(self).__name__}()"

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        x2, phi, ld, shape = _elementwise(self.phi, x, 2)
        y, ladj = _uni_call(E.ZK_UNI_AFFINE, 0, 5.0, self.slope, x2, phi, ld)
        return y.reshape(shape), ladj.reshape(shape)

    def _inverse(self, y: Tensor) -> Tensor:
        _no_grad_inverse(y, self.phi)
        y2, phi, ld, shape = _elementwise(self.phi.detach(), y.detach(), 2)
        x = torch.empty_like(y2)
        with torch.cuda.device(y2.device):
            E.check(E.lib().zk_affine_inverse(y2.data_ptr(), 1, phi.data_ptr(), ld, y2.shape[0], 1, self.slope,
                                              x.data_ptr(), 1, E.stream_ptr(y2.device)))  # fmt: skip
        return x.reshape(shape)


def bisection_steps(bound: float, eps: float) -> int:
    """Iterations of the reference's bisection inverse on ``[-bound, bound]`` (transforms.py:609-617)."""
    return math.ceil(math.log2(2 * bound / eps))


class GaussianizationTransform(EngineTransform):
    """``f(x) = Phi^-1(c/K sum_k Phi(exp(a_k) x + b_k))``, ``c = 1 - 1e-6``, with ``shift`` b and unconstrained
    ``scale`` a of shape ``(*, K)`` (zuko/transforms.py:834-875).  ``zk_gaussianization_forward`` evaluates y and the
    closed-form ladj; the inverse runs the reference's ``ceil(log2(2 bound / eps))`` bisection steps on
    ``[-bound, bound]`` (transforms.py:609-617) in ``zk_gaussianization_inverse``."""

    domain = constraints.real
    codomain = constraints.real

    def __init__(self, shift: Tensor, scale: Tensor, bound: float = 10.0, eps: float = 1e-6) -> None:
        super().__init__()
        shift, scale = torch.broadcast_tensors(shift, scale)
        self.phi = torch.cat((shift, scale), dim=-1)  # (*, 2K): layout of flows/gaussianization.py:91-92
        self.components = shift.shape[-1]
        self.bound, self.eps = float(bound), float(eps)
        self.iterations = bisection_steps(self.bound, self.eps)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(components={self.components})"

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        x2, phi, ld, shape = _elementwise(self.phi, x, 2 * self.components)
        y, ladj = _uni_call(E.ZK_UNI_GAUSS, self.components, self.bound, 1e-3, x2, phi, ld)
        return y.reshape(shape), ladj.reshape(shape)

    def _inverse(self, y: Tensor) -> Tensor:
        _no_grad_inverse(y, self.phi)
        y2, phi, ld, shape = _elementwise(self.phi.detach(), y.detach(), 2 * self.components)
        x = torch.empty_like(y2)
        with torch.cuda.device(y2.device):
            E.check(E.lib().zk_gaussianization_inverse(y2.data_ptr(), 1, phi.data_ptr(), ld, y2.shape[0], 1, self.components,
                                                       self.bound, self.iterations, x.data_ptr(), 1, E.stream_ptr(y2.device)))  # fmt: skip
        return x.reshape(shape)


class SOSPolynomialTransform(EngineTransform):
    """Sum-of-squares polynomial bijector ``f(x) = int_0^x (1/K) sum_k (1 + sum_j a_kj (u / bound)^j)^2 du + slope x``
    with coefficients ``a`` of shape ``(*, K, L + 1)`` (zuko/transforms.py:931-963).  ``zk_sosp_forward`` evaluates
    the reference's ``L + 1``-node Gauss-Legendre quadrature and ``ladj = log g(x)``; the inverse runs the
    reference's ``ceil(log2(2 bound / eps))`` bisection steps on ``[-bound, bound]`` (transforms.py:609-617) in
    ``zk_sosp_inverse``.  Gradients: ``zk_sosp_backward``."""

    domain = constraints.real
    codomain = constraints.real

    def __init__(self, a: Tensor, slope: float = 1e-3, bound: float = 10.0, eps: float = 1e-6) -> None:
        super().__init__()
        self._setup(a, a.new_zeros(()), slope, bound, eps)

    def _setup(self, a: Tensor, constant: Tensor, slope: float, bound: float, eps: float) -> None:
        self.polynomials, n = a.shape[-2:]
        self.degree = n - 1
        batch = torch.broadcast_shapes(a.shape[:-2], constant.shape)
        a = a.expand(*batch, self.polynomials, n).flatten(-2)
        # (*, K (L + 1) + 1): the layout of MaskedAutoregressiveTransform's split for shapes [(K, L + 1), ()]
        self.phi = torch.cat((a, constant.expand(batch)[..., None].to(a.dtype)), dim=-1)
        self.slope, self.bound, self.eps = float(slope), float(bound), float(eps)
        self.iterations = bisection_steps(self.bound, self.eps)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(polynomials={self.polynomials}, degree={self.degree})"

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        x2, phi, ld, shape = _elementwise(self.phi, x, self.phi.shape[-1])
        y, ladj = _uni_call(E.ZK_UNI_SOSP, (self.polynomials, self.degree), self.bound, self.slope, x2, phi, ld)
        return y.reshape(shape), ladj.reshape(shape)

    def _inverse(self, y: Tensor) -> Tensor:
        _no_grad_inverse(y, self.phi)
        y2, phi, ld, shape = _elementwise(self.phi.detach(), y.detach(), self.phi.shape[-1])
        x = torch.empty_like(y2)
        with torch.cuda.device(y2.device):
            E.check(E.lib().zk_sosp_inverse(y2.data_ptr(), 1, phi.data_ptr(), ld, y2.shape[0], 1, self.polynomials, self.degree,
                                            self.bound, self.slope, self.iterations, x.data_ptr(), 1, E.stream_ptr(y2.device)))  # fmt: skip
        return x.reshape(shape)


def ShiftedSOSPTransform(a: Tensor, constant: Tensor, slope: float = 1e-3) -> Transform:
    """``SOSPolynomialTransform(a, slope)`` followed by ``AdditiveTransform(constant)`` (zuko/flows/polynomial.py:23-28)
    as ONE engine transform: the constant is the last parameter of each pair and the kernels add it (forward) or
    subtract it before the bisection (inverse)."""
    t = SOSPolynomialTransform.__new__(SOSPolynomialTransform)
    EngineTransform.__init__(t)
    t._setup(a, constant, slope, 10.0, 1e-6)
    return t


class BoundedBernsteinTransform(EngineTransform):
    """Bounded Bernstein polynomial bijector of BPF with unconstrained parameters ``theta`` of shape
    ``(*, degree + 1)`` (zuko/transforms.py:780-831): the coefficients rise from ``-bound`` to ``bound``
    through a softmax, the polynomial of order ``degree + 5`` maps ``[-bound, bound]`` onto itself, and two
    linear branches of slope 1 continue it beyond (``x -+ 2 bound eps``).  ``zk_bernstein_forward`` evaluates
    it and ``ladj = log f'(x)``; the inverse returns the linear branches for ``|y| >= bound`` and otherwise
    runs the reference's ``ceil(log2(2 bound / eps))`` bisection steps on ``[-bound, bound]``
    (``zk_bernstein_inverse``).  Gradients: ``zk_bernstein_backward``."""

    domain = constraints.real
    codomain = constraints.real

    def __init__(self, theta: Tensor, bound: float = 5.0, eps: float = 1e-6) -> None:
        super().__init__()
        self.phi = theta
        self.degree = theta.shape[-1] - 1
        self.bound, self.eps = float(bound), float(eps)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(degree={self.degree}, bound={self.bound})"

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        x2, phi, ld, shape = _elementwise(self.phi, x, self.degree + 1)
        y, ladj = _uni_call(E.ZK_UNI_BERNSTEIN, (self.degree, self.eps), self.bound, 1e-3, x2, phi, ld)
        return y.reshape(shape), ladj.reshape(shape)

    def _inverse(self, y: Tensor) -> Tensor:
        _no_grad_inverse(y, self.phi)
        y2, phi, ld, shape = _elementwise(self.phi.detach(), y.detach(), self.degree + 1)
        x = torch.empty_like(y2)
        with torch.cuda.device(y2.device):
            E.check(E.lib().zk_bernstein_inverse(y2.data_ptr(), 1, phi.data_ptr(), ld, y2.shape[0], 1, self.degree,
                                                 self.bound, self.eps, x.data_ptr(), 1, E.stream_ptr(y2.device)))  # fmt: skip
        return x.reshape(shape)


class SoftclipTransform(EngineTransform):
    """``f(x) = x / (1 + |x / B|)`` mapping R to (-B, B) (zuko/transforms.py:286-316)."""

    def __init__(self, bound: float = 1.0) -> None:
        super().__init__()
        self.bound = float(bound)
        self.domain = constraints.real
        self.codomain = constraints.interval(-bound, bound)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(bound={self.bound})"

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        E.require_cuda(x, "input")
        x2 = x.reshape(-1, 1).contiguous()
        y, ladj = _uni_call(0, 0, self.bound, 1e-3, x2, None, 0)
        return y.reshape(x.shape), ladj.reshape(x.shape)

    def _inverse(self, y: Tensor) -> Tensor:
        E.require_cuda(y, "input")
        _no_grad_inverse(y)
        y = y.detach()
        y2 = y.reshape(-1, 1).contiguous()
        x = torch.empty_like(y2)
        with torch.cuda.device(y.device):
            E.check(E.lib().zk_softclip_inverse(y2.data_ptr(), 1, y2.shape[0], 1, self.bound, x.data_ptr(), 1,
                                                E.stream_ptr(y.device)))  # fmt: skip
        return x.reshape(y.shape)

    def _layer_desc(self, D: int):
        return E.LayerDesc(kind=E.ZK_LAYER_SOFTCLIP, features=D, bound=self.bound, slope=1e-3), []


class _CircularShiftFunction(torch.autograd.Function):
    """y = remainder(x, 2B) - B is a translation almost everywhere: dy/dx = 1."""

    @staticmethod
    def forward(ctx, x2, bound):  # noqa: ANN001
        y = torch.empty_like(x2)
        with torch.cuda.device(x2.device):
            E.check(E.lib().zk_circular_shift(x2.data_ptr(), 1, x2.shape[0], 1, bound, y.data_ptr(), 1, E.stream_ptr(x2.device)))
        return y

    @staticmethod
    def backward(ctx, gy):  # noqa: ANN001
        return gy, None


class CircularShiftTransform(EngineTransform):
    """``f(x) = (x mod 2B) - B``: circular shift of ``[-B, B]`` by half a period, its own inverse,
    ladj 0 (zuko/transforms.py:319-351; evaluated by ``zk_circular_shift``)."""

    def __init__(self, bound: float = 1.0) -> None:
        super().__init__()
        self.bound = float(bound)
        self.domain = constraints.interval(-bound, bound)
        self.codomain = constraints.interval(-bound, bound)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(bound={self.bound})"

    def _shift(self, x: Tensor) -> Tensor:
        E.require_cuda(x, "input")
        x2 = x.reshape(-1, 1).contiguous()
        return _CircularShiftFunction.apply(x2, self.bound).reshape(x.shape)

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        return self._shift(x), torch.zeros_like(x)

    def _inverse(self, y: Tensor) -> Tensor:
        return self._shift(y)


def CircularRQSTransform(*phi: Tensor, slope: float = 1e-3) -> Transform:
    """Circular rational-quadratic spline: a circular shift of ``[-pi, pi]`` followed by the monotonic
    RQS over the same interval (zuko/flows/spline.py:65-72).  Inside ``NCSF`` the engine evaluates
    the pair as one univariate kind (``ZK_UNI_CRQS``)."""
    return ComposedTransform(
        CircularShiftTransform(bound=math.pi),
        MonotonicRQSTransform(*phi, bound=math.pi, slope=slope),
    )


# --------------------------------------------------------------------------- #
# linear maps
# --------------------------------------------------------------------------- #


class _VectorLayer(EngineTransform):
    """A parameter-free / explicit-parameter map on feature vectors that the engine knows as a
    ``zk_layer``: evaluated as a one-layer flow call, which also gives it the autograd seam."""

    def _single(self, D: int) -> _ops.FlowCall:
        ref = _simple_layer_handle(self, D)
        cache = self.__dict__.setdefault("_single_calls", {})
        if D not in cache or cache[D][0] is not ref:
            src = self._grad_source() if hasattr(self, "_grad_source") else {}
            cache[D] = (ref, _ops.FlowCall([ref.handle], D, 0, None, None, sources=[src], keep=[ref]))
        return cache[D][1]


class PermutationTransform(_VectorLayer):
    """``y = x[..., order]`` — a bit-exact gather (zuko/transforms.py:1182-1214)."""

    domain = constraints.real_vector
    codomain = constraints.real_vector

    def __init__(self, order: LongTensor) -> None:
        super().__init__()
        if order.dim() != 1:
            raise NotImplementedError("zuko_b200: batched permutation orders are not supported")
        self.order = order

    def __repr__(self) -> str:
        order = self.order.tolist()
        if len(order) > 10:
            order = str(order[:5] + [...] + order[-5:]).replace("Ellipsis", "...")
        return f"{type(self).__name__}({order})"

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        return self._single(self.order.shape[0]).forward(x, None)

    def _inverse(self, y: Tensor) -> Tensor:
        return self._single(self.order.shape[0]).inverse(y, None)

    def _layer_desc(self, D: int):
        host = self.order.detach().to("cpu", torch.int64).contiguous()
        arr = (ctypes.c_int64 * D)(*host.tolist())
        return E.LayerDesc(kind=E.ZK_LAYER_PERMUTATION, features=D, slope=1e-3, bound=1.0, order=arr), [arr]


class RotationTransform(_VectorLayer):
    """``y = R x`` with ``R = exp(A - A^T)`` orthogonal (zuko/transforms.py:1217-1244).
    ``matrix_exp`` of the (D, D) generator is one-time torch plumbing; the batched
    product runs in ``zk_rotate``."""

    domain = constraints.real_vector
    codomain = constraints.real_vector

    def __init__(self, A: Tensor) -> None:
        super().__init__()
        if A.dim() != 2:
            raise NotImplementedError("zuko_b200: batched rotation generators are not supported")
        # R carries its autograd history: the engine returns dL/dR and torch chains through matrix_exp
        self.R = torch.linalg.matrix_exp(A - A.mT).contiguous()

    def _grad_source(self) -> dict:
        return {"R": self.R} if self.R.requires_grad else {}

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        return self._single(self.R.shape[0]).forward(x, None)

    def _inverse(self, y: Tensor) -> Tensor:
        return self._single(self.R.shape[0]).inverse(y, None)

    def _layer_desc(self, D: int):
        R = self.R.detach()
        return E.LayerDesc(kind=E.ZK_LAYER_ROTATION, features=D, slope=1e-3, bound=1.0, rotation=R.data_ptr()), [R]


# --------------------------------------------------------------------------- #
# packed conditional layers
# --------------------------------------------------------------------------- #


class _PackedLayerTransform(EngineTransform):
    """A ``zk_layer`` handle (owned by a lazy module) bound to a context ``c``."""

    domain = constraints.real_vector
    codomain = constraints.real_vector

    def __init__(self, owner, c: Tensor | None) -> None:  # noqa: ANN001
        super().__init__()
        self._owner = owner
        self._c = c
        self.features = owner.features

    def _layer_handle(self, D: int | None = None):
        return self._owner._zk_layer()

    def _layer_ref(self, D: int | None = None):
        return self._owner._zk_layer_ref()

    def _grad_source(self) -> dict:
        return self._owner._grad_source()

    def _single(self) -> _ops.FlowCall:
        """This layer alone as a flow-level call (gives it the autograd seam of _ops.FlowCall)."""
        ref = self._layer_ref()
        cached = self.__dict__.get("_single_call")
        if cached is None or cached[0] is not ref:
            call = _ops.FlowCall([ref.handle], self.features, self._owner.context, None, None,
                                 sources=[self._grad_source()], keep=[ref])  # fmt: skip
            cached = (ref, call)
            self.__dict__["_single_call"] = cached
        return cached[1]

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        return self._single().forward(x, self._c)

    def _inverse(self, y: Tensor) -> Tensor:
        return self._single().inverse(y, self._c)

    def __repr__(self) -> str:
        return f"{type(self).__name__}()"


class AutoregressiveTransform(_PackedLayerTransform):
    """``y_i = f(x_i | x_<i, c)`` with a masked conditioner (zuko/transforms.py:966-1007).
    The inverse runs the reference's ``passes`` fixed-point sweeps (:994-1000)."""

    @property
    def passes(self) -> int:
        return self._owner.passes


class CouplingTransform(_PackedLayerTransform):
    """``y_a = x_a, y_b = f(x_b | x_a, c)`` (zuko/transforms.py:1010-1073)."""


class DependentTransform(_PackedLayerTransform):
    """Element-wise univariate transformation whose ladj is summed over the feature
    dimension (zuko/transforms.py:163-220 wrapping flows/gaussianization.py:86-94)."""


# --------------------------------------------------------------------------- #
# composition
# --------------------------------------------------------------------------- #


def _simple_layer_handle(t: Transform, D: int):
    """Creates (and caches on the transform object) a zk_layer for a parameter-free /
    explicit-parameter transform so that it can join a fused flow call."""
    cache = t.__dict__.setdefault("_zk_layers", {})
    key = D
    if key not in cache:
        desc, keep = t._layer_desc(D)
        h = ctypes.c_void_p()
        E.check(E.lib().zk_layer_create(ctypes.byref(desc), ctypes.byref(h)))
        cache[key] = _OwnedLayer(h)
        del keep
    return cache[key]


_FOLD_PERMS: dict = {}


def _fold_perm_handle(q: tuple):
    """The gather layer that materialises a pending re-indexing ``q`` (ComposedTransform._folded): the composed
    transform is rebuilt on every ``flow(c)`` call, so these handles are kept per (device, q) — no allocation per call."""
    key = (torch.cuda.current_device() if torch.cuda.is_available() else -1, q)
    ref = _FOLD_PERMS.get(key)
    if ref is None:
        if len(_FOLD_PERMS) >= 64:
            _FOLD_PERMS.clear()
        ref = _simple_layer_handle(PermutationTransform(torch.tensor(q, dtype=torch.long)), len(q))
        _FOLD_PERMS[key] = ref
    return ref


class _OwnedLayer:
    def __init__(self, handle) -> None:  # noqa: ANN001
        self.handle = handle

    def __del__(self) -> None:
        try:
            E.lib().zk_layer_destroy(self.handle)
        except Exception:
            pass


def plan_permutation_fold(kinds: Sequence[str], sigmas: Sequence, D: int):
    """Bookkeeping of ComposedTransform._folded, free of engine objects (CPU-tested).  ``kinds[i]`` says what member i
    is: ``"perm"`` (``y = x[sigmas[i]]``), ``"reindex"`` (an autoregressive layer: ``T(P x) = P T~_q(x)``),
    ``"commute"`` (``S(P x) = P S(x)``) or ``"fixed"`` (needs the true feature order).  The stored vector ``s`` and
    the true one ``t`` are related by a pending re-indexing ``t[j] = s[q[j]]``.  Returns the list of actions
    ``("member", i, q or None)`` (run member i, re-indexed by q unless None) / ``("gather", q)`` (``s <- s[q]``), or
    ``None`` when a permutation is malformed or no kernel is saved."""
    ident = tuple(range(D))
    q = ident
    plan: list[tuple] = []
    for i, kind in enumerate(kinds):
        if kind == "perm":
            sigma = list(sigmas[i])
            if sorted(sigma) != list(ident):
                return None
            q = tuple(q[j] for j in sigma)  # t'[j] = t[sigma[j]] = s[q[sigma[j]]]
        elif kind == "reindex":
            plan.append(("member", i, None if q == ident else q))
        elif kind == "commute":
            plan.append(("member", i, None))
        else:
            if q != ident:
                plan.append(("gather", q))
                q = ident
            plan.append(("member", i, None))
    if q != ident:
        plan.append(("gather", q))
    return plan if len(plan) < len(kinds) else None


class ComposedTransform(EngineTransform):
    """``f = f_n ∘ ... ∘ f_0`` (zuko/transforms.py:59-160).

    When every member is an engine layer bound to the same context, the whole stack runs
    as ONE flow-level engine call per direction (``zk_flow_forward`` / ``zk_flow_inverse``);
    otherwise members are applied one after the other with the reference's event-dim
    bookkeeping (transforms.py:141-150)."""

    def __init__(self, *transforms: Transform) -> None:
        super().__init__()
        assert transforms, "'transforms' cannot be empty"
        event_dim = 0
        for t in reversed(transforms):
            event_dim = t.domain.event_dim + max(event_dim - t.codomain.event_dim, 0)
        self.domain_dim = event_dim
        for t in transforms:
            event_dim += t.codomain.event_dim - t.domain.event_dim
        self.codomain_dim = event_dim
        self.transforms = list(transforms)

    def __repr__(self) -> str:
        lines = "\n".join(f"({i}): {t}" for i, t in enumerate(self.transforms))
        return f"{type(self).__name__}(\n" + indent(lines, "  ") + "\n)"

    @property
    def domain(self) -> constraints.Constraint:
        dom = self.transforms[0].domain
        extra = self.domain_dim - dom.event_dim
        return constraints.independent(dom, extra) if extra > 0 else dom

    @property
    def codomain(self) -> constraints.Constraint:
        cod = self.transforms[-1].codomain
        extra = self.codomain_dim - cod.event_dim
        return constraints.independent(cod, extra) if extra > 0 else cod

    # -- fused path ----------------------------------------------------------
    def _fused(self, D: int):
        """Returns a FlowCall when all members can run inside one engine call."""
        key = ("_fused", D)
        if key in self.__dict__:
            return self.__dict__[key]
        call = None
        ctx = None
        handles, refs, sources, inverted = [], [], [], []
        ok = self.domain_dim == 1 and self.codomain_dim == 1
        C = 0
        for t in self.transforms if ok else ():
            inv = isinstance(t, _InverseOf) and isinstance(t._t, AutoregressiveTransform)
            if inv:  # LazyInverse of an autoregressive layer (zuko/lazy.py:81-98): an inverted member of the engine call
                t = t._t
                if not E.lib().zk_layer_sequential_inverse(t._layer_handle()):
                    ok = False
                    break
            inverted.append(inv)
            if isinstance(t, _PackedLayerTransform):
                if t.features != D:
                    ok = False
                    break
                if t._owner.context:
                    if ctx is not None and ctx is not t._c:
                        ok = False
                        break
                    ctx = t._c
                    C = t._owner.context
                refs.append(t._layer_ref())
                sources.append(t._grad_source())
            elif hasattr(t, "_layer_desc"):
                refs.append(_simple_layer_handle(t, D))
                sources.append(t._grad_source() if hasattr(t, "_grad_source") else {})
            else:
                ok = False
                break
        if ok:
            handles = [r.handle for r in refs]
            call = (_ops.FlowCall(handles, D, C, None, None, sources=sources, keep=refs, inverted=inverted), ctx)
            call[0].folded = self._folded(D, C, refs, inverted)
        self.__dict__[key] = call
        return call

    def _folded(self, D: int, C: int, refs: list, inverted: list):
        """The same bijection with every ``PermutationTransform`` that feeds an autoregressive layer folded INTO that
        layer (SURVEY K8; zuko/transforms.py:1193-1214): with ``(P x)_i = x_{q[i]}``, ``T(P x) = P T~(x)`` for the
        layer ``T~`` re-indexed by ``q`` (``MaskedAutoregressiveTransform._zk_layer_ref_reindexed``), and a soft clip
        commutes with ``P`` — so the permutation is carried along as a pending re-indexing ``q`` of the stored vector,
        and a gather kernel runs only where a member that cannot be re-indexed (coupling, rotation, element-wise
        tables) needs the true order, or at the end when ``q`` is not the identity (two reversals cancel).  A
        forward-only ``FlowCall`` (no gradient sources), or ``None`` when nothing folds."""
        from .flows.autoregressive import MaskedAutoregressiveTransform

        members = []
        for t in self.transforms:
            members.append(t._t if isinstance(t, _InverseOf) and isinstance(t._t, AutoregressiveTransform) else t)
        if not any(isinstance(t, PermutationTransform) for t in members):
            return None
        kinds, sigmas = [], []
        for t in members:
            sigma = None
            if isinstance(t, PermutationTransform):
                kind = "perm"
                sigma = t.__dict__.get("_order_host")  # the object is cached by its lazy module: one download, not one per call
                if sigma is None:
                    sigma = t.__dict__["_order_host"] = t.order.detach().to("cpu", torch.int64).tolist()
            elif isinstance(t, AutoregressiveTransform) and isinstance(t._owner, MaskedAutoregressiveTransform):
                kind = "reindex"
            elif isinstance(t, SoftclipTransform):
                kind = "commute"  # element-wise with one bound: S(P x) = P S(x), the ladj sum does not see the order
            else:
                kind = "fixed"
            kinds.append(kind)
            sigmas.append(sigma)
        plan = plan_permutation_fold(kinds, sigmas, D)
        if plan is None:
            return None
        out_refs, out_inv = [], []
        for act in plan:
            if act[0] == "gather":
                out_refs.append(_fold_perm_handle(act[1]))
                out_inv.append(False)
            else:
                _, i, q = act
                out_refs.append(refs[i] if q is None else members[i]._owner._zk_layer_ref_reindexed(q))
                out_inv.append(inverted[i])
        return _ops.FlowCall([r.handle for r in out_refs], D, C, None, None, sources=None, keep=out_refs, inverted=out_inv)

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        fused = self._fused(x.shape[-1]) if x.dim() >= 1 else None
        if fused is not None and fused[0].usable(x, fused[1]):
            call, ctx = fused
            return call.best(x, ctx).forward(x, ctx)
        event_dim = self.domain_dim
        acc = 0
        for t in self.transforms:
            x, ladj = t.call_and_ladj(x)
            acc = acc + _sum_rightmost(ladj, event_dim - t.domain.event_dim)
            event_dim += t.codomain.event_dim - t.domain.event_dim
        return x, acc

    def _inverse(self, y: Tensor) -> Tensor:
        fused = self._fused(y.shape[-1]) if y.dim() >= 1 else None
        if fused is not None and fused[0].usable(y, fused[1]):
            call, ctx = fused
            return call.best(y, ctx).inverse(y, ctx)
        for t in reversed(self.transforms):
            y = t.inv(y)
        return y

    def forward_shape(self, shape: Size) -> Size:
        for t in self.transforms:
            shape = t.forward_shape(shape)
        return shape

    def inverse_shape(self, shape: Size) -> Size:
        for t in reversed(self.transforms):
            shape = t.inverse_shape(shape)
        return shape


# --------------------------------------------------------------------------- #
# continuous flow
# --------------------------------------------------------------------------- #


class FreeFormJacobianTransform(EngineTransform):
    """Free-form Jacobian transformation ``x(t1) = x(t0) + int_t0^t1 f(t, x(t)) dt`` (transforms.py:1095-1179),
    integrated by the engine's Dormand-Prince kernel (``zk_cnf_integrate``) with the step size shared by the
    batch, as the reference does.  ``f`` is the vector field of :class:`zuko_b200.flows.FFJTransform` (built by
    its ``forward``); an arbitrary Python callable is refused.  Leading dimensions are flattened into one batch,
    which is integrated as a whole: the result of a row depends on the others through the step sequence.

    ``exact=False`` estimates the trace with Hutchinson's ``eps^T (df/dx) eps``, ``eps = randn_like(x)`` drawn
    once per call.  Gradients through the integration (the reference's adaptive checkpoint adjoint, second-order
    terms of the trace included) are opt-in: with ``adjoint=True`` a call that can need them becomes one autograd
    node whose backward is one ``zk_cnf_backward`` call; with ``adjoint=False`` (the default) such a call is
    refused with ``NotImplementedError``.  Gradients reach ``x`` and the tensors of ``phi`` (the context and, in
    training mode, the ODE parameters), never ``t0`` / ``t1``.  After ``max_trials`` trials without reaching
    ``t1`` a call raises ``RuntimeError``."""

    domain = constraints.real_vector
    codomain = constraints.real_vector

    def __init__(self, f, t0: float | Tensor = 0.0, t1: float | Tensor = 1.0, phi: Sequence[Tensor] = (),  # noqa: ANN001
                 atol: float = 1e-6, rtol: float = 1e-5, exact: bool = True, max_trials: int = 10000,
                 adjoint: bool = False) -> None:  # fmt: skip
        super().__init__()
        if not hasattr(f, "cnf_handle"):
            raise NotImplementedError(
                "zuko_b200: FreeFormJacobianTransform integrates the vector field of zuko_b200.flows.FFJTransform "
                "only; an arbitrary Python callable is outside the engine"
            )
        self.f = f
        self.t0, self.t1 = t0, t1
        self.phi = tuple(p for p in phi if p.requires_grad)
        self.atol, self.rtol, self.exact = atol, rtol, exact
        self.max_trials = max_trials
        self.adjoint = adjoint
        self.stats = None  # (trials, accepted) of the last call

    def __repr__(self) -> str:
        return f"FreeFormJacobianTransform(exact={self.exact})"

    @property
    def inv(self) -> Transform:
        return FreeFormJacobianTransform(self.f, self.t1, self.t0, self.phi, self.atol, self.rtol, self.exact, self.max_trials,
                                         self.adjoint)  # fmt: skip

    def _needs_grad(self, x: Tensor) -> bool:
        # the rule of call_and_ladj's create_graph (transforms.py:1150): phi holds c and the ODE parameters in
        # training mode only (flows/continuous.py:99-103)
        if not (torch.is_grad_enabled() and (x.requires_grad or bool(self.phi))):
            return False
        if not self.adjoint:
            raise NotImplementedError(
                "zuko_b200: gradients through the CNF integration (the adaptive checkpoint adjoint of "
                "zuko/utils.py:556-593) are opt-in: pass adjoint=True (or set transform.adjoint = True), call under "
                "torch.no_grad(), or use flow.eval() with an input that does not require grad"
            )
        if any(isinstance(t, Tensor) and t.requires_grad for t in (self.t0, self.t1)):
            raise NotImplementedError("zuko_b200: gradients with respect to the CNF integration times are not implemented")
        return True

    def _launch(self, x2: Tensor, lead: Size, trace: int, step_log: Tensor | None = None):
        """One zk_cnf_integrate call on the rows x2 (B, D): (y, ladj or None, eps or None, c, ldc, trials, accepted)."""
        B, D = x2.shape
        dev = x2.device
        times = torch.stack([torch.as_tensor(self.t0, device=dev), torch.as_tensor(self.t1, device=dev)]).float()
        eps = torch.randn_like(x2) if trace == E.ZK_CNF_TRACE_HUTCHINSON else None
        c, ldc = self.f.context(lead, B)
        y = torch.empty(B, D, device=dev, dtype=torch.float32)
        ladj = torch.empty(B, device=dev, dtype=torch.float32) if trace != E.ZK_CNF_TRACE_NONE else None
        counts = torch.zeros(2, device=dev, dtype=torch.int32)
        if B == 0:  # nothing to integrate; the empty ladj and eps would reach the engine as NULL pointers
            self.stats = (0, 0)
            return y, ladj, eps, c, ldc, 0, 0
        with torch.cuda.device(dev):
            h = self.f.cnf_handle()
            need = E.lib().zk_cnf_workspace_bytes(h, B, trace)
            ws = E.Workspace.get(dev, need, need)
            E.check(
                E.lib().zk_cnf_integrate(
                    h, x2.data_ptr(), x2.stride(0), c.data_ptr() if c is not None else None, ldc, B, times.data_ptr(),
                    self.atol, self.rtol, trace, eps.data_ptr() if eps is not None else None, D, self.max_trials,
                    y.data_ptr(), D, ladj.data_ptr() if ladj is not None else None, counts.data_ptr(),
                    step_log.data_ptr() if step_log is not None else None, ws.data_ptr(), ws.numel(), E.stream_ptr(dev),
                )
            )  # fmt: skip
        trials, accepted = counts.tolist()  # the one device-to-host read of a call
        if accepted < 0:
            raise RuntimeError(
                f"zuko_b200: the CNF integration did not reach t1: {trials} trials (max_trials = {self.max_trials}), "
                f"{-1 - accepted} accepted steps; the step size collapsed or the trial budget ran out"
            )
        self.stats = (trials, accepted)
        return y, ladj, eps, c, ldc, trials, accepted

    def _integrate(self, x: Tensor, trace: int) -> tuple[Tensor, Tensor | None]:
        grad = self._needs_grad(x)
        E.require_cuda(x, "CNF input")
        D = x.shape[-1]
        lead = x.shape[:-1]
        if grad:
            out = _CNFAdjoint.apply(self, trace, x, *self.phi)
            return (out, None) if trace == E.ZK_CNF_TRACE_NONE else out
        x2 = x.reshape(-1, D)
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        y, ladj = self._launch(x2, lead, trace)[:2]
        return y.reshape(*lead, D), (ladj.reshape(lead) if ladj is not None else None)

    def _call(self, x: Tensor) -> Tensor:
        return self._integrate(x, E.ZK_CNF_TRACE_NONE)[0]

    def _inverse(self, y: Tensor) -> Tensor:
        return self.inv._call(y)

    def call_and_ladj(self, x: Tensor) -> tuple[Tensor, Tensor]:
        return self._integrate(x, E.ZK_CNF_TRACE_EXACT if self.exact else E.ZK_CNF_TRACE_HUTCHINSON)

    def log_abs_det_jacobian(self, x: Tensor, y: Tensor) -> Tensor:
        return self.call_and_ladj(x)[1]


class _CNFAdjoint(torch.autograd.Function):
    """One CNF integration as an autograd node with inputs ``(x, *phi)``: the forward logs its steps, the backward
    is one ``zk_cnf_backward`` call (the adaptive checkpoint adjoint of zuko/utils.py:556-593).  The ODE
    parameters are saved, so that modifying them in place between forward and backward raises as torch does, and
    the handle looked up in backward is the forward's."""

    @staticmethod
    def forward(ctx, T: FreeFormJacobianTransform, trace: int, x: Tensor, *phi: Tensor):  # noqa: ANN001, ANN205
        D = x.shape[-1]
        lead = x.shape[:-1]
        x2 = x.detach().reshape(-1, D)
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        B = x2.shape[0]
        dev = x.device
        owner = T.f.owner
        with torch.cuda.device(dev):  # refuse a shape whose backward does not fit now, not at .backward()
            E.check(E.lib().zk_cnf_backward_plan(T.f.cnf_handle(), 0, trace, 0, 0, None, None, None, None))
        step_log = torch.empty(max(T.max_trials, 1), 4, device=dev, dtype=torch.float32)
        y, ladj, eps, c, ldc, trials, accepted = T._launch(x2, lead, trace, step_log)
        params = [t for m in owner.ode._linears() for t in (m.weight, m.bias) if t is not None]
        ctx.save_for_backward(x2, c, eps, step_log, *params)
        ctx.T, ctx.trace, ctx.lead, ctx.ldc = T, trace, lead, ldc
        ctx.counts = (trials, accepted)
        y = y.reshape(*lead, D)
        if trace == E.ZK_CNF_TRACE_NONE:
            return y
        return y, ladj.reshape(lead)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy: Tensor, gl: Tensor | None = None):  # noqa: ANN001, ANN205
        x2, c, eps, step_log, *_ = ctx.saved_tensors
        T, trace, lead, ldc = ctx.T, ctx.trace, ctx.lead, ctx.ldc
        trials, accepted = ctx.counts
        phi = T.phi
        B, D = x2.shape
        dev = x2.device
        lins = T.f.owner.ode._linears()
        gw = [torch.zeros_like(m.weight) if any(p is m.weight for p in phi) else None for m in lins]
        gb = [torch.zeros_like(m.bias) if m.bias is not None and any(p is m.bias for p in phi) else None for m in lins]
        cin = T.f.c
        want_c = cin is not None and any(p is cin for p in phi)
        gc = None
        if want_c and c is not None:
            gc = torch.empty(B, c.shape[-1], device=dev) if ldc else torch.empty(c.shape[-1], device=dev)
        gx = torch.empty(B, D, device=dev) if ctx.needs_input_grad[2] else None
        gy2 = None if gy is None else gy.reshape(B, D).float().contiguous()
        gl2 = None
        if trace != E.ZK_CNF_TRACE_NONE:
            gl2 = torch.zeros(B, device=dev) if gl is None else gl.reshape(B).float().contiguous()
        n = len(lins)
        wp = (ctypes.c_void_p * n)(*[None if g is None else g.data_ptr() for g in gw])
        bp = (ctypes.c_void_p * n)(*[None if g is None else g.data_ptr() for g in gb])
        grads = E.LayerGrads()
        grads.grad_weight, grads.grad_bias = wp, bp
        if B:
            with torch.cuda.device(dev):
                h = T.f.cnf_handle()
                lib = E.lib()
                need = lib.zk_cnf_backward_workspace_bytes(h, B, trace, accepted)
                ws = E.Workspace.get(dev, need, lib.zk_cnf_backward_min_workspace_bytes(h, trace, accepted))
                E.check(
                    lib.zk_cnf_backward(
                        h, x2.data_ptr(), x2.stride(0), None if c is None else c.data_ptr(), ldc, B, step_log.data_ptr(),
                        trials, accepted, trace, None if eps is None else eps.data_ptr(), D,
                        None if gy2 is None else gy2.data_ptr(), D, None if gl2 is None else gl2.data_ptr(),
                        None if gx is None else gx.data_ptr(), D, None if gc is None else gc.data_ptr(),
                        c.shape[-1] if c is not None else 0, ctypes.byref(grads), ws.data_ptr(), ws.numel(),
                        E.stream_ptr(dev),
                    )
                )  # fmt: skip
        else:  # no rows: every gradient is zero, the broadcast context's included
            for g in (gx, gc):
                if g is not None:
                    g.zero_()
        out = []
        for p in phi:
            g = None
            if p is cin:
                if gc is None:
                    g = torch.zeros_like(p)
                elif ldc:
                    g = gc.reshape(*lead, gc.shape[-1]).sum_to_size(p.shape)  # -1 is ambiguous when B = 0
                else:
                    g = gc.reshape(p.shape)
            else:
                for m, w, b in zip(lins, gw, gb, strict=True):
                    if p is m.weight:
                        g = w
                    elif p is m.bias:
                        g = b
            out.append(g)
        return (None, None, None if gx is None else gx.reshape(*lead, D), *out)
