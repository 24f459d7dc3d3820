"""Distributions of the flow hot path: ``NormalizingFlow`` and ``DiagNormal``.

Host-side mirror of zuko/distributions.py:39-138 (NormalizingFlow) and :337-363
(DiagNormal).  Densities and inverse passes run in the H100 engine; torch provides the
random numbers (``torch.randn`` on the device) and owns all memory.
"""

from __future__ import annotations

__all__ = ["BoxUniform", "DiagNormal", "NormalizingFlow"]

from textwrap import indent

import torch
from torch import Size, Tensor
from torch.distributions import Distribution, Transform, constraints

from . import _engine as E
from . import _ops
from .transforms import ComposedTransform

Distribution.set_default_validate_args(False)  # like zuko/distributions.py:35


class DiagNormal(Distribution):
    """Multivariate normal with diagonal covariance, ``loc`` / ``scale`` of shape ``(D,)``
    (zuko/distributions.py:337-363 = Independent(Normal(loc, scale), 1)).

    ``log_prob`` is evaluated by ``zk_diag_normal_log_prob`` (the arithmetic of
    torch/distributions/normal.py:87-102 summed over the event dimension)."""

    has_rsample = True
    arg_constraints = {}

    def __init__(self, loc: Tensor, scale: Tensor, ndims: int = 1) -> None:
        loc, scale = torch.as_tensor(loc), torch.as_tensor(scale)
        if ndims != 1 or loc.dim() != 1 or scale.shape != loc.shape:
            raise NotImplementedError("zuko_b200: DiagNormal supports 1-d loc/scale and ndims=1 only")
        self.loc, self.scale = loc, scale
        super().__init__(batch_shape=Size(), event_shape=loc.shape, validate_args=False)

    def __repr__(self) -> str:
        return f"DiagNormal(loc: {self.loc.shape}, scale: {self.scale.shape})"

    @property
    def support(self) -> constraints.Constraint:
        return constraints.real_vector

    @property
    def mean(self) -> Tensor:
        return self.loc.expand(self.batch_shape + self.event_shape)

    @property
    def stddev(self) -> Tensor:
        return self.scale.expand(self.batch_shape + self.event_shape)

    def expand(self, batch_shape: Size, new: Distribution | None = None) -> Distribution:
        new = self._get_checked_instance(DiagNormal, new)
        new.loc, new.scale = self.loc, self.scale
        Distribution.__init__(new, batch_shape=Size(batch_shape), event_shape=self.event_shape, validate_args=False)
        return new

    def rsample(self, shape: Size = ()) -> Tensor:
        full = Size(shape) + self.batch_shape + self.event_shape
        eps = torch.randn(full, device=self.loc.device, dtype=self.loc.dtype)  # torch RNG (normal.py:82-85)
        return self.loc + eps * self.scale

    def sample(self, shape: Size = ()) -> Tensor:
        with torch.no_grad():
            return self.rsample(shape)

    def log_prob(self, z: Tensor) -> Tensor:
        E.require_cuda(z, "input")
        D = self.loc.shape[0]
        lead = torch.broadcast_shapes(z.shape[:-1], self.batch_shape)
        z2 = z.expand(*lead, D).reshape(-1, D).contiguous()
        E.require_cuda(self.loc, "base loc")
        if torch.is_grad_enabled() and (z2.requires_grad or self.loc.requires_grad or self.scale.requires_grad):
            # the unfused path of NormalizingFlow.log_prob (`base.log_prob(z) + ladj`) and direct users
            # differentiate through the base term: autograd seam around the same kernel
            return _DiagNormalLogProb.apply(z2, self.loc, self.scale).reshape(lead)
        return _diag_normal_log_prob(z2.detach(), self.loc.detach(), self.scale.detach()).reshape(lead)


def _diag_normal_log_prob(z2: Tensor, loc: Tensor, scale: Tensor) -> Tensor:
    D = loc.shape[0]
    out = torch.empty(z2.shape[0], device=z2.device, dtype=torch.float32)
    loc, scale = loc.contiguous(), scale.contiguous()
    with torch.cuda.device(z2.device):
        E.check(E.lib().zk_diag_normal_log_prob(z2.data_ptr(), D, loc.data_ptr(), scale.data_ptr(), None,
                                                z2.shape[0], D, out.data_ptr(), E.stream_ptr(z2.device)))  # fmt: skip
    return out


class _DiagNormalLogProb(torch.autograd.Function):
    """``DiagNormal(loc, scale).log_prob(z)`` with its gradient (torch/distributions/normal.py:87-102,
    independent.py:120-122): forward = ``zk_diag_normal_log_prob``; backward = the analytic
    ``d/dz = -(z - loc) / scale^2``, ``d/dloc = -d/dz`` summed over the batch, ``d/dscale = ((z - loc)^2 /
    scale^2 - 1) / scale`` summed over the batch."""

    @staticmethod
    def forward(ctx, z2, loc, scale):  # noqa: ANN001
        ctx.save_for_backward(z2, loc, scale)
        return _diag_normal_log_prob(z2.detach(), loc.detach(), scale.detach())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):  # noqa: ANN001
        z2, loc, scale = ctx.saved_tensors
        need = ctx.needs_input_grad
        u = (z2 - loc) / scale
        gu = g.reshape(-1, 1) * u
        gz = -gu / scale if need[0] else None
        g_loc = (gu / scale).sum(0) if need[1] else None
        g_scale = (g.reshape(-1, 1) * (u * u - 1.0) / scale).sum(0) if need[2] else None
        return gz, g_loc, g_scale


class BoxUniform(Distribution):
    """Uniform distribution over the box ``lower_i <= x_i < upper_i`` (zuko/distributions.py:366-396 =
    Independent(Uniform(lower, upper), 1)); the base of ``NCSF`` (flows/spline.py:111-116).

    ``log_prob`` is evaluated by ``zk_box_uniform_log_prob``: ``-sum log(upper - lower)`` inside the
    box, ``-inf`` outside (torch/distributions/uniform.py)."""

    has_rsample = True
    arg_constraints = {}

    def __init__(self, lower: Tensor, upper: Tensor, ndims: int = 1) -> None:
        lower, upper = torch.as_tensor(lower), torch.as_tensor(upper)
        if ndims != 1 or lower.dim() != 1 or upper.shape != lower.shape:
            raise NotImplementedError("zuko_b200: BoxUniform supports 1-d lower/upper and ndims=1 only")
        self.lower, self.upper = lower, upper
        super().__init__(batch_shape=Size(), event_shape=lower.shape, validate_args=False)

    def __repr__(self) -> str:
        return f"BoxUniform(lower: {self.lower.shape}, upper: {self.upper.shape})"

    def expand(self, batch_shape: Size, new: Distribution | None = None) -> Distribution:
        new = self._get_checked_instance(BoxUniform, new)
        new.lower, new.upper = self.lower, self.upper
        Distribution.__init__(new, batch_shape=Size(batch_shape), event_shape=self.event_shape, validate_args=False)
        return new

    def rsample(self, shape: Size = ()) -> Tensor:
        full = Size(shape) + self.batch_shape + self.event_shape
        u = torch.rand(full, device=self.lower.device, dtype=self.lower.dtype)  # torch RNG (uniform.py)
        return self.lower + u * (self.upper - self.lower)

    def sample(self, shape: Size = ()) -> Tensor:
        with torch.no_grad():
            return self.rsample(shape)

    def log_prob(self, z: Tensor) -> Tensor:
        E.require_cuda(z, "input")
        D = self.lower.shape[0]
        lead = torch.broadcast_shapes(z.shape[:-1], self.batch_shape)
        z2 = z.detach().expand(*lead, D).reshape(-1, D).contiguous()
        out = torch.empty(z2.shape[0], device=z.device, dtype=torch.float32)
        lo, hi = self.lower.detach().contiguous(), self.upper.detach().contiguous()
        E.require_cuda(lo, "lower bound")
        with torch.cuda.device(z.device):
            E.check(E.lib().zk_box_uniform_log_prob(z2.data_ptr(), D, lo.data_ptr(), hi.data_ptr(), None,
                                                    z2.shape[0], D, out.data_ptr(), E.stream_ptr(z.device)))  # fmt: skip
        return out.reshape(lead)


class NormalizingFlow(Distribution):
    """Normalizing flow ``p(x) = p_Z(f(x)) |det df/dx|`` (zuko/distributions.py:39-138).

    With a composed stack of engine layers and a ``DiagNormal`` base, ``log_prob``,
    ``rsample`` and ``rsample_and_log_prob`` are each ONE engine call
    (``zk_flow_log_prob`` / ``zk_flow_inverse``)."""

    has_rsample = True
    arg_constraints = {}

    def __init__(self, transform: Transform, base: Distribution) -> None:
        super().__init__(validate_args=False)
        reinterpreted = transform.codomain.event_dim - len(base.event_shape)
        if reinterpreted > 0:
            raise NotImplementedError("zuko_b200: base distributions with fewer event dims than the transform are not supported")
        self.transform = transform
        self.base = base
        self.reinterpreted = max(-reinterpreted, 0)

    def __repr__(self) -> str:
        lines = indent(f"(transform): {self.transform}\n(base): {self.base}", "  ")
        return f"{type(self).__name__}(\n{lines}\n)"

    @property
    def batch_shape(self) -> Size:
        return self.base.batch_shape

    @property
    def event_shape(self) -> Size:
        return self.transform.inverse_shape(self.base.event_shape)

    def expand(self, batch_shape: Size, new: Distribution | None = None) -> Distribution:
        new = self._get_checked_instance(NormalizingFlow, new)
        new.transform = self.transform
        new.base = self.base.expand(batch_shape)
        new.reinterpreted = self.reinterpreted
        Distribution.__init__(new, validate_args=False)
        return new

    # -- fused engine path -----------------------------------------------------
    def _flow_call(self):
        if "_fc" in self.__dict__:
            return self.__dict__["_fc"]
        fc = None
        t, base = self.transform, self.base
        if isinstance(t, ComposedTransform) and isinstance(base, (DiagNormal, BoxUniform)) and self.reinterpreted == 0:
            box = isinstance(base, BoxUniform)
            first, second = (base.lower, base.upper) if box else (base.loc, base.scale)
            fused = t._fused(first.shape[0])
            if fused is not None:
                call, ctx = fused
                kind = E.ZK_BASE_BOX_UNIFORM if box else E.ZK_BASE_DIAG_NORMAL
                fc = (_ops.FlowCall(call._handles, call.D, call.C, first, second, sources=call._sources, keep=call._keep,
                                    base_kind=kind, inverted=call._inverted), ctx)  # fmt: skip
                if call.folded is not None:  # permutations folded into the layers: forward-only sibling, same base
                    f = call.folded
                    fc[0].folded = _ops.FlowCall(f._handles, f.D, f.C, first.detach(), second.detach(), sources=None,
                                                 keep=f._keep, base_kind=kind, inverted=f._inverted)  # fmt: skip
        self.__dict__["_fc"] = fc
        return fc

    def log_prob(self, x: Tensor) -> Tensor:
        fc = self._flow_call()
        if fc is not None and fc[0].usable(x, fc[1]):
            call, ctx = fc
            lp = call.best(x, ctx).log_prob(x, ctx)
            return lp.expand(torch.broadcast_shapes(lp.shape, self.batch_shape)) if self.batch_shape else lp
        z, ladj = self.transform.call_and_ladj(x)
        if self.reinterpreted:
            ladj = ladj.sum(dim=tuple(range(-self.reinterpreted, 0)))
        return self.base.log_prob(z) + ladj

    def log_prob_and_sum(self, x: Tensor, sum_out: Tensor | None = None) -> tuple[Tensor, Tensor]:
        """``(log_prob(x), sum(log_prob(x)) as a device double[1])`` — the per-rank term of
        the mean NLL, produced by a fixed-order reduction inside the same engine call (written
        into ``sum_out``, e.g. ``dist.NllRing.slot(count)``, when given)."""
        fc = self._flow_call()
        if fc is None or not fc[0].usable(x, fc[1]):
            lp = self.log_prob(x)
            total = lp.detach().double().sum().reshape(1)
            if sum_out is not None:
                sum_out.copy_(total)
                total = sum_out
            return lp, total
        call, ctx = fc
        return call.best(x, ctx).log_prob(x, ctx, with_sum=True, sum_out=sum_out)

    def rsample(self, shape: Size = ()) -> Tensor:
        z = self.base.rsample(shape) if self.base.has_rsample else self.base.sample(shape)
        fc = self._flow_call()
        if fc is not None and fc[0].usable(z, fc[1]):
            call, ctx = fc
            return call.best(z, ctx).inverse(z, ctx)
        return self.transform.inv(z)

    def sample(self, shape: Size = ()) -> Tensor:
        with torch.no_grad():
            return self.rsample(shape)

    def rsample_and_log_prob(self, shape: Size = ()) -> tuple[Tensor, Tensor]:
        z = self.base.rsample(shape) if self.base.has_rsample else self.base.sample(shape)
        fc = self._flow_call()
        if fc is not None and fc[0].usable(z, fc[1], inverse_log_prob=True):
            call, ctx = fc
            return call.best(z, ctx).inverse(z, ctx, with_log_prob=True)
        x, ladj = self.transform.inv.call_and_ladj(z)
        if self.reinterpreted:
            ladj = ladj.sum(dim=tuple(range(-self.reinterpreted, 0)))
        return x, self.base.log_prob(z) - ladj
