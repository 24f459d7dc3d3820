"""Distributions of the hot path: ``NormalizingFlow``, ``DiagNormal`` and the Gaussian ``Mixture``.

Host-side mirror of zuko/distributions.py:39-138 (NormalizingFlow), :216-290 (Mixture) and :337-363
(DiagNormal).  Densities and inverse passes run in the H100 engine; torch provides the
random numbers (``torch.randn`` on the device) and owns all memory.
"""

from __future__ import annotations

__all__ = ["BoxUniform", "DiagNormal", "Mixture", "NormalizingFlow"]

from textwrap import indent

import ctypes
from math import prod

import torch
from torch import Size, Tensor
from torch.distributions import Distribution, Independent, MultivariateNormal, Normal, Transform, constraints

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


class _GMMCall:
    """The components of ``GMM(c)``: the model and its context (``None`` when unconditional).  The
    base a :class:`Mixture` is built over."""

    def __init__(self, gmm, c: Tensor | None) -> None:  # noqa: ANN001
        self.gmm, self.c = gmm, c
        self.batch_shape = Size(()) if c is None else c.shape[:-1]

    def phi(self) -> tuple[Tensor, ...]:
        """The parameter tensors with the reference's shapes, detached (inspection only)."""
        from .utils import unpack

        gmm = self.gmm
        if self.c is None:
            return tuple(p.detach() for p in gmm.phi)
        with torch.no_grad():
            return unpack(gmm.hyper(self.c), gmm.shapes)


class Mixture(Distribution):
    r"""Mixture of Gaussian components (zuko/distributions.py:216-290), built by :class:`zuko_b200.mixtures.GMM`.

    .. math:: p(X = x) = \frac{1}{\sum_i w_i} \sum_i w_i \, p(Z_i = x)

    ``log_prob`` is one engine call (``zk_gmm_log_prob``) behind an autograd function whose backward is
    one ``zk_gmm_backward`` call: gradients reach ``x``, the context (reduced to its own shape) and every
    parameter of the model.  ``sample(shape)`` draws ``u = torch.rand(n)`` then ``z = torch.randn(n, D)``
    on the device and makes one ``zk_gmm_sample`` call.  As in the reference there is no ``rsample``.

    ``logits`` and ``base`` (a ``MultivariateNormal``, or an ``Independent(Normal)`` for diagonal and
    spherical covariances) are materialised on access, detached, with the reference's shapes: they are
    for inspection and carry no gradient.  Only the components of a ``GMM`` are accepted as base.
    """

    has_rsample = False
    arg_constraints = {}

    def __init__(self, base: _GMMCall, logits: Tensor | None = None) -> None:
        if not isinstance(base, _GMMCall) or logits is not None:
            raise NotImplementedError("zuko_b200: Mixture is implemented for the components of zuko_b200.mixtures.GMM only")
        self._call = base
        self._batch = base.batch_shape
        super().__init__(validate_args=False)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.base})"

    @property
    def batch_shape(self) -> Size:
        return self._batch

    @property
    def event_shape(self) -> Size:
        return Size((self._call.gmm.features,))

    @property
    def support(self) -> constraints.Constraint:
        return constraints.real_vector

    def expand(self, batch_shape: Size, new: Distribution | None = None) -> Distribution:
        new = self._get_checked_instance(Mixture, new)
        new._call = self._call
        new._batch = Size(batch_shape)
        Distribution.__init__(new, validate_args=False)
        return new

    @property
    def logits(self) -> Tensor:
        logits = self._call.phi()[0]
        return logits.expand(*self._batch, logits.shape[-1])

    @property
    def base(self) -> Distribution:
        gmm = self._call.gmm
        phi = self._call.phi()
        K, D = gmm.components, gmm.features
        loc = phi[1].expand(*self._batch, K, D)
        scale = phi[2].exp() + gmm.epsilon
        if gmm.covariance_type == "full":
            tril = torch.diag_embed(scale)
            mask = torch.tril(torch.ones_like(tril, dtype=bool), diagonal=-1)
            tril = torch.masked_scatter(tril, mask, phi[3])
            return MultivariateNormal(loc=loc, scale_tril=tril.expand(*self._batch, K, D, D))
        return Independent(Normal(loc, scale.expand(*self._batch, K, D)), 1)

    def _rows(self, lead: Size) -> tuple[Tensor | None, int]:
        """The context as engine rows for the batch ``lead``: (c (n, C), ldc), one broadcast row (ldc = 0)
        for a context without batch dimensions, ``(None, 0)`` when unconditional."""
        c = self._call.c
        if c is None:
            return None, 0
        E.require_cuda(c, "context")
        if c.dim() == 1:
            return c.contiguous(), 0
        C = c.shape[-1]
        return c.expand(*lead, C).reshape(-1, C).contiguous(), C

    def log_prob(self, x: Tensor) -> Tensor:
        E.require_cuda(x, "input")
        gmm = self._call.gmm
        D = gmm.features
        lead = torch.broadcast_shapes(x.shape[:-1], self._batch)
        x2 = x.expand(*lead, D).reshape(-1, D).contiguous()
        c2, ldc = self._rows(lead)
        return _MixtureLogProb.apply(gmm, ldc, x2, c2, *gmm.params()).reshape(lead)

    def sample(self, shape: Size = ()) -> Tensor:
        gmm = self._call.gmm
        D = gmm.features
        lead = Size(shape) + self._batch
        params = gmm.params()
        device = params[0].device
        n = prod(lead)
        with torch.no_grad():
            u = torch.rand(n, device=device)
            z = torch.randn(n, D, device=device)
            c2, ldc = self._rows(lead)
            x = torch.empty(n, D, device=device)
            with torch.cuda.device(device):
                h = gmm.handle(params)
                table = _table(gmm, params)
                need = E.lib().zk_gmm_workspace_bytes(h, n)
                ws = E.Workspace.get(device, need, E.lib().zk_gmm_min_workspace_bytes(h))
                E.check(E.lib().zk_gmm_sample(h, _ptr(c2), ldc, _ptr(table), u.data_ptr(), z.data_ptr(), D, n,
                                              x.data_ptr(), D, ws.data_ptr(), ws.numel(), E.stream_ptr(device)))  # fmt: skip
        return x.reshape(*lead, D)


def _ptr(t: Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def _table(gmm, params) -> Tensor | None:  # noqa: ANN001
    """The unconditional parameter row (``phi`` flattened in unpack order); ``None`` for a conditional model."""
    if hasattr(gmm, "hyper"):
        return None
    return torch.cat([p.detach().reshape(-1) for p in params]).contiguous()


class _MixtureLogProb(torch.autograd.Function):
    """``Mixture.log_prob`` on engine rows: forward = ``zk_gmm_log_prob``, backward = ``zk_gmm_backward``
    (gradients of x, of the context rows and of every tensor of ``GMM.params()``)."""

    @staticmethod
    def forward(ctx, gmm, ldc, x2, c2, *params):  # noqa: ANN001
        E.require_cuda(x2, "input")
        B, D = x2.shape
        device = x2.device
        out = torch.empty(B, device=device, dtype=torch.float32)
        with torch.cuda.device(device):
            h = gmm.handle(params)
            table = _table(gmm, params)
            need = E.lib().zk_gmm_workspace_bytes(h, B)
            ws = E.Workspace.get(device, need, E.lib().zk_gmm_min_workspace_bytes(h))
            E.check(E.lib().zk_gmm_log_prob(h, x2.data_ptr(), D, _ptr(c2), ldc, _ptr(table), B, out.data_ptr(),
                                            ws.data_ptr(), ws.numel(), E.stream_ptr(device)))  # fmt: skip
        ctx.gmm, ctx.ldc, ctx.has_c = gmm, ldc, c2 is not None
        ctx.save_for_backward(x2, *(() if c2 is None else (c2,)), *params)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):  # noqa: ANN001
        gmm, ldc = ctx.gmm, ctx.ldc
        saved = ctx.saved_tensors
        x2, c2 = saved[0], (saved[1] if ctx.has_c else None)
        params = saved[2 if ctx.has_c else 1 :]
        need = ctx.needs_input_grad
        B, D = x2.shape
        device = x2.device
        g = g.contiguous()
        gx = torch.empty_like(x2) if need[2] else None
        gc = torch.zeros_like(c2) if c2 is not None and need[3] else None
        grads = [torch.zeros_like(p) for p in params]
        keep = []
        if hasattr(gmm, "hyper"):
            weights, biases = gmm._split(grads)
            W = (ctypes.c_void_p * len(weights))(*[w.data_ptr() for w in weights])
            Bv = (ctypes.c_void_p * len(biases))(*[None if b is None else b.data_ptr() for b in biases])
            keep += [W, Bv]
            layer_grads = E.LayerGrads(ctypes.cast(W, ctypes.POINTER(ctypes.c_void_p)), ctypes.cast(Bv, ctypes.POINTER(ctypes.c_void_p)), None, None)  # noqa: E501
            flat = None
        else:
            flat = torch.zeros(gmm.total, device=device)
            layer_grads = E.LayerGrads(None, None, flat.data_ptr(), None)
        with torch.cuda.device(device):
            h = gmm.handle(params)
            table = _table(gmm, params)
            want = E.lib().zk_gmm_backward_workspace_bytes(h, B)
            ws = E.Workspace.get(device, want, E.lib().zk_gmm_min_workspace_bytes(h))
            E.check(E.lib().zk_gmm_backward(h, x2.data_ptr(), D, _ptr(c2), ldc, _ptr(table), B, g.data_ptr(), _ptr(gx), D,
                                            _ptr(gc), 0 if c2 is None else c2.shape[-1], ctypes.byref(layer_grads),
                                            ws.data_ptr(), ws.numel(), E.stream_ptr(device)))  # fmt: skip
        if flat is not None:
            grads = [part.reshape(p.shape) for part, p in zip(flat.split([p.numel() for p in params]), params, strict=True)]
        return (None, None, gx, gc, *[gr if n else None for gr, n in zip(grads, need[4:], strict=True)])
