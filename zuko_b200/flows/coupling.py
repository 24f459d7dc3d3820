"""Coupling transformations and flows (zuko/flows/coupling.py)."""

from __future__ import annotations

__all__ = ["NICE", "GeneralCouplingTransform", "RealNVP"]

import ctypes
from collections.abc import Callable, Sequence

import torch
from torch import BoolTensor, Size, Tensor
from torch.distributions import Transform

from .. import _engine as E
from ..distributions import DiagNormal
from ..lazy import Flow, LazyTransform, UnconditionalDistribution
from ..nn import MLP
from ..transforms import CouplingTransform, MonotonicAffineTransform
from ._packed import PackedLayerMixin, refuse_autoregressive_only, refuse_elementwise_only, resolve_univariate, total_of
from .elementwise import ElementWiseTransform


class GeneralCouplingTransform(PackedLayerMixin, LazyTransform):
    """Lazy coupling transformation ``y_a = x_a``, ``y_b = f(x_b | x_a, c)``
    (zuko/flows/coupling.py:25-139).  ``mask`` marks the constant split ``x_a``; the
    default is the checkered mask ``arange(features) % 2 == 1``.  The conditioner is a
    dense :class:`zuko_b200.nn.MLP` on ``cat(x_a, c)``."""

    def __new__(cls, features: int | None = None, context: int = 0, mask: BoolTensor | None = None, *args, **kwargs) -> LazyTransform:  # fmt: skip
        if features is None or features > 1:
            return super().__new__(cls)
        return ElementWiseTransform(features, context, *args, **kwargs)

    def __init__(
        self,
        features: int,
        context: int = 0,
        mask: BoolTensor | None = None,
        univariate: Callable[..., Transform] = MonotonicAffineTransform,
        shapes: Sequence[Size] = ((), ()),
        **kwargs,
    ) -> None:
        super().__init__()
        self.univariate, self.shapes = univariate, shapes
        self.total = total_of(shapes)
        self._uni = resolve_univariate(univariate, shapes)
        refuse_elementwise_only(self._uni, "GeneralCouplingTransform")
        refuse_autoregressive_only(self._uni, "GeneralCouplingTransform")
        self.features, self.context = features, context
        mask = torch.arange(features) % 2 == 1 if mask is None else torch.as_tensor(mask, dtype=bool)
        assert mask.ndim == 1, "'mask' should be a vector."
        assert mask.shape[0] == features, f"'mask' should have {features} elements."
        n_const = int(mask.sum())
        assert 0 < n_const < features
        self.register_buffer("mask", mask)
        self.hyper = MLP(n_const + context, (features - n_const) * self.total, **kwargs)

    def extra_repr(self) -> str:
        mask = self.mask.int().tolist()
        if len(mask) > 10:
            mask = str(mask[:5] + [...] + mask[-5:]).replace("Ellipsis", "...")
        return f"(base): {self._describe_base()}\n(mask): {mask}"

    def _layer_tensors(self) -> list:
        return super()._layer_tensors() + [self.mask]

    def _layer_desc(self):
        hyper, keep = self.hyper.mlp_desc()
        desc = self._base_desc(E.ZK_LAYER_COUPLING)
        desc.hyper = ctypes.pointer(hyper)
        host = self.mask.detach().to("cpu", torch.uint8).tolist()
        arr = (ctypes.c_uint8 * self.features)(*host)
        desc.coupling_mask = arr
        return desc, [hyper, keep, arr]

    def forward(self, c: Tensor | None = None) -> Transform:
        return CouplingTransform(self, c)


class NICE(Flow):
    """NICE / RealNVP flow (zuko/flows/coupling.py:142-196): ``transforms`` coupling layers
    with alternating checkered masks (random with ``randmask=True``), affine by default."""

    def __init__(self, features: int, context: int = 0, transforms: int = 3, randmask: bool = False, **kwargs) -> None:
        layers = []
        for i in range(transforms):
            positions = torch.randperm(features) if randmask else torch.arange(features)
            layers.append(GeneralCouplingTransform(features=features, context=context, mask=positions % 2 == i % 2, **kwargs))
        base = UnconditionalDistribution(DiagNormal, loc=torch.zeros(features), scale=torch.ones(features), buffer=True)
        super().__init__(layers, base)


class RealNVP(NICE):
    pass
