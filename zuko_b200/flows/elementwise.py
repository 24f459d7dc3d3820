"""Element-wise lazy transformation (zuko/flows/gaussianization.py:28-94)."""

from __future__ import annotations

__all__ = ["ElementWiseTransform"]

import ctypes
from collections.abc import Callable, Sequence

import torch
import torch.nn as nn
from torch import Size, Tensor
from torch.distributions import Transform

from .. import _engine as E
from ..lazy import LazyTransform
from ..nn import MLP
from ..transforms import DependentTransform, MonotonicAffineTransform
from ._packed import PackedLayerMixin, refuse_autoregressive_only, resolve_univariate, total_of


class ElementWiseTransform(PackedLayerMixin, LazyTransform):
    """Applies an independent univariate bijector to every feature.  Without context the
    per-feature parameters are learnable tensors (one shared ``(D, P)`` table staged once
    per CTA by the engine); with context they come from a dense ``MLP(c)``."""

    def __init__(
        self,
        features: int,
        context: int = 0,
        univariate: Callable[..., Transform] = MonotonicAffineTransform,
        shapes: Sequence[Size] = ((), ()),
        **kwargs,
    ) -> None:
        super().__init__()
        self.univariate, self.shapes = univariate, shapes
        self.total = total_of(shapes)
        self._uni = resolve_univariate(univariate, shapes)
        refuse_autoregressive_only(self._uni, "ElementWiseTransform")
        self.features, self.context = features, context
        if context > 0:
            self.hyper = MLP(context, features * self.total, **kwargs)
        else:
            self.phi = nn.ParameterList(torch.randn(features, *s) for s in shapes)

    def extra_repr(self) -> str:
        return f"(base): {self._describe_base()}"

    def _layer_desc(self):
        desc = self._base_desc(E.ZK_LAYER_ELEMENTWISE)
        if self.context > 0:
            hyper, keep = self.hyper.mlp_desc()
            desc.hyper = ctypes.pointer(hyper)
            return desc, [hyper, keep]
        table = torch.cat([p.detach().reshape(self.features, -1) for p in self.phi], dim=-1).contiguous()
        E.require_cuda(table, "element-wise parameters")
        desc.phi = table.data_ptr()
        return desc, [table]

    def forward(self, c: Tensor | None = None) -> Transform:
        return DependentTransform(self, c)
