"""Lazy distributions and transformations — the drop-in boundary.

Host-side mirror of zuko/lazy.py: a lazy module builds the distribution
``p(X | c)`` / transformation ``y = f(x | c)`` inside ``forward(c)`` so that it can be
conditional and own parameters.  ``Flow.forward(c)`` (zuko/lazy.py:156-172) is the seam
the H100 engine plugs in at: it returns a ``NormalizingFlow`` whose ``log_prob`` /
``rsample`` are engine calls.
"""

from __future__ import annotations

__all__ = [
    "Flow",
    "LazyComposedTransform",
    "LazyDistribution",
    "LazyInverse",
    "LazyTransform",
    "UnconditionalDistribution",
    "UnconditionalTransform",
]

import abc
from collections.abc import Callable, Sequence

import torch
import torch.nn as nn
from torch import Tensor
from torch.distributions import Distribution, Transform

from . import _engine as E
from .distributions import NormalizingFlow
from .transforms import ComposedTransform
from .utils import Partial


class LazyDistribution(nn.Module, abc.ABC):
    """A module whose ``forward(c)`` returns a distribution ``p(X | c)`` (zuko/lazy.py:29-49)."""

    @abc.abstractmethod
    def forward(self, c: Tensor | None = None) -> Distribution: ...


class LazyTransform(nn.Module, abc.ABC):
    """A module whose ``forward(c)`` returns a transformation ``y = f(x | c)``
    (zuko/lazy.py:52-78)."""

    @abc.abstractmethod
    def forward(self, c: Tensor | None = None) -> Transform: ...

    @property
    def inv(self) -> LazyTransform:
        return LazyInverse(self)


class LazyInverse(LazyTransform):
    """Lazy inverse ``x = f^{-1}(y | c)`` of a lazy transformation (zuko/lazy.py:81-98)."""

    def __init__(self, transform: LazyTransform) -> None:
        super().__init__()
        self.transform = transform

    def forward(self, c: Tensor | None = None) -> Transform:
        return self.transform(c).inv

    @property
    def inv(self) -> LazyTransform:
        return self.transform


class LazyComposedTransform(LazyTransform):
    """Lazy composition ``f_n ∘ ... ∘ f_0`` (zuko/lazy.py:101-128)."""

    def __init__(self, *transforms: LazyTransform) -> None:
        super().__init__()
        self.transforms = nn.ModuleList(transforms)

    def __repr__(self) -> str:
        return repr(self.transforms).replace("ModuleList", "LazyComposedTransform", 1)

    def forward(self, c: Tensor | None = None) -> Transform:
        return ComposedTransform(*(t(c) for t in self.transforms))


class Flow(LazyDistribution):
    """Lazy normalizing flow: ``flow(c)`` is ``NormalizingFlow(transform(c), base(c))``,
    with the base expanded to the batch shape of ``c`` (zuko/lazy.py:131-172)."""

    def __init__(self, transform: LazyTransform | Sequence[LazyTransform], base: LazyDistribution) -> None:
        super().__init__()
        if isinstance(transform, LazyTransform):
            self.transform = transform
        else:
            self.transform = LazyComposedTransform(*transform)
        self.base = base

    def forward(self, c: Tensor | None = None) -> NormalizingFlow:
        transform = self.transform(c)
        base = self.base(c)
        if c is not None:
            base = base.expand(c.shape[:-1])
        return NormalizingFlow(transform, base)


class _Unconditional(Partial):
    """Caches the built object while the registered tensors are unchanged, so that packed
    engine handles created from it survive across ``forward`` calls."""

    def _tensor_signature(self) -> tuple:
        sig = []
        for v in list(self.args) + list(self.kwargs.values()):
            sig.append((v.data_ptr(), v._version, v.device, v.dtype) if torch.is_tensor(v) else v)
        return tuple(sig)

    def _build(self):
        if torch.is_grad_enabled() and any(
            torch.is_tensor(v) and v.requires_grad for v in list(self.args) + list(self.kwargs.values())
        ):
            # the object may hold tensors computed from the arguments (e.g. R = exp(A - A^T)): its
            # autograd graph belongs to this forward call, so it is not cached
            return Partial.forward(self)
        sig = self._tensor_signature()
        cached = self.__dict__.get("_built")
        if cached is not None and cached[0] == sig:
            return cached[1]
        obj = Partial.forward(self)
        self.__dict__["_built"] = (sig, obj, E.hold_storage(list(self.args) + list(self.kwargs.values())))
        return obj

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_built", None)
        return state

    def extra_repr(self) -> str:
        return "" if isinstance(self.f, nn.Module) else repr(Partial.forward(self))


class UnconditionalDistribution(_Unconditional, LazyDistribution):
    """Unconditional lazy distribution built from a constructor whose tensor arguments are
    registered as buffers / parameters (zuko/lazy.py:242-287).  The context is ignored."""

    def __init__(self, f: Callable[..., Distribution], *args, buffer: bool = False, **kwargs) -> None:
        super().__init__(f, *args, buffer=buffer, **kwargs)

    def forward(self, c: Tensor | None = None) -> Distribution:
        return self._build()


class UnconditionalTransform(_Unconditional, LazyTransform):
    """Unconditional lazy transformation built from a constructor (zuko/lazy.py:290-335).
    The context is ignored."""

    def __init__(self, f: Callable[..., Transform], *args, buffer: bool = False, **kwargs) -> None:
        super().__init__(f, *args, buffer=buffer, **kwargs)

    def forward(self, c: Tensor | None = None) -> Transform:
        return self._build()
