"""Gaussianization flow (zuko/flows/gaussianization.py:97-155)."""

from __future__ import annotations

__all__ = ["GF"]

import torch

from ..distributions import DiagNormal
from ..lazy import Flow, UnconditionalDistribution, UnconditionalTransform
from ..transforms import GaussianizationTransform, RotationTransform
from .elementwise import ElementWiseTransform


class GF(Flow):
    """Gaussianization flow: ``transforms`` element-wise layers of the Gaussianization bijector with
    ``components`` mixture components, separated by trainable rotations, over a standard
    ``DiagNormal`` base.  Same arguments, state-dict keys and seeded initialisation as the reference.

    The inverse is a bisection on ``[-10, 10]``: features beyond that interval are not recovered
    (standardise them first, as the reference recommends)."""

    def __init__(self, features: int, context: int = 0, transforms: int = 3, components: int = 8, **kwargs) -> None:
        layers = [
            ElementWiseTransform(
                features=features,
                context=context,
                univariate=GaussianizationTransform,
                shapes=[(components,), (components,)],
                **kwargs,
            )
            for _ in range(transforms)
        ]
        # the rotation generators are drawn after every element-wise layer, last one first
        for i in reversed(range(1, len(layers))):
            layers.insert(i, UnconditionalTransform(RotationTransform, A=torch.randn(features, features)))
        base = UnconditionalDistribution(
            DiagNormal,
            loc=torch.zeros(features),
            scale=torch.ones(features),
            buffer=True,
        )
        super().__init__(layers, base)
