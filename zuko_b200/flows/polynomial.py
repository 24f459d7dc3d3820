"""Polynomial flows (zuko/flows/polynomial.py): the sum-of-squares polynomial flow."""

from __future__ import annotations

__all__ = ["SOSPF", "ShiftedSOSPTransform"]

from functools import partial

from ..lazy import UnconditionalTransform
from ..transforms import ShiftedSOSPTransform, SoftclipTransform
from .autoregressive import MAF


class SOSPF(MAF):
    """Sum-of-squares polynomial flow: a :class:`MAF` whose univariate bijector is ``ShiftedSOSPTransform``
    with ``polynomials`` polynomials of degree ``degree`` (P = polynomials (degree + 1) + 1 parameters per
    feature), with a ``SoftclipTransform(bound=11)`` between consecutive autoregressive layers.  Same arguments,
    module tree, state-dict keys and seeded initialisation as the reference.

    The inverse is a bisection on ``[-10, 10]``: features beyond that interval are not recovered
    (standardise them first, as the reference recommends)."""

    def __init__(
        self,
        features: int,
        context: int = 0,
        degree: int = 4,
        polynomials: int = 3,
        slope: float = 1e-3,
        **kwargs,
    ) -> None:
        super().__init__(
            features=features,
            context=context,
            univariate=partial(ShiftedSOSPTransform, slope=slope),
            shapes=[(polynomials, degree + 1), ()],
            **kwargs,
        )

        transforms = self.transform.transforms

        for i in reversed(range(1, len(transforms))):
            transforms.insert(i, UnconditionalTransform(SoftclipTransform, bound=11.0))
