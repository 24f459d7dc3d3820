"""Polynomial flows (zuko/flows/polynomial.py): the sum-of-squares polynomial flow and the Bernstein
polynomial flow."""

from __future__ import annotations

__all__ = ["BPF", "SOSPF", "ShiftedSOSPTransform"]

from functools import partial

from ..lazy import UnconditionalTransform
from ..transforms import BoundedBernsteinTransform, ShiftedSOSPTransform, SoftclipTransform
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


class BPF(MAF):
    """Bernstein polynomial flow: a :class:`MAF` whose univariate bijector is ``BoundedBernsteinTransform``
    (bound 5) with ``degree + 1`` unconstrained parameters per feature.  Same arguments, module tree,
    state-dict keys and seeded initialisation as the reference.

    The polynomial acts on ``[-5, 5]``; beyond it the map is linear with slope 1 (``x -+ 1e-5``), so
    standardise the features first, as the reference recommends.  Degree 16 inverts with the
    dimension-sequential kernel, other degrees with the ``passes`` sweeps."""

    def __init__(
        self,
        features: int,
        context: int = 0,
        degree: int = 16,
        **kwargs,
    ) -> None:
        super().__init__(
            features=features,
            context=context,
            univariate=BoundedBernsteinTransform,
            shapes=[(degree + 1,)],
            **kwargs,
        )
