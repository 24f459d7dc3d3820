"""Flow zoo of the hot path (zuko/flows/__init__.py, restricted to SURVEY §8)."""

from .autoregressive import MAF, MaskedAutoregressiveTransform
from .continuous import CNF, FFJTransform
from .coupling import NICE, GeneralCouplingTransform, RealNVP
from .elementwise import ElementWiseTransform
from .gaussianization import GF
from .polynomial import BPF, SOSPF
from .spline import NCSF, NSF
from ..lazy import Flow, UnconditionalDistribution, UnconditionalTransform

__all__ = [
    "GF",
    "MAF",
    "NCSF",
    "NICE",
    "NSF",
    "BPF",
    "CNF",
    "SOSPF",
    "ElementWiseTransform",
    "FFJTransform",
    "Flow",
    "GeneralCouplingTransform",
    "MaskedAutoregressiveTransform",
    "RealNVP",
    "UnconditionalDistribution",
    "UnconditionalTransform",
]
