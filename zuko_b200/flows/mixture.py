"""Alias of :mod:`zuko_b200.mixtures` under ``flows``, as the reference keeps it (zuko/flows/mixture.py)."""

__all__ = ["GMM"]

from ..mixtures import GMM
