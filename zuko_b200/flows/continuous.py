"""Continuous flows (zuko/flows/continuous.py): the free-form Jacobian transformation and the continuous
normalizing flow."""

from __future__ import annotations

__all__ = ["CNF", "FFJTransform"]

import ctypes
from math import pi

import torch
import torch.nn as nn
from torch import Size, Tensor
from torch.distributions import Transform

from .. import _engine as E
from ..distributions import DiagNormal
from ..lazy import Flow, LazyTransform, UnconditionalDistribution
from ..nn import MLP
from ..transforms import FreeFormJacobianTransform


class _VectorField:
    """``FFJTransform.f`` with its context bound (flows/continuous.py:88-97): what
    ``FreeFormJacobianTransform`` hands to the engine."""

    def __init__(self, owner: FFJTransform, c: Tensor | None) -> None:
        self.owner, self.c = owner, c

    def cnf_handle(self) -> ctypes.c_void_p:
        return self.owner._cnf_handle()

    def context(self, lead: Size, B: int) -> tuple[Tensor | None, int]:
        """(c as B rows or one broadcast row, its row stride)."""
        c = self.c
        if c is None or c.shape[-1] == 0:
            return None, 0
        E.require_cuda(c, "CNF context")
        if c.dim() == 1 or c.shape[:-1].numel() == 1:
            return c.reshape(1, -1).contiguous(), 0
        c2 = c.expand(*lead, c.shape[-1]).reshape(B, c.shape[-1])  # -1 is ambiguous when B = 0
        if c2.stride(-1) != 1:
            c2 = c2.contiguous()
        return c2, c2.stride(0)


class FFJTransform(LazyTransform):
    """Lazy free-form Jacobian (FFJ) transformation (FFJORD, Grathwohl et al., 2018): the vector field
    ``ode(cat(cos(freqs t), sin(freqs t), x, c))`` of an :class:`zuko_b200.nn.MLP` (ELU by default) integrated
    from ``times[0]`` to ``times[1]``.  Same arguments, module tree (``ode``), buffers (``times``, ``freqs``),
    state-dict keys and seeded initialisation as the reference.  ``normalize=True`` and activations outside the
    engine raise ``NotImplementedError``.  ``adjoint=True`` (an engine extension, also settable afterwards) lets
    the transforms it builds carry gradients through the integration: see :class:`FreeFormJacobianTransform`."""

    def __init__(
        self,
        features: int,
        context: int = 0,
        freqs: int = 3,
        atol: float = 1e-6,
        rtol: float = 1e-5,
        exact: bool = True,
        adjoint: bool = False,
        **kwargs,
    ) -> None:
        super().__init__()

        kwargs.setdefault("activation", nn.ELU)

        self.ode = MLP(features + context + 2 * freqs, features, **kwargs)

        self.register_buffer("times", torch.tensor((0.0, 1.0)))
        self.register_buffer("freqs", torch.arange(1, freqs + 1) * pi)

        self.atol = atol
        self.rtol = rtol
        self.exact = exact
        self.adjoint = adjoint

    def _cnf_handle(self) -> ctypes.c_void_p:
        """The ``zk_cnf`` handle of the current weights, re-packed when a parameter or ``freqs`` changes."""
        fr = self.freqs
        sig = (self.ode._signature(), fr.data_ptr(), fr._version, fr.device)
        cached = self.__dict__.get("_zk_cnf")
        if cached is not None and cached[0] == sig:
            return cached[1]
        self._release()
        E.require_cuda(fr, "CNF freqs")
        desc, keep = self.ode.mlp_desc()
        D = self.ode.out_features
        F = fr.numel()
        freqs = fr.detach().contiguous()
        h = ctypes.c_void_p()
        E.check(E.lib().zk_cnf_create(ctypes.byref(desc), D, self.ode.in_features - D - 2 * F, F,
                                      freqs.data_ptr() if F else None, ctypes.byref(h)))  # fmt: skip
        del keep
        self.__dict__["_zk_cnf"] = (sig, h, self.ode._held_storage() + E.hold_storage([fr]))
        return h

    def _release(self) -> None:
        cached = self.__dict__.pop("_zk_cnf", None)
        if cached is not None:
            E.lib().zk_cnf_destroy(cached[1])

    def __del__(self) -> None:
        try:
            self._release()
        except Exception:
            pass

    def __getstate__(self):  # handles are not picklable
        state = self.__dict__.copy()
        state.pop("_zk_cnf", None)
        return state

    def forward(self, c: Tensor | None = None) -> Transform:
        if self.training:
            phi = self.parameters() if c is None else (c, *self.parameters())
        else:
            phi = () if c is None else (c,)

        return FreeFormJacobianTransform(
            f=_VectorField(self, c),
            t0=self.times[0],
            t1=self.times[1],
            phi=phi,
            atol=self.atol,
            rtol=self.rtol,
            exact=self.exact,
            adjoint=self.adjoint,
        )


class CNF(Flow):
    """Continuous normalizing flow (Chen et al., 2018; Grathwohl et al., 2018): one :class:`FFJTransform` on a
    standard ``DiagNormal`` base.  ``kwargs`` go to :class:`FFJTransform`."""

    def __init__(
        self,
        features: int,
        context: int = 0,
        **kwargs,
    ) -> None:
        transform = FFJTransform(
            features=features,
            context=context,
            **kwargs,
        )

        base = UnconditionalDistribution(
            DiagNormal,
            loc=torch.zeros(features),
            scale=torch.ones(features),
            buffer=True,
        )

        super().__init__(transform, base)
