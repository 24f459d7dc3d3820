"""Shared plumbing of the lazy layers: resolving the ``univariate`` / ``shapes`` hooks to an
engine bijector and packing the layer into a ``zk_layer`` handle."""

from __future__ import annotations

import ctypes
from collections.abc import Callable, Sequence
from functools import partial
from math import prod

import torch
from torch import Size

from .. import _engine as E
import math

from ..transforms import (
    BoundedBernsteinTransform,
    CircularRQSTransform,
    GaussianizationTransform,
    MonotonicAffineTransform,
    MonotonicRQSTransform,
    ShiftedSOSPTransform,
    bisection_steps,
)


def resolve_univariate(univariate: Callable, shapes: Sequence[Size]) -> dict:
    """Maps the reference's ``univariate=`` / ``shapes=`` constructor hooks
    (zuko/flows/autoregressive.py:95-104, flows/coupling.py:84-93,
    flows/gaussianization.py:64-72) onto an engine bijector."""
    kwargs = {}
    f = univariate
    while isinstance(f, partial):
        if f.args:
            raise NotImplementedError("zuko_b200: positional arguments bound to `univariate` are not supported")
        kwargs = {**f.keywords, **kwargs}
        f = f.func
    shapes = [tuple(s) for s in shapes]
    if f is MonotonicAffineTransform:
        if shapes != [(), ()]:
            raise ValueError(f"MonotonicAffineTransform expects shapes [(), ()], got {shapes}")
        extra = set(kwargs) - {"slope"}
        if extra:
            raise NotImplementedError(f"zuko_b200: unsupported MonotonicAffineTransform arguments {sorted(extra)}")
        return dict(kind=E.ZK_UNI_AFFINE, bins=0, bound=5.0, slope=float(kwargs.get("slope", 1e-3)), total=2)
    if f is MonotonicRQSTransform:
        if len(shapes) != 3 or shapes[0] != shapes[1] or len(shapes[0]) != 1 or shapes[2] != (shapes[0][0] - 1,):
            raise ValueError(f"MonotonicRQSTransform expects shapes [(K,), (K,), (K-1,)], got {shapes}")
        extra = set(kwargs) - {"slope", "bound"}
        if extra:
            raise NotImplementedError(f"zuko_b200: unsupported MonotonicRQSTransform arguments {sorted(extra)}")
        K = shapes[0][0]
        return dict(kind=E.ZK_UNI_RQS, bins=K, bound=float(kwargs.get("bound", 5.0)),
                    slope=float(kwargs.get("slope", 1e-3)), total=3 * K - 1)  # fmt: skip
    if f is CircularRQSTransform:  # flows/spline.py:65-72: CircularShift(pi) then RQS(bound=pi)
        if len(shapes) != 3 or shapes[0] != shapes[1] or len(shapes[0]) != 1 or shapes[2] != (shapes[0][0] - 1,):
            raise ValueError(f"CircularRQSTransform expects shapes [(K,), (K,), (K-1,)], got {shapes}")
        extra = set(kwargs) - {"slope"}
        if extra:
            raise NotImplementedError(f"zuko_b200: unsupported CircularRQSTransform arguments {sorted(extra)}")
        K = shapes[0][0]
        return dict(kind=E.ZK_UNI_CRQS, bins=K, bound=math.pi, slope=float(kwargs.get("slope", 1e-3)), total=3 * K - 1)
    if f is GaussianizationTransform:
        if len(shapes) != 2 or shapes[0] != shapes[1] or len(shapes[0]) != 1:
            raise ValueError(f"GaussianizationTransform expects shapes [(K,), (K,)], got {shapes}")
        extra = set(kwargs) - {"bound", "eps"}
        if extra:
            raise NotImplementedError(f"zuko_b200: unsupported GaussianizationTransform arguments {sorted(extra)}")
        K = shapes[0][0]
        bound, eps = float(kwargs.get("bound", 10.0)), float(kwargs.get("eps", 1e-6))
        return dict(kind=E.ZK_UNI_GAUSS, bins=K, bound=bound, slope=1e-3, total=2 * K, iterations=bisection_steps(bound, eps))
    if f is ShiftedSOSPTransform:  # flows/polynomial.py:23-28, 66-72: SOSPolynomialTransform's bound / eps defaults
        if len(shapes) != 2 or len(shapes[0]) != 2 or shapes[1] != ():
            raise ValueError(f"ShiftedSOSPTransform expects shapes [(K, L+1), ()], got {shapes}")
        extra = set(kwargs) - {"slope"}
        if extra:
            raise NotImplementedError(f"zuko_b200: unsupported ShiftedSOSPTransform arguments {sorted(extra)}")
        K, n = shapes[0]
        if K < 1 or not 1 <= n <= 16 or K * n + 1 > 1024:
            raise NotImplementedError(f"zuko_b200: ShiftedSOSPTransform with {K} polynomials of degree {n - 1} "
                                      "(the engine takes degree <= 15 and K (degree + 1) + 1 <= 1024)")  # fmt: skip
        return dict(kind=E.ZK_UNI_SOSP, bins=K, degree=n - 1, bound=10.0, slope=float(kwargs.get("slope", 1e-3)),
                    total=K * n + 1, iterations=bisection_steps(10.0, 1e-6))  # fmt: skip
    if f is BoundedBernsteinTransform:  # flows/polynomial.py:79-117: shapes [(degree + 1,)]
        if len(shapes) != 1 or len(shapes[0]) != 1 or shapes[0][0] < 1:
            raise ValueError(f"BoundedBernsteinTransform expects shapes [(degree + 1,)], got {shapes}")
        extra = set(kwargs) - {"bound", "eps"}
        if extra:
            raise NotImplementedError(f"zuko_b200: unsupported BoundedBernsteinTransform arguments {sorted(extra)}")
        degree = shapes[0][0] - 1
        bound, eps = float(kwargs.get("bound", 5.0)), float(kwargs.get("eps", 1e-6))
        if eps != 1e-6:
            raise NotImplementedError(f"zuko_b200: BoundedBernsteinTransform in a flow layer takes eps = 1e-6 only, got {eps}")
        if degree > 59:
            raise NotImplementedError(f"zuko_b200: BoundedBernsteinTransform of degree {degree} (the engine takes degree <= 59)")
        if not bound > 0:
            raise ValueError(f"BoundedBernsteinTransform expects a positive bound, got {bound}")
        return dict(kind=E.ZK_UNI_BERNSTEIN, bins=0, degree=degree, bound=bound, slope=1e-3, total=degree + 1,
                    iterations=bisection_steps(bound, eps))  # fmt: skip
    if getattr(f, "__name__", None) == "BernsteinTransform":
        raise NotImplementedError("zuko_b200: the unbounded BernsteinTransform is not implemented by the engine "
                                  "(BPF uses BoundedBernsteinTransform)")  # fmt: skip
    raise NotImplementedError(
        f"zuko_b200: univariate transformation {getattr(f, '__name__', f)!r} is not implemented by the engine "
        "(supported: MonotonicAffineTransform, MonotonicRQSTransform, CircularRQSTransform, GaussianizationTransform, "
        "ShiftedSOSPTransform, BoundedBernsteinTransform)"
    )


def refuse_elementwise_only(uni: dict, layer: str) -> None:
    """The Gaussianization bijector's bisection inverse runs per element: the engine takes it in
    element-wise layers only (flows/gaussianization.py:97-155)."""
    if uni["kind"] == E.ZK_UNI_GAUSS:
        raise NotImplementedError(f"zuko_b200: GaussianizationTransform is supported in element-wise layers only, not in {layer}")


def refuse_autoregressive_only(uni: dict, layer: str) -> None:
    """The sum-of-squares polynomial bijector runs in masked autoregressive layers only
    (flows/polynomial.py:31-76)."""
    if uni["kind"] == E.ZK_UNI_SOSP:
        raise NotImplementedError(f"zuko_b200: ShiftedSOSPTransform is supported in autoregressive layers only, not in {layer}")
    if uni["kind"] == E.ZK_UNI_BERNSTEIN:
        raise NotImplementedError(f"zuko_b200: BoundedBernsteinTransform is supported in autoregressive layers only, not in {layer}")


class OwnedLayer:
    """Owns one ``zk_layer`` handle; destroys it when the last reference goes away.  ``generation``
    counts the in-place weight refreshes (``zk_layer_update_weights``): an autograd graph built
    before a refresh and back-propagated after it would differentiate the new weights — the
    engine's seam raises instead, as torch does for tensors modified in place."""

    def __init__(self, handle: ctypes.c_void_p) -> None:
        self.handle = handle
        self.generation = 0

    def __del__(self) -> None:
        try:
            E.lib().zk_layer_destroy(self.handle)
        except Exception:
            pass


class PackedLayerMixin:
    """Gives a lazy layer a cached ``zk_layer`` handle, rebuilt when any tensor it was
    packed from changes (data pointer / version / device; the cache holds the storage it was packed from, so a
    data pointer is never reused by another tensor while cached) — optimizer steps,
    ``load_state_dict``, ``.to()``, Bayesian re-parameterisation (zuko/bayesian.py:161-166)."""

    def _layer_tensors(self) -> list:
        ts = []
        hyper = getattr(self, "hyper", None)
        if hyper is not None:
            ts.append(hyper.gemm_mode)
            ts.append(hyper._activation_code())
            for m in hyper._linears():
                ts += [m.weight, m.bias, getattr(m, "mask", None)]
        for p in getattr(self, "phi", []) or []:
            ts.append(p)
        order = getattr(self, "order", None)
        if torch.is_tensor(order):
            ts.append(order)
        return ts

    def _layer_signature(self) -> tuple:
        return tuple(
            (t.data_ptr(), t._version, t.device, t.dtype) if torch.is_tensor(t) else t for t in self._layer_tensors()
        )

    def _weights_only_change(self, old: tuple, new: tuple) -> bool:
        """True when the two signatures differ only in the ``_version`` of conditioner weights / biases
        (an optimizer step): same storage, device, dtype, masks, options."""
        hyper = getattr(self, "hyper", None)
        if hyper is None or len(old) != len(new):
            return False
        n_lin = len(hyper._linears())
        wb = {2 + 3 * i + j for i in range(n_lin) for j in (0, 1)}  # positions of (weight, bias) in _layer_tensors
        for k, (a, b) in enumerate(zip(old, new)):
            if a == b:
                continue
            if k not in wb or a is None or b is None or (a[0], a[2], a[3]) != (b[0], b[2], b[3]):
                return False
        return True

    def _zk_layer_ref(self) -> OwnedLayer:
        """The packed handle as a reference-counted owner.  A change of anything structural (storage,
        masks, options, device) builds a new handle — calls that outlive it keep the one they were built
        with; an optimizer step (only the weights' versions moved) refreshes the packed copies IN PLACE
        with stream-ordered kernels (``zk_layer_update_weights``: no mask download, no allocation, no
        host synchronisation).

        Writes through ``.data`` (EMA copies, weight clipping) do not bump ``_version`` and are invisible
        here: call :func:`zuko_b200.invalidate` on the module afterwards."""
        sig = self._layer_signature()
        cached = self.__dict__.get("_zk_cache")
        if cached is not None and cached[0] == sig:
            return cached[1]
        dev = next((t.device for t in self._layer_tensors() if torch.is_tensor(t) and t.is_cuda), None)
        if cached is not None and dev is not None and self._weights_only_change(cached[0], sig):
            ref = cached[1]
            lins = self.hyper._linears()
            n = len(lins)
            keep = [m.weight.detach().contiguous() for m in lins]
            keep += [None if m.bias is None else m.bias.detach().contiguous() for m in lins]
            W = (ctypes.c_void_p * n)(*[t.data_ptr() for t in keep[:n]])
            Bv = (ctypes.c_void_p * n)(*[None if t is None else t.data_ptr() for t in keep[n:]])
            with torch.cuda.device(dev):
                E.check(E.lib().zk_layer_update_weights(ref.handle, W, Bv, E.stream_ptr(dev)))
            ref.generation += 1
            self.__dict__["_zk_cache"] = (sig, ref, E.hold_storage(self._layer_tensors()))
            return ref
        self._zk_release()
        desc, keep = self._layer_desc()
        h = ctypes.c_void_p()
        if dev is not None:
            with torch.cuda.device(dev):
                E.lib().zk_set_pack_stream(E.stream_ptr(dev))  # the pack kernels wait for work queued on this stream
                try:
                    E.check(E.lib().zk_layer_create(ctypes.byref(desc), ctypes.byref(h)))
                finally:
                    E.lib().zk_set_pack_stream(None)
        else:
            E.check(E.lib().zk_layer_create(ctypes.byref(desc), ctypes.byref(h)))
        del keep
        ref = OwnedLayer(h)
        self.__dict__["_zk_cache"] = (sig, ref, E.hold_storage(self._layer_tensors()))
        return ref

    def _zk_layer(self) -> ctypes.c_void_p:
        return self._zk_layer_ref().handle

    def _zk_release(self) -> None:
        self.__dict__.pop("_zk_cache", None)  # the handle is destroyed with its last reference
        self.__dict__.pop("_zk_reindexed", None)

    def _grad_source(self) -> dict:
        """Tensors the engine's parameter gradients of this layer belong to (see _ops.FlowCall)."""
        hyper = getattr(self, "hyper", None)
        if hyper is not None:
            lins = hyper._linears()
            return {"weights": [m.weight for m in lins], "biases": [m.bias for m in lins]}
        phi = getattr(self, "phi", None)
        if phi is not None:
            return {"phi": list(phi)}
        return {}

    def __del__(self) -> None:
        try:
            self._zk_release()
        except Exception:
            pass

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_zk_cache", None)
        state.pop("_zk_reindexed", None)
        return state

    def _base_desc(self, kind: int) -> E.LayerDesc:
        u = self._uni
        return E.LayerDesc(kind=kind, features=self.features, context=self.context, univariate=u["kind"],
                           bins=u["bins"], bound=u["bound"], slope=u["slope"], passes=getattr(self, "passes", 0),
                           iterations=u.get("iterations", 0), degree=u.get("degree", 0))  # fmt: skip

    def _describe_base(self) -> str:
        if self._uni["kind"] == E.ZK_UNI_BERNSTEIN:
            return "BoundedBernsteinTransform(degree=%d, bound=%g)" % (self._uni["degree"], self._uni["bound"])
        if self._uni["kind"] == E.ZK_UNI_SOSP:
            return "ShiftedSOSPTransform(polynomials=%d, degree=%d)" % (self._uni["bins"], self._uni["degree"])
        if self._uni["kind"] == E.ZK_UNI_GAUSS:
            return "GaussianizationTransform(components=%d)" % self._uni["bins"]
        if self._uni["kind"] == E.ZK_UNI_CRQS:
            return "CircularRQSTransform(bins=%d)" % self._uni["bins"]
        return "MonotonicRQSTransform(bins=%d)" % self._uni["bins"] if self._uni["kind"] == E.ZK_UNI_RQS else "MonotonicAffineTransform()"


def total_of(shapes: Sequence[Size]) -> int:
    return sum(prod(s) for s in shapes)
