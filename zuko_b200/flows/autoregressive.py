"""Masked autoregressive transformations and flows.

Host-side mirror of zuko/flows/autoregressive.py: ``MaskedAutoregressiveTransform``
(:24-218) and ``MAF`` (:221-316).  Construction (orders, adjacency, masks, parameter
initialisation) reproduces the reference bit for bit; evaluation is handed to the H100
engine as one packed ``zk_layer`` (conditioner GEMMs + fused bijector/ladj kernel).
"""

from __future__ import annotations

__all__ = ["MAF", "MaskedAutoregressiveTransform"]

from collections.abc import Callable, Sequence
from math import ceil

from functools import partial

import torch
from torch import BoolTensor, LongTensor, Size, Tensor
from torch.distributions import Transform

from .. import _engine as E
from ..distributions import DiagNormal
from ..lazy import Flow, LazyTransform, UnconditionalDistribution
from ..nn import MaskedMLP
from ..transforms import AutoregressiveTransform, MonotonicAffineTransform
from ._packed import PackedLayerMixin, refuse_elementwise_only, resolve_univariate, total_of
from .elementwise import ElementWiseTransform


def dag_diameter(adjacency: BoolTensor) -> int:
    """Number of topological generations of the DAG ``adjacency`` (``[i, j]``: i depends
    on j) = sequential passes the inverse needs (zuko/flows/autoregressive.py:154-185).
    Raises if the graph has a cycle."""
    n = adjacency.shape[0]
    pending = adjacency.sum(dim=1).tolist()  # unresolved dependencies per node
    frontier = [i for i in range(n) if pending[i] == 0]
    generations = 0
    resolved = 0
    while frontier:
        generations += 1
        resolved += len(frontier)
        nxt = []
        for node in frontier:
            for child in adjacency[:, node].nonzero().flatten().tolist():
                pending[child] -= 1
                if pending[child] == 0:
                    nxt.append(child)
        frontier = nxt
    assert resolved == n, "The graph contains cycles."
    return generations


def reindex_conditioner(i: int, n: int, w: Tensor, b: Tensor | None, mask: Tensor | None, *, qi: Tensor, D: int, P: int):
    """Tensors of linear layer ``i`` of ``n`` of an autoregressive conditioner re-indexed by the feature permutation
    ``q`` (``qi`` as a LongTensor): the layer ``T~`` with ``T(P x) = P T~(x)`` for ``(P x)_j = x_{q[j]}`` reads
    feature ``q[j]`` where ``T`` read its input ``j`` (first layer: ``W~[:, q[j]] = W[:, j]`` for the D x-columns, the
    context columns stay) and emits the parameters of feature ``q[j]`` where ``T`` emitted those of ``j`` (last
    layer: block ``q[j]`` of P rows = block ``j``)."""
    if i == 0:
        w2 = w.clone()
        w2[:, qi] = w[:, :D]
        w = w2
        if mask is not None:
            m2 = mask.clone()
            m2[:, qi] = mask[:, :D]
            mask = m2
    if i == n - 1:
        w2 = torch.empty_like(w)
        w2.view(D, P, -1)[qi] = w.view(D, P, -1)
        w = w2
        if b is not None:
            b2 = torch.empty_like(b)
            b2.view(D, P)[qi] = b.view(D, P)
            b = b2
        if mask is not None:
            m2 = torch.empty_like(mask)
            m2.view(D, P, -1)[qi] = mask.view(D, P, -1)
            mask = m2
    return w, b, mask


class MaskedAutoregressiveTransform(PackedLayerMixin, LazyTransform):
    """Lazy masked autoregressive transformation ``y_i = f(x_i | x_<i, c)``.

    Arguments follow zuko/flows/autoregressive.py:88-99: ``features``, ``context``,
    ``passes`` (None = fully autoregressive, 2 = coupling), ``order``, ``adjacency``
    (custom dependency DAG; overrides ``order`` / ``passes``), ``univariate`` / ``shapes``
    (engine bijectors: ``MonotonicAffineTransform``, ``MonotonicRQSTransform``) and
    ``**kwargs`` for :class:`zuko_b200.nn.MaskedMLP`.
    """

    def __new__(cls, features: int | None = None, context: int = 0, passes: int | None = None,
                order: LongTensor | None = None, adjacency: BoolTensor | None = None, *args, **kwargs) -> LazyTransform:  # fmt: skip
        if features is None or features > 1:
            return super().__new__(cls)
        return ElementWiseTransform(features, context, *args, **kwargs)  # single feature: nothing to mask

    def __init__(
        self,
        features: int,
        context: int = 0,
        passes: int | None = None,
        order: LongTensor | None = None,
        adjacency: BoolTensor | None = None,
        univariate: Callable[..., Transform] = MonotonicAffineTransform,
        shapes: Sequence[Size] = ((), ()),
        **kwargs,
    ) -> None:
        super().__init__()
        self.univariate, self.shapes = univariate, shapes
        self.total = total_of(shapes)
        self._uni = resolve_univariate(univariate, shapes)
        refuse_elementwise_only(self._uni, "MaskedAutoregressiveTransform")
        self.features, self.context = features, context
        self.register_buffer("order", None)

        ctx_cols = None
        if adjacency is None:
            passes = features if passes is None else passes
            order = torch.arange(features) if order is None else torch.as_tensor(order, dtype=int)
            assert order.ndim == 1, "'order' should be a vector."
            assert order.shape[0] == features, f"'order' should have {features} elements."
            self.passes = min(max(passes, 1), features)
            # features sharing an order class are transformed in the same pass
            self.order = torch.div(order, ceil(features / self.passes), rounding_mode="floor")
            deps = self.order[:, None] > self.order
        else:
            adjacency = torch.as_tensor(adjacency, dtype=bool)
            assert adjacency.ndim == 2, "'adjacency' should be a matrix."
            assert adjacency.shape[0] == features, f"'adjacency' should have {features} rows."
            assert adjacency.shape[1] in (features, features + context), (
                f"'adjacency' should have {features} or {features + context} columns."
            )
            if adjacency.shape[1] > features:
                ctx_cols = adjacency[:, features:]
            deps = adjacency[:, :features]
            assert deps.diag().all(), "'adjacency' should have ones on the diagonal."
            deps = deps * ~torch.eye(features, dtype=bool)
            self.passes = dag_diameter(deps)

        if context > 0:
            if ctx_cols is None:
                ctx_cols = torch.ones((features, context), dtype=bool)
            deps = torch.cat((deps, ctx_cols), dim=1)

        # one conditioner output row per (feature, parameter): row index d * total + p
        self.hyper = MaskedMLP(torch.repeat_interleave(deps, repeats=self.total, dim=0), **kwargs)

    def extra_repr(self) -> str:
        if self.order is None:
            return f"(base): {self._describe_base()}\n(passes): {self.passes}"
        order = self.order.tolist()
        if len(order) > 10:
            order = str(order[:5] + [...] + order[-5:]).replace("Ellipsis", "...")
        return f"(base): {self._describe_base()}\n(order): {order}"

    def _layer_desc(self):
        hyper, keep = self.hyper.mlp_desc()
        desc = self._base_desc(E.ZK_LAYER_AUTOREGRESSIVE)
        import ctypes

        desc.hyper = ctypes.pointer(hyper)
        keep = [hyper, keep]
        if self.order is not None:  # order classes let the engine run the dimension-sequential inverse
            host = self.order.detach().to("cpu", torch.int64).tolist()
            arr = (ctypes.c_int64 * self.features)(*host)
            desc.order = arr
            keep.append(arr)
        return desc, keep

    def _zk_layer_ref_reindexed(self, q: tuple):
        """The handle of this layer conjugated by a feature permutation: with ``(P x)_i = x_{q[i]}``,
        ``T(P x) = P T~(x)`` where ``T~`` is the same layer with the conditioner's x-input columns and its per-dimension
        output blocks re-indexed (``W0~[:, q] = W0[:, :D]``, block ``q[i]`` of the last layer = block ``i``, ``order~[q] =
        order``) — a permutation in front of an autoregressive layer (zuko/transforms.py:1193-1214 feeding
        flows/autoregressive.py:207-215) costs nothing but this re-packing.  Forward-only (no gradient sources);
        cached per (layer signature, q)."""
        from ._packed import OwnedLayer

        sig = (self._layer_signature(), tuple(q))
        cache = self.__dict__.setdefault("_zk_reindexed", {})
        hit = cache.get(tuple(q))
        if hit is not None and hit[0] == sig:
            return hit[1]
        import ctypes

        D, P = self.features, self.total
        dev = self.hyper._linears()[0].weight.device
        qi = torch.as_tensor(list(q), dtype=torch.long, device=dev)

        reindex = partial(reindex_conditioner, qi=qi, D=D, P=P)

        hyper, keep = self.hyper.mlp_desc(reindex)
        desc = self._base_desc(E.ZK_LAYER_AUTOREGRESSIVE)
        desc.hyper = ctypes.pointer(hyper)
        keep = [hyper, keep]
        if self.order is not None:
            host = self.order.detach().to("cpu", torch.int64)
            ro = torch.empty_like(host)
            ro[torch.as_tensor(list(q), dtype=torch.long)] = host
            arr = (ctypes.c_int64 * D)(*ro.tolist())
            desc.order = arr
            keep.append(arr)
        h = ctypes.c_void_p()
        with torch.cuda.device(dev):
            E.lib().zk_set_pack_stream(E.stream_ptr(dev))
            try:
                E.check(E.lib().zk_layer_create(ctypes.byref(desc), ctypes.byref(h)))
            finally:
                E.lib().zk_set_pack_stream(None)
        del keep
        ref = OwnedLayer(h)
        if len(cache) > 8:
            cache.clear()
        cache[tuple(q)] = (sig, ref, E.hold_storage(self._layer_tensors()))
        return ref

    def forward(self, c: Tensor | None = None) -> Transform:
        return AutoregressiveTransform(self, c)


class MAF(Flow):
    """Masked autoregressive flow (zuko/flows/autoregressive.py:221-316): ``transforms``
    autoregressive layers whose feature order alternates ascending / descending (or is
    random with ``randperm=True``), over a standard ``DiagNormal`` base."""

    def __init__(self, features: int, context: int = 0, transforms: int = 3, randperm: bool = False, **kwargs) -> None:
        ascending = torch.arange(features)
        layers = []
        for i in range(transforms):
            if randperm:
                order = torch.randperm(features)
            else:
                order = ascending if i % 2 == 0 else ascending.flip(0)
            layers.append(MaskedAutoregressiveTransform(features=features, context=context, order=order, **kwargs))
        base = UnconditionalDistribution(DiagNormal, loc=torch.zeros(features), scale=torch.ones(features), buffer=True)
        super().__init__(layers, base)
