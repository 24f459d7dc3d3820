"""``accelerate(flow)`` — put the H100 engine behind an *existing* reference flow.

The reference has no plugin registry; its stable seam for the hot path is
``LazyDistribution.forward(c) -> Distribution`` (zuko/lazy.py:39-49, SURVEY §8b).
``accelerate`` takes a flow built by the reference constructors (``zuko.flows.MAF / NSF /
NICE / RealNVP`` or a hand-composed ``zuko.lazy.Flow``) and returns an engine-backed
``LazyDistribution`` with the same module tree and the same state-dict keys that **shares the
reference's own parameters and buffers** (weights, biases, the reference-built masks, orders,
base ``loc`` / ``scale``): optimizer steps, ``load_state_dict`` and re-parameterisations of the
original are seen by the accelerated flow, whose packed weights are re-built when a tensor's
``(data_ptr, _version)`` changes.

The reference package is never imported: modules are recognised by class name and by the
attributes their constructors set (file:line cited per converter), so the same code accepts
``zuko_b200``'s own modules.  Options the engine does not implement (residual conditioners,
activation modules outside ZK_ACT_*, other univariate bijectors, other bases) raise ``NotImplementedError``
here, at ``accelerate()`` time — never a silent eager fallback.
"""

from __future__ import annotations

__all__ = ["AcceleratedFlow", "accelerate"]

from functools import partial

import torch
import torch.nn as nn

from . import distributions as _D
from . import transforms as _T
from .flows.autoregressive import MaskedAutoregressiveTransform
from .flows.continuous import FFJTransform
from .flows.coupling import GeneralCouplingTransform
from .flows.elementwise import ElementWiseTransform
from .lazy import (
    Flow,
    LazyComposedTransform,
    LazyDistribution,
    LazyInverse,
    LazyTransform,
    UnconditionalDistribution,
    UnconditionalTransform,
)

# constructors a reference `Unconditional*` / `univariate=` hook may name -> engine classes
_ENGINE_CALLABLES = {
    "DiagNormal": _D.DiagNormal,
    "BoxUniform": _D.BoxUniform,
    "CircularRQSTransform": _T.CircularRQSTransform,
    "CircularShiftTransform": _T.CircularShiftTransform,
    "GaussianizationTransform": _T.GaussianizationTransform,
    "MonotonicAffineTransform": _T.MonotonicAffineTransform,
    "MonotonicRQSTransform": _T.MonotonicRQSTransform,
    "SoftclipTransform": _T.SoftclipTransform,
    "ShiftedSOSPTransform": _T.ShiftedSOSPTransform,
    "SOSPolynomialTransform": _T.SOSPolynomialTransform,
    "BoundedBernsteinTransform": _T.BoundedBernsteinTransform,
    "PermutationTransform": _T.PermutationTransform,
    "RotationTransform": _T.RotationTransform,
}


def _unsupported(what: str) -> NotImplementedError:
    return NotImplementedError(f"zuko_b200.accelerate: {what} is outside the accelerated hot path (SURVEY §8)")


def _engine_callable(f):  # noqa: ANN001, ANN202
    """Maps a reference constructor (possibly wrapped in ``functools.partial``) to the engine's."""
    if isinstance(f, partial):
        return partial(_engine_callable(f.func), *f.args, **f.keywords)
    name = getattr(f, "__name__", type(f).__name__)
    if name not in _ENGINE_CALLABLES:
        raise _unsupported(f"constructor {name!r}")
    return _ENGINE_CALLABLES[name]


def _conditioner_kwargs(hyper: nn.Module) -> tuple[dict, list]:
    """Recovers ``hidden_features`` from a reference ``MLP`` / ``MaskedMLP`` (an ``nn.Sequential``
    of linear layers and activations, zuko/nn.py:160-192, 295-318) and rejects the options the
    engine does not implement."""
    from .nn import activation_code

    linears = []
    activation = None
    block_widths = []  # residual conditioners: one block per hidden depth (zuko/nn.py:297-309)
    flat = []
    for m in hyper:
        if type(m).__name__ == "Residual":
            inner = list(m)
            if len(inner) != 3 or not hasattr(inner[0], "weight") or hasattr(inner[1], "weight") or not hasattr(inner[2], "weight"):
                raise _unsupported("a residual block that is not Linear-activation-Linear")
            block_widths.append(inner[0].weight.shape[0])
            flat += inner
        else:
            flat.append(m)
    for m in flat:
        if hasattr(m, "weight") and isinstance(getattr(m, "weight", None), torch.Tensor):
            if m.weight.dim() != 2:
                raise _unsupported("a stacked / non-matrix linear layer in the conditioner")
            linears.append(m)
        elif any(True for _ in m.children()):
            raise _unsupported(f"conditioner module {type(m).__name__}")
        else:
            try:
                activation_code(m)
            except NotImplementedError as e:
                raise _unsupported(f"conditioner module {type(m).__name__} ({e})") from None
            if activation is not None and activation is not type(m):
                raise _unsupported("a conditioner mixing different activations")
            activation = type(m)
    if not linears:
        raise _unsupported("a conditioner without linear layers")
    kwargs = dict(hidden_features=[m.weight.shape[0] for m in linears[:-1]])
    if block_widths:
        kwargs = dict(hidden_features=block_widths, residual=True)
    if activation is not None and activation is not nn.ReLU:
        kwargs["activation"] = activation
    return kwargs, linears


def _convert(m: nn.Module, passthrough: bool = True) -> nn.Module:
    """Builds the engine-backed mirror of the reference module ``m`` (fresh tensors; ``_share``
    then rebinds them to the reference's)."""
    if passthrough and isinstance(m, (LazyDistribution, LazyTransform)):
        return m  # already an engine module
    kind = type(m).__name__

    if hasattr(m, "transform") and hasattr(m, "base"):  # Flow and its subclasses — zuko/lazy.py:131-172
        return Flow(_convert(m.transform, passthrough), _convert(m.base, passthrough))
    if kind == "LazyComposedTransform":  # zuko/lazy.py:101-128
        return LazyComposedTransform(*(_convert(t, passthrough) for t in m.transforms))
    if kind == "LazyInverse":  # zuko/lazy.py:81-98
        return LazyInverse(_convert(m.transform, passthrough))

    if kind == "MaskedAutoregressiveTransform":  # zuko/flows/autoregressive.py:88-152
        kwargs, linears = _conditioner_kwargs(m.hyper)
        features = linears[-1].weight.shape[0] // m.total
        context = linears[0].weight.shape[1] - features
        out = MaskedAutoregressiveTransform(
            features, context, passes=m.passes, univariate=_engine_callable(m.univariate), shapes=m.shapes, **kwargs
        )
        out.passes = m.passes
        if m.order is None:  # built from an `adjacency=` DAG: no order classes, inverse by sweeps
            out.order = None
        return out
    if kind == "GeneralCouplingTransform":  # zuko/flows/coupling.py:79-111
        kwargs, linears = _conditioner_kwargs(m.hyper)
        mask = m.mask.detach().to("cpu", torch.bool)
        context = linears[0].weight.shape[1] - int(mask.sum())
        return GeneralCouplingTransform(
            mask.numel(), context, mask=mask, univariate=_engine_callable(m.univariate), shapes=m.shapes, **kwargs
        )
    if kind == "ElementWiseTransform":  # zuko/flows/gaussianization.py:60-77
        if hasattr(m, "hyper"):
            kwargs, linears = _conditioner_kwargs(m.hyper)
            return ElementWiseTransform(
                linears[-1].weight.shape[0] // m.total, linears[0].weight.shape[1],
                univariate=_engine_callable(m.univariate), shapes=m.shapes, **kwargs,
            )  # fmt: skip
        return ElementWiseTransform(m.phi[0].shape[0], 0, univariate=_engine_callable(m.univariate), shapes=m.shapes)

    if kind == "FFJTransform":  # zuko/flows/continuous.py:70-86
        kwargs, linears = _conditioner_kwargs(m.ode)
        kwargs.setdefault("activation", nn.ReLU)  # the reference's conditioner was built without an ELU default
        F = m.freqs.numel()
        D = linears[-1].weight.shape[0]
        return FFJTransform(D, linears[0].weight.shape[1] - D - 2 * F, freqs=F, atol=m.atol, rtol=m.rtol, exact=m.exact,
                            **kwargs)  # fmt: skip

    if kind in ("UnconditionalDistribution", "UnconditionalTransform"):  # zuko/lazy.py:242-335, utils.py:58-86
        if isinstance(m.f, nn.Module):
            raise _unsupported("an Unconditional wrapper around a module")
        tensors = [v for v in list(m.args) + list(m.kwargs.values()) if torch.is_tensor(v)]
        buffer = bool(tensors) and all(not isinstance(v, nn.Parameter) for v in tensors)
        cls = UnconditionalDistribution if kind == "UnconditionalDistribution" else UnconditionalTransform
        args = [v.detach() if torch.is_tensor(v) else v for v in m.args]
        kw = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in m.kwargs.items()}
        return cls(_engine_callable(m.f), *args, buffer=buffer, **kw)

    raise _unsupported(f"module {kind}")


def _owner(root: nn.Module, dotted: str) -> tuple[nn.Module, str]:
    *path, leaf = dotted.split(".")
    mod = root
    for name in path:
        mod = mod._modules[name]
    return mod, leaf


def _share(mirror: nn.Module, source: nn.Module) -> None:
    """Rebinds every parameter / buffer of ``mirror`` to the tensor object ``source`` owns under
    the same name.  The two trees have the same state-dict layout by construction (the engine
    classes reproduce the reference's constructors; tests/test_host.py checks key-for-key)."""
    src_keys, dst_keys = set(source.state_dict().keys()), set(mirror.state_dict().keys())
    if src_keys != dst_keys:
        diff = sorted(src_keys ^ dst_keys)
        raise _unsupported(f"a module whose state-dict layout differs from the engine's mirror ({diff[:4]} ...)")
    for name, p in source.named_parameters(remove_duplicate=False):
        mod, leaf = _owner(mirror, name)
        if mod._parameters[leaf].shape != p.shape:
            raise ValueError(f"zuko_b200.accelerate: shape mismatch for {name}")
        mod._parameters[leaf] = p
    for name, b in source.named_buffers(remove_duplicate=False):
        mod, leaf = _owner(mirror, name)
        if leaf not in mod._buffers:
            raise ValueError(f"zuko_b200.accelerate: missing buffer {name}")
        mod._buffers[leaf] = b


class AcceleratedFlow(Flow):
    """What ``accelerate(flow)`` returns: a :class:`zuko_b200.lazy.Flow` on the reference's own
    tensors.  ``accel(c)`` is a ``NormalizingFlow`` whose ``log_prob`` / ``rsample`` /
    ``rsample_and_log_prob`` are engine calls (zuko/distributions.py:115-138)."""

    def __init__(self, mirror: Flow, source: nn.Module) -> None:
        super().__init__(mirror.transform, mirror.base)
        object.__setattr__(self, "_source", source)  # not a sub-module: keeps the state-dict layout
        self.resync()

    def resync(self) -> None:
        """Re-adopts the source's tensors (needed after ``source.to(...)`` / ``.cuda()``, which
        replace buffer objects — parameters are updated in place by torch)."""
        _share(self, self._source)
        pairs = []
        for name, _ in self._source.named_buffers(remove_duplicate=False):
            (dst, leaf), (src, _) = _owner(self, name), _owner(self._source, name)
            pairs.append((dst, src, leaf, "_buffers"))
        for name, _ in self._source.named_parameters(remove_duplicate=False):
            (dst, leaf), (src, _) = _owner(self, name), _owner(self._source, name)
            pairs.append((dst, src, leaf, "_parameters"))
        self.__dict__["_pairs"] = pairs

    def _stale(self) -> bool:
        return any(getattr(d, kind)[leaf] is not getattr(s, kind).get(leaf) for d, s, leaf, kind in self._pairs)

    def forward(self, c=None):  # noqa: ANN001, ANN201
        if self._stale():
            self.resync()
        return super().forward(c)


def _accelerate_gmm(gmm: nn.Module) -> nn.Module:
    """The engine's ``GMM`` on the reference model's own parameters (``hyper.*`` or ``phi.*``)."""
    from .mixtures import GMM

    for name, t in gmm.named_parameters():
        if t.dtype != torch.float32:
            raise TypeError(f"zuko_b200.accelerate: {name} is {t.dtype}; the engine computes in float32")
    kwargs, context = {}, 0
    if hasattr(gmm, "hyper"):
        kwargs, linears = _conditioner_kwargs(gmm.hyper)
        context = linears[0].weight.shape[1]
    with torch.random.fork_rng(devices=[]):
        mirror = GMM(gmm.shapes[1][1], context, components=gmm.components, covariance_type=gmm.covariance_type,
                     tied=gmm.tied, epsilon=gmm.epsilon, **kwargs)  # fmt: skip
    _share(mirror, gmm)
    return mirror


def accelerate(flow: nn.Module) -> nn.Module:
    """Returns an engine-backed drop-in for ``flow`` (a reference ``zuko.lazy.Flow`` such as
    ``zuko.flows.NSF(...)``) that shares its parameters and buffers.

    A reference ``zuko.mixtures.GMM`` gives the engine's :class:`~zuko_b200.mixtures.GMM` on the reference's
    own parameters.  A reference ``zuko.bayesian.BayesianModel`` gives an engine :class:`~zuko_b200.bayesian.BayesianModel`
    over ``accelerate(model.base)`` whose ``means`` / ``logvars`` are the reference's own.

    Move ``flow`` to its CUDA device first (or call ``.resync()`` / just call the result — buffer
    replacement is detected).  The engine is fp32-only: other parameter dtypes raise ``TypeError``
    (the reference's tests default to fp64, tests/conftest.py:12).
    """
    if type(flow).__name__ == "BayesianModel":  # zuko/bayesian.py:48-100
        from .bayesian import BayesianModel

        model = BayesianModel(accelerate(flow.base), include_params=())  # no parameters, no draws
        model.means, model.logvars = flow.means, flow.logvars
        return model
    if type(flow).__name__ == "GMM":  # zuko/mixtures.py:25-99
        return _accelerate_gmm(flow)
    if not (hasattr(flow, "transform") and hasattr(flow, "base")):
        raise TypeError("accelerate() expects a lazy Flow (an object with .transform and .base)")
    for name, t in list(flow.named_parameters()) + list(flow.named_buffers()):
        if t.is_floating_point() and t.dtype != torch.float32:
            raise TypeError(f"zuko_b200.accelerate: {name} is {t.dtype}; the engine computes in float32")
    # the mirror's constructors draw fresh initial weights (rebound to the reference's right after): keep
    # the caller's global RNG stream untouched
    with torch.random.fork_rng(devices=[]):
        mirror = _convert(flow, passthrough=False)
    return AcceleratedFlow(mirror, flow)
