"""Conditioner networks of the flow hot path: ``MaskedMLP`` and ``MLP``.

Host-side mirror of zuko/nn.py:122-192 (MLP), :202-218 (MaskedLinear) and :221-318
(MaskedMLP).  The modules own the same parameters / buffers under the same state-dict
keys as the reference (``{2j}.weight``, ``{2j}.bias``, ``{2j}.mask``) and are initialised
by the same torch initialisers in the same order, so a reference checkpoint loads
unchanged and ``torch.manual_seed(s)`` yields bit-identical weights.

``forward`` does not run torch ops: it hands the weights to the H100 engine
(``zk_mlp_forward`` — pre-masked, packed once per parameter version).
"""

from __future__ import annotations

__all__ = ["MLP", "Linear", "MaskedLinear", "MaskedMLP", "Residual"]

import ctypes
import warnings
from collections.abc import Callable, Sequence

import torch
import torch.nn as nn
from torch import BoolTensor, Tensor

from . import _engine as E


class Linear(nn.Module):
    """Dense affine layer ``y = x W^T + b`` with U(-1/sqrt(in), 1/sqrt(in)) initialisation
    (zuko/nn.py:51-119, ``stack`` is not supported by the engine)."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, stack: int | None = None) -> None:
        super().__init__()
        if stack is not None:
            raise NotImplementedError("zuko_b200: stacked Linear operators are outside the accelerated path")
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.empty(out_features)) if bias else None
        self.in_features, self.out_features = in_features, out_features
        self.reset_parameters()

    def reset_parameters(self) -> None:
        k = self.weight.shape[-1] ** -0.5
        nn.init.uniform_(self.weight, -k, k)
        if self.bias is not None:
            nn.init.uniform_(self.bias, -k, k)

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}"


class MaskedLinear(nn.Linear):
    """``y = x (W * A)^T + b`` for a boolean adjacency ``A`` (out, in) — zuko/nn.py:202-218.
    The product ``mask * weight`` is formed once, when the engine packs the layer."""

    def __init__(self, adjacency: BoolTensor, **kwargs) -> None:
        out_features, in_features = adjacency.shape
        super().__init__(in_features, out_features, **kwargs)
        self.register_buffer("mask", adjacency)


# activation modules the engine implements (with torch's default arguments) -> ZK_ACT_* code
_ACTIVATION_CODES = {
    "ReLU": (E.ZK_ACT_RELU, {}),
    "ELU": (E.ZK_ACT_ELU, {"alpha": 1.0}),
    "Tanh": (E.ZK_ACT_TANH, {}),
    "SiLU": (E.ZK_ACT_SILU, {}),
    "GELU": (E.ZK_ACT_GELU, {"approximate": "none"}),
    "LeakyReLU": (E.ZK_ACT_LEAKY_RELU, {"negative_slope": 0.01}),
    "Softplus": (E.ZK_ACT_SOFTPLUS, {"beta": 1.0, "threshold": 20.0}),
    "Sigmoid": (E.ZK_ACT_SIGMOID, {}),
}


def activation_code(module: nn.Module) -> int:
    """ZK_ACT_* of an activation module instance; raises for modules / arguments the engine does not
    implement (the reference accepts any constructor, zuko/nn.py:264-265)."""
    name = type(module).__name__
    if name not in _ACTIVATION_CODES or any(True for _ in module.children()):
        raise NotImplementedError(
            f"zuko_b200: activation {name} is not implemented by the engine "
            f"(supported with their default arguments: {', '.join(_ACTIVATION_CODES)})"
        )
    code, defaults = _ACTIVATION_CODES[name]
    for k, v in defaults.items():
        if getattr(module, k, v) != v:
            raise NotImplementedError(f"zuko_b200: {name}({k}={getattr(module, k)!r}) is not implemented (engine: {k}={v!r})")
    return code


class Residual(nn.Sequential):
    """Residual block ``x + block(x)`` (zuko/nn.py:195-199).  Inside an engine conditioner the block is
    ``MaskedLinear -> activation -> MaskedLinear`` and runs as two GEMM layers, the second one adding
    the block's input in its epilogue."""


def _relu_only(activation: Callable[[], nn.Module] | None) -> Callable[[], nn.Module]:
    """Validates the ``activation=`` constructor hook (name kept for history: ReLU is the default)."""
    if activation is None:
        return nn.ReLU
    activation_code(activation())  # raises NotImplementedError for unsupported modules
    return activation


class _EngineMLP(nn.Sequential):
    """Shared engine plumbing for MLP / MaskedMLP: packs the linear layers into a
    ``zk_mlp`` handle, re-packing whenever a parameter / mask changes (optimizer step,
    ``load_state_dict``, ``.to()``, re-parameterisation)."""

    gemm_mode = "auto"  # "auto" | "fp32" | "bf16x3" | "bf16x1"

    def _linears(self) -> list[nn.Module]:
        """Linear layers in execution order (residual blocks flattened)."""
        out: list[nn.Module] = []
        for m in self:
            if isinstance(m, Residual):
                out += [k for k in m if hasattr(k, "weight")]
            elif hasattr(m, "weight"):
                out.append(m)
        return out

    def _layer_flags(self) -> tuple[list[int], list[int]] | None:
        """Per linear layer: the activation applied to its output (0 = none, else ZK_ACT_* with ReLU = 1) and
        whether the input of the PREVIOUS linear layer is added to its output (second layer of a residual
        block).  ``None`` for the plain pattern (activation after every layer but the last)."""
        mods = list(self)
        if not any(isinstance(m, Residual) for m in mods):
            return None
        acts: list[int] = []
        res: list[int] = []
        for j, m in enumerate(mods):
            if isinstance(m, Residual):
                inner = list(m)
                if len(inner) != 3 or not hasattr(inner[0], "weight") or hasattr(inner[1], "weight") or not hasattr(inner[2], "weight"):
                    raise NotImplementedError("zuko_b200: residual blocks other than Linear-activation-Linear are not implemented")
                acts += [activation_code(inner[1]) or 1, 0]
                res += [0, 1]
            elif hasattr(m, "weight"):
                nxt = mods[j + 1] if j + 1 < len(mods) else None
                follows = nxt is not None and not hasattr(nxt, "weight") and not isinstance(nxt, Residual)
                acts.append((activation_code(nxt) or 1) if follows else 0)
                res.append(0)
        return acts, res

    _warned_detached = False

    def _activation_code(self) -> int:
        acts = [k for m in self for k in (m if isinstance(m, Residual) else [m]) if not hasattr(k, "weight")]
        codes = {activation_code(m) for m in acts}
        if len(codes) > 1:
            raise NotImplementedError("zuko_b200: a conditioner mixing different activations is not implemented")
        return codes.pop() if codes else E.ZK_ACT_RELU

    def _signature(self) -> tuple:
        flags = self._layer_flags()
        sig = [self.gemm_mode, self._activation_code(), None if flags is None else (tuple(flags[0]), tuple(flags[1]))]
        for m in self._linears():
            for t in (m.weight, m.bias, getattr(m, "mask", None)):
                sig.append(None if t is None else (t.data_ptr(), t._version, t.device, t.dtype))
        return tuple(sig)

    def _held_storage(self) -> list:
        """What a cache keyed on ``_signature()`` keeps alive with its entry (``_engine.hold_storage``)."""
        return E.hold_storage([t for m in self._linears() for t in (m.weight, m.bias, getattr(m, "mask", None))])

    def mlp_desc(self, reindex=None) -> tuple[E.MlpDesc, list]:
        """Builds the ``zk_mlp_desc`` for the current parameters. Returns (desc, keepalive).
        ``reindex(i, n, weight, bias, mask)`` may substitute the tensors of linear layer ``i`` of ``n`` (used to
        re-index a conditioner's input columns / output rows when a permutation is folded into the layer)."""
        lins = self._linears()
        n = len(lins)
        keep: list = []
        dims = (ctypes.c_int * (n + 1))(lins[0].weight.shape[1], *[m.weight.shape[0] for m in lins])
        W = (ctypes.c_void_p * n)()
        Bv = (ctypes.c_void_p * n)()
        M = (ctypes.c_void_p * n)()
        for i, m in enumerate(lins):
            E.require_cuda(m.weight, "conditioner weight")
            w_src, b_src, mask = m.weight.detach(), (None if m.bias is None else m.bias.detach()), getattr(m, "mask", None)
            if reindex is not None:
                w_src, b_src, mask = reindex(i, n, w_src, b_src, mask)
            w = w_src.contiguous()
            keep.append(w)
            W[i] = w.data_ptr()
            if b_src is not None:
                b = b_src.contiguous()
                keep.append(b)
                Bv[i] = b.data_ptr()
            if mask is not None:
                mk = mask.detach().to(torch.uint8).contiguous()
                keep.append(mk)
                M[i] = mk.data_ptr()
        flags = self._layer_flags()
        la = lr = None
        if flags is not None:
            la, lr = (ctypes.c_int * n)(*flags[0]), (ctypes.c_int * n)(*flags[1])
        desc = E.MlpDesc(n, dims, W, Bv, M, E.GEMM_MODES[self.gemm_mode], self._activation_code(), la, lr)
        keep += [dims, W, Bv, M, la, lr]
        return desc, keep

    def _handle(self) -> ctypes.c_void_p:
        sig = self._signature()
        cached = self.__dict__.get("_zk_cache")
        if cached is not None and cached[0] == sig:
            return cached[1]
        self._release()
        desc, keep = self.mlp_desc()
        h = ctypes.c_void_p()
        dev = self._linears()[0].weight.device
        with torch.cuda.device(dev):
            E.lib().zk_set_pack_stream(E.stream_ptr(dev))  # the pack kernels wait for work queued on this stream
            try:
                E.check(E.lib().zk_mlp_create(ctypes.byref(desc), ctypes.byref(h)))
            finally:
                E.lib().zk_set_pack_stream(None)
        del keep
        self.__dict__["_zk_cache"] = (sig, h, self._held_storage())
        return h

    def _release(self) -> None:
        cached = self.__dict__.pop("_zk_cache", None)
        if cached is not None:
            E.lib().zk_mlp_destroy(cached[1])

    def __del__(self) -> None:
        try:
            self._release()
        except Exception:
            pass

    def __getstate__(self):  # handles are not picklable (torch.save of the whole module)
        state = self.__dict__.copy()
        state.pop("_zk_cache", None)
        return state

    def forward(self, x: Tensor) -> Tensor:
        E.require_cuda(x, "conditioner input")
        if torch.is_grad_enabled():
            # the stand-alone conditioner call has no autograd seam (gradients flow through the flow-level calls,
            # _ops._FlowFunction).  An input that asks for gradients is refused; parameters that merely still
            # carry requires_grad (the default of a freshly built module used for inference) get one warning.
            if x.requires_grad:
                raise NotImplementedError(
                    "zuko_b200: MLP / MaskedMLP called on its own is forward-only; differentiate through "
                    "flow(c).log_prob / transform.call_and_ladj / rsample, or detach the input"
                )
            if not _EngineMLP._warned_detached and any(p.requires_grad for p in self.parameters()):
                _EngineMLP._warned_detached = True
                warnings.warn(
                    "zuko_b200: MLP / MaskedMLP called on its own returns a tensor that is NOT connected to its "
                    "parameters in the autograd graph (forward-only); use torch.no_grad() to silence this",
                    RuntimeWarning, stacklevel=2,
                )  # fmt: skip
        lead = x.shape[:-1]
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        B = x2.shape[0]
        out = torch.empty(B, self.out_features, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            h = self._handle()
            need = E.lib().zk_mlp_workspace_bytes(h, B)
            ws = E.Workspace.get(x.device, need, need) if need else None
            E.check(
                E.lib().zk_mlp_forward(
                    h, x2.data_ptr(), x2.shape[1], x2.shape[1], None, 0, 0, B, out.data_ptr(),
                    self.out_features, ws.data_ptr() if ws is not None else None,
                    ws.numel() if ws is not None else 0, E.stream_ptr(x.device),
                )
            )  # fmt: skip
        return out.reshape(*lead, self.out_features)


class MLP(_EngineMLP):
    """Dense multi-layer perceptron ``in -> hidden... -> out`` with an element-wise activation between
    layers (zuko/nn.py:122-192; ReLU by default, see ``_ACTIVATION_CODES``; ``normalize`` is not
    implemented)."""

    def __init__(
        self,
        in_features: int,
        out_features: int,
        hidden_features: Sequence[int] = (64, 64),
        activation: Callable[[], nn.Module] | None = None,
        normalize: bool = False,
        **kwargs,
    ) -> None:
        act = _relu_only(activation)
        if normalize:
            raise NotImplementedError("zuko_b200: LayerNorm between MLP layers is outside the accelerated path")
        widths = [in_features, *hidden_features, out_features]
        layers: list[nn.Module] = []
        for fan_in, fan_out in zip(widths[:-1], widths[1:], strict=True):
            layers += [Linear(fan_in, fan_out, **kwargs), act()]
        super().__init__(*layers[:-1])
        self.in_features, self.out_features = in_features, out_features


def masked_mlp_masks(adjacency: BoolTensor, hidden_features: Sequence[int], blocks: bool = False):
    """Masks of the masked MLP realising ``adjacency`` (out, in): every output may only
    depend on the inputs its adjacency row allows.  Restates zuko/nn.py:270-293.

    Outputs with identical dependency sets are merged into *classes* (unique rows).  Class
    ``j`` precedes class ``i`` when ``deps(j) ⊆ deps(i)``.  Hidden unit ``u`` of every hidden
    layer is assigned the class ``reachable[u mod #reachable]`` — cyclically over the classes
    with a non-empty dependency set; it listens to the units of the previous layer whose
    class precedes its own.  The output layer restores the original row multiplicity.

    With ``blocks=True`` also returns, per depth, the square mask of the residual block that follows
    that layer (zuko/nn.py:297-309): unit ``u`` may listen to unit ``v`` of the same layer when
    ``class(v)`` precedes ``class(u)``.
    """
    adjacency = torch.as_tensor(adjacency, dtype=torch.bool)
    classes, inverse = torch.unique(adjacency, dim=0, return_inverse=True)
    as_f64 = classes.to(torch.float64)
    overlap = as_f64 @ as_f64.T  # |deps(i) ∩ deps(j)|
    precedes = overlap == classes.sum(dim=-1)  # [i, j]: deps(j) ⊆ deps(i)

    masks: list[BoolTensor] = []
    block_masks: list[BoolTensor | None] = []
    unit_class = None
    widths = [*hidden_features, adjacency.shape[0]]
    for depth, width in enumerate(widths):
        table = classes if depth == 0 else precedes[:, unit_class]
        if not table.any():
            raise ValueError("The adjacency matrix leads to a null Jacobian.")
        if depth < len(hidden_features):
            reachable = table.any(dim=-1).nonzero().squeeze(-1)
            unit_class = reachable[torch.arange(width) % len(reachable)]
            masks.append(table[unit_class])
        else:
            masks.append(table[inverse])
        # the block after the output layer reuses the last hidden layer's classes: the reference builds it
        # (drawing its initial weights) and drops it again
        block_masks.append(None if unit_class is None else precedes[unit_class, :][:, unit_class])
    return (masks, block_masks) if blocks else masks


class MaskedMLP(_EngineMLP):
    """Masked multi-layer perceptron whose Jacobian ``dy_i/dx_j`` is null wherever
    ``adjacency[i, j]`` is False (zuko/nn.py:221-318).  ``residual=True`` builds the reference's residual
    blocks (:class:`Residual`); activations: see ``_ACTIVATION_CODES``."""

    def __init__(
        self,
        adjacency: BoolTensor,
        hidden_features: Sequence[int] = (64, 64),
        activation: Callable[[], nn.Module] | None = None,
        residual: bool = False,
    ) -> None:
        act = _relu_only(activation)
        out_features, in_features = adjacency.shape
        layers: list[nn.Module] = []
        if residual:
            if len(hidden_features) == 0:
                raise ValueError("zuko_b200: residual=True needs at least one hidden layer")
            masks, block_masks = masked_mlp_masks(adjacency, hidden_features, blocks=True)
            for depth, (mask, block) in enumerate(zip(masks, block_masks, strict=True)):
                # same construction order as zuko/nn.py:295-313, so that torch.manual_seed(s) yields the same
                # tensors: a hidden layer whose mask is square is built and replaced by its residual block,
                # and the block after the output layer is built and dropped
                layers.append(MaskedLinear(adjacency=mask))
                if 0 < depth < len(hidden_features) and mask.shape[0] == mask.shape[1]:
                    layers.pop()
                layers.append(Residual(MaskedLinear(adjacency=block), act(), MaskedLinear(adjacency=block)))
            layers.pop()
            super().__init__(*layers)
        else:
            for mask in masked_mlp_masks(adjacency, hidden_features):
                layers += [MaskedLinear(adjacency=mask), act()]
            super().__init__(*layers[:-1])
        self.in_features, self.out_features = in_features, out_features
