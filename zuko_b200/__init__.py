"""zuko_b200 — H100-native (sm_90a) log-density and sampling engine for Zuko's flow hot path.

The public surface mirrors the reference (probabilists/zuko) for the hot path only:
``zuko_b200.flows.{MAF, NSF, NICE, ...}``, ``zuko_b200.lazy.Flow``,
``zuko_b200.distributions.NormalizingFlow`` — ``flow(c).log_prob(x)`` and
``flow(c).rsample(shape)`` run as hand-written CUDA kernels behind a C ABI
(``include/zuko_b200.h``).  There is no CPU fallback.
"""

__version__ = "0.1.0"

from . import bayesian, distributions, flows, lazy, nn, transforms, utils  # noqa: F401
from .accel import AcceleratedFlow, accelerate  # noqa: F401


def invalidate(module) -> None:
    """Drops every packed engine handle cached under ``module`` (a flow, a layer, a conditioner), so that
    the next call re-packs from the current tensors.

    The caches are keyed on ``(data_ptr, _version, device, dtype)`` of the tensors they were packed from:
    optimizer steps, ``load_state_dict``, ``.to()`` are seen.  In-place writes through ``.data`` (EMA /
    Polyak copies ``ema.data.mul_(a).add_(p.data)``, ``p.data.clamp_()``) do NOT bump ``_version`` — call
    this after them, or write through ``torch.no_grad()`` + the tensor itself instead of ``.data``."""
    import torch.nn as _nn

    mods = module.modules() if isinstance(module, _nn.Module) else [module]
    for m in mods:
        if hasattr(m, "_release"):  # conditioner used on its own: it owns (and destroys) its zk_mlp handle
            m._release()
        for key in ("_zk_cache", "_zk_reindexed", "_built"):
            m.__dict__.pop(key, None)
