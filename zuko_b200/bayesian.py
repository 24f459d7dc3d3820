r"""Bayesian flows: a Gaussian mean-field posterior over a module's parameters (zuko/bayesian.py).

:class:`BayesianModel` wraps a base module (a flow, a conditioner) and keeps, per included parameter,
a posterior mean (initialised to the parameter) and a log-variance.  ``reparameterize()`` swaps a
posterior draw ``mean + exp(softclip(logvar, 18) / 2) * eps`` into the base for the duration of a
context, so that the base's engine calls differentiate through the draw to ``means`` / ``logvars``.

Constructor, pattern rules, state-dict keys, initialisation and the order of the random draws follow the
reference, so a seeded model and a seeded draw give the reference's tensors.

The local reparameterization trick (``reparameterize(local_trick=True)``) is not implemented by the
engine: requesting it on a model with a linear layer it would apply to raises ``NotImplementedError``
rather than silently sampling weights.
"""

from __future__ import annotations

__all__ = ["BayesianModel"]

import copy
import math
import re
from collections.abc import Iterator, Sequence
from contextlib import contextmanager
from typing import Any

import torch
import torch.nn as nn
from torch import Tensor

from .nn import Linear, MaskedLinear

# module classes whose forward the local reparameterization trick replaces (matched by exact type)
_LOCAL_TRICK_TYPES = (nn.Linear, Linear, MaskedLinear)


def _compile(prefix: str) -> re.Pattern:
    """A parameter-name prefix as a regular expression: ``*`` is one name component, ``**`` any
    dot-separated run of components; the pattern matches every name that starts with the prefix."""
    if re.fullmatch(r"[\w.*]*", prefix) is None:
        raise ValueError(f"Invalid prefix {prefix!r}: only word characters, '.' and '*' are allowed")
    pattern = prefix.replace(".", r"\.").replace("**", r"[\w\.]+").replace("*", r"\w+")
    return re.compile(pattern + ".*")


def _match(pattern: re.Pattern, string: str) -> bool:
    return pattern.fullmatch(string) is not None


def _softclip(x: Tensor, bound: float) -> Tensor:
    """``x / sqrt(1 + (x / bound)^2)``: keeps the log-variances in (-bound, bound)."""
    return x * (1 + (x / bound).square()).rsqrt()


class BayesianModel(nn.Module):
    r"""Creates a Bayesian wrapper around a base model.

    Arguments:
        base: A base model.
        init_logvar: The mean of the initial log-variances.
        include_params: Parameter name prefixes to include. In a prefix, ``*`` matches one
            alphanumeric name component and ``**`` matches dot-separated components. By default,
            all parameters are included.
        exclude_params: Parameter name prefixes to exclude.
    """

    def __init__(
        self,
        base: nn.Module,
        init_logvar: float = -9.0,
        include_params: Sequence[str] = ("",),
        exclude_params: Sequence[str] = (),
    ) -> None:
        super().__init__()
        self.base = base
        self.means = nn.ParameterDict()
        self.logvars = nn.ParameterDict()

        include = [_compile(p) for p in include_params]
        exclude = [_compile(p) for p in exclude_params]
        for name, param in base.named_parameters():
            if any(_match(p, name) for p in include) and not any(_match(p, name) for p in exclude):
                key = name.replace(".", "-")
                self.means[key] = nn.Parameter(torch.empty_like(param))
                self.logvars[key] = nn.Parameter(torch.empty_like(param))

        self._reset_bayesian_parameters(logvar_mean=init_logvar)

    def _reset_bayesian_parameters(self, logvar_mean: float = -9.0, logvar_std: float = 1e-3) -> None:
        """Means from the base's parameters, log-variances ~ N(logvar_mean, logvar_std^2), in the
        base's parameter order."""
        for name, param in self.base.named_parameters():
            key = name.replace(".", "-")
            if key in self.means:
                self.means[key].data.copy_(param.data)
                self.logvars[key].data.normal_(logvar_mean, logvar_std)

    def forward(self, *args, **kwargs) -> None:
        raise RuntimeError(
            "'forward' method of BayesianModel should not be called directly. "
            "Use 'sample_model' or 'reparameterize' instead."
        )

    def sample_params(self) -> dict[str, Tensor]:
        r"""Returns model parameters sampled from the posterior, one ``randn_like`` draw per
        parameter in the order of ``means``."""
        params = {}
        for key, mean in self.means.items():
            std = _softclip(self.logvars[key], 18.0).div(2.0).exp()
            params[key.replace("-", ".")] = mean + std * torch.randn_like(mean)
        return params

    def sample_model(self) -> nn.Module:
        r"""Returns a standalone copy of the base model with parameters sampled from the posterior.

        Gradients of the copy do not reach the Bayesian model's parameters: train through
        :meth:`reparameterize`.
        """
        with torch.no_grad():
            params = self.sample_params()
        model = copy.deepcopy(self.base)
        model.load_state_dict(params, strict=False)
        return model

    @contextmanager
    def reparameterize(self, local_trick: bool = False) -> Iterator[nn.Module]:
        r"""Reparameterizes the base model from the posterior.

        Within the context the base model holds one posterior draw and is deterministic; gradients
        of what it computes reach ``means`` and ``logvars``.

        Arguments:
            local_trick: Whether to use the local reparameterization trick for linear layers. The
                engine does not implement it: ``True`` raises ``NotImplementedError`` when the model
                has an included linear layer it would apply to.
        """
        if local_trick:
            self._refuse_local_trick()
        params = self.sample_params()
        target = self.base
        # an accelerated reference flow re-adopts its source's tensors when they change: swap the draw into
        # the source, which the accelerated flow then follows for the duration of the context
        source = self.base.__dict__.get("_source")
        if source is not None:
            target = source
        try:
            with torch.nn.utils.stateless._reparametrize_module(target, params):
                yield self.base
        finally:
            if source is not None:
                self.base.resync()  # back on the source's own parameters

    def _refuse_local_trick(self) -> None:
        for name, module in self.base.named_modules():
            if type(module) in _LOCAL_TRICK_TYPES and name.replace(".", "-") + "-weight" in self.means:
                raise NotImplementedError(
                    f"zuko_b200: the local reparameterization trick (layer {name!r}) is not implemented by the "
                    "engine; use reparameterize() to sample the weights"
                )

    def kl_divergence(self, prior_var: float = 1.0) -> Tensor:
        r"""Returns the KL divergence between the posterior and the prior ``N(0, prior_var)``."""
        kl = 0.0
        for key, mean in self.means.items():
            log_var = _softclip(self.logvars[key], 18.0)
            var = log_var.exp()
            kl = kl + 0.5 * (var / prior_var + mean.square() / prior_var + math.log(prior_var) - log_var - 1.0).sum()
        return kl

    def __getattr__(self, name: str) -> Any:  # noqa: ANN401
        r"""Looks attributes missing from the Bayesian model up in the base model."""
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self.base, name)
