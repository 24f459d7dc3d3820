r"""Mixture models: the Gaussian mixture model ``GMM`` (zuko/mixtures.py).

``GMM(c)`` returns a :class:`~zuko_b200.distributions.Mixture` whose ``log_prob``, its gradients and
``sample`` are engine calls (``zk_gmm_log_prob`` / ``zk_gmm_backward`` / ``zk_gmm_sample``).  The
conditioner ``MLP(context -> total)`` runs inside those calls.

Constructor, state-dict keys (``hyper.{2j}.weight`` / ``.bias`` or ``phi.{i}``), seeded initial tensors
and ``initialize`` follow the reference: ``initialize`` is torch plumbing that makes the reference's torch
calls in the reference's order, so that it gives the same tensors on the CPU bit for bit.

Covered shapes: up to 64 features and 32 components; others raise ``NotImplementedError`` at construction.
"""

from __future__ import annotations

__all__ = ["GMM"]

import ctypes
from collections.abc import Sequence
from math import prod
from typing import Literal

import torch
import torch.nn as nn
from torch import Tensor

from . import _engine as E
from .distributions import Mixture, _GMMCall
from .lazy import LazyDistribution
from .nn import MLP

COVARIANCE_CODES = {"full": E.ZK_COV_FULL, "diagonal": E.ZK_COV_DIAGONAL, "spherical": E.ZK_COV_SPHERICAL}


class GMM(LazyDistribution):
    r"""Creates a Gaussian mixture model (GMM).

    .. math:: p(X | c) = \sum_{i = 1}^K w_i(c) \, \mathcal{N}(X | \mu_i(c), \Sigma_i(c))

    Arguments:
        features: The number of features :math:`D` (at most 64).
        context: The number of context features.
        components: The number of components :math:`K` in the mixture (at most 32).
        covariance_type: The type of covariance matrix parameterization to use.
        tied: Whether to tie the covariance parameters across components.
        epsilon: A numerical stability term.
        kwargs: Keyword arguments passed to :class:`zuko_b200.nn.MLP`.
    """

    def __init__(
        self,
        features: int,
        context: int = 0,
        components: int = 2,
        covariance_type: Literal["full", "diagonal", "spherical"] = "full",
        tied: bool = False,
        epsilon: float = 1e-6,
        **kwargs,
    ) -> None:
        super().__init__()

        self.components = components
        self.covariance_type = covariance_type
        self.tied = tied
        self.epsilon = epsilon

        shapes = _gmm_shapes(components, features, covariance_type, tied)
        E.check(E.lib().zk_gmm_plan(features, components, COVARIANCE_CODES[covariance_type], int(tied),
                                    None, None, None, None, None))  # fmt: skip

        self.shapes = shapes
        self.total = sum(prod(s) for s in shapes)

        if context > 0:
            self.hyper = MLP(context, self.total, **kwargs)
        else:
            self.phi = nn.ParameterList(torch.randn(*s) for s in shapes)

    @property
    def features(self) -> int:
        return self.shapes[1][1]

    @property
    def context(self) -> int:
        return self.hyper.in_features if hasattr(self, "hyper") else 0

    def forward(self, c: Tensor | None = None) -> Mixture:
        if c is None and hasattr(self, "hyper"):
            raise ValueError("zuko_b200: a conditional GMM needs its context c")
        if c is not None and not hasattr(self, "hyper"):
            raise ValueError("zuko_b200: an unconditional GMM takes no context")
        if self.covariance_type not in COVARIANCE_CODES:
            raise NotImplementedError(f"Unknown covariance type '{self.covariance_type}'.")
        return Mixture(_GMMCall(self, c))

    # -- engine handle ---------------------------------------------------------------------------------------------
    def params(self) -> list[Tensor]:
        """The tensors the engine reads: the conditioner's weights and biases in layer order, or the ``phi``
        tensors."""
        if hasattr(self, "hyper"):
            return [t for m in self.hyper._linears() for t in (m.weight, m.bias) if t is not None]
        return list(self.phi)

    def _structure(self, params: Sequence[Tensor]) -> tuple:
        h = self.hyper
        flags = h._layer_flags()
        return (h.gemm_mode, h._activation_code(), flags, tuple((p.shape, p.device, p.dtype) for p in params))

    def _split(self, params: Sequence[Tensor]) -> tuple[list[Tensor], list[Tensor | None]]:
        """(weights, biases) of the conditioner's linear layers from the flat list ``params()``."""
        weights, biases, it = [], [], iter(params)
        for m in self.hyper._linears():
            weights.append(next(it))
            biases.append(next(it) if m.bias is not None else None)
        return weights, biases

    def handle(self, params: Sequence[Tensor]) -> ctypes.c_void_p:
        """The ``zk_gmm`` handle for these conditioner tensors (``params()`` at the time of a call).

        Keyed on the tensors' ``(data_ptr, _version)`` and holding their storage (``_engine.hold_storage``).
        New weights of the same structure (an optimizer step, a posterior draw) are copied into the
        existing handle with ``zk_gmm_update_weights``."""
        conditional = hasattr(self, "hyper")
        device = params[0].device
        structure = self._structure(params) if conditional else (device,)
        key = tuple((p.data_ptr(), p._version) for p in params) if conditional else ()
        cached = self.__dict__.get("_zk_cache")
        if cached is not None and cached[0] == structure and cached[1] == key:
            return cached[2]
        with torch.cuda.device(device):
            if cached is not None and cached[0] == structure:
                weights, biases = self._split([p.detach().contiguous() for p in params])
                W = (ctypes.c_void_p * len(weights))(*[w.data_ptr() for w in weights])
                Bv = (ctypes.c_void_p * len(biases))(*[None if b is None else b.data_ptr() for b in biases])
                E.check(E.lib().zk_gmm_update_weights(cached[2], W, Bv, E.stream_ptr(device)))
                self.__dict__["_zk_cache"] = (structure, key, cached[2], E.hold_storage([*weights, *biases]))
                return cached[2]
            self._release()
            h = ctypes.c_void_p()
            mlp = None
            if conditional:
                for p in params:
                    E.require_cuda(p, "GMM conditioner parameter")
                weights, biases = self._split(params)
                mlp, keep = self.hyper.mlp_desc(reindex=lambda i, n, w, b, mask: (weights[i].detach(), None if biases[i] is None else biases[i].detach(), mask))  # noqa: E501
                mlp = ctypes.pointer(mlp)
            desc = E.GmmDesc(self.features, self.context, self.components, COVARIANCE_CODES[self.covariance_type],
                             int(self.tied), self.epsilon, mlp)  # fmt: skip
            E.lib().zk_set_pack_stream(E.stream_ptr(device))  # the pack kernels wait for work queued on this stream
            try:
                E.check(E.lib().zk_gmm_create(ctypes.byref(desc), ctypes.byref(h)))
            finally:
                E.lib().zk_set_pack_stream(None)
        self.__dict__["_zk_cache"] = (structure, key, h, E.hold_storage(params) if conditional else [])
        return h

    def _release(self) -> None:
        cached = self.__dict__.pop("_zk_cache", None)
        if cached is not None:
            E.lib().zk_gmm_destroy(cached[2])

    def __del__(self) -> None:
        try:
            self._release()
        except Exception:
            pass

    def __getstate__(self):  # handles are not picklable (torch.save of the whole module)
        state = self.__dict__.copy()
        state.pop("_zk_cache", None)
        return state

    # -- initialisation (torch plumbing, no engine call) -----------------------------------------------------------
    @torch.no_grad()
    def initialize(self, x: Tensor, strategy: Literal["random", "kmeans", "kmeans++"]) -> None:
        r"""Initializes the components of the model from the samples ``x`` (N, D) clustered by ``strategy``:
        the mixture weights, means and covariances of the clusters become the unconditional parameters, or
        the bias of the conditioner's last layer (whose weight is scaled by :math:`10^{-2}`)."""
        N, _ = x.shape

        assert N > self.components, (
            f"The number of samples ({N}) should be larger than the number of components ({self.components})."
        )

        clusterings = {"random": _cluster_random, "kmeans": _cluster_kmeans, "kmeans++": _cluster_kmeans_pp}
        if strategy not in clusterings:
            raise NotImplementedError(f"Unknown clustering strategy '{strategy}'.")
        centers = clusterings[strategy](x, self.components)

        nearest = torch.cdist(x, centers).argmin(dim=-1)
        onehot = torch.nn.functional.one_hot(nearest, num_classes=self.components).to(dtype=x.dtype)

        weights = torch.sum(onehot, dim=0) / torch.sum(onehot)
        means = torch.sum(onehot[:, :, None] * x[:, None, :], dim=0) / torch.sum(onehot[:, :, None], dim=0)

        estimators = {"full": _full_covariance, "diagonal": _diagonal_covariance, "spherical": _spherical_covariance}
        if self.covariance_type not in estimators:
            raise NotImplementedError(f"Unknown covariance type '{self.covariance_type}'.")
        cov = estimators[self.covariance_type](x, onehot, self.tied)

        params = (weights.log(), means, *(cov if isinstance(cov, tuple) else (cov,)))

        assert all(p.shape == s for p, s in zip(params, self.shapes, strict=True))

        if hasattr(self, "hyper"):
            self.hyper[-1].weight.mul_(1e-2)
            self.hyper[-1].bias.copy_(torch.cat([p.flatten() for p in params]))
        else:
            for p, value in zip(self.phi, params, strict=True):
                p.copy_(value)


def _gmm_shapes(components: int, features: int, covariance_type: str, tied: bool) -> list[tuple[int, ...]]:
    """Parameter shapes in unpack order: logits (K,), loc (K, D), then the covariance's diagonal (L, D) or
    (L, 1) and, for a full covariance, its strict lower triangle (L, D (D - 1) / 2), L = 1 if tied else K."""
    L = 1 if tied else components
    covariance = {
        "full": [(L, features), (L, features * (features - 1) // 2)],
        "diagonal": [(L, features)],
        "spherical": [(L, 1)],
    }
    if covariance_type not in covariance:
        raise NotImplementedError(f"Unknown covariance type '{covariance_type}'.")
    return [(components,), (components, features), *covariance[covariance_type]]


def _full_covariance(x: Tensor, onehot: Tensor, tied: bool) -> tuple[Tensor, Tensor]:
    """Log-diagonal and strict lower triangle of the Cholesky factors of the clusters' weighted covariances."""
    D = x.shape[1]
    covs = torch.stack([torch.cov(x.T, aweights=onehot[:, k]) for k in range(onehot.shape[1])])
    if tied:
        covs = covs.mean(dim=0, keepdim=True)
    chol = torch.linalg.cholesky(covs)
    return torch.diagonal(chol, dim1=-2, dim2=-1).log(), chol[(..., *torch.tril_indices(D, D, offset=-1))]


def _diagonal_covariance(x: Tensor, onehot: Tensor, tied: bool) -> Tensor:
    """Log of the clusters' weighted per-feature variances (L, D)."""
    K, D = onehot.shape[1], x.shape[1]
    variances = torch.stack([torch.cov(x[:, d], aweights=onehot[:, k]) for k in range(K) for d in range(D)])
    variances = variances.reshape(K, D)
    if tied:
        variances = variances.mean(dim=0, keepdim=True)
    return variances.log()


def _spherical_covariance(x: Tensor, onehot: Tensor, tied: bool) -> Tensor:
    """Log of the mean per-feature variance (L, 1)."""
    return _diagonal_covariance(x, onehot, tied).exp().mean(dim=-1, keepdim=True).log()


def _cluster_random(x: Tensor, components: int) -> Tensor:
    """``components`` distinct samples drawn uniformly."""
    picks = torch.multinomial(torch.ones(x.shape[0], device=x.device), components)
    return x[picks]


def _cluster_kmeans(x: Tensor, components: int, iterations: int = 7) -> Tensor:
    """Lloyd's iterations from k-means++ seeds; a cluster left empty takes a fresh random sample."""
    N = x.shape[0]
    centers = _cluster_kmeans_pp(x, components)
    for _ in range(iterations):
        nearest = torch.cdist(x, centers).argmin(dim=-1)
        onehot = torch.nn.functional.one_hot(nearest, num_classes=components).to(dtype=x.dtype)
        picks = torch.multinomial(torch.ones(N, device=x.device), components)
        counts = torch.sum(onehot[:, :, None], dim=0)
        centers = torch.where(counts > 0, torch.sum(onehot[:, :, None] * x[:, None, :], dim=0) / counts, x[picks])
    return centers


def _cluster_kmeans_pp(x: Tensor, components: int) -> Tensor:
    """k-means++ seeding: each new center drawn with probability proportional to the squared distance to
    the nearest center chosen so far (a sample already chosen has distance 0)."""
    N = x.shape[0]
    picks = torch.multinomial(torch.ones(N, device=x.device), components)
    centers = x[picks]
    chosen = torch.zeros((N, components), dtype=torch.bool, device=x.device)
    chosen[picks, 0] = True
    for k in range(1, components):
        dist = torch.cdist(x, centers[:k])
        dist[chosen[:, :k]] = 0
        dist = dist.min(dim=-1).values
        pick = torch.multinomial(dist.square(), 1)
        centers[k] = x[pick]
        chosen[pick, k] = True
    return centers
