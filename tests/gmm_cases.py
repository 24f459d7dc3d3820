"""Cases of the Gaussian mixture goldens (tests/golden/make_golden_gmm.py), shared by the CPU and GPU tests.
Each builder takes the package (the reference's ``zuko`` or ``zuko_b200``) so that both sides construct the
same model under the same seed."""

from __future__ import annotations

import torch

# name -> (seed, GMM args, GMM kwargs, x shape, c shape or None)
GMM_CASES = {
    **{
        f"{cov}_{'tied' if tied else 'untied'}": (0, (3, 5), dict(covariance_type=cov, tied=tied), (64, 3), (64, 5))
        for cov in ("full", "diagonal", "spherical")
        for tied in (False, True)
    },
    "uncond": (1, (3,), dict(components=3), (64, 3), None),
    "wide": (2, (16, 8), dict(components=8, hidden_features=[256] * 3), (8, 16), (8, 8)),
    "bcast": (3, (3, 5), {}, (64, 3), (5,)),
    "batched": (4, (3, 5), {}, (256, 4, 3), (4, 5)),
    "d1k1": (5, (1, 2), dict(components=1), (64, 1), (64, 2)),
    "illcond": (6, (4, 3), dict(components=3), (128, 4), (128, 3)),
}

INIT_CASES = {  # name -> (seed, GMM args, GMM kwargs, strategy)
    f"init_{tag}_{s.replace('+', 'p')}": (7, args, kw, s)
    for s in ("random", "kmeans", "kmeans++")
    for tag, args, kw in (("uncond", (3,), dict(components=3)), ("cond", (3, 5), dict(covariance_type="diagonal", tied=True)))
}

ADAM_STEPS = 30


def build(zuko, name: str):  # noqa: ANN001, ANN201
    """The case's model, in fp32, built under its seed."""
    seed, args, kw, *_ = GMM_CASES[name] if name in GMM_CASES else INIT_CASES[name]
    torch.manual_seed(seed)
    gmm = zuko.mixtures.GMM(*args, **kw)
    if name == "illcond":  # an ill-conditioned scale: the off-diagonal outputs of the conditioner x3
        with torch.no_grad():
            at = sum(s[0] * (s[1] if len(s) > 1 else 1) for s in gmm.shapes[:3])
            gmm.hyper[-1].weight[at:] *= 3
            gmm.hyper[-1].bias[at:] *= 3
    return gmm


def inputs(name: str) -> tuple[torch.Tensor, torch.Tensor | None, torch.Tensor]:
    """(x, c, w) of a case in fp32: samples, context, and the weights of the gradient target sum(w * log_prob)."""
    _, _, _, xs, cs = GMM_CASES[name]
    g = torch.Generator().manual_seed(100)
    x = torch.randn(*xs, generator=g) * 1.5
    c = None if cs is None else torch.randn(*cs, generator=g)
    w = torch.rand(*torch.broadcast_shapes(xs[:-1], () if cs is None else cs[:-1]), generator=g) + 0.5
    return x, c, w


def init_data() -> torch.Tensor:
    g = torch.Generator().manual_seed(200)
    return torch.cat([torch.randn(100, 3, generator=g) + 3, torch.randn(150, 3, generator=g) * 0.5 - 2])


def adam_model(zuko):  # noqa: ANN001, ANN201
    torch.manual_seed(8)
    return zuko.mixtures.GMM(2, 2, components=4, hidden_features=[32, 32])


def adam_batches() -> list[tuple[torch.Tensor, torch.Tensor]]:
    """Seeded conditional data: x = a rotation of c-shifted blobs."""
    g = torch.Generator().manual_seed(300)
    out = []
    for _ in range(ADAM_STEPS):
        c = torch.randn(256, 2, generator=g)
        k = torch.randint(0, 3, (256, 1), generator=g).float()
        x = torch.cat([c[:, :1] + k, c[:, 1:] * 0.5 - k], dim=1) + 0.3 * torch.randn(256, 2, generator=g)
        out.append((x, c))
    return out


def adam_curve(gmm, batches, device=None) -> list[float]:  # noqa: ANN001
    opt = torch.optim.Adam(gmm.parameters(), lr=1e-2)
    losses = []
    for x, c in batches:
        if device is not None:
            x, c = x.to(device), c.to(device)
        loss = -gmm(c).log_prob(x).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return losses
