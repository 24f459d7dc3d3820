"""GPU tests of the Gaussian mixture model: every golden case of the unmodified reference
(tests/golden/make_golden_gmm.py) in both GEMM modes, sampling against the fp64 restatement
(tests/gmm_reference.py) and in distribution, the reference's own GMM properties, batch and stride edges, the
largest covered shape, reproducibility, chunking, ``accelerate``, ``BayesianModel`` draws and an Adam curve."""

import ctypes
import io

import gmm_reference as R
import numpy as np
import pytest
import torch
from cases import load
from gmm_cases import GMM_CASES, adam_batches, adam_curve, adam_model, build, inputs

import zuko_b200 as zuko
from zuko_b200 import _engine as E

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EPS = 1e-6


def set_mode(module, mode):
    for m in module.modules():
        if hasattr(m, "gemm_mode") and hasattr(m, "_linears"):
            m.gemm_mode = mode


def spec(name):
    _, args, kw, *_ = GMM_CASES[name]
    return args[0], kw.get("components", 2), kw.get("covariance_type", "full"), kw.get("tied", False)


def rel_to_max(ours, ref):
    return float(np.max(np.abs(ours - ref)) / max(np.max(np.abs(ref)), 1e-30))


def recorded(G, key):
    """A recorded fp64 gradient; a wide layer's weight gradient is stored as the reference's two factors, the
    layer's output gradient and its input (grad = gout^T @ input)."""
    if key in G:
        return G[key].astype(np.float64)
    return G[f"gout/{key}"].T @ G[f"input/{key}"]


@pytest.mark.parametrize("mode", ["fp32", "auto"])
@pytest.mark.parametrize("name", list(GMM_CASES))
def test_golden_log_prob_and_gradients(name, mode):
    G = load(f"gmm_{name}")
    gmm = build(zuko, name).to(DEV)
    set_mode(gmm, mode)
    x, c, w = inputs(name)
    x = x.to(DEV).requires_grad_()
    c = None if c is None else c.to(DEV).requires_grad_()
    lp = gmm(c).log_prob(x)
    assert lp.shape == tuple(G["lp"].shape)
    err32 = np.max(np.abs(G["lp32"] - G["lp"]) / np.maximum(np.abs(G["lp"]), 1.0))
    err = np.max(np.abs(lp.detach().cpu().double().numpy() - G["lp"]) / np.maximum(np.abs(G["lp"]), 1.0))
    assert err <= max(1e-5, 2 * err32), f"log_prob: {err:.3e}"
    (w.to(DEV) * lp).sum().backward()
    checks = [("gx", x.grad)] + ([("gc", c.grad)] if c is not None else [])
    checks += [(f"grad/{k}", p.grad) for k, p in gmm.named_parameters()]
    for key, t in checks:
        assert t is not None, key
        e = rel_to_max(t.detach().cpu().double().numpy(), recorded(G, key))
        bar = max(5e-5, 3 * float(G[f"err32/{key}"]))
        assert e <= bar, f"{key}: {e:.3e} > {bar:.3e}"


def table(gmm):
    return None if hasattr(gmm, "hyper") else torch.cat([p.detach().reshape(-1) for p in gmm.params()])


def ws_for(h, bytes_=None):
    n = bytes_ if bytes_ is not None else 256 << 20
    return torch.empty(n, dtype=torch.uint8, device=DEV)


def sample_raw(gmm, c, ldc, u, z, ws=None):
    h = gmm.handle(gmm.params())
    B, D = z.shape
    x = torch.empty(B, D, device=DEV)
    ws = ws if ws is not None else ws_for(h)
    t = table(gmm)
    E.check(E.lib().zk_gmm_sample(h, None if c is None else c.data_ptr(), ldc, None if t is None else t.data_ptr(),
                                  u.data_ptr(), z.data_ptr(), D, B, x.data_ptr(), D, ws.data_ptr(), ws.numel(),
                                  E.stream_ptr(DEV)))  # fmt: skip
    return x


@pytest.mark.parametrize("name", ["full_untied", "full_tied", "diagonal_untied", "spherical_tied", "uncond", "d1k1", "wide"])
def test_sample_against_restatement(name):
    G = load(f"gmm_{name}")
    D, K, cov, tied = spec(name)
    gmm = build(zuko, name).to(DEV)
    _, c, _ = inputs(name)
    g = torch.Generator().manual_seed(5)
    B = c.shape[0] if c is not None else 4096
    u = torch.rand(B, generator=g)
    z = torch.randn(B, D, generator=g)
    x = sample_raw(gmm, None if c is None else c.to(DEV), 0 if c is None else c.shape[-1], u.to(DEV), z.to(DEV))
    ref, _, margin = R.sample(G["phi"], u.double().numpy(), z.double().numpy(), D, K, cov, tied, EPS)
    ok = margin > 1e-6
    print(f"{name}: {int((~ok).sum())} of {B} rows within 1e-6 of a CDF boundary excluded")
    assert ok.mean() > 0.99
    np.testing.assert_allclose(x.cpu().double().numpy()[ok], ref[ok], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("cov,tied", [("full", False), ("diagonal", True), ("spherical", False)])
def test_sample_statistics(cov, tied):
    """2^20 samples: component frequencies, means and covariances against the analytic ones."""
    torch.manual_seed(0)
    gmm = zuko.mixtures.GMM(3, components=3, covariance_type=cov, tied=tied).to(DEV)
    n = 1 << 20
    torch.manual_seed(1)
    x = gmm().sample((n,)).double().cpu().numpy()
    phi = table(gmm).double().cpu().numpy()
    logits = phi[:3]
    p = np.exp(logits - logits.max())
    p /= p.sum()
    loc, L = R.scale_tril(phi, 3, 3, cov, tied, EPS)
    covs = L @ np.swapaxes(L, -1, -2)
    mean = (p[:, None] * loc).sum(0)
    cov_total = (p[:, None, None] * (covs + loc[:, :, None] * loc[:, None, :])).sum(0) - np.outer(mean, mean)
    sd = np.sqrt(np.diag(cov_total))
    # means within 6 standard errors; covariances within 18 sqrt(3) sd_i sd_j / sqrt(n), a loose bar on the
    # standard error of a product moment
    assert np.all(np.abs(x.mean(0) - mean) <= 6 * sd / np.sqrt(n))
    emp = np.cov(x.T)
    assert np.all(np.abs(emp - cov_total) <= 6 * np.sqrt(3.0) * np.outer(sd, sd) / np.sqrt(n) * 3)
    # component frequencies: the sampler's choice depends on u alone, so with z = 0 every draw lands on its
    # component's mean, which identifies it
    u = torch.rand(n, device=DEV)
    z = torch.zeros(n, 3, device=DEV)
    xs = sample_raw(gmm, None, 0, u, z).double().cpu().numpy()
    k = np.argmin(np.abs(xs[:, None, :] - loc[None]).sum(-1), axis=1)
    freq = np.bincount(k, minlength=3) / n
    assert np.all(np.abs(freq - p) <= 6 * np.sqrt(p * (1 - p) / n))


@pytest.mark.parametrize("context", [0, 5])
@pytest.mark.parametrize("batch", [(), (4,)])
@pytest.mark.parametrize("cov", ["full", "diagonal", "spherical"])
@pytest.mark.parametrize("tied", [False, True])
def test_reference_properties_shapes(context, batch, cov, tied):
    gmm = zuko.mixtures.GMM(3, context, components=2, covariance_type=cov, tied=tied).to(DEV)
    c = torch.randn(*batch, context, device=DEV) if context else None
    batch = batch if context else ()
    d = gmm(c)
    assert d.batch_shape == batch and d.event_shape == (3,)
    assert d.logits.shape == (*batch, 2)
    if cov == "full":
        assert d.base.loc.shape == (*batch, 2, 3)
        assert d.base.covariance_matrix.shape == (*batch, 2, 3, 3)
    else:
        assert d.base.base_dist.loc.shape == (*batch, 2, 3)
        assert d.base.base_dist.scale.shape == (*batch, 2, 3)
    if context == 0 and tied:
        covs = d.base.covariance_matrix if cov == "full" else d.base.base_dist.scale
        assert torch.allclose(covs[0], covs[1])


def test_reference_properties_training_sampling_saving(tmp_path):
    gmm = zuko.mixtures.GMM(3, 5).to(DEV)
    x, c = torch.randn(256, 3, device=DEV), torch.randn(5, device=DEV)
    lp = gmm(c).log_prob(x)
    assert lp.shape == (256,) and lp.requires_grad
    gmm.zero_grad(set_to_none=True)
    (-lp.mean()).backward()
    for name, p in gmm.named_parameters():
        assert p.grad is not None, name
    assert gmm(c).sample((32,)).shape == (32, 3)
    assert not gmm(c).has_rsample
    with pytest.raises(NotImplementedError):
        gmm(c).rsample()
    buf = io.BytesIO()
    torch.save(gmm, buf)
    buf.seek(0)
    bis = torch.load(buf, weights_only=False)
    x, c = torch.randn(3, device=DEV), torch.randn(5, device=DEV)
    assert torch.allclose(gmm(c).log_prob(x), bis(c).log_prob(x))
    assert repr(gmm) and repr(gmm(c)).startswith("Mixture(MultivariateNormal(")


def test_empty_batch_broadcast_context_and_padded_strides():
    torch.manual_seed(0)
    gmm = zuko.mixtures.GMM(3, 5, components=3).to(DEV)
    h = gmm.handle(gmm.params())
    ws = ws_for(h)
    out = torch.full((1,), 7.0, device=DEV)
    E.check(E.lib().zk_gmm_log_prob(h, None, 3, torch.zeros(1, 5, device=DEV).data_ptr(), 5, None, 0, out.data_ptr(),
                                    ws.data_ptr(), ws.numel(), E.stream_ptr(DEV)))  # fmt: skip
    assert out.item() == 7.0
    assert gmm(torch.randn(5, device=DEV)).log_prob(torch.randn(0, 3, device=DEV)).shape == (0,)
    x = torch.randn(300, 3, device=DEV)
    c = torch.randn(5, device=DEV)
    ref = gmm(c.expand(300, 5)).log_prob(x)
    assert torch.allclose(gmm(c).log_prob(x), ref, rtol=1e-6, atol=1e-6)
    # padded rows: x with row stride 8, c with row stride 9
    xp = torch.zeros(300, 8, device=DEV)
    xp[:, :3] = x
    cp = torch.zeros(300, 9, device=DEV)
    cp[:, :5] = c
    lp = torch.empty(300, device=DEV)
    E.check(E.lib().zk_gmm_log_prob(h, xp.data_ptr(), 8, cp.data_ptr(), 9, None, 300, lp.data_ptr(), ws.data_ptr(),
                                    ws.numel(), E.stream_ptr(DEV)))  # fmt: skip
    torch.testing.assert_close(lp, ref, rtol=0, atol=0)
    gx = torch.zeros(300, 7, device=DEV)
    gc = torch.zeros(300, 9, device=DEV)
    g = torch.ones(300, device=DEV)
    grads = E.LayerGrads(None, None, None, None)
    E.check(E.lib().zk_gmm_backward(h, xp.data_ptr(), 8, cp.data_ptr(), 9, None, 300, g.data_ptr(), gx.data_ptr(), 7,
                                    gc.data_ptr(), 9, ctypes.byref(grads), ws.data_ptr(), ws.numel(), E.stream_ptr(DEV)))  # fmt: skip
    xr, cr = x.clone().requires_grad_(), c.expand(300, 5).clone().requires_grad_()
    gmm(cr).log_prob(xr).sum().backward()
    torch.testing.assert_close(gx[:, :3], xr.grad, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(gc[:, :5], cr.grad, rtol=1e-5, atol=1e-5)
    assert gx[:, 3:].abs().max().item() == 0 and gc[:, 5:].abs().max().item() == 0


@pytest.mark.parametrize("cov", ["full", "diagonal", "spherical"])
def test_largest_covered_shape(cov):
    D, K = 64, 32
    torch.manual_seed(0)
    gmm = zuko.mixtures.GMM(D, components=K, covariance_type=cov).to(DEV)
    with torch.no_grad():
        for p in gmm.phi[2:]:
            p.mul_(0.1)
    x = torch.randn(1000, D, device=DEV).requires_grad_()
    lp = gmm().log_prob(x)
    phi = table(gmm).double().cpu().numpy()
    xn = x.detach().double().cpu().numpy()
    ref = R.log_prob(xn, phi, D, K, cov, False, EPS)
    assert np.max(np.abs(lp.detach().cpu().double().numpy() - ref) / np.maximum(np.abs(ref), 1.0)) <= 1e-4
    lp.sum().backward()
    gx, gphi = R.grads(xn, phi, np.ones(1000), D, K, cov, False, EPS)
    assert rel_to_max(x.grad.double().cpu().numpy(), gx) <= 1e-4
    ours = torch.cat([p.grad.reshape(-1) for p in gmm.phi]).double().cpu().numpy()
    assert rel_to_max(ours, gphi.sum(0)) <= 1e-4


def test_bitwise_repeat_and_chunked_workspace():
    torch.manual_seed(0)
    gmm = zuko.mixtures.GMM(8, 4, components=5, hidden_features=[64, 64]).to(DEV)
    B = 5000
    x, c = torch.randn(B, 8, device=DEV), torch.randn(B, 4, device=DEV)

    def run(ws_bytes):
        h = gmm.handle(gmm.params())
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
        lp = torch.empty(B, device=DEV)
        E.check(E.lib().zk_gmm_log_prob(h, x.data_ptr(), 8, c.data_ptr(), 4, None, B, lp.data_ptr(), ws.data_ptr(),
                                        ws_bytes, E.stream_ptr(DEV)))  # fmt: skip
        gx = torch.empty(B, 8, device=DEV)
        gw = [torch.zeros_like(m.weight) for m in gmm.hyper._linears()]
        W = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in gw])
        grads = E.LayerGrads(ctypes.cast(W, ctypes.POINTER(ctypes.c_void_p)), None, None, None)
        g = torch.ones(B, device=DEV)
        E.check(E.lib().zk_gmm_backward(h, x.data_ptr(), 8, c.data_ptr(), 4, None, B, g.data_ptr(), gx.data_ptr(), 8,
                                        None, 0, ctypes.byref(grads), ws.data_ptr(), ws_bytes, E.stream_ptr(DEV)))  # fmt: skip
        torch.cuda.synchronize()
        return lp, gx, gw

    h = gmm.handle(gmm.params())
    full = max(E.lib().zk_gmm_workspace_bytes(h, B), E.lib().zk_gmm_backward_workspace_bytes(h, B))
    small = E.lib().zk_gmm_min_workspace_bytes(h) + E.lib().zk_gmm_backward_workspace_bytes(h, 700) // 2
    assert E.lib().zk_gmm_chunk_rows(h, B, 1, small) < B
    a, b, s = run(full), run(full), run(small)
    for t1, t2 in zip([a[0], a[1], *a[2]], [b[0], b[1], *b[2]], strict=True):
        assert torch.equal(t1, t2)
    torch.testing.assert_close(s[0], a[0], rtol=0, atol=0)  # rows are independent
    torch.testing.assert_close(s[1], a[1], rtol=0, atol=0)
    for t1, t2 in zip(s[2], a[2], strict=True):
        torch.testing.assert_close(t1, t2, rtol=1e-5, atol=1e-5 * t2.abs().max().item())


def test_accelerate_reference_gmm():
    """The engine's GMM stands in for the reference's class (recognised by class name)."""
    torch.manual_seed(0)
    ref = zuko.mixtures.GMM(3, 5, components=3, covariance_type="diagonal").to(DEV)
    acc = zuko.accelerate(ref)
    assert acc is not ref and isinstance(acc, zuko.mixtures.GMM)
    for (k1, p1), (k2, p2) in zip(ref.named_parameters(), acc.named_parameters(), strict=True):
        assert k1 == k2 and p1 is p2
    x, c = torch.randn(100, 3, device=DEV), torch.randn(100, 5, device=DEV)
    torch.testing.assert_close(acc(c).log_prob(x), ref(c).log_prob(x), rtol=0, atol=0)
    uncond = zuko.mixtures.GMM(3, components=2).to(DEV)
    assert [p is q for p, q in zip(uncond.parameters(), zuko.accelerate(uncond).parameters(), strict=True)] == [True] * 4
    with pytest.raises(TypeError):
        zuko.accelerate(torch.nn.Linear(2, 2))


def test_bayesian_draws_are_never_stale():
    from zuko_b200.bayesian import BayesianModel

    torch.manual_seed(0)
    model = BayesianModel(zuko.mixtures.GMM(3, 5, components=3), init_logvar=-2.0).to(DEV)
    x, c = torch.randn(200, 3, device=DEV), torch.randn(200, 5, device=DEV)
    draws = []
    for seed in (1, 2, 1):
        torch.manual_seed(seed)
        with model.reparameterize() as gmm:
            draws.append(gmm(c).log_prob(x).detach().clone())
    assert not torch.equal(draws[0], draws[1])
    assert torch.equal(draws[0], draws[2])
    torch.manual_seed(1)
    with model.reparameterize() as gmm:
        (-gmm(c).log_prob(x).mean()).backward()
    for name, p in [*model.means.items(), *model.logvars.items()]:
        assert p.grad is not None and torch.isfinite(p.grad).all(), name


def test_adam_curve_matches_reference():
    ref = load("gmm_adam")["losses"]
    gmm = adam_model(zuko).to(DEV)
    set_mode(gmm, "fp32")
    ours = np.array(adam_curve(gmm, adam_batches(), DEV))
    assert np.max(np.abs(ours - ref)) <= 1e-3, np.abs(ours - ref)
