"""CPU tests of the Gaussian mixture model: the fp64 restatement (tests/gmm_reference.py) against the reference's
goldens (tests/golden/make_golden_gmm.py), the kernels' row math (zuko_b200/csrc/gmm_math.cuh, compiled by g++)
against the restatement, constructor / state-dict / initialize parity with the reference, its error messages,
the refusals beyond the covered shapes and the launch plan."""

import ctypes
import subprocess
from pathlib import Path

import gmm_reference as R
import numpy as np
import pytest
import torch
from cases import crc, load
from gmm_cases import GMM_CASES, INIT_CASES, build, init_data

import zuko_b200 as zuko
from zuko_b200 import _engine as E
from zuko_b200.distributions import Mixture

ROOT = Path(__file__).resolve().parent.parent
_P = ctypes.c_void_p
EPS = 1e-6


def spec(name: str) -> tuple[int, int, str, bool]:
    """(D, K, covariance, tied) of a golden case."""
    _, args, kw, *_ = GMM_CASES[name]
    return args[0], kw.get("components", 2), kw.get("covariance_type", "full"), kw.get("tied", False)


def rows(name: str) -> tuple[np.ndarray, np.ndarray, np.ndarray, bool]:
    """(x (B, D), phi (B, P) or (P,), w (B,), shared) of a golden case, fp64."""
    G = load(f"gmm_{name}")
    D = spec(name)[0]
    x, phi, w = G["x"].astype(np.float64), G["phi"], G["w"].astype(np.float64)
    lead = np.broadcast_shapes(x.shape[:-1], phi.shape[:-1], w.shape)
    shared = phi.ndim == 1
    x2 = np.broadcast_to(x, (*lead, D)).reshape(-1, D)
    phi2 = phi if shared else np.broadcast_to(phi, (*lead, phi.shape[-1])).reshape(-1, phi.shape[-1])
    return x2, phi2, np.broadcast_to(w, lead).reshape(-1), shared


def sum_rows(gphi: np.ndarray, name: str) -> np.ndarray:
    """Per-sample phi gradients reduced to the shape of the golden's phi."""
    G = load(f"gmm_{name}")
    phi = G["phi"]
    if phi.ndim == 1:
        return gphi.sum(0)
    lead = np.broadcast_shapes(G["x"].shape[:-1], phi.shape[:-1])
    g = gphi.reshape(*lead, -1)
    return g.sum(axis=tuple(range(len(lead) - (phi.ndim - 1))))


@pytest.mark.parametrize("name", list(GMM_CASES))
def test_restatement_against_reference(name):
    G = load(f"gmm_{name}")
    D, K, cov, tied = spec(name)
    x, phi, w, _ = rows(name)
    lp = R.log_prob(x, phi, D, K, cov, tied, EPS)
    ref = G["lp"].reshape(-1)
    assert np.max(np.abs(lp - ref) / np.maximum(np.abs(ref), 1.0)) <= 1e-10
    gx, gphi = R.grads(x, phi, w, D, K, cov, tied, EPS)
    for ours, theirs, what in ((gx.reshape(G["gx"].shape) if G["x"].ndim == 2 else None, G["gx"], "gx"),
                               (sum_rows(gphi, name), G["gphi"], "gphi")):  # fmt: skip
        if ours is None:  # x broadcast against a batched context: compare the summed gradient
            ours = gx.reshape(*np.broadcast_shapes(G["x"].shape[:-1], G["phi"].shape[:-1]), D).reshape(G["gx"].shape)
        err = np.max(np.abs(ours - theirs)) / max(np.max(np.abs(theirs)), 1e-300)
        assert err <= 1e-10, f"{what}: {err:.3e}"


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libgmm_host.so"
    src = ROOT / "tests" / "native" / "gmm_math_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so), "-lm"], check=True)
    return ctypes.CDLL(str(so))


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(_P)


def _args(D, K, cov, tied):
    return [ctypes.c_int(D), ctypes.c_int(K), ctypes.c_int(R.COV[cov]), ctypes.c_int(int(tied)), ctypes.c_float(EPS)]


@pytest.mark.parametrize("name", list(GMM_CASES))
def test_row_math_against_restatement(harness, name):
    D, K, cov, tied = spec(name)
    x, phi, w, shared = rows(name)
    x32, phi32, w32 = (np.ascontiguousarray(a, np.float32) for a in (x, phi, w))
    B, P = x.shape[0], phi.shape[-1]
    ld = 0 if shared else P
    out = np.empty(B, np.float32)
    harness.gmm_log_prob_rows(_ptr(x32), _ptr(phi32), ctypes.c_int64(ld), ctypes.c_int64(B), *_args(D, K, cov, tied), _ptr(out))
    # the restatement on the fp32-rounded inputs
    xr, pr = x32.astype(np.float64), phi32.astype(np.float64)
    ref = R.log_prob(xr, pr, D, K, cov, tied, EPS)
    assert np.max(np.abs(out - ref) / np.maximum(np.abs(ref), 1.0)) <= 2e-5
    gx = np.empty((B, D), np.float32)
    gphi = np.empty((B, P), np.float32)
    harness.gmm_backward_rows(_ptr(x32), _ptr(phi32), ctypes.c_int64(ld), ctypes.c_int64(B), *_args(D, K, cov, tied), _ptr(w32),
                              _ptr(gx), _ptr(gphi))  # fmt: skip
    rgx, rgphi = R.grads(xr, pr, w32.astype(np.float64), D, K, cov, tied, EPS)
    for ours, theirs, what in ((gx, rgx, "gx"), (gphi, rgphi, "gphi")):
        scale = np.maximum(np.abs(theirs).max(axis=-1, keepdims=True), 1.0)
        err = np.max(np.abs(ours - theirs) / scale)
        assert err <= 5e-5 if name != "illcond" else 2e-4, f"{what}: {err:.3e}"


@pytest.mark.parametrize("name", ["full_untied", "diagonal_tied", "spherical_untied", "uncond", "d1k1"])
def test_row_sample_against_restatement(harness, name):
    D, K, cov, tied = spec(name)
    _, phi, _, shared = rows(name)
    g = np.random.default_rng(0)
    B = 4096 if shared else phi.shape[0]
    phi32 = np.ascontiguousarray(phi, np.float32)
    u = g.random(B).astype(np.float32)
    z = g.standard_normal((B, D)).astype(np.float32)
    x = np.empty((B, D), np.float32)
    harness.gmm_sample_rows(_ptr(phi32), ctypes.c_int64(0 if shared else phi.shape[-1]), _ptr(u), _ptr(z), ctypes.c_int64(B),
                            *_args(D, K, cov, tied), _ptr(x))  # fmt: skip
    ref, _, margin = R.sample(phi32.astype(np.float64), u.astype(np.float64), z.astype(np.float64), D, K, cov, tied, EPS)
    ok = margin > 1e-6
    assert ok.mean() > 0.99
    np.testing.assert_allclose(x[ok], ref[ok], rtol=1e-5, atol=1e-5)


def selection_uniforms(logits: np.ndarray) -> np.ndarray:
    """u at 0, 2^-24, 1/2, the fp32 running sums of softmax(logits) and 1 - j 2^-24 for j = 1..64: the values
    where the running sum's rounding decides the component (those below 1: u is drawn from [0, 1))."""
    p = np.exp(logits.astype(np.float64) - logits.max())
    p32 = (p / p.sum()).astype(np.float32)
    sums = np.cumsum(p32, dtype=np.float32)[:-1]
    top = 1.0 - np.arange(1, 65) * 2.0**-24
    u = np.concatenate([[0.0, 2.0**-24, 0.5], sums, top]).astype(np.float32)
    return u[u < 1]


def check_selection(logits: np.ndarray, u: np.ndarray, k: np.ndarray, what: str, floor: float = 1e-30) -> None:
    """Each draw k has an fp64 weight of at least `floor` and u lies in its fp64 CDF interval, up to the rounding of
    the fp32 running sum (K 2^-23).  At u = 0 the inverse CDF takes the first component, whatever its weight."""
    K = logits.size
    p = np.exp(logits.astype(np.float64) - logits.max())
    p /= p.sum()
    hi = np.cumsum(p)
    lo = hi - p
    tol = K * 2.0**-23
    ok = (lo[k] - tol <= u) & (u < hi[k] + tol) & ((p[k] >= floor) | ((u == 0) & (k == 0)))
    assert ok.all(), f"{what}: u {u[~ok].tolist()} drew {k[~ok].tolist()} (weights {p[k[~ok]].tolist()})"


@pytest.mark.parametrize("K", range(2, 33))
def test_select_component_never_draws_a_zero_weight(harness, K):
    """K - 1 equal logits and one at -200 or -1e4 (fp32 weight 0: exp(-200) is 1e-87) last, first or in the
    middle, through select_component and row_sample (D = 1, means 10 k, z = 0, so x names the component).
    Rounding leaves the fp32 running sum of the first K - 1 weights below u = 1 - 2^-24 for several K (6, 12,
    16, 24 with glibc's expf); the last component must then not be drawn when its weight is zero."""
    harness.gmm_select_component.restype = ctypes.c_int
    for dead in (-200.0, -1e4):
        for at in sorted({K - 1, 0, K // 2}):
            logits = np.zeros(K, np.float32)
            logits[at] = dead
            u = selection_uniforms(logits)
            k = np.array([harness.gmm_select_component(_ptr(logits), K, ctypes.c_float(v)) for v in u])
            check_selection(logits, u, k, f"K={K} dead={dead} at {at}")
            phi = np.concatenate([logits, 10.0 * np.arange(K), np.zeros(K)]).astype(np.float32)  # diagonal, untied
            z = np.zeros((u.size, 1), np.float32)
            x = np.empty((u.size, 1), np.float32)
            harness.gmm_sample_rows(_ptr(phi), ctypes.c_int64(0), _ptr(u), _ptr(z), ctypes.c_int64(u.size),
                                    *_args(1, K, "diagonal", False), _ptr(x))  # fmt: skip
            np.testing.assert_array_equal(x[:, 0], 10.0 * k)


@pytest.mark.parametrize("name", list(GMM_CASES))
def test_constructor_and_state_dict_match_reference(name):
    G = load(f"gmm_{name}")
    gmm = build(zuko, name)
    assert list(gmm.state_dict().keys()) == list(G["keys"])
    assert [crc(t) for t in gmm.state_dict().values()] == list(G["crc"])


def test_flows_export_the_mixture():
    from zuko_b200.flows.mixture import GMM

    assert zuko.flows.GMM is zuko.mixtures.GMM is GMM


@pytest.mark.parametrize("name", list(INIT_CASES))
def test_initialize_is_bit_identical_to_reference(name):
    I = load("gmm_init")
    gmm = build(zuko, name)
    torch.manual_seed(11)
    gmm.initialize(init_data(), INIT_CASES[name][3])
    for k, t in gmm.state_dict().items():
        np.testing.assert_array_equal(t.numpy(), I[f"{name}/{k}"], err_msg=k)


def test_reference_error_messages():
    gmm = zuko.mixtures.GMM(features=3, components=7, covariance_type="full")
    with pytest.raises(AssertionError, match="The number of samples"):
        gmm.initialize(torch.randn(6, 3), strategy="random")
    gmm = zuko.mixtures.GMM(features=3, components=2, covariance_type="full")
    with pytest.raises(NotImplementedError, match="Unknown clustering strategy"):
        gmm.initialize(torch.randn(16, 3), strategy="invalid")
    with pytest.raises(NotImplementedError, match="Unknown covariance type"):
        zuko.mixtures.GMM(features=3, components=2, covariance_type="invalid")
    gmm.covariance_type = "invalid"
    with pytest.raises(NotImplementedError, match="Unknown covariance type"):
        gmm.initialize(torch.randn(16, 3), strategy="random")


@pytest.mark.parametrize("features,components", [(65, 2), (3, 33), (0, 2), (3, 0)])
def test_shapes_beyond_the_plan_are_refused(features, components):
    with pytest.raises(NotImplementedError, match="outside the covered"):
        zuko.mixtures.GMM(features, 4, components=components)


def test_mixture_over_other_bases_is_refused():
    base = torch.distributions.Normal(torch.zeros(2), torch.ones(2))
    with pytest.raises(NotImplementedError):
        Mixture(base, torch.zeros(2))


def plan_restated(D: int, K: int, cov: int, tied: int) -> tuple[int, int, int, int, int]:
    T = 128
    while T > 32 and T * (2 * D + K) * 4 > 48 * 1024:
        T //= 2
    return T, T, T * (D + K) * 4, T * (2 * D + K) * 4, cov * 2 + tied


@pytest.mark.parametrize("D,K", [(1, 1), (3, 2), (16, 8), (33, 17), (64, 1), (40, 32), (64, 32)])
@pytest.mark.parametrize("cov", ["full", "diagonal", "spherical"])
@pytest.mark.parametrize("tied", [False, True])
def test_plan_restated(D, K, cov, tied):
    c = R.COV[cov]
    threads, rows_, instantiated = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    s1, s2 = ctypes.c_size_t(), ctypes.c_size_t()
    E.check(E.lib().zk_gmm_plan(D, K, c, int(tied), ctypes.byref(threads), ctypes.byref(rows_), ctypes.byref(s1),
                                ctypes.byref(s2), ctypes.byref(instantiated)))  # fmt: skip
    assert (threads.value, rows_.value, s1.value, s2.value, instantiated.value) == plan_restated(D, K, c, int(tied))
    assert s2.value <= 48 * 1024
    assert E.lib().zk_gmm_params_per_row(D, K, c, int(tied)) == R.total(D, K, cov, tied)


def test_plan_refusals():
    assert E.lib().zk_gmm_plan(65, 2, 0, 0, None, None, None, None, None) == E.ZK_EUNSUPPORTED
    assert E.lib().zk_gmm_plan(3, 33, 0, 0, None, None, None, None, None) == E.ZK_EUNSUPPORTED
    assert E.lib().zk_gmm_plan(3, 2, 3, 0, None, None, None, None, None) == E.ZK_EINVAL
