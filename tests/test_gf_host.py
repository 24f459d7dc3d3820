"""CPU tests of the Gaussianization flow (GF): the fp64 restatement of tests/gf_reference.py against the
reference's goldens (tests/golden/make_golden_gf.py), the per-pair reverse-mode math of
zuko_b200/csrc/bijector_grad.cuh compiled by g++, constructor parity with the reference under the same
seed, and the layers that refuse the bijector."""

import ctypes
import subprocess
from functools import partial
from pathlib import Path

import numpy as np
import pytest
import torch

import gf_reference as R
from cases import crc, load
from zuko_b200 import _engine as E
from zuko_b200.flows import GF, GeneralCouplingTransform, MaskedAutoregressiveTransform
from zuko_b200.flows._packed import resolve_univariate
from zuko_b200.transforms import GaussianizationTransform

ROOT = Path(__file__).resolve().parent.parent
UG = load("units_gf")
UNIT_TAGS = ["k1", "k8", "k16", "shared8", "partial8"]

# name -> (constructor, components); must mirror tests/golden/make_golden_gf.py:CASES
GF_CASES = {
    "gf53": (lambda: GF(5, 3, hidden_features=[32, 32]), 8),
    "gf35_row": (lambda: GF(3, 5), 8),
    "gf6_uncond": (lambda: GF(6, 0, transforms=4, components=16), 16),
    "gf53_stress": (lambda: GF(5, 3, hidden_features=[32, 32]), 8),
    "gf16_wide": (lambda: GF(16, 8, components=8, hidden_features=[256] * 3), 8),
}


def build_gf(name: str):
    torch.manual_seed(0)
    return GF_CASES[name][0]().eval()


def reference_of(name: str, flow) -> R.Flow:
    sd = {k: v.detach().numpy() for k, v in flow.state_dict().items()}
    t0 = flow.transform.transforms[0]
    return R.Flow(sd, t0.features, t0.context, GF_CASES[name][1])


def rel(ours, ref):
    ours, ref = np.asarray(ours, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(ours - ref) / np.maximum(np.abs(ref), 1.0)))


@pytest.mark.parametrize("name", list(GF_CASES))
def test_constructor_matches_reference_state_dict(name):
    g = load(f"flow_{name}")
    sd = build_gf(name).state_dict()
    assert list(sd.keys()) == [str(k) for k in g["sd_keys"]]
    assert [crc(v) for v in sd.values()] == [int(v) for v in g["sd_crc"]]
    for k, v in g.items():
        if k.startswith("sd/"):
            np.testing.assert_array_equal(sd[k[3:]].numpy(), v)


def test_rotation_generators_are_parameters():
    flow = GF(4, 0, transforms=3)
    names = [n for n, _ in flow.named_parameters()]
    assert "transform.transforms.1.A" in names and "transform.transforms.3.A" in names
    assert "transform.transforms.0.phi.0" in names and "transform.transforms.0.phi.1" in names


@pytest.mark.parametrize("name", list(GF_CASES))
def test_fp64_restatement_against_goldens(name):
    g = load(f"flow_{name}")
    ref = reference_of(name, build_gf(name))
    c = g.get("c")
    assert rel(ref.log_prob(g["x"], c), g["log_prob64"]) < 1e-10
    z, ladj = ref.call_and_ladj(g["x"], c)
    assert rel(z, g["z64"]) < 1e-10
    assert rel(ladj, g["ladj64"]) < 1e-10
    ci = None if c is None else (c if c.ndim == 1 else c[: g["zin"].shape[0]])
    np.testing.assert_allclose(ref.inverse(g["zin"], ci), g["xinv64"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_unit_forward_inverse_and_gradients(tag):
    shift, scale, x, z = UG[f"{tag}_shift"], UG[f"{tag}_scale"], UG[f"{tag}_x"], UG[f"{tag}_z"]
    y, ladj = R.forward(x, shift, scale)
    assert rel(y, UG[f"{tag}_y64"]) < 1e-12
    assert rel(ladj, UG[f"{tag}_ladj64"]) < 1e-10
    bound, eps = float(UG[f"{tag}_bound"]), float(UG[f"{tag}_eps"])
    np.testing.assert_array_equal(R.inverse(z, shift, scale, bound, eps), UG[f"{tag}_xinv64"])
    gx, gs, ga = R.grad(x, shift, scale, UG[f"{tag}_gy"], UG[f"{tag}_gl"])
    if shift.ndim == 1:  # one shared parameter vector: autograd sums over the batch
        gs, ga = gs.sum(0), ga.sum(0)
    for ours, key in ((gx, "gx"), (gs, "gshift"), (ga, "gscale")):
        ref = UG[f"{tag}_{key}"]
        assert np.max(np.abs(ours - ref)) <= 1e-9 * max(1.0, np.abs(ref).max()), key


def test_out_of_range_inverse_returns_reference_edge():
    """A y beyond the range of f comes back as +-(bound - half the final interval)."""
    z, xi = UG["k8_z"], UG["k8_xinv64"]
    n = R.steps(10.0, 1e-6)
    edge = 10.0 - 10.0 / 2**n
    for v in (4.9, 6.0, 100.0):
        np.testing.assert_array_equal(xi[z == np.float32(v)], edge)
    for v in (-4.9, -6.0):
        np.testing.assert_array_equal(xi[z == np.float32(v)], -edge)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libgaussgrad_host.so"
    src = ROOT / "tests" / "native" / "gauss_grad_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so), "-lm"], check=True)
    return ctypes.CDLL(str(so))


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_pair_backward_harness(harness, tag):
    """fp32 pair math with y taken from the goldens, against the reference's fp64 autograd."""
    shift, scale = UG[f"{tag}_shift"], UG[f"{tag}_scale"]
    K = shift.shape[-1]
    x = UG[f"{tag}_x"].astype(np.float32)
    y = UG[f"{tag}_y64"].astype(np.float32)
    gy, gl = UG[f"{tag}_gy"].astype(np.float32), UG[f"{tag}_gl"].astype(np.float32)
    phi = np.ascontiguousarray(np.concatenate([shift, scale], -1).astype(np.float32))
    n = x.size
    ld = 0 if phi.ndim == 1 else 2 * K
    gx = np.empty(n, np.float32)
    gphi = np.empty((n, 2 * K), np.float32)
    harness.gauss_backward_pairs(_ptr(x), _ptr(y), _ptr(phi), ctypes.c_int64(ld), _ptr(gy), _ptr(gl), ctypes.c_int64(n), K,
                                 _ptr(gx), _ptr(gphi))  # fmt: skip
    ref_gx = UG[f"{tag}_gx"]
    ref_gphi = np.concatenate([UG[f"{tag}_gshift"], UG[f"{tag}_gscale"]], -1)
    if ld == 0:
        gphi = gphi.astype(np.float64).sum(0)
    scale_x = np.maximum(np.abs(ref_gx), 1.0)
    assert np.max(np.abs(gx - ref_gx) / scale_x) < 2e-4
    scale_p = np.maximum(np.abs(ref_gphi).max(-1, keepdims=True), 1.0)
    assert np.max(np.abs(gphi - ref_gphi) / scale_p) < 2e-4


def test_resolve_univariate_binds_bound_and_eps():
    u = resolve_univariate(GaussianizationTransform, [(8,), (8,)])
    assert (u["kind"], u["bins"], u["total"], u["bound"], u["iterations"]) == (E.ZK_UNI_GAUSS, 8, 16, 10.0, 25)
    u = resolve_univariate(partial(GaussianizationTransform, bound=5.0, eps=1e-4), [(4,), (4,)])
    assert (u["bins"], u["total"], u["bound"], u["iterations"]) == (4, 8, 5.0, R.steps(5.0, 1e-4))
    with pytest.raises(ValueError):
        resolve_univariate(GaussianizationTransform, [(8,), (7,)])
    with pytest.raises(NotImplementedError):
        resolve_univariate(partial(GaussianizationTransform, slope=1e-3), [(8,), (8,)])


def test_autoregressive_and_coupling_layers_refuse_it():
    shapes = [(8,), (8,)]
    with pytest.raises(NotImplementedError, match="element-wise"):
        MaskedAutoregressiveTransform(3, 2, univariate=GaussianizationTransform, shapes=shapes)
    with pytest.raises(NotImplementedError, match="element-wise"):
        GeneralCouplingTransform(4, 0, univariate=GaussianizationTransform, shapes=shapes)


def test_layer_desc_carries_the_bisection_steps():
    flow = GF(3, 0, transforms=1, components=4)
    desc = flow.transform.transforms[0]._base_desc(E.ZK_LAYER_ELEMENTWISE)
    assert (desc.univariate, desc.bins, desc.iterations, desc.bound) == (E.ZK_UNI_GAUSS, 4, 25, 10.0)
    assert "GaussianizationTransform(components=4)" in repr(flow)
