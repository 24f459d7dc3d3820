"""CPU tests of the sum-of-squares polynomial flow (SOSPF): the fp64 restatement of tests/sospf_reference.py
against the reference's goldens (tests/golden/make_golden_sospf.py), the per-pair math of
zuko_b200/csrc/sosp_math.cuh and its host Gauss-Legendre routine compiled by g++, constructor parity with the
reference under the same seed, the layers that refuse the bijector, and the C-ABI additions."""

import ctypes
import subprocess
from functools import partial
from pathlib import Path

import numpy as np
import pytest
import torch

import sospf_reference as R
from cases import crc, load
from zuko_b200 import _engine as E
from zuko_b200.flows import SOSPF, ElementWiseTransform, GeneralCouplingTransform, MaskedAutoregressiveTransform
from zuko_b200.flows._packed import resolve_univariate
from zuko_b200.flows.polynomial import ShiftedSOSPTransform

ROOT = Path(__file__).resolve().parent.parent
US = load("units_sospf")
UNIT_TAGS = ["k1l0", "k3l4", "k2l7", "k4l15", "shared34"]

# name -> (constructor, polynomials, degree); must mirror tests/golden/make_golden_sospf.py:CASES
SOSPF_CASES = {
    "sospf53": (lambda: SOSPF(5, 3, hidden_features=[32, 32]), 3, 4),
    "sospf35_row": (lambda: SOSPF(3, 5), 3, 4),
    "sospf6_uncond": (lambda: SOSPF(6, 0, transforms=4, degree=3, polynomials=2), 2, 3),
    "sospf53_stress": (lambda: SOSPF(5, 3, hidden_features=[32, 32]), 3, 4),
    "sospf16_wide": (lambda: SOSPF(16, 8, hidden_features=[256] * 3), 3, 4),
}


def build_sospf(name: str):
    torch.manual_seed(0)
    return SOSPF_CASES[name][0]().eval()


def reference_of(name: str, flow) -> R.Flow:
    sd = {k: v.detach().numpy() for k, v in flow.state_dict().items()}
    t0 = flow.transform.transforms[0]
    return R.Flow(sd, t0.features, t0.context, SOSPF_CASES[name][1], SOSPF_CASES[name][2])


def rel(ours, ref):
    ours, ref = np.asarray(ours, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(ours - ref) / np.maximum(np.abs(ref), 1.0)))


def unit(tag):
    a, const = US[f"{tag}_a"], US[f"{tag}_const"]
    return a, const


@pytest.mark.parametrize("name", list(SOSPF_CASES))
def test_constructor_matches_reference_state_dict(name):
    g = load(f"flow_{name}")
    sd = build_sospf(name).state_dict()
    assert list(sd.keys()) == [str(k) for k in g["sd_keys"]]
    assert [crc(v) for v in sd.values()] == [int(v) for v in g["sd_crc"]]
    for k, v in g.items():
        if k.startswith("sd/"):
            np.testing.assert_array_equal(sd[k[3:]].numpy(), v)


def test_softclips_sit_between_the_autoregressive_layers():
    flow = SOSPF(4, 0, transforms=3)
    kinds = [type(t).__name__ for t in flow.transform.transforms]
    assert kinds == ["MaskedAutoregressiveTransform", "UnconditionalTransform"] * 2 + ["MaskedAutoregressiveTransform"]
    assert flow.transform.transforms[1].kwargs["bound"] == 11.0
    assert "ShiftedSOSPTransform(polynomials=3, degree=4)" in repr(flow)


@pytest.mark.parametrize("name", list(SOSPF_CASES))
def test_fp64_restatement_against_goldens(name):
    g = load(f"flow_{name}")
    ref = reference_of(name, build_sospf(name))
    c = g.get("c")
    assert rel(ref.log_prob(g["x"], c), g["log_prob64"]) < 1e-10
    z, ladj = ref.call_and_ladj(g["x"], c)
    assert rel(z, g["z64"]) < 1e-10
    assert rel(ladj, g["ladj64"]) < 1e-10
    ci = None if c is None else (c if c.ndim == 1 else c[: g["zin"].shape[0]])
    np.testing.assert_allclose(ref.inverse(g["zin"], ci), g["xinv64"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_unit_forward_inverse_and_gradients(tag):
    a, const = unit(tag)
    x, z = US[f"{tag}_x"], US[f"{tag}_z"]
    y, ladj = R.forward(x, a, const)
    assert rel(y, US[f"{tag}_y64"]) < 1e-12
    assert rel(ladj, US[f"{tag}_ladj64"]) < 1e-12
    np.testing.assert_array_equal(R.inverse(z, a, const), US[f"{tag}_xinv64"])
    gx, ga, gc = R.grad(x, a, const, US[f"{tag}_gy"], US[f"{tag}_gl"])
    if not bool(US[f"{tag}_batched"]):  # one shared coefficient set: autograd sums over the batch
        ga = ga.sum(0)
    if not bool(US[f"{tag}_shifted"]):
        gc = np.zeros_like(gc)
    for ours, key in ((gx, "gx"), (ga, "ga"), (gc, "gconst")):
        ref = US[f"{tag}_{key}"]
        assert np.max(np.abs(ours - ref)) <= 1e-9 * max(1.0, np.abs(ref).max()), key


def test_out_of_range_inverse_returns_reference_edge():
    """A y beyond f([-10, 10]) comes back as +-(bound - half the final interval)."""
    z, xi = US["k3l4_z"], US["k3l4_xinv64"]
    edge = 10.0 - 10.0 / 2 ** R.steps()
    np.testing.assert_array_equal(xi[z == np.float32(1e6)], edge)
    np.testing.assert_array_equal(xi[z == np.float32(-1e6)], -edge)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libsospgrad_host.so"
    src = ROOT / "tests" / "native" / "sosp_grad_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so), "-lm"], check=True)
    return ctypes.CDLL(str(so))


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def phi_of(tag):
    a, const = unit(tag)
    K, n = a.shape[-2:]
    if a.ndim == 2:  # shared coefficients, constant 0
        return np.ascontiguousarray(np.append(a.reshape(-1), 0.0).astype(np.float32)), 0, K, n - 1
    phi = np.concatenate([a.reshape(a.shape[0], -1), const[:, None]], -1)
    return np.ascontiguousarray(phi.astype(np.float32)), K * n + 1, K, n - 1


def test_gauss_legendre_nodes_match_numpy(harness):
    for n in range(1, 17):
        t, w = np.empty(n), np.empty(n)
        harness.sosp_nodes(n, _ptr(t), _ptr(w))
        tr, wr = R.nodes(n)
        np.testing.assert_allclose(t, tr, rtol=0, atol=1e-14)
        np.testing.assert_allclose(w, wr, rtol=0, atol=1e-14)


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_pair_forward_and_inverse_harness(harness, tag):
    phi, ld, K, L = phi_of(tag)
    x = US[f"{tag}_x"].astype(np.float32)
    n = x.size
    y, ladj = np.empty(n, np.float32), np.empty(n, np.float32)
    harness.sosp_forward_pairs(_ptr(x), _ptr(phi), ctypes.c_int64(ld), ctypes.c_int64(n), K, L, _ptr(y), _ptr(ladj))
    for ours, key in ((y, "y"), (ladj, "ladj")):
        ref64, ref32 = US[f"{tag}_{key}64"], US[f"{tag}_{key}32"].astype(np.float64)
        tol = np.maximum(1e-5 * np.maximum(np.abs(ref64), 1.0), 2 * np.abs(ref32 - ref64))
        assert np.all(np.abs(ours - ref64) <= tol), key
    z = US[f"{tag}_z"].astype(np.float32)
    xi = np.empty(n, np.float32)
    harness.sosp_inverse_pairs(_ptr(z), _ptr(phi), ctypes.c_int64(ld), ctypes.c_int64(n), K, L, _ptr(xi))
    ref64, ref32 = US[f"{tag}_xinv64"], US[f"{tag}_xinv32"].astype(np.float64)
    tol = np.maximum(np.maximum(1e-5 * np.maximum(np.abs(ref64), 1.0), 2 * np.abs(ref32 - ref64)), 2 * 20.0 / 2**25)
    assert np.mean(np.abs(xi - ref64) > tol) <= 0.01


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_pair_backward_harness(harness, tag):
    """fp32 pair math against the reference's fp64 autograd."""
    phi, ld, K, L = phi_of(tag)
    P = K * (L + 1) + 1
    x = US[f"{tag}_x"].astype(np.float32)
    gy, gl = US[f"{tag}_gy"].astype(np.float32), US[f"{tag}_gl"].astype(np.float32)
    n = x.size
    gx = np.empty(n, np.float32)
    gphi = np.empty((n, P), np.float32)
    harness.sosp_backward_pairs(_ptr(x), _ptr(phi), ctypes.c_int64(ld), _ptr(gy), _ptr(gl), ctypes.c_int64(n), K, L,
                                _ptr(gx), _ptr(gphi))  # fmt: skip
    ref_gx = US[f"{tag}_gx"]
    ga = US[f"{tag}_ga"]
    np.testing.assert_array_equal(gphi[:, -1], gy)  # d y / d constant = 1
    if ld == 0:  # one shared coefficient set: autograd summed over the batch
        ours_a, ref_a = gphi[:, :-1].astype(np.float64).sum(0)[None], ga.reshape(1, -1)
    else:
        ours_a, ref_a = gphi[:, :-1], ga.reshape(n, -1)
        if bool(US[f"{tag}_shifted"]):
            np.testing.assert_allclose(gy, US[f"{tag}_gconst"], rtol=1e-7)
    scale_x = np.maximum(np.abs(ref_gx), 1.0)
    assert np.max(np.abs(gx - ref_gx) / scale_x) < 2e-4
    scale_p = np.maximum(np.abs(ref_a).max(-1, keepdims=True), 1.0)
    assert np.max(np.abs(ours_a - ref_a) / scale_p) < 2e-4
    if ld:  # in place, as uni_bwd_kernel writes it: the same result
        blk, gx2 = phi.copy(), np.empty(n, np.float32)
        harness.sosp_backward_in_place(_ptr(x), _ptr(blk), _ptr(gy), _ptr(gl), ctypes.c_int64(n), K, L, _ptr(gx2))
        np.testing.assert_allclose(blk.reshape(n, P), gphi, rtol=1e-6, atol=1e-6 * np.abs(gphi).max())


def test_resolve_univariate():
    u = resolve_univariate(partial(ShiftedSOSPTransform, slope=1e-3), [(3, 5), ()])
    assert (u["kind"], u["bins"], u["degree"], u["total"], u["bound"], u["iterations"]) == (E.ZK_UNI_SOSP, 3, 4, 16, 10.0, 25)
    u = resolve_univariate(partial(ShiftedSOSPTransform, slope=1e-2), [(2, 8), ()])
    assert (u["bins"], u["degree"], u["total"], u["slope"]) == (2, 7, 17, 1e-2)
    with pytest.raises(ValueError):
        resolve_univariate(ShiftedSOSPTransform, [(3, 5)])
    with pytest.raises(NotImplementedError):
        resolve_univariate(partial(ShiftedSOSPTransform, bound=5.0), [(3, 5), ()])
    with pytest.raises(NotImplementedError):
        resolve_univariate(ShiftedSOSPTransform, [(3, 17), ()])  # degree 16


def test_coupling_and_elementwise_layers_refuse_it():
    shapes = [(3, 5), ()]
    with pytest.raises(NotImplementedError, match="autoregressive"):
        GeneralCouplingTransform(4, 0, univariate=ShiftedSOSPTransform, shapes=shapes)
    with pytest.raises(NotImplementedError, match="autoregressive"):
        ElementWiseTransform(4, 2, univariate=ShiftedSOSPTransform, shapes=shapes)
    t = MaskedAutoregressiveTransform(3, 2, univariate=ShiftedSOSPTransform, shapes=shapes)
    assert t.total == 16


def test_layer_desc_layout():
    names = [f[0] for f in E.LayerDesc._fields_]
    assert names[-2:] == ["iterations", "degree"]
    flow = SOSPF(3, 0, transforms=1, degree=5, polynomials=2)
    desc = flow.transform.transforms[0]._base_desc(E.ZK_LAYER_AUTOREGRESSIVE)
    assert (desc.univariate, desc.bins, desc.degree, desc.iterations, desc.bound) == (E.ZK_UNI_SOSP, 2, 5, 25, 10.0)
    assert abs(desc.slope - 1e-3) < 1e-9


def test_c_abi_symbols():
    assert E.ZK_UNI_SOSP == 5
    header = (ROOT / "include" / "zuko_b200.h").read_text()
    assert "#define ZK_UNI_SOSP 5" in header
    for sym in ("zk_sosp_forward", "zk_sosp_inverse", "zk_sosp_backward"):
        assert sym in E.EXPORTED_SYMBOLS and f"zk_status {sym}(" in header
    lib = E.lib()
    for sym in ("zk_sosp_forward", "zk_sosp_inverse", "zk_sosp_backward"):
        assert hasattr(lib, sym)
