"""CPU tests of the Bernstein polynomial flow (BPF): the fp64 restatement of tests/bpf_reference.py against
the reference's goldens (tests/golden/make_golden_bpf.py), the per-pair math of
zuko_b200/csrc/bernstein_math.cuh compiled by g++, constructor parity with the reference under the same
seed, the refusals, and the C-ABI additions."""

import ctypes
import subprocess
from functools import partial
from pathlib import Path

import numpy as np
import pytest
import torch

import bpf_reference as R
from cases import crc, load
from zuko_b200 import _engine as E
from zuko_b200.accel import _engine_callable
from zuko_b200.flows import BPF, MAF, ElementWiseTransform, GeneralCouplingTransform, MaskedAutoregressiveTransform
from zuko_b200.flows._packed import resolve_univariate
from zuko_b200.transforms import BoundedBernsteinTransform

ROOT = Path(__file__).resolve().parent.parent
US = load("units_bpf")
UNIT_TAGS = ["d0", "d4", "d16", "d16x10", "d40", "shared16", "eps4_b3"]

# name -> (constructor, degree, bound); must mirror tests/golden/make_golden_bpf.py:CASES
BPF_CASES = {
    "bpf53": (lambda: BPF(5, 3, hidden_features=[32, 32]), 16, 5.0),
    "bpf35_row": (lambda: BPF(3, 5), 16, 5.0),
    "bpf6_uncond": (lambda: BPF(6, 0, transforms=4, degree=7), 7, 5.0),
    "bpf53_stress": (lambda: BPF(5, 3, hidden_features=[32, 32]), 16, 5.0),
    "bpf16_wide": (lambda: BPF(16, 8, hidden_features=[256] * 3), 16, 5.0),
    "bpf42_b3": (lambda: MAF(4, 2, univariate=partial(BoundedBernsteinTransform, bound=3.0), shapes=[(9,)]), 8, 3.0),
}


def build_bpf(name: str):
    torch.manual_seed(0)
    return BPF_CASES[name][0]().eval()


def reference_of(name: str, flow) -> R.Flow:
    sd = {k: v.detach().numpy() for k, v in flow.state_dict().items()}
    t0 = flow.transform.transforms[0]
    return R.Flow(sd, t0.features, t0.context, BPF_CASES[name][1], BPF_CASES[name][2])


def rel(ours, ref):
    ours, ref = np.asarray(ours, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(ours - ref) / np.maximum(np.abs(ref), 1.0)))


def unit(tag):
    return US[f"{tag}_u"], float(US[f"{tag}_bound"]), float(US[f"{tag}_eps"])


@pytest.mark.parametrize("name", list(BPF_CASES))
def test_constructor_matches_reference_state_dict(name):
    g = load(f"flow_{name}")
    sd = build_bpf(name).state_dict()
    assert list(sd.keys()) == [str(k) for k in g["sd_keys"]]
    assert [crc(v) for v in sd.values()] == [int(v) for v in g["sd_crc"]]
    for k, v in g.items():
        if k.startswith("sd/"):
            np.testing.assert_array_equal(sd[k[3:]].numpy(), v)


def test_module_tree():
    flow = BPF(4, 2, transforms=2, degree=5)
    kinds = [type(t).__name__ for t in flow.transform.transforms]
    assert kinds == ["MaskedAutoregressiveTransform"] * 2
    assert flow.transform.transforms[0].total == 6
    assert "BoundedBernsteinTransform(degree=5, bound=5)" in repr(flow)


@pytest.mark.parametrize("name", list(BPF_CASES))
def test_fp64_restatement_against_goldens(name):
    g = load(f"flow_{name}")
    ref = reference_of(name, build_bpf(name))
    c = g.get("c")
    assert rel(ref.log_prob(g["x"], c), g["log_prob64"]) < 1e-10
    z, ladj = ref.call_and_ladj(g["x"], c)
    assert rel(z, g["z64"]) < 1e-10
    assert rel(ladj, g["ladj64"]) < 1e-10
    ci = None if c is None else (c if c.ndim == 1 else c[: g["zin"].shape[0]])
    np.testing.assert_allclose(ref.inverse(g["zin"], ci), g["xinv64"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_unit_forward_inverse_and_gradients(tag):
    u, bound, eps = unit(tag)
    x, z = US[f"{tag}_x"], US[f"{tag}_z"]
    y, ladj = R.forward(x, u, bound, eps)
    assert rel(y, US[f"{tag}_y64"]) < 1e-10
    assert np.max(np.abs(ladj - US[f"{tag}_ladj64"])) < 1e-10
    # within one final bisection interval: a midpoint test may flip on the last bits of the fp64 polynomial
    np.testing.assert_allclose(R.inverse(z, u, bound, eps), US[f"{tag}_xinv64"], rtol=0, atol=2 * bound / 2 ** R.steps(bound, eps))
    gx, gu = R.grad(x, u, US[f"{tag}_gy"], US[f"{tag}_gl"], bound, eps)
    if not bool(US[f"{tag}_batched"]):  # one shared parameter row: autograd sums over the batch
        gu = gu.sum(0)
    for ours, key in ((gx, "gx"), (gu, "gu")):
        ref = US[f"{tag}_{key}"]
        assert np.max(np.abs(ours - ref)) <= 1e-9 * max(1.0, np.abs(ref).max()), key


def test_linear_branches_are_not_the_identity():
    """Beyond [-B, B] the reference maps x to x -+ 2B eps, and inverts y beyond it exactly."""
    x, y = US["d16_x"], US["d16_y32"]
    for v, off in ((-7.0, -1.0014e-5), (7.0, 1.0014e-5), (-1e3, -1e-5), (1e3, 1e-5)):
        i = np.flatnonzero(x == np.float32(v))[0]
        assert abs((float(y[i]) - v) - off) < 2e-6 * max(1.0, abs(v) / 5)
    z, xi = US["d16_z"], US["d16_xinv64"]
    for v in (1e3, -1e3, 5.0, -5.0):
        i = np.flatnonzero(z == np.float32(v))[0]
        expect = ((v + 5) / 10 + 1e-6) * 10 - 5 if v < 0 else ((v - 5) / 10 - 1e-6 + 1) * 10 - 5
        assert abs(xi[i] - expect) < 1e-9


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libberngrad_host.so"
    src = ROOT / "tests" / "native" / "bernstein_grad_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so), "-lm"],
                   check=True)  # fmt: skip
    return ctypes.CDLL(str(so))


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def same_branch(x, bound, eps):
    """Rows whose fp32 t = (x + B) / 2B takes the branch the fp64 autograd golden took: at the branch
    boundary the two precisions can disagree, and the gradient jumps there."""
    t32 = (x.astype(np.float32) + np.float32(bound)) / np.float32(2 * bound)
    t64 = (x.astype(np.float64) + bound) / (2 * bound)
    b32 = np.where(t32 <= np.float32(eps), 0, np.where(t32 >= np.float32(1 - eps), 2, 1))
    b64 = np.where(t64 <= eps, 0, np.where(t64 >= 1 - eps, 2, 1))
    return b32 == b64


def phi_of(tag):
    u = US[f"{tag}_u"]
    P = u.shape[-1]
    return np.ascontiguousarray(u.astype(np.float32)), (P if u.ndim == 2 else 0), P - 1


def value_tol(ref64, ref32):
    return np.maximum(1e-5 * np.maximum(np.abs(ref64), 1.0), 2 * np.abs(ref32 - ref64))


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_pair_forward_and_inverse_harness(harness, tag):
    phi, ld, degree = phi_of(tag)
    _, bound, eps = unit(tag)
    x = US[f"{tag}_x"].astype(np.float32)
    n = x.size
    y, ladj = np.empty(n, np.float32), np.empty(n, np.float32)
    harness.bern_forward_pairs(_ptr(x), _ptr(phi), ctypes.c_int64(ld), ctypes.c_int64(n), degree, ctypes.c_float(bound),
                               ctypes.c_float(eps), _ptr(y), _ptr(ladj))  # fmt: skip
    for ours, key in ((y, "y"), (ladj, "ladj")):
        ref64, ref32 = US[f"{tag}_{key}64"], US[f"{tag}_{key}32"].astype(np.float64)
        assert np.all(np.abs(ours - ref64) <= value_tol(ref64, ref32)), key
    z = US[f"{tag}_z"].astype(np.float32)
    xi = np.empty(n, np.float32)
    harness.bern_inverse_pairs(_ptr(z), _ptr(phi), ctypes.c_int64(ld), ctypes.c_int64(n), degree, ctypes.c_float(bound),
                               ctypes.c_float(eps), _ptr(xi))  # fmt: skip
    ref64, ref32 = US[f"{tag}_xinv64"], US[f"{tag}_xinv32"].astype(np.float64)
    tol = np.maximum(value_tol(ref64, ref32), 2 * 2 * bound / 2 ** R.steps(bound, eps))
    assert np.all(np.abs(xi - ref64) <= tol)
    out = np.abs(z) >= bound  # the linear branches: the reference's fp32 operations, bit for bit
    np.testing.assert_array_equal(xi[out], US[f"{tag}_xinv32"][out])


@pytest.mark.parametrize("tag", UNIT_TAGS)
def test_pair_backward_harness(harness, tag):
    """fp32 pair math against the reference's fp64 autograd."""
    phi, ld, degree = phi_of(tag)
    _, bound, eps = unit(tag)
    P = degree + 1
    x = US[f"{tag}_x"].astype(np.float32)
    gy, gl = US[f"{tag}_gy"].astype(np.float32), US[f"{tag}_gl"].astype(np.float32)
    n = x.size
    gx = np.empty(n, np.float32)
    gphi = np.empty((n, P), np.float32)
    harness.bern_backward_pairs(_ptr(x), _ptr(phi), ctypes.c_int64(ld), _ptr(gy), _ptr(gl), ctypes.c_int64(n), degree,
                                ctypes.c_float(bound), ctypes.c_float(eps), _ptr(gx), _ptr(gphi))  # fmt: skip
    ok = same_branch(x, bound, eps)
    assert ok.sum() >= n - 2
    ref_gx, gu = US[f"{tag}_gx"], US[f"{tag}_gu"]
    if ld == 0:  # one shared parameter row: autograd summed over the batch (rows off the branch re-derived in fp64)
        _, gu_fix = R.grad(x[~ok].astype(np.float32).astype(np.float64), US[f"{tag}_u"], gy[~ok], gl[~ok], bound, eps)
        ours_u = gphi[ok].astype(np.float64).sum(0)[None] + gu_fix.sum(0)
        ref_u = gu.reshape(1, -1)
    else:
        ours_u, ref_u = gphi[ok], gu.reshape(n, -1)[ok]
    assert np.max(np.abs(gx - ref_gx)[ok]) <= 1e-4 * np.abs(ref_gx).max()
    assert np.max(np.abs(ours_u - ref_u)) <= 1e-4 * np.abs(ref_u).max()
    if ld:  # in place, as uni_bwd_kernel writes it: the same result
        blk, gx2 = phi.copy(), np.empty(n, np.float32)
        harness.bern_backward_in_place(_ptr(x), _ptr(blk), _ptr(gy), _ptr(gl), ctypes.c_int64(n), degree, ctypes.c_float(bound),
                                       ctypes.c_float(eps), _ptr(gx2))  # fmt: skip
        np.testing.assert_allclose(blk.reshape(n, P), gphi, rtol=1e-6, atol=1e-6 * np.abs(gphi).max())
        np.testing.assert_allclose(gx2, gx, rtol=1e-6, atol=1e-6 * np.abs(gx).max())


def test_resolve_univariate():
    u = resolve_univariate(BoundedBernsteinTransform, [(17,)])
    assert (u["kind"], u["degree"], u["total"], u["bound"], u["iterations"]) == (E.ZK_UNI_BERNSTEIN, 16, 17, 5.0, 24)
    u = resolve_univariate(partial(BoundedBernsteinTransform, bound=3.0), [(9,)])
    assert (u["degree"], u["total"], u["bound"], u["iterations"]) == (8, 9, 3.0, 23)
    u = resolve_univariate(BoundedBernsteinTransform, [(60,)])
    assert u["degree"] == 59
    with pytest.raises(ValueError):
        resolve_univariate(BoundedBernsteinTransform, [(3,), ()])
    with pytest.raises(NotImplementedError, match="eps"):
        resolve_univariate(partial(BoundedBernsteinTransform, eps=1e-4), [(17,)])
    with pytest.raises(NotImplementedError, match="degree"):
        resolve_univariate(BoundedBernsteinTransform, [(61,)])  # degree 60


def test_unbounded_bernstein_is_refused():
    class BernsteinTransform:  # the reference's unbounded class, recognised by name
        pass

    with pytest.raises(NotImplementedError, match="unbounded"):
        resolve_univariate(BernsteinTransform, [(17,)])
    with pytest.raises(NotImplementedError):
        _engine_callable(BernsteinTransform)
    assert _engine_callable(partial(BoundedBernsteinTransform, bound=3.0)).func is BoundedBernsteinTransform


def test_coupling_and_elementwise_layers_refuse_it():
    shapes = [(17,)]
    with pytest.raises(NotImplementedError, match="autoregressive"):
        GeneralCouplingTransform(4, 0, univariate=BoundedBernsteinTransform, shapes=shapes)
    with pytest.raises(NotImplementedError, match="autoregressive"):
        ElementWiseTransform(4, 2, univariate=BoundedBernsteinTransform, shapes=shapes)
    t = MaskedAutoregressiveTransform(3, 2, univariate=BoundedBernsteinTransform, shapes=shapes)
    assert t.total == 17


def test_layer_desc_fields():
    names = [f[0] for f in E.LayerDesc._fields_]
    assert names[-2:] == ["iterations", "degree"]
    flow = BPF(3, 0, transforms=1, degree=7)
    desc = flow.transform.transforms[0]._base_desc(E.ZK_LAYER_AUTOREGRESSIVE)
    assert (desc.univariate, desc.degree, desc.iterations, desc.bound) == (E.ZK_UNI_BERNSTEIN, 7, 24, 5.0)


def test_c_abi_symbols():
    assert E.ZK_UNI_BERNSTEIN == 6
    header = (ROOT / "include" / "zuko_b200.h").read_text()
    assert "#define ZK_UNI_BERNSTEIN 6" in header
    syms = ("zk_bernstein_forward", "zk_bernstein_inverse", "zk_bernstein_backward")
    for sym in syms:
        assert sym in E.EXPORTED_SYMBOLS and f"zk_status {sym}(" in header
    lib = E.lib()
    for sym in syms:
        assert hasattr(lib, sym)
