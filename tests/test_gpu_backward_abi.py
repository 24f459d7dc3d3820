"""GPU tests of the backward C ABI below the flow level:

* ``zk_layer_backward`` on every layer kind of the composed golden flows and on one tensor-core
  autoregressive layer: values against the fp64 gradient oracle (oracle_grad.layer_backward), and
  the documented contracts — strided rows, ``+=`` into parameter gradients and per-row grad_c, one
  summed grad_c row for a broadcast context (ldc == 0), grad_x overwritten, NULL grad_ladj / grads,
  B = 0, and the workspace size check;
* the stand-alone bijector backward (``zk_rqs_backward`` / ``zk_affine_backward``) at D > 1 with
  strided x / grad_y / grad_x, a padded per-sample parameter row (phi_ld > D * P), in-place
  grad_phi, and a shared table whose per-row gradients pass through a workspace of 1 or 7 rows;
  ``zk_gaussianization_backward`` / ``zk_sosp_backward`` at D > 1 against their D = 1 calls.

Rows at a ReLU kink or spline knot get zero weight on both sides (cases.relu_kink_rows)."""

import ctypes
import types

import numpy as np
import pytest
import torch

from cases import build_flow, relu_kink_rows
from oracle import oracle as O
from oracle import oracle_grad as OG
from test_gpu_backward import close, cpu, dev_t
from test_gpu_backward_edges import assert_tensor_core_path, make_flow
from zuko_b200 import _engine as E

pytestmark = pytest.mark.gpu

NAN = float("nan")
EPS32 = 2.0**-23

# (flow, member index): every layer kind of the composed golden flows, and a tensor-core layer
LAYERS = {
    "ar_affine": ("composed", 0),
    "softclip": ("composed", 1),
    "permutation": ("composed", 2),
    "ar_rqs": ("composed", 3),
    "rotation": ("composed", 4),
    "coupling": ("composed", 5),
    "elementwise_cond": ("composed", 6),
    "elementwise_table_rqs": ("composed_uncond", 0),
    "ar_uncond": ("composed_uncond", 1),
    "elementwise_table_affine": ("composed_uncond", 3),
    "ar_tensor_core": ("nsf5", 0),
}


class LayerCase:
    """One flow member: its engine handle, its oracle layer, its input rows (per-row context, or one
    broadcast context row) and upstream gradients, with zero weight on rows at a kink or knot."""

    def __init__(self, key, device, B=300, broadcast=False):
        name, i = LAYERS[key]
        cpu_flow = build_flow(name) if name.startswith("composed") else make_flow(name)
        self.flow = (build_flow(name) if name.startswith("composed") else make_flow(name)).to(device)
        if key == "ar_tensor_core":
            assert_tensor_core_path(self.flow)
        spec = O.flowspec_from_module(cpu_flow)
        self.layer = spec.layers[i]
        self.D, self.C = spec.layers[0].features, self.flow.transform.transforms[0].context
        self.broadcast = broadcast and self.C > 0
        gen = torch.Generator().manual_seed(i)
        c = None
        if self.C:
            c = torch.randn(self.C, generator=gen).numpy() if self.broadcast else torch.randn(B, self.C, generator=gen).numpy()
        z = torch.randn(B, self.D, generator=gen).numpy().astype(np.float64)
        for layer in spec.layers[:i]:  # the input of member i
            z, _ = layer.forward(z, c, np.float64)
        self.x, self.c = np.asarray(z, np.float32), c
        self.gy = torch.randn(B, self.D, generator=gen).numpy()
        self.gl = torch.randn(B, generator=gen).numpy()
        kink = relu_kink_rows(types.SimpleNamespace(layers=[self.layer]), self.x, c)
        self.gy[kink], self.gl[kink] = 0.0, 0.0
        self.conditioned = self.layer.hyper is not None and self.C > 0
        probe = None if c is None else dev_t(c if self.broadcast else c[:1], device)
        self.fc = self.flow(probe)._flow_call()[0]
        self.handle, self.src = self.fc._handles[i], self.fc._sources[i]
        self.B, self.device = B, device

    def oracle(self):
        """(grad_x, grad_c (summed over the batch for a broadcast row), {buffer name: parameter gradient})."""
        gx, gc, lg = OG.layer_backward(self.layer, self.x.astype(np.float64), self.c, self.gy, self.gl)
        if gc is not None and self.broadcast:
            gc = gc.sum(0)
        out = {}
        if lg.hyper is not None:
            for j, (w, b) in enumerate(zip(lg.hyper.weights, lg.hyper.biases, strict=True)):
                out[f"w{j}"] = w
                if b is not None:
                    out[f"b{j}"] = b
        if lg.phi is not None:
            out["phi"] = lg.phi
        if lg.R is not None:
            out["R"] = lg.R
        return gx, gc, out

    def grad_buffers(self):
        """Zeroed parameter-gradient buffers and the zk_layer_grads pointing at them."""
        f32 = dict(device=self.device, dtype=torch.float32)
        bufs = {}
        for j, w in enumerate(self.src.get("weights") or []):
            bufs[f"w{j}"] = torch.zeros(w.shape, **f32)
        for j, b in enumerate(self.src.get("biases") or []):
            if b is not None:
                bufs[f"b{j}"] = torch.zeros(b.shape, **f32)
        if self.src.get("phi"):
            bufs["phi"] = torch.zeros(self.D, sum(int(t[0].numel()) for t in self.src["phi"]), **f32)
        if self.layer.kind == "rotation":  # dL/dR also for a rotation held in a buffer
            bufs["R"] = torch.zeros(self.D, self.D, **f32)
        lg = E.LayerGrads()
        n = len(self.src.get("weights") or [])
        if n:
            lg.grad_weight = (ctypes.c_void_p * n)(*[bufs[f"w{j}"].data_ptr() for j in range(n)])
            lg.grad_bias = (ctypes.c_void_p * n)(*[bufs[f"b{j}"].data_ptr() if f"b{j}" in bufs else None for j in range(n)])
        if "phi" in bufs:
            lg.grad_phi = bufs["phi"].data_ptr()
        if "R" in bufs:
            lg.grad_rotation = bufs["R"].data_ptr()
        return bufs, lg

    def call(self, *, ldx=None, ldc=None, ldg=None, ldgc=None, gx_fill=0.0, gc_fill=0.0, grads=True, bufs=None,
             null_gl=False, B=None, ws_bytes=None, check=True):  # fmt: skip
        """One zk_layer_backward call on padded device buffers (pad columns NaN).  grad_x / grad_c start as
        `gx_fill` / `gc_fill` (scalars or arrays); `bufs` = (buffers, zk_layer_grads) to accumulate into.
        Returns (status, grad_x with its pads, grad_c with its pads or None, parameter gradients or None)."""
        B = self.B if B is None else B
        D, C, dev = self.D, self.C, self.device
        ldx, ldg = ldx or D, ldg or D
        ldc = 0 if self.broadcast else (ldc or C)
        ldgc = ldgc or C

        def padded(a, ld, fill=NAN):
            t = torch.full((max(a.shape[0], 1), ld), fill, device=dev)
            t[: a.shape[0], : a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a, np.float32))
            return t

        x, gy = padded(self.x[:B], ldx), padded(self.gy[:B], ldg)
        gl = None if null_gl else dev_t(self.gl[:B], dev)
        gx = torch.full((max(B, 1), ldg), NAN, device=dev)
        gx[:, :D] = torch.as_tensor(np.asarray(gx_fill, np.float32)).to(dev)
        c = gc = None
        if C:
            if self.broadcast:
                c = dev_t(self.c, dev)
                gc = torch.full((C,), NAN, device=dev)
                gc[:] = torch.as_tensor(np.asarray(gc_fill, np.float32)).to(dev)
            else:
                c = padded(self.c[:B], ldc)
                gc = torch.full((max(B, 1), ldgc), NAN, device=dev)
                gc[:, :C] = torch.as_tensor(np.asarray(gc_fill, np.float32)).to(dev)
        if grads and bufs is None:
            bufs = self.grad_buffers()
        L = E.lib()
        need = L.zk_layer_backward_workspace_bytes(self.handle, B)
        nbytes = need if ws_bytes is None else ws_bytes
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        st = L.zk_layer_backward(self.handle, p(x), ldx, p(c), ldc, B, p(gy), ldg, p(gl), p(gx), ldg, p(gc), ldgc,
                                 ctypes.byref(bufs[1]) if grads else None, p(ws), nbytes, E.stream_ptr(dev))  # fmt: skip
        torch.cuda.synchronize(dev)
        if check:
            E.check(st)
        pg = {k: cpu(v) for k, v in bufs[0].items()} if grads else None
        return st, cpu(gx), (None if gc is None else cpu(gc)), pg


def _within_adds(got, T, g, n, what):
    """got == T + n g where every add rounds once in fp32 (an FMA-contracted add too)."""
    T, g = np.asarray(T, np.float64), np.asarray(g, np.float64)
    ref = T + n * g
    tol = n * EPS32 * (np.abs(T) + n * np.abs(g)) + 1e-37
    err = np.abs(np.asarray(got, np.float64) - ref)
    assert (err <= tol).all(), f"{what}: {int((err > tol).sum())} entries off T + {n} g, worst {err.max():.3e}"


@pytest.mark.parametrize("key", list(LAYERS))
def test_layer_backward_vs_oracle(device, key):
    case = LayerCase(key, device)
    D, C = case.D, case.C
    _, gx, gc, pg = case.call()
    ogx, ogc, ref = case.oracle()
    close(gx[:, :D], ogx, 5e-5, f"{key} grad_x")
    if case.conditioned:
        close(gc[:, :C], ogc, 5e-5, f"{key} grad_c")
    assert set(pg) == set(ref), f"{key}: buffers {sorted(pg)} vs oracle {sorted(ref)}"
    for k in ref:
        close(pg[k], ref[k], 5e-5, f"{key} d/d{k}")


@pytest.mark.parametrize("key", list(LAYERS))
def test_layer_backward_strided_rows(device, key):
    """ld = D + 3 for x / grad_y / grad_x and C + 2 for c / grad_c: the pads stay NaN and the values
    equal the contiguous call bit for bit."""
    case = LayerCase(key, device)
    D, C = case.D, case.C
    _, gx0, gc0, pg0 = case.call()
    _, gx1, gc1, pg1 = case.call(ldx=D + 3, ldg=D + 3, ldc=C + 2, ldgc=C + 2)
    assert np.isnan(gx1[:, D:]).all(), f"{key}: grad_x pad written"
    assert np.array_equal(gx1[:, :D], gx0[:, :D])
    if C:
        assert np.isnan(gc1[:, C:]).all(), f"{key}: grad_c pad written"
        assert np.array_equal(gc1[:, :C], gc0[:, :C])
    for k in pg0:
        assert np.array_equal(pg1[k], pg0[k]), f"{key}: d/d{k} depends on the strides"


@pytest.mark.parametrize("broadcast", [False, True], ids=["rows", "broadcast"])
@pytest.mark.parametrize("key", list(LAYERS))
def test_layer_backward_accumulates(device, key, broadcast):
    """Parameter gradients and grad_c accumulate: T + g after one call, T + 2 g after two.  With a broadcast
    context (ldc == 0) grad_c is one row that gains the batch sum.  grad_x is overwritten: a NaN fill comes
    back finite."""
    case = LayerCase(key, device, broadcast=broadcast)
    if broadcast and not case.conditioned:
        pytest.skip(f"{key} reads no context")
    D, C = case.D, case.C
    _, gx0, gc0, g = case.call()  # from zero: g
    gen = torch.Generator().manual_seed(1)
    bufs = case.grad_buffers()
    T = {}
    for k, t in bufs[0].items():
        t.copy_(torch.randn(t.shape, generator=gen))
        T[k] = cpu(t)
    Tc = None if gc0 is None else torch.randn(gc0.shape, generator=gen).numpy()
    _, gx1, gc1, r1 = case.call(bufs=bufs, gx_fill=NAN, gc_fill=0.0 if Tc is None else Tc[..., :C])
    assert np.isfinite(gx1[:, :D]).all() and np.array_equal(gx1[:, :D], gx0[:, :D]), f"{key}: grad_x not overwritten"
    _, _, gc2, r2 = case.call(bufs=bufs, gc_fill=0.0 if gc1 is None else gc1[..., :C])
    for k in T:
        _within_adds(r1[k], T[k], g[k], 1, f"{key} d/d{k} (one call)")
        _within_adds(r2[k], T[k], g[k], 2, f"{key} d/d{k} (two calls)")
    if case.conditioned:
        _within_adds(gc1[..., :C], Tc[..., :C], gc0[..., :C], 1, f"{key} grad_c (one call)")
        _within_adds(gc2[..., :C], Tc[..., :C], gc0[..., :C], 2, f"{key} grad_c (two calls)")
    if broadcast:
        _, ogc, ref = case.oracle()
        close(gc0, ogc, 5e-5, f"{key} grad_c summed over the batch")
        for k in ref:
            close(g[k], ref[k], 5e-5, f"{key} d/d{k} (broadcast context)")


@pytest.mark.parametrize("key", list(LAYERS))
def test_layer_backward_nulls_empty_batch_and_workspace(device, key):
    case = LayerCase(key, device)
    D, C = case.D, case.C
    _, gx, _, _ = case.call()
    # a NULL grad_ladj is the same as zeros
    _, gx_n, gc_n, pg_n = case.call(null_gl=True)
    saved = case.gl.copy()
    case.gl[:] = 0.0
    _, gx_z, gc_z, pg_z = case.call()
    case.gl[:] = saved
    assert np.array_equal(gx_n, gx_z, equal_nan=True) and (gc_n is None or np.array_equal(gc_n, gc_z, equal_nan=True))
    assert all(np.array_equal(pg_n[k], pg_z[k]) for k in pg_z)
    # NULL grads: grad_x unchanged
    _, gx_g, _, _ = case.call(grads=False)
    assert np.array_equal(gx_g[:, :D], gx[:, :D])
    # B = 0: ZK_OK and nothing written
    st, gx_e, gc_e, pg_e = case.call(B=0, gx_fill=7.0, gc_fill=7.0)
    assert st == E.ZK_OK
    assert (gx_e[:, :D] == 7.0).all() and (gc_e is None or (gc_e[:, :C] == 7.0).all())
    assert all((v == 0.0).all() for v in pg_e.values())
    # the workspace size is checked on the host: exactly enough is accepted, one byte less refused
    need = E.lib().zk_layer_backward_workspace_bytes(case.handle, case.B)
    assert case.call(ws_bytes=need)[0] == E.ZK_OK
    if need:
        st = case.call(ws_bytes=need - 1, check=False)[0]
        assert st == E.ZK_EINVAL, f"{key}: a workspace one byte short returned {st}"


# --------------------------------------------------------------------------- #
# F. stand-alone bijector backward at D > 1
# --------------------------------------------------------------------------- #

BOUND, SLOPE = 5.0, 1e-3
UNIS = {"rqs8": 8, "rqs16": 16, "rqs5": 5, "affine": 0}
# unconstrained spline parameters of scale 0.1 and the matching bar of test_rqs_backward_per_sample ("s01");
# at scale 1 some of the ~10^4 elements per call sit in bins narrow enough that fp32 itself is off by 1e-4.
# Sixteen bins halve the bin widths, and fp32 error in a knot position is divided by them twice: worst
# per-element grad_x error measured on an H100 80GB HBM3 (700 W): 5.4e-6 (K = 5), 9.2e-6 (8), 4.2e-5 (16)
PHI_SCALE, AFFINE_TOL = 0.1, 1e-5
RQS_TOL = {5: 2e-5, 8: 2e-5, 16: 1e-4}


def uni_inputs(kind, B, D, seed):
    P = 3 * UNIS[kind] - 1 if kind != "affine" else 2
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, D, generator=gen) * 2.5).numpy()  # some beyond +-bound: the identity tails
    phi = (torch.randn(B, D, P, generator=gen) * PHI_SCALE).numpy()
    table = (torch.randn(D, P, generator=gen) * PHI_SCALE).numpy()
    gy = torch.randn(B, D, generator=gen).numpy()
    gl = torch.randn(B, generator=gen).numpy()
    return P, x, phi, table, gy, gl


def uni_oracle(kind, x, phi, gy, gl):
    x64 = x.astype(np.float64)
    gl_el = np.broadcast_to(gl.astype(np.float64)[:, None], x.shape)
    if kind == "affine":
        return OG.affine_backward(x64, phi, gy, gl_el, SLOPE)
    return OG.rqs_backward(x64, phi, gy, gl_el, UNIS[kind], BOUND, SLOPE)


def off_knot(kind, x, phi):
    """Elements away from the spline's knots (the ladj is only C0 there)."""
    if kind == "affine":
        return np.ones(x.shape, bool)
    B, D = x.shape
    X, _, _ = O.rqs_knots(np.broadcast_to(np.asarray(phi, np.float64), (B, D, phi.shape[-1])), UNIS[kind], BOUND, SLOPE)
    return np.abs(x.astype(np.float64)[..., None] - X).min(-1) >= 5e-5


def uni_call(kind, x, ldx, phi, phi_ld, gy, ldgy, gl, gx, ldgx, gphi, ws, B, D, device, K=None, degree=None):
    L = E.lib()
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    nb = 0 if ws is None else ws.numel()
    common = (p(gy), ldgy, p(gl), p(gx), ldgx, p(gphi), p(ws), nb, E.stream_ptr(device))
    if kind == "affine":
        st = L.zk_affine_backward(p(x), ldx, p(phi), phi_ld, B, D, SLOPE, *common)
    elif kind == "gauss":
        st = L.zk_gaussianization_backward(p(x), ldx, p(phi), phi_ld, B, D, K, *common)
    elif kind == "sosp":
        st = L.zk_sosp_backward(p(x), ldx, p(phi), phi_ld, B, D, K, degree, 10.0, SLOPE, *common)
    else:
        st = L.zk_rqs_backward(p(x), ldx, p(phi), phi_ld, B, D, UNIS[kind], BOUND, SLOPE, *common)
    E.check(st)
    torch.cuda.synchronize(device)


def padded_dev(a, ld, device):
    t = torch.full((a.shape[0], ld), NAN, device=device)
    t[:, : a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a, np.float32))
    return t


def check_uni(kind, gx, gphi, ref_gx, ref_gphi, ok, what):
    tol = AFFINE_TOL if kind == "affine" else RQS_TOL[UNIS[kind]]
    assert np.all((np.abs(gx - ref_gx) <= tol * np.maximum(np.abs(ref_gx), 1.0))[ok]), f"{what}: grad_x"
    scale = np.maximum(np.abs(ref_gphi).max(-1, keepdims=True), 1.0)
    assert np.all((np.abs(gphi - ref_gphi) / scale <= tol)[ok]), f"{what}: grad_phi"


@pytest.mark.parametrize("D", [3, 7, 64])
@pytest.mark.parametrize("B", [1, 255, 1000])
@pytest.mark.parametrize("kind", list(UNIS))
def test_bijector_backward_strided_per_sample(device, kind, B, D):
    """ldx = ldgy = ldgx = D + 5, phi_ld = D * P + 3 (grad_phi stays (B, D * P) contiguous), and the
    in-place grad_phi == phi with phi_ld == D * P."""
    P, x, phi, _, gy, gl = uni_inputs(kind, B, D, seed=B * 100 + D)
    ld = D + 5
    xd, gyd = padded_dev(x, ld, device), padded_dev(gy, ld, device)
    gxd = torch.full((B, ld), NAN, device=device)
    phid = padded_dev(phi.reshape(B, D * P), D * P + 3, device)
    gphid = torch.full((B, D * P), NAN, device=device)
    gld = dev_t(gl, device)
    uni_call(kind, xd, ld, phid, D * P + 3, gyd, ld, gld, gxd, ld, gphid, None, B, D, device)
    ref_gx, ref_gphi = uni_oracle(kind, x, phi, gy, gl)
    ok = off_knot(kind, x, phi)
    what = f"{kind} B={B} D={D} strided"
    gx = cpu(gxd)
    assert np.isnan(gx[:, D:]).all(), f"{what}: grad_x pad written"
    assert np.isnan(cpu(phid)[:, D * P :]).all()
    check_uni(kind, gx[:, :D], cpu(gphid).reshape(B, D, P), ref_gx, ref_gphi, ok, what)
    # in place: grad_phi overwrites phi (phi_ld == D * P)
    inplace = dev_t(phi.reshape(B, D * P), device)
    gx2 = torch.full((B, ld), NAN, device=device)
    uni_call(kind, xd, ld, inplace, D * P, gyd, ld, gld, gx2, ld, inplace, None, B, D, device)
    assert np.array_equal(cpu(gx2)[:, :D], gx[:, :D])
    check_uni(kind, cpu(gx2)[:, :D], cpu(inplace).reshape(B, D, P), ref_gx, ref_gphi, ok, f"{kind} B={B} D={D} in place")


@pytest.mark.parametrize("rows", [1, 7])
@pytest.mark.parametrize("D", [3, 7, 64])
@pytest.mark.parametrize("B", [1, 255, 1000])
@pytest.mark.parametrize("kind", list(UNIS))
def test_bijector_backward_shared_table_row_chunks(device, kind, B, D, rows):
    """A shared (D, P) table with a workspace of `rows` rows: the row-chunk loop of uni_backward_entry."""
    _shared_table(device, kind, B, D, rows)


def test_bijector_backward_wide_shared_table(device):
    """D = 256, K = 16: one row per tile and ~94 KB of shared memory (the opt-in above 48 KB)."""
    _shared_table(device, "rqs16", 300, 256, 7)


def _shared_table(device, kind, B, D, rows):
    P, x, _, table, gy, gl = uni_inputs(kind, B, D, seed=B * 100 + D + 1)
    ok = off_knot(kind, x, table).all(1)  # rows with an element on a knot get zero weight
    gy[~ok], gl[~ok] = 0.0, 0.0
    ld = D + 5
    xd, gyd = padded_dev(x, ld, device), padded_dev(gy, ld, device)
    gxd = torch.full((B, ld), NAN, device=device)
    gphid = torch.zeros(D, P, device=device)
    need = E.lib().zk_univariate_backward_workspace_bytes(rows, D, P, 0)
    ws = torch.empty(need, dtype=torch.uint8, device=device)
    uni_call(kind, xd, ld, dev_t(table, device), 0, gyd, ld, dev_t(gl, device), gxd, ld, gphid, ws, B, D, device)
    ref_gx, ref_gphi = uni_oracle(kind, x, table, gy, gl)
    what = f"{kind} B={B} D={D} table in {rows}-row chunks"
    gx = cpu(gxd)
    assert np.isnan(gx[:, D:]).all(), f"{what}: grad_x pad written"
    tol = AFFINE_TOL if kind == "affine" else RQS_TOL[UNIS[kind]]
    assert np.all(np.abs(gx[:, :D] - ref_gx) <= tol * np.maximum(np.abs(ref_gx), 1.0)), f"{what}: grad_x"
    close(cpu(gphid), ref_gphi, tol, f"{what}: grad_phi (summed over the batch)")


@pytest.mark.parametrize("shared", [False, True], ids=["per_sample", "table"])
@pytest.mark.parametrize("kind,K,degree", [("gauss", 8, 0), ("gauss", 5, 0), ("sosp", 3, 4), ("sosp", 2, 7)])
def test_gf_sosp_backward_strided_matches_one_column(device, kind, K, degree, shared):
    """No per-element fp64 oracle here: the strided D > 1 call against D = 1 calls on contiguous
    columns (the path the GF / SOSPF tests pin), to 1e-6 relative."""
    B, D = 255, 7
    P = 2 * K if kind == "gauss" else K * (degree + 1) + 1
    gen = torch.Generator().manual_seed(K * 10 + degree)
    x = (torch.randn(B, D, generator=gen) * 2.0).numpy()
    phi = (torch.randn(B, D, P, generator=gen) * 0.5).numpy()
    table = (torch.randn(D, P, generator=gen) * 0.5).numpy()
    gy, gl = torch.randn(B, D, generator=gen).numpy(), torch.randn(B, generator=gen).numpy()
    ld = D + 5
    rows = 7
    L = E.lib()
    gld = dev_t(gl, device)
    xd, gyd = padded_dev(x, ld, device), padded_dev(gy, ld, device)
    gxd = torch.full((B, ld), NAN, device=device)
    kw = dict(K=K, degree=degree)
    if shared:
        gphid = torch.zeros(D, P, device=device)
        ws = torch.empty(L.zk_univariate_backward_workspace_bytes(rows, D, P, 0), dtype=torch.uint8, device=device)
        uni_call(kind, xd, ld, dev_t(table, device), 0, gyd, ld, gld, gxd, ld, gphid, ws, B, D, device, **kw)
    else:
        phid = padded_dev(phi.reshape(B, D * P), D * P + 3, device)
        gphid = torch.full((B, D * P), NAN, device=device)
        uni_call(kind, xd, ld, phid, D * P + 3, gyd, ld, gld, gxd, ld, gphid, None, B, D, device, **kw)
    gx = cpu(gxd)
    assert np.isnan(gx[:, D:]).all()
    gphi = cpu(gphid).reshape(D, P) if shared else cpu(gphid).reshape(B, D, P)
    for d in range(D):
        xc, gyc = dev_t(x[:, d : d + 1], device), dev_t(gy[:, d : d + 1], device)
        gxc = torch.empty(B, 1, device=device)
        if shared:
            gpc = torch.zeros(1, P, device=device)
            ws = torch.empty(L.zk_univariate_backward_workspace_bytes(rows, 1, P, 0), dtype=torch.uint8, device=device)
            uni_call(kind, xc, 1, dev_t(table[d : d + 1], device), 0, gyc, 1, gld, gxc, 1, gpc, ws, B, 1, device, **kw)
            close(gphi[d], cpu(gpc)[0], 1e-6, f"{kind} column {d} grad_phi (table)")
        else:
            gpc = torch.empty(B, P, device=device)
            uni_call(kind, xc, 1, dev_t(phi[:, d], device), P, gyc, 1, gld, gxc, 1, gpc, None, B, 1, device, **kw)
            close(gphi[:, d], cpu(gpc), 1e-6, f"{kind} column {d} grad_phi")
        close(gx[:, d], cpu(gxc)[:, 0], 1e-6, f"{kind} column {d} grad_x")
