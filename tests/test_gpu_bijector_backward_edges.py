"""GPU tests of the bijector backward kernel (uni_bwd_kernel, backward.cu) at its tile-plan, shared-table,
instantiation, batch, stride and aliasing edges, against the fp64 gradient references.

* `uni_bwd_plan_of` restates in numpy what uni_bwd_plan decides for a call: the refusals, the rows per tile R (the
  24 KB rule, the ceil(256 / D) floor, the 96 KB cap counting a shared table, R = 1 up to 200 KB, the batch cap), the
  dynamic shared memory, whether a shared table is rewritten in place (R = 1) and the compile-time instantiation.
  Tests without a GPU check that the case table reaches every cell and that every shared-table shape the forward plan
  accepts the backward plan accepts too; on the GPU `zk_univariate_backward_plan` must report the same plan.
* Oracle parity through the stand-alone `zk_{rqs,affine,gaussianization,sosp,bernstein}_backward`: every case at
  batches 0, 1, R - 1, R, R + 1, 2R - 1 and 3R + 77, in both zk_set_fast_math modes, per-sample (contiguous, and with
  NaN-padded phi_ld, ldx, ldgy and ldgx), and with a shared table (one chunk, a 1-row workspace, and a workspace whose
  row count does not divide B).  Inputs include +-bound and its float32 neighbours, bound + 1, +-1e30 (RQS, affine,
  Bernstein) and the Bernstein t = eps / 1 - eps edges; rows on an RQS knot, on a Bernstein branch boundary where
  float32 and fp64 disagree (test_bpf_host.same_branch), or where the Gaussianization map is ill-conditioned
  (test_gpu_bijector_edges.gauss_ok) get zero upstream gradient.
* Contracts: prefix batches bit-identical to the full batch, shared-table reductions bit-reproducible, NULL outputs
  and NULL upstream gradients, the documented in-place grad_phi == phi, every refusal (overlapping grad_phi included,
  with NaN-filled outputs left untouched), shared tables between 100 and 200 KB, and the layer paths through the same
  kernel (an element-wise GF layer with a 128 KB table, a coupling layer's dim_map, an NCSF layer's circular shift).

Bars, with the worst case measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit over every form, batch and
both math modes:
* RQS and affine at parameter scale 0.1 (test_gpu_backward_abi.py): grad_x within tol max(|ref|, 1) per element and
  grad_phi within tol of max(max_p |ref|, 1) per (row, dim); the table gradient within tol of its largest entry.
  Affine 1e-5 (measured 4.7e-7); RQS 5 and 8 bins 2e-5 (6.1e-6), 16 bins 1e-4 (1.2e-5).  64 random bins: 4e-4
  (2.1e-4 on grad_x: fp32 error in a knot is divided by the bin width twice, a quarter of 16 bins').  More than 256
  bins draw uniform bins, whose knots are exact (random float32 knot sums drift ~1e-5 at K = 1024): 1024 bins 5e-5
  (2.1e-5 on grad_x: the spline is the identity, and the fp32 rounding of the position in a bin 10 / 1024 wide is
  left in the ladj term, which is exactly 0 in fp64).
* Gaussianization and SOSP: 5e-5 of the largest entry of each tensor (measured 1.5e-6 at K = 256, 1.3e-6 at
  P = 1009); Bernstein: 1e-4 (test_gpu_bpf.py; measured 2.1e-6 at degree 59)."""

import ctypes
import types
import zlib

import numpy as np
import pytest
import torch

import bpf_reference as BR
import gf_reference as GR
import sospf_reference as SR
from cases import build_flow, relu_kink_rows
from oracle import oracle as O
from oracle import oracle_grad as OG
from test_bpf_host import same_branch
from test_gpu_backward_abi import AFFINE_TOL, RQS_TOL
from test_gpu_bijector_edges import (AFFINE, BERN, GAUSS, KIND_NAMES, RQS, SOSP, THREADS, gauss_ok, math_mode,  # noqa: F401
                                     n_params, uni_plan_of)  # fmt: skip
from zuko_b200 import _engine as E

SLOPE, RQS_BOUND, BISECT_BOUND, BERN_BOUND, BERN_EPS = 1e-3, 5.0, 10.0, 5.0, 1e-6
NAN = float("nan")
PAD = 5
KB = 1024
# RQS bars by bins: 5 / 8 / 16 from test_gpu_backward_abi.py; 64 random bins of scale 0.1, 1024 uniform bins (docstring)
RQS_BAR = {**RQS_TOL, 64: 4e-4, 1024: 5e-5}
FAMILY_BAR = {GAUSS: 5e-5, SOSP: 5e-5, BERN: 1e-4}


# --------------------------------------------------------------------------- #
# the plan, restated
# --------------------------------------------------------------------------- #


def uni_bwd_plan_of(kind, B, D, K, degree, phi_ld):
    """What uni_bwd_plan decides.  Returns {"ok": False, "why": ...} for a refusal, else rows / smem / bins / in_place
    and the rule that set R before the batch cap ("24k", "floor", "cap96")."""
    if B < 0 or D <= 0:
        return {"ok": False, "why": "shape"}
    if B == 0:
        return {"ok": True, "rows": 0, "smem": 0, "bins": 0, "rule": None, "capped": False, "in_place": False}
    if kind not in KIND_NAMES:
        return {"ok": False, "why": "kind"}
    if kind in (RQS, GAUSS) and not 1 <= K <= 1024:
        return {"ok": False, "why": "K"}
    if kind == SOSP and not (1 <= K <= 1023 and 0 <= degree <= 15 and K * (degree + 1) + 1 <= 1024):
        return {"ok": False, "why": "degree"}
    if kind == BERN and not 0 <= degree <= 59:
        return {"ok": False, "why": "degree"}
    P = n_params(kind, K, degree)
    if phi_ld != 0 and phi_ld < D * P:
        return {"ok": False, "why": "phi_ld"}
    row = D * P * 4
    table = row if phi_ld == 0 else 0
    if row > 200 * KB:
        return {"ok": False, "why": "row"}
    r24, floor = 24 * KB // row, -(-THREADS // D)
    R = max(r24, floor)
    rule = "24k" if r24 >= floor else "floor"
    while R > 1 and R * row + table > 96 * KB:
        R -= 1
        rule = "cap96"
    R = max(R, 1)
    capped = R > B
    R = min(R, B)
    in_place = phi_ld == 0 and R == 1
    bins = {RQS: K if K in (8, 16) else 0, GAUSS: K if K in (8, 16) else 0, AFFINE: 0,
            SOSP: 3 if (K, degree) == (3, 4) else 0, BERN: 17 if degree == 16 else 0}[kind]  # fmt: skip
    return {"ok": True, "rows": R, "smem": R * row + (0 if in_place else table), "bins": bins, "rule": rule,
            "capped": capped, "in_place": in_place, "P": P}  # fmt: skip


# name -> (kind, K or polynomials, degree, D)
CASES = {
    "affine_d1": (AFFINE, 0, 0, 1),        # 24 KB rule: R = 3072
    "affine_d7": (AFFINE, 0, 0, 7),
    "rqs8_d1": (RQS, 8, 0, 1),             # 24 KB rule: R = 267
    "rqs8_d3": (RQS, 8, 0, 3),             # shared table beside R = 89 rows
    "rqs16_d64": (RQS, 16, 0, 64),         # floor: R = 4, 48128 B (attribute raised)
    "rqs5_d7": (RQS, 5, 0, 7),             # runtime bins
    "rqs64_d32": (RQS, 64, 0, 32),         # 96 KB cap: R = 4 per sample, R = 3 beside a table
    "rqs1024_d2": (RQS, 1024, 0, 2),       # 96 KB cap: R = 4, 98272 B
    "rqs1024_d16": (RQS, 1024, 0, 16),     # R = 1, 196544 B; a shared table is rewritten in place
    "gauss8_d4": (GAUSS, 8, 0, 4),
    "gauss16_d3": (GAUSS, 16, 0, 3),
    "gauss5_d7": (GAUSS, 5, 0, 7),         # runtime components
    "gauss256_d64": (GAUSS, 256, 0, 64),   # R = 1, 128 KB table in place
    "sosp_d4": (SOSP, 3, 4, 4),            # (3, 4) instantiation
    "sosp23_d5": (SOSP, 2, 3, 5),          # runtime shape
    "sosp1009_d2": (SOSP, 63, 15, 2),      # P = 1009
    "bern16_d4": (BERN, 0, 16, 4),         # P = 17 instantiation
    "bern7_d3": (BERN, 0, 7, 3),
    "bern59_d5": (BERN, 0, 59, 5),         # P = 60
}  # fmt: skip
FORMS = ("dense", "padded", "shared")


def phi_ld_of(name, form):
    kind, K, deg, D = CASES[name]
    P = n_params(kind, K, deg)
    return {"dense": D * P, "padded": D * P + PAD, "shared": 0}[form]


def plan_of(name, form, B=1 << 20):
    kind, K, deg, D = CASES[name]
    return uni_bwd_plan_of(kind, B, D, K, deg, phi_ld_of(name, form))


def batches_of(R):
    return sorted({0, 1, max(R - 1, 1), R, R + 1, 2 * R - 1, 3 * R + 77})


REFUSALS = {
    "rqs_k0": ((RQS, 10, 4, 0, 0, 0), "K"),
    "rqs_k1025": ((RQS, 10, 4, 1025, 0, 0), "K"),
    "gauss_k0": ((GAUSS, 10, 4, 0, 0, 0), "K"),
    "sosp_degree16": ((SOSP, 10, 4, 3, 16, 0), "degree"),
    "sosp_too_many": ((SOSP, 10, 4, 512, 1, 0), "degree"),
    "bern_degree60": ((BERN, 10, 4, 0, 60, 0), "degree"),
    "phi_ld_short": ((RQS, 10, 4, 8, 0, 4 * 23 - 1), "phi_ld"),
    "row_over_200k": ((RQS, 10, 17, 1024, 0, 17 * 3071), "row"),
    "row_over_200k_shared": ((RQS, 10, 17, 1024, 0, 0), "row"),
    "kind_crqs": ((E.ZK_UNI_CRQS, 10, 4, 8, 0, 0), "kind"),
    "d0": ((RQS, 10, 0, 8, 0, 0), "shape"),
}


def test_plan_table_reaches_every_cell():
    """The case table reaches every rule, both table layouts, the in-place rewrite, the batch cap, every instantiation
    and every refusal (no GPU)."""
    rules, inst, capped, big_r1, in_place, beside = set(), set(), False, False, set(), False
    for name, (kind, K, deg, D) in CASES.items():
        for form in FORMS:
            p = plan_of(name, form)
            assert p["ok"], (name, form)
            rules.add(p["rule"])
            inst.add((kind, p["bins"]))
            big_r1 |= p["rows"] == 1 and p["smem"] > 96 * KB
            if form == "shared":
                if p["in_place"]:
                    in_place.add(p["smem"])
                beside |= p["rows"] > 1
            for B in batches_of(p["rows"]):
                capped |= B > 0 and plan_of(name, form, B)["capped"]
    assert rules == {"24k", "floor", "cap96"} and capped and big_r1 and beside, (rules, capped, big_r1, beside)
    assert in_place == {128 * KB, 196544}, in_place
    assert inst == {(AFFINE, 0), (RQS, 8), (RQS, 16), (RQS, 0), (GAUSS, 8), (GAUSS, 16), (GAUSS, 0), (SOSP, 3),
                    (SOSP, 0), (BERN, 17), (BERN, 0)}, inst  # fmt: skip
    # the cells by value
    assert plan_of("affine_d1", "dense")["rows"] == 3072 and plan_of("affine_d1", "dense")["rule"] == "24k"
    assert plan_of("rqs8_d1", "dense")["rows"] == 267 and plan_of("rqs8_d1", "dense")["rule"] == "24k"
    p = plan_of("rqs16_d64", "dense")
    assert (p["rows"], p["smem"], p["rule"]) == (4, 48128, "floor") and p["smem"] > 40 * KB
    p = plan_of("rqs1024_d2", "dense")
    assert (p["rows"], p["smem"], p["rule"]) == (4, 98272, "cap96")
    p = plan_of("rqs64_d32", "shared")
    assert (p["rows"], p["rule"], p["in_place"]) == (3, "cap96", False) and plan_of("rqs64_d32", "dense")["rows"] == 4
    p = plan_of("rqs1024_d16", "dense")
    assert (p["rows"], p["smem"]) == (1, 196544)
    p = plan_of("rqs8_d3", "shared")
    assert (p["rows"], p["in_place"], p["smem"]) == (89, False, 90 * 276)
    p = plan_of("gauss256_d64", "shared")
    assert (p["rows"], p["smem"], p["in_place"]) == (1, 128 * KB, True)
    p = plan_of("rqs1024_d16", "shared")
    assert (p["rows"], p["smem"], p["in_place"]) == (1, 196544, True)
    p = uni_bwd_plan_of(RQS, 5, 3, 8, 0, 0)  # batch cap
    assert (p["rows"], p["capped"], p["in_place"]) == (5, True, False)
    assert uni_bwd_plan_of(RQS, 1, 3, 8, 0, 0)["in_place"]  # one row: the table is rewritten in place
    for name, (args, why) in REFUSALS.items():
        assert uni_bwd_plan_of(*args) == {"ok": False, "why": why}, name


def test_backward_accepts_every_shared_table_the_forward_accepts():
    """Walk (kind, D, K or degree) with a shared table: every shape uni_plan takes, uni_bwd_plan takes too (no GPU).
    Under the old rule (table + one row <= 200 KB) tables above 100 KB were refused."""
    walked = newly = 0
    shapes = [(RQS, K, 0) for K in (*range(1, 40), 64, 100, 128, 256, 300, 512, 700, 1000, 1024)]
    shapes += [(GAUSS, K, 0) for K in (*range(1, 40), 64, 100, 128, 256, 300, 512, 700, 1000, 1024)]
    shapes += [(AFFINE, 0, 0)] + [(BERN, 0, deg) for deg in range(60)]
    shapes += [(SOSP, K, deg) for deg in range(16) for K in range(1, 1024) if K * (deg + 1) + 1 <= 1024 and (K < 40 or K % 37 == 0)]
    for kind, K, deg in shapes:
        P = n_params(kind, K, deg)
        for D in (*range(1, 70), 100, 128, 200, 256, 300, 512, 1000, 4096, 12800, 25600, 51200):
            if uni_plan_of(kind, 1000, D, K, deg, 0)["ok"]:
                walked += 1
                assert uni_bwd_plan_of(kind, 1000, D, K, deg, 0)["ok"], (KIND_NAMES[kind], K, deg, D)
                newly += 2 * D * P * 4 > 200 * KB
    assert walked > 5000 and newly > 100, (walked, newly)


# --------------------------------------------------------------------------- #
# GPU helpers
# --------------------------------------------------------------------------- #


def cpu(t):
    return t.detach().cpu().numpy().astype(np.float64)


def dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(device)


def query(kind, B, D, K, deg, phi_ld):
    R, smem, bins = ctypes.c_int(-1), ctypes.c_size_t(0), ctypes.c_int(-1)
    st = E.lib().zk_univariate_backward_plan(kind, B, D, K, deg, phi_ld, ctypes.byref(R), ctypes.byref(smem), ctypes.byref(bins))
    return st, (R.value, smem.value, bins.value)


def want(p):
    return p["rows"], p["smem"], p["bins"]


def backward_abi(kind, K, deg, x, ldx, phi, phi_ld, B, D, gy, ldgy, gl, gx, ldgx, gphi, ws, device, bound=None,
                 slope=SLOPE, eps=BERN_EPS):  # fmt: skip
    """One stand-alone backward call; tensors or raw addresses (int) or None."""
    L, st = E.lib(), E.stream_ptr(device)
    p = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
    nb = 0 if ws is None else ws.numel()
    tail = (p(gy), ldgy, p(gl), p(gx), ldgx, p(gphi), p(ws), nb, st)
    if kind == RQS:
        return L.zk_rqs_backward(p(x), ldx, p(phi), phi_ld, B, D, K, bound or RQS_BOUND, slope, *tail)
    if kind == AFFINE:
        return L.zk_affine_backward(p(x), ldx, p(phi), phi_ld, B, D, slope, *tail)
    if kind == GAUSS:
        return L.zk_gaussianization_backward(p(x), ldx, p(phi), phi_ld, B, D, K, *tail)
    if kind == SOSP:
        return L.zk_sosp_backward(p(x), ldx, p(phi), phi_ld, B, D, K, deg, bound or BISECT_BOUND, slope, *tail)
    return L.zk_bernstein_backward(p(x), ldx, p(phi), phi_ld, B, D, deg, bound or BERN_BOUND, eps, *tail)


def bound_of(kind):
    return {RQS: RQS_BOUND, AFFINE: RQS_BOUND, GAUSS: BISECT_BOUND, SOSP: BISECT_BOUND, BERN: BERN_BOUND}[kind]


def params_of(kind, K, deg, n_rows, D, g):
    """Parameters (n_rows, D, P), float32; RQS and affine at scale 0.1 (uniform bins beyond 256 bins)."""
    P = n_params(kind, K, deg)
    r = g.standard_normal((n_rows, D, P))
    if kind in (RQS, AFFINE):
        r *= 0.1 if K <= 256 else 0.0
    elif kind == GAUSS:
        r[..., K:] *= 0.3
    elif kind == SOSP:
        r[..., :-1] *= 0.3
    return r.astype(np.float32)


def outside_edges(kind):
    """Inputs at and beyond the bound that every family differentiates like its interior (or as the identity)."""
    b = np.float32(bound_of(kind))
    up, down = np.float32(np.inf), np.float32(-np.inf)
    e = [b + 1, -b - 1]
    if kind != RQS:  # RQS: on its outer knots (inputs_of)
        e += [np.nextafter(b, up), np.nextafter(-b, down)]
    if kind in (RQS, AFFINE, BERN):  # the polynomial and mixture maps overflow float32 there
        e += [1e30, -1e30]
    if kind in (AFFINE, SOSP, GAUSS, BERN):
        e += [b, -b, np.nextafter(b, np.float32(0)), np.nextafter(-b, np.float32(0))]
    if kind == BERN:  # t = eps and t = 1 - eps, and their float32 neighbours
        for v in (np.float32(2 * BERN_BOUND * BERN_EPS - BERN_BOUND), np.float32(BERN_BOUND - 2 * BERN_BOUND * BERN_EPS)):
            e += [v, np.nextafter(v, up), np.nextafter(v, down)]
    return np.array(e, np.float32)


def inputs_of(kind, K, phi, n, D, g):
    """x (n, D): randn * bound / 2 (randn for Gaussianization); rows 1 mod 3 hold the edges; for RQS rows 2 mod 3 hold
    +-bound, its float32 neighbours and knots of their own spline (zero weight: the ladj is only C0 there, and the
    float32 outer knots may round past +-bound)."""
    spread = 1.0 if kind == GAUSS else bound_of(kind) / 2
    x = (g.standard_normal((n, D)) * spread).astype(np.float32)
    e = outside_edges(kind)
    rows = np.arange(1, n, 3)
    x[rows] = e[(np.arange(rows.size)[:, None] * D + np.arange(D)) % e.size]
    if kind == RQS:
        b = np.float32(RQS_BOUND)
        on = np.array([b, -b, np.nextafter(b, np.float32(0)), np.nextafter(-b, np.float32(0)), np.nextafter(b, np.float32(np.inf)),
                       np.nextafter(-b, np.float32(-np.inf))], np.float32)  # fmt: skip
        X = O.rqs_knots(np.asarray(phi, np.float64), K, RQS_BOUND, SLOPE)[0]  # (n, D, K + 1)
        for r in range(2, n, 3):
            for d in range(D):
                x[r, d] = on[(r // 3 + d) % on.size] if (r + d) % 2 else X[r, d, (r * 7 + d) % (K + 1)]
    return x


def weight_rows(kind, K, deg, x, phi):
    """Rows that keep their upstream gradient (module docstring)."""
    x64 = x.astype(np.float64)
    if kind == RQS:
        X = O.rqs_knots(np.asarray(phi, np.float64), K, RQS_BOUND, SLOPE)[0]
        ok = np.abs(x64[..., None] - X).min(-1) >= 5e-5
    elif kind == GAUSS:
        ok = gauss_ok(x64, np.asarray(phi[..., :K], np.float64), np.asarray(phi[..., K:], np.float64))
    elif kind == BERN:
        ok = same_branch(x, BERN_BOUND, BERN_EPS)
    else:
        ok = np.ones(x.shape, bool)
    return ok.all(-1)


def reference(kind, K, deg, x, phi, gy, gl):
    """fp64 (grad_x (n, D), grad_phi (n, D, P)) of <gy, y> + <gl, ladj summed over D>; phi (n, D, P)."""
    x64, phi64 = x.astype(np.float64), np.asarray(phi, np.float64)
    gy = gy.astype(np.float64)
    gle = np.broadcast_to(gl.astype(np.float64)[:, None], x.shape)
    if kind == RQS:
        return OG.rqs_backward(x64, phi64, gy, gle, K, RQS_BOUND, SLOPE)
    if kind == AFFINE:
        return OG.affine_backward(x64, phi64, gy, gle, SLOPE)
    if kind == GAUSS:
        gx, gs, gc = GR.grad(x64, phi64[..., :K], phi64[..., K:], gy, gle)
        return gx, np.concatenate([gs, gc], -1)
    if kind == SOSP:
        a = phi64[..., :-1].reshape(*phi64.shape[:-1], K, deg + 1)
        gx, ga, gc = SR.grad(x64, a, phi64[..., -1], gy, gle, SLOPE, BISECT_BOUND)
        return gx, np.concatenate([ga.reshape(*ga.shape[:-2], -1), gc[..., None]], -1)
    return BR.grad(x64, phi64, gy, gle, BERN_BOUND, BERN_EPS)


def _fail(what, bad, ours, ref):
    i = tuple(int(v) for v in np.argwhere(bad)[0])
    raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} off the reference; first at {i}: ours {ours[i]!r} ref {ref[i]!r}")


def check_grads(kind, K, what, gx, gphi, ref_gx, ref_gphi):
    """grad_x (B, D) and per-sample grad_phi (B, D, P) against the family's bar (module docstring)."""
    if kind in (RQS, AFFINE):
        tol = AFFINE_TOL if kind == AFFINE else RQS_BAR[K]
        with np.errstate(invalid="ignore"):
            bad = ~(np.abs(gx - ref_gx) <= tol * np.maximum(np.abs(ref_gx), 1.0))
        if bad.any():
            _fail(what + " grad_x", bad, gx, ref_gx)
        if gphi is not None:
            scale = np.maximum(np.abs(ref_gphi).max(-1, keepdims=True), 1.0)
            with np.errstate(invalid="ignore"):
                bad = ~(np.abs(gphi - ref_gphi) <= tol * scale)
            if bad.any():
                _fail(what + " grad_phi", bad, gphi, ref_gphi)
        return
    check_tensor(kind, what + " grad_x", gx, ref_gx)
    if gphi is not None:
        check_tensor(kind, what + " grad_phi", gphi, ref_gphi)


def check_tensor(kind, what, ours, ref):
    """Gaussianization, SOSP and Bernstein: max |ours - ref| within the bar times max |ref| (at least 1)."""
    bar = FAMILY_BAR[kind]
    scale = max(float(np.abs(ref).max(initial=0.0)), 1.0)
    with np.errstate(invalid="ignore"):
        bad = ~(np.abs(ours - ref) <= bar * scale)
    if bad.any():
        _fail(f"{what} (bar {bar:.0e} of {scale:.3e})", bad, ours, ref)


def check_table(kind, K, what, gphi, ref_sum):
    """A shared table's gradient, summed over the batch, at the family's bar of the largest entry."""
    bar = AFFINE_TOL if kind == AFFINE else RQS_BAR[K] if kind == RQS else FAMILY_BAR[kind]
    scale = max(float(np.abs(ref_sum).max(initial=0.0)), 1.0)
    with np.errstate(invalid="ignore"):
        bad = ~(np.abs(gphi - ref_sum) <= bar * scale)
    if bad.any():
        _fail(f"{what} table gradient (bar {bar:.0e} of {scale:.3e})", bad, gphi, ref_sum)


class Data:
    """Seeded inputs of one case at its largest batch, with the fp64 references for per-sample parameters and for
    the shared table (rows are independent: every batch is a prefix)."""

    def __init__(self, name):
        kind, K, deg, D = CASES[name]
        self.kind, self.K, self.deg, self.D = kind, K, deg, D
        self.P = n_params(kind, K, deg)
        self.n = max(3 * plan_of(name, f)["rows"] + 77 for f in FORMS)
        g = np.random.default_rng(zlib.crc32(name.encode()))
        self.phi = params_of(kind, K, deg, self.n, D, g)
        self.table = params_of(kind, K, deg, 1, D, g)[0]
        full = np.broadcast_to(self.table, self.phi.shape)
        self.gy = g.standard_normal((self.n, D)).astype(np.float32)
        self.gl = g.standard_normal(self.n).astype(np.float32)
        self.x = inputs_of(kind, K, self.phi, self.n, D, g)
        self.xs = inputs_of(kind, K, full, self.n, D, np.random.default_rng(zlib.crc32(name.encode()) + 1))
        # zero weight on rows off the fp32 / fp64 agreement (module docstring), per parameter layout
        self.gy_p, self.gl_p = self.gy.copy(), self.gl.copy()
        w = weight_rows(kind, K, deg, self.x, self.phi)
        self.gy_p[~w], self.gl_p[~w] = 0.0, 0.0
        self.gy_s, self.gl_s = self.gy.copy(), self.gl.copy()
        ws = weight_rows(kind, K, deg, self.xs, full)
        self.gy_s[~ws], self.gl_s[~ws] = 0.0, 0.0
        assert w.mean() > 0.4 and ws.mean() > 0.4, (name, w.mean(), ws.mean())
        self.gx64, self.gphi64 = reference(kind, K, deg, self.x, self.phi, self.gy_p, self.gl_p)
        self.gxs64, gphis = reference(kind, K, deg, self.xs, full, self.gy_s, self.gl_s)
        self.gphis_cum = np.concatenate([np.zeros((1, D, self.P)), np.cumsum(gphis, 0)])  # prefix sums over rows


_DATA = {}


def data(name):
    if name not in _DATA:
        _DATA.clear()
        _DATA[name] = Data(name)
    return _DATA[name]


def padded(a, ld, device, fill=NAN):
    a = np.ascontiguousarray(a, np.float32)
    t = torch.full((max(a.shape[0], 1), ld), fill, device=device)
    t[: a.shape[0], : a.shape[1]] = torch.from_numpy(a).to(device)
    return t


def run_per_sample(d, device, B, form):
    """(grad_x (B, D), grad_phi (B, D P)) device tensors of one per-sample call, and the NaN pads that must survive."""
    D, P = d.D, d.P
    DP = D * P
    if form == "dense":
        ldx = ldgy = ldgx = D
        phi_ld = DP
    else:
        ldx, ldgy, ldgx, phi_ld = D + 3, D + 2, D + 4, DP + PAD
    x, gy = padded(d.x[:B], ldx, device), padded(d.gy_p[:B], ldgy, device)
    phi = padded(d.phi[:B].reshape(B, DP), phi_ld, device)
    gl = dev(d.gl_p[:B], device) if B else torch.zeros(1, device=device)
    gx = torch.full((max(B, 1), ldgx), NAN, device=device)
    gphi = torch.full((max(B, 1), DP), NAN, device=device)
    E.check(backward_abi(d.kind, d.K, d.deg, x, ldx, phi, phi_ld, B, D, gy, ldgy, gl, gx, ldgx, gphi, None, device))
    return gx, gphi, phi


def run_shared(d, device, B, rows, ld_extra=0):
    """grad_x (B, D) and the accumulated table gradient (D, P) of one shared-table call through a workspace of
    `rows` rows."""
    D, P = d.D, d.P
    ld = D + ld_extra
    x, gy = padded(d.xs[:B], ld, device), padded(d.gy_s[:B], ld, device)
    gl = dev(d.gl_s[:B], device) if B else torch.zeros(1, device=device)
    gx = torch.full((max(B, 1), ld), NAN, device=device)
    gphi = torch.zeros(D, P, device=device)
    ws = torch.empty(E.lib().zk_univariate_backward_workspace_bytes(max(rows, 1), D, P, 0), dtype=torch.uint8, device=device)
    E.check(backward_abi(d.kind, d.K, d.deg, x, ld, dev(d.table, device), 0, B, D, gy, ld, gl, gx, ld, gphi, ws, device))
    return gx, gphi


def odd_rows(B):
    """A workspace row count that does not divide B (None for B < 3)."""
    return next((r for r in range(2, B) if B % r), None)


# --------------------------------------------------------------------------- #
# plan query and oracle parity
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
def test_plan_query_matches_restatement(device):
    for name, (kind, K, deg, D) in CASES.items():
        for form in FORMS:
            for B in batches_of(plan_of(name, form)["rows"]):
                p = uni_bwd_plan_of(kind, B, D, K, deg, phi_ld_of(name, form))
                st, got = query(kind, B, D, K, deg, phi_ld_of(name, form))
                assert st == E.ZK_OK and got == want(p), (name, form, B, got, want(p))
    for name, (args, _) in REFUSALS.items():
        assert query(*args)[0] == E.ZK_EINVAL, name


MATRIX = [(n, f) for n in CASES for f in (1, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,fast", MATRIX, ids=[f"{n}-{'fast' if f else 'ieee'}" for n, f in MATRIX])
def test_oracle_parity_matrix(device, math_mode, name, fast):
    math_mode(fast)
    d = data(name)
    kind, K, D, P = d.kind, d.K, d.D, d.P
    mode = "fast" if fast else "ieee"
    # per sample, contiguous and padded; the full batch first: every prefix must give its first rows bit for bit
    gx_full, gphi_full, _ = run_per_sample(d, device, d.n, "dense")
    gx_full, gphi_full = cpu(gx_full), cpu(gphi_full)
    check_grads(kind, K, f"{name} {mode} B={d.n}", gx_full, gphi_full.reshape(d.n, D, P), d.gx64, d.gphi64)
    for B in batches_of(plan_of(name, "dense")["rows"]):
        what = f"{name} {mode} B={B}"
        gx, gphi, _ = run_per_sample(d, device, B, "dense")
        gxp, gphip, phip = run_per_sample(d, device, B, "padded")
        gx, gphi, gxp, gphip = cpu(gx), cpu(gphi), cpu(gxp), cpu(gphip)
        assert np.isnan(gxp[:, D:]).all() and np.isnan(cpu(phip)[:, D * P :]).all(), what + ": a pad was written"
        if B == 0:
            assert np.isnan(gx).all() and np.isnan(gphi).all() and np.isnan(gxp).all(), what + ": B = 0 wrote"
            continue
        assert np.array_equal(gx, gx_full[:B]) and np.array_equal(gphi, gphi_full[:B]), what + ": prefix differs"
        assert np.array_equal(gxp[:, :D], gx) and np.array_equal(gphip, gphi), what + ": padded rows differ"
    # shared table: one chunk, 1-row chunks, and chunks that do not divide the batch
    for B in batches_of(plan_of(name, "shared")["rows"]):
        what = f"{name} {mode} shared B={B}"
        gx1, gt1 = run_shared(d, device, B, B, ld_extra=3)
        gx1, gt1 = cpu(gx1), cpu(gt1)
        if B == 0:
            assert np.isnan(gx1).all() and not gt1.any(), what + ": B = 0 wrote"
            continue
        assert np.isnan(gx1[:, D:]).all(), what + ": grad_x pad written"
        check_grads(kind, K, what, gx1[:, :D], None, d.gxs64[:B], None)
        check_table(kind, K, what + " (one chunk)", gt1, d.gphis_cum[B])
        for rows in (1, odd_rows(B)):
            if rows is None or rows >= B:
                continue
            gxr, gtr = run_shared(d, device, B, rows)
            assert np.array_equal(cpu(gxr), gx1[:, :D]), f"{what}: grad_x depends on the {rows}-row workspace"
            check_table(kind, K, f"{what} ({rows}-row chunks)", cpu(gtr), d.gphis_cum[B])


@pytest.mark.gpu
def test_refusals_of_the_entry_points(device):
    """Each refusal returns ZK_EINVAL before anything runs: grad_x, grad_phi and phi keep their NaN / values."""
    x = torch.zeros(64 * 64, device=device)
    phi = torch.zeros(17 * 3071 + 64, device=device)
    gy, gl = torch.zeros_like(x), torch.zeros(64, device=device)
    ws = torch.empty(E.lib().zk_univariate_backward_workspace_bytes(2, 17, 3071, 0), dtype=torch.uint8, device=device)
    gx, gphi = torch.full_like(x, NAN), torch.full((64 * 3071,), NAN, device=device)

    def call(kind, K, deg, phi_ld, B, D, gp=None, w=None, **kw):
        return backward_abi(kind, K, deg, x, D, phi, phi_ld, B, D, gy, D, gl, gx, D, gp, w, device, **kw)

    refusals = {
        "rqs bins 0": call(RQS, 0, 0, 0, 4, 4),
        "rqs bins 1025": call(RQS, 1025, 0, 4 * 3074, 4, 4),
        "gauss components 0": call(GAUSS, 0, 0, 0, 4, 4),
        "gauss components 1025": call(GAUSS, 1025, 0, 0, 4, 4),
        "sosp degree 16": call(SOSP, 3, 16, 0, 4, 4),
        "sosp 512 x 2": call(SOSP, 512, 1, 0, 4, 4),
        "sosp bound 0": call(SOSP, 3, 4, 4 * 16, 4, 4, bound=-1.0),
        "bernstein degree 60": call(BERN, 0, 60, 0, 4, 4),
        "bernstein eps 0": call(BERN, 0, 16, 4 * 17, 4, 4, eps=0.0),
        "bernstein eps 1/2": call(BERN, 0, 16, 4 * 17, 4, 4, eps=0.5),
        "slope 0": call(RQS, 8, 0, 4 * 23, 4, 4, slope=0.0),
        "slope 1": call(AFFINE, 0, 0, 4 * 2, 4, 4, slope=1.0),
        "phi_ld short": call(RQS, 8, 0, 4 * 23 - 1, 4, 4),
        "row over 200 KB": call(RQS, 1024, 0, 17 * 3071, 2, 17),
        "shared row over 200 KB": call(RQS, 1024, 0, 0, 2, 17),
        "shared row over 200 KB, grad_phi": call(RQS, 1024, 0, 0, 2, 17, gp=gphi, w=ws),
        "rqs bins 1025, grad_phi": call(RQS, 1025, 0, 4 * 3074, 4, 4, gp=gphi),
    }
    torch.cuda.synchronize(device)
    for what, st in refusals.items():
        assert st == E.ZK_EINVAL, f"{what}: status {st}"
    assert torch.isnan(gx).all() and torch.isnan(gphi).all(), "a refused call wrote"
    big = torch.empty(E.lib().zk_univariate_backward_workspace_bytes(2, 16, 3071, 0), dtype=torch.uint8, device=device)
    assert call(RQS, 1024, 0, 0, 2, 16, gp=gphi, w=big) == E.ZK_OK  # the largest shared RQS table that fits, in place
    torch.cuda.synchronize(device)


def _alias_case(device, B=40, D=3, K=8):
    g = np.random.default_rng(11)
    P = 3 * K - 1
    phi = params_of(RQS, K, 0, B, D, g)
    x = (g.standard_normal((B, D)) * 2).astype(np.float32)
    gy, gl = g.standard_normal((B, D)).astype(np.float32), g.standard_normal(B).astype(np.float32)
    return P, phi, dev(x, device), dev(gy, device), dev(gl, device)


@pytest.mark.gpu
def test_overlapping_grad_phi_is_refused(device):
    """grad_phi overlapping phi is refused (ZK_EINVAL, nothing written, phi intact) unless it is phi itself with
    phi_ld == D P; a grad_phi that starts right after phi's last element is accepted."""
    B, D, K = 40, 3, 8
    P, phi, x, gy, gl = _alias_case(device, B, D, K)
    DP = D * P
    ws = torch.empty(E.lib().zk_univariate_backward_workspace_bytes(7, D, P, 0), dtype=torch.uint8, device=device)

    def call(ph, phi_ld, gp, w=None):
        gx = torch.full((B, D), NAN, device=device)
        st = backward_abi(RQS, K, 0, x, D, ph, phi_ld, B, D, gy, D, gl, gx, D, gp, w, device)
        torch.cuda.synchronize(device)
        return st, gx

    # per-sample rows with phi_ld > D P: grad_phi == phi, or inside phi's rows, or overlapping its tail
    buf = torch.full((B * (DP + PAD) + 2 * B * DP,), NAN, device=device)
    rows = buf[: B * (DP + PAD)].view(B, DP + PAD)
    rows[:, :DP] = dev(phi.reshape(B, DP), device)
    base, f4 = rows.data_ptr(), 4
    last = (B - 1) * (DP + PAD) + DP  # one past phi's last element
    cases = {
        "same pointer, phi_ld > D P": (rows, DP + PAD, base),
        "inside the rows": (rows, DP + PAD, base + f4 * (DP + 1)),
        "over the tail": (rows, DP + PAD, base + f4 * (last - 1)),
        "dense, one element on": (rows, DP, base + f4),
        "dense, starts before phi": (buf[B * DP :], DP, base + f4 * DP),
    }
    before = rows.clone()
    for what, (ph, ld, gp) in cases.items():
        st, gx = call(ph, ld, gp)
        assert st == E.ZK_EINVAL, f"{what}: status {st}"
        assert torch.isnan(gx).all(), f"{what}: grad_x written"
        assert torch.equal(torch.nan_to_num(rows, 7.0), torch.nan_to_num(before, 7.0)), f"{what}: phi written"
    # right after phi's last element: no overlap, accepted (the pads of the last row are not phi)
    st, _ = call(rows, DP + PAD, base + f4 * last)
    assert st == E.ZK_OK
    # shared table: grad_phi == phi, or overlapping the table, with a workspace
    tbuf = torch.full((3 * DP,), NAN, device=device)
    table = tbuf[DP : 2 * DP]
    table.copy_(dev(phi[0].reshape(-1), device))
    tb = table.clone()
    for what, gp in (("table itself", table.data_ptr()), ("table + 1", table.data_ptr() + f4), ("table - 1", table.data_ptr() - f4)):
        st, gx = call(table, 0, gp, ws)
        assert st == E.ZK_EINVAL, f"shared {what}: status {st}"
        assert torch.isnan(gx).all() and torch.equal(torch.nan_to_num(table, 7.0), torch.nan_to_num(tb, 7.0)), what
    st, _ = call(table, 0, table.data_ptr() + f4 * DP, ws)
    assert st == E.ZK_OK


# --------------------------------------------------------------------------- #
# contracts
# --------------------------------------------------------------------------- #

CONTRACT_CASES = ["affine_d7", "rqs8_d3", "rqs5_d7", "rqs16_d64", "gauss8_d4", "gauss5_d7", "sosp_d4", "sosp23_d5",
                  "bern16_d4", "bern7_d3"]  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("name", CONTRACT_CASES)
def test_nulls_in_place_and_reproducible_reduction(device, name):
    """NULL grad_y / grad_ladj equal zeros, NULL grad_x / grad_phi leave the other output bit for bit, grad_phi == phi
    (phi_ld == D P) equals the out-of-place call, and two shared-table reductions agree bit for bit."""
    d = data(name)
    kind, K, deg, D, P = d.kind, d.K, d.deg, d.D, d.P
    B = 2 * plan_of(name, "dense")["rows"] + 5
    B = min(B, d.n)
    DP = D * P
    x, gy, gl = dev(d.x[:B], device), dev(d.gy_p[:B], device), dev(d.gl_p[:B], device)
    zy, zl = torch.zeros_like(gy), torch.zeros_like(gl)
    phi = dev(d.phi[:B].reshape(B, DP), device)

    def call(gyv, glv, want_x=True, want_phi=True, ph=None, gp=None):
        gx = torch.full((B, D), NAN, device=device) if want_x else None
        gphi = gp if gp is not None else (torch.full((B, DP), NAN, device=device) if want_phi else None)
        E.check(backward_abi(kind, K, deg, x, D, phi if ph is None else ph, DP, B, D, gyv, D, glv, gx, D, gphi, None, device))
        return gx, gphi

    gx0, gp0 = call(gy, gl)
    for what, (gx1, gp1), (gx2, gp2) in (("grad_y", call(None, gl), call(zy, gl)), ("grad_ladj", call(gy, None), call(gy, zl))):
        assert torch.equal(gx1, gx2) and torch.equal(gp1, gp2), f"{name}: NULL {what} is not zeros"
    gxn, _ = call(gy, gl, want_phi=False)
    _, gpn = call(gy, gl, want_x=False)
    assert torch.equal(gxn, gx0) and torch.equal(gpn, gp0), f"{name}: a NULL output changes the other"
    inplace = phi.clone()
    gxi, _ = call(gy, gl, ph=inplace, gp=inplace)
    torch.cuda.synchronize(device)
    assert torch.equal(gxi, gx0) and torch.equal(inplace, gp0), f"{name}: grad_phi == phi differs from out of place"
    # shared table: two runs, and NULL grad_phi leaving grad_x
    Bs = min(d.n, 3 * plan_of(name, "shared")["rows"] + 1)
    r = odd_rows(Bs) or 1
    (ga, ta), (gb, tb) = run_shared(d, device, Bs, r), run_shared(d, device, Bs, r)
    assert torch.equal(ga, gb) and torch.equal(ta, tb), f"{name}: two shared-table reductions differ"
    xs, gys, gls = dev(d.xs[:Bs], device), dev(d.gy_s[:Bs], device), dev(d.gl_s[:Bs], device)
    gxs = torch.full((Bs, D), NAN, device=device)
    E.check(backward_abi(kind, K, deg, xs, D, dev(d.table, device), 0, Bs, D, gys, D, gls, gxs, D, None, None, device))
    torch.cuda.synchronize(device)
    assert torch.equal(gxs, ga), f"{name}: NULL grad_phi changes the shared-table grad_x"


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
@pytest.mark.parametrize("name", ["gauss256_d64", "rqs1024_d16"])
def test_shared_table_rewritten_in_place(device, math_mode, name, fast):
    """Tables of 128 KB and 192 KB (one row per tile, rewritten in place): grad_x equals the per-sample call on the
    table broadcast to every row bit for bit, and the table gradient matches the fp64 reference; the forward runs the
    same shapes."""
    math_mode(fast)
    d = data(name)
    kind, K, deg, D, P = d.kind, d.K, d.deg, d.D, d.P
    p = plan_of(name, "shared")
    assert p["in_place"] and p["smem"] > 100 * KB and query(kind, 50, D, K, deg, 0) == (E.ZK_OK, (1, p["smem"], 0))
    B = 50
    x, gy, gl = dev(d.xs[:B], device), dev(d.gy_s[:B], device), dev(d.gl_s[:B], device)
    table = dev(d.table, device)
    gx_t, gt = run_shared(d, device, B, 7)
    full = table.reshape(1, -1).expand(B, -1).contiguous()
    gx_b = torch.full((B, D), NAN, device=device)
    gp_b = torch.full((B, D * P), NAN, device=device)
    E.check(backward_abi(kind, K, deg, x, D, full, D * P, B, D, gy, D, gl, gx_b, D, gp_b, None, device))
    y, ladj = torch.empty(B, D, device=device), torch.empty(B, device=device)
    L, st = E.lib(), E.stream_ptr(device)
    if kind == RQS:
        E.check(L.zk_rqs_forward(x.data_ptr(), D, table.data_ptr(), 0, B, D, K, RQS_BOUND, SLOPE, y.data_ptr(), D, ladj.data_ptr(), 0, st))
    else:
        E.check(L.zk_gaussianization_forward(x.data_ptr(), D, table.data_ptr(), 0, B, D, K, y.data_ptr(), D, ladj.data_ptr(), 0, st))
    torch.cuda.synchronize(device)
    assert torch.equal(gx_t, gx_b), f"{name}: the in-place table changes grad_x"
    check_table(kind, K, name, cpu(gt), d.gphis_cum[B])
    check_table(kind, K, name + " (rows summed)", cpu(gp_b).reshape(B, D, P).sum(0), d.gphis_cum[B])
    assert torch.isfinite(y).all() and torch.isfinite(ladj).all()


# --------------------------------------------------------------------------- #
# layer paths through the same kernel
# --------------------------------------------------------------------------- #


def _layer_call(handle, x, c, gy, gl, device, grads=None):
    L = E.lib()
    B, D = x.shape
    ws = torch.empty(max(L.zk_layer_backward_workspace_bytes(handle, B), 1), dtype=torch.uint8, device=device)
    gx = torch.full((B, D), NAN, device=device)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    C = 0 if c is None else c.shape[1]
    E.check(L.zk_layer_backward(handle, p(x), D, p(c), C, B, p(gy), D, p(gl), p(gx), D, None, C,
                                None if grads is None else ctypes.byref(grads), p(ws), ws.numel(), E.stream_ptr(device)))  # fmt: skip
    torch.cuda.synchronize(device)
    return cpu(gx)


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
def test_gf_layer_with_a_128k_table(device, math_mode, fast):
    """An unconditional element-wise GF layer, D = 64 and K = 256 (a 128 KB table), through zk_layer_backward: grad_x
    and the table gradient summed over the batch against gf_reference.grad at the GF bar."""
    from zuko_b200.flows import GF

    math_mode(fast)
    torch.manual_seed(0)
    D, K, B = 64, 256, 300
    flow = GF(D, transforms=1, components=K).to(device)
    shift = flow.transform.transforms[0].phi[0].detach()
    scale = flow.transform.transforms[0].phi[1].detach()
    g = np.random.default_rng(5)
    x = g.standard_normal((B, D)).astype(np.float32)
    gy, gl = g.standard_normal((B, D)).astype(np.float32), g.standard_normal(B).astype(np.float32)
    sh, sc = cpu(shift), cpu(scale)
    w = gauss_ok(x.astype(np.float64), sh, sc).all(-1)
    assert w.mean() > 0.5
    gy[~w], gl[~w] = 0.0, 0.0
    fc = flow()._flow_call()[0]
    handle = fc._handles[0]
    gphi = torch.zeros(D, 2 * K, device=device)
    lg = E.LayerGrads()
    lg.grad_phi = gphi.data_ptr()
    gx = _layer_call(handle, dev(x, device), None, dev(gy, device), dev(gl, device), device, lg)
    rgx, rgs, rgc = GR.grad(x.astype(np.float64), sh, sc, gy.astype(np.float64), np.broadcast_to(gl[:, None].astype(np.float64), x.shape))
    check_tensor(GAUSS, f"GF layer {'fast' if fast else 'ieee'} grad_x", gx, rgx)
    check_table(GAUSS, K, f"GF layer {'fast' if fast else 'ieee'}", cpu(gphi), np.concatenate([rgs, rgc], -1).sum(0))


@pytest.mark.gpu
def test_gf_flow_with_256_components_trains(device):
    """GF(64, components=256): log_prob(x).sum().backward() runs and leaves finite gradients on every parameter."""
    from zuko_b200.flows import GF

    torch.manual_seed(0)
    flow = GF(64, components=256).to(device)
    x = torch.randn(257, 64, generator=torch.Generator().manual_seed(1)).to(device)
    flow().log_prob(x).sum().backward()
    grads = [p.grad for p in flow.parameters()]
    assert grads and all(gr is not None and torch.isfinite(gr).all() for gr in grads)


def _rqs_coupling():
    from zuko_b200.distributions import DiagNormal
    from zuko_b200.flows import GeneralCouplingTransform
    from zuko_b200.lazy import Flow, UnconditionalDistribution
    from zuko_b200.transforms import MonotonicRQSTransform

    torch.manual_seed(0)
    mask = torch.tensor([1, 0, 0, 1, 0, 1, 0, 0, 0, 0], dtype=torch.bool)  # 7 transformed columns, not contiguous
    t = GeneralCouplingTransform(10, 3, mask=mask, univariate=MonotonicRQSTransform, shapes=[(8,), (8,), (7,)],
                                 hidden_features=[64, 64])  # fmt: skip
    return Flow([t], UnconditionalDistribution(DiagNormal, torch.zeros(10), torch.ones(10), buffer=True)).eval()


# (flow, member): a coupling layer (its transformed columns reached through dim_map) and an NCSF layer (the
# circular shift in front of the spline)
LAYER_PATHS = {"coupling": (_rqs_coupling, 0), "ncsf": (lambda: build_flow("ncsf34"), 0)}


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(LAYER_PATHS))
def test_layer_paths(device, key):
    """zk_layer_backward against oracle_grad.layer_backward at B = R - 1, R + 1 and 3R + 77 (R: the backward tile of the
    layer's transformed dims), 5e-5 of the largest entry per tensor (test_gpu_backward_abi.py)."""
    make, i = LAYER_PATHS[key]
    flow = make()
    spec = O.flowspec_from_module(flow)
    layer = spec.layers[i]
    D = spec.layers[0].features
    C = flow.transform.transforms[0].context
    nt = int((~np.asarray(layer.mask)).sum()) if layer.kind == "coupling" else D
    R = uni_bwd_plan_of(RQS, 1 << 20, nt, layer.bins, 0, nt * (3 * layer.bins - 1))["rows"]
    assert layer.univariate == ("crqs" if key == "ncsf" else "rqs"), layer.univariate
    flow = flow.to(device)
    for B in (R - 1, R + 1, 3 * R + 77):
        gen = torch.Generator().manual_seed(B)
        c = torch.randn(B, C, generator=gen).numpy() if C else None
        z = (torch.randn(B, D, generator=gen) * 2).numpy().astype(np.float64)
        for lay in spec.layers[:i]:
            z, _ = lay.forward(z, c, np.float64)
        x = np.asarray(z, np.float32)
        gy, gl = torch.randn(B, D, generator=gen).numpy(), torch.randn(B, generator=gen).numpy()
        kink = relu_kink_rows(types.SimpleNamespace(layers=[layer]), x, c)
        gy[kink], gl[kink] = 0.0, 0.0
        fc = flow(None if c is None else dev(c[:1], device))._flow_call()[0]
        gx = _layer_call(fc._handles[i], dev(x, device), None if c is None else dev(c, device), dev(gy, device), dev(gl, device), device)
        ogx, _, _ = OG.layer_backward(layer, x.astype(np.float64), c, gy, gl)
        scale = max(float(np.abs(ogx).max()), 1e-30)
        err = float(np.abs(gx - ogx).max()) / scale
        assert err <= 5e-5, f"{key} B={B}: grad_x max err {err:.3e} of {scale:.3e}"
