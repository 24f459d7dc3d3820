"""GPU tests of the stand-alone bijector kernel (uni_kernel, bijectors.cu) and its small element-wise neighbours at
their tile-plan, staging, reduction, instantiation, batch and stride edges, against fp64 references.

* `uni_plan_of` restates in numpy what uni_plan (bijectors.cu) decides for a call: the refusals, the rows per tile R
  (the 24 KB rule, the ceil(256 / D) floor, the 96 KB cap, the batch cap), the dynamic shared memory, the bulk-staging
  verdict, the ladj reduction (warp shuffle or fixed order) and the compile-time instantiation.  A test without a GPU
  checks that the case table reaches every cell; on the GPU `zk_univariate_plan` must report the same plan.
* Oracle parity: every case at batches 0, 1, R - 1, R, R + 1, 2R - 1 and 3R + 77, in both zk_set_fast_math modes,
  forward (y and the summed ladj) and inverse, on inputs at +-bound, its float32 neighbours, bound + 1, +-1e30, on
  RQS knots and at the Bernstein eps / 1 - eps branch edges.
* The C ABI (padded rows of x, y and phi, y aliasing x, NULL outputs, accumulate), bitwise properties, the layer paths
  that run the kernel (coupling, element-wise with a broadcast context, an unfused last layer with the DiagNormal term)
  and the small kernels (softclip, permute, rotate, circular shift, box uniform, diag normal).

Bars, per family, those of the existing unit tests (none looser):
* RQS (test_gpu_parity.py::test_rqs_forward_inverse, its s01 case): y within max(5e-6 max(|y64|, 1), 3 |y32 - y64|),
  each element's ladj within max(2e-5, 3 |l32 - l64|) (the summed ladj within the sum of those), the inverse within
  max(2e-5 max(|x64|, 1), 3 |x32 - x64|); ref32 is the oracle evaluated in float32.
* Affine (test_gpu_parity.py::test_affine): y and x within 5e-6 max(|ref|, 1); 5e-6 per element of the ladj.
* Gaussianization, SOSP, Bernstein (test_gpu_gf.py, test_gpu_sospf.py, test_gpu_bpf.py): 1e-5 max(|ref64|, 1) for y and
  per element of the ladj, without the 2 |ref32 - ref64| term those tests add (the fp64 restatements have no float32
  twin).  The bisection inverses add two final intervals 2 (2 bound / 2^n) to the absolute term.
  Compared only where the fp64 map is well-conditioned (the float32 rounding of f cannot move the answer past the
  bar): for the inverses f'(x64) >= 0.5 and |x64| <= bound - 2 intervals; for Gaussianization, forward and inverse,
  |C mean_k erf(u_k / sqrt 2)| <= 0.99, where erfinv's derivative is at most 24 (beyond it the reference's own float32
  forward drifts, which test_gpu_gf.py's ref32 term records).  Bernstein ladj: where the float32 t takes the fp64
  branch (test_bpf_host.same_branch)."""

import ctypes
import math
import zlib

import numpy as np
import pytest
import torch
from scipy.special import erf

import bpf_reference as BR
import gf_reference as GR
import sospf_reference as SR
from oracle import oracle as O
from test_bpf_host import same_branch
from zuko_b200 import _engine as E

SEED = 0
THREADS = 256
AFFINE, RQS, GAUSS, SOSP, BERN = E.ZK_UNI_AFFINE, E.ZK_UNI_RQS, E.ZK_UNI_GAUSS, E.ZK_UNI_SOSP, E.ZK_UNI_BERNSTEIN
KIND_NAMES = {AFFINE: "affine", RQS: "rqs", GAUSS: "gauss", SOSP: "sosp", BERN: "bernstein"}
SLOPE, RQS_BOUND, BISECT_BOUND, BERN_BOUND, BERN_EPS = 1e-3, 5.0, 10.0, 5.0, 1e-6
STEPS_10 = math.ceil(math.log2(2 * BISECT_BOUND / 1e-6))  # 25
F32_MAX = float(np.finfo(np.float32).max)


def n_params(kind, K, degree):
    return {AFFINE: 2, RQS: 3 * K - 1, GAUSS: 2 * K, SOSP: K * (degree + 1) + 1, BERN: degree + 1}[kind]


# --------------------------------------------------------------------------- #
# the plan, restated
# --------------------------------------------------------------------------- #


def uni_plan_of(kind, B, D, K, degree, phi_ld, phi_addr=0):
    """What uni_plan decides.  Returns {"ok": False, "why": ...} for a refusal, else rows / smem / bulk / shuffle /
    bins and the rule that set R before the batch cap ("24k", "floor", "cap96")."""
    if B < 0 or D <= 0:
        return {"ok": False, "why": "shape"}
    if B == 0:
        return {"ok": True, "rows": 0, "smem": 0, "bulk": 0, "shuffle": 0, "bins": 0, "rule": None, "capped": False}
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
    row_bytes = D * P * 4
    if row_bytes + 4 * D > 200 * 1024:
        return {"ok": False, "why": "row"}
    r24, floor = 24 * 1024 // row_bytes, -(-THREADS // D)
    R = max(r24, floor)
    rule = "24k" if r24 >= floor else "floor"
    while R > 1 and R * (row_bytes + 4 * D) > 96 * 1024:
        R -= 1
        rule = "cap96"
    R = max(R, 1)
    capped = R > B
    R = min(R, B)
    bins = {RQS: K if K in (4, 8, 16) else 0, GAUSS: K if K in (8, 16) else 0, AFFINE: 0,
            SOSP: 3 if (K, degree) == (3, 4) else 0, BERN: 17 if degree == 16 else 0}[kind]  # fmt: skip
    bulk = phi_ld == D * P and phi_addr % 16 == 0 and (R * row_bytes) % 16 == 0
    smem = (row_bytes if phi_ld == 0 else R * row_bytes) + R * D * 4
    return {"ok": True, "rows": R, "smem": smem, "bulk": int(bulk), "shuffle": int(D <= 32 and D & (D - 1) == 0),
            "bins": bins, "rule": rule, "capped": capped, "P": P, "row_bytes": row_bytes}  # fmt: skip


def staging_of(plan, B, layout, offset):
    """The staging path the kernel takes for the tiles of a batch of B rows: a set of cells."""
    if layout == "shared":
        return {"shared"}
    if layout == "strided":
        return {"strided"}
    if offset % 4:
        return {"misaligned"}
    if not plan["bulk"]:
        return {"tile_bytes"}
    last = B % plan["rows"]
    return {"bulk", "bulk_partial"} if last and (last * plan["row_bytes"]) % 16 else {"bulk"}


# name -> (kind, K, degree, D, layout, phi offset in floats); layout "dense" (phi_ld = D P), "strided" (phi_ld = D P + 5,
# NaN pads) or "shared" (phi_ld = 0)
CASES = {
    "affine_d1": (AFFINE, 0, 0, 1, "dense", 0),            # 24 KB rule: R = 3072, 12 pair iterations; bulk + partial
    "affine_d2_off2": (AFFINE, 0, 0, 2, "dense", 2),       # misaligned phi
    "affine_d33_strided": (AFFINE, 0, 0, 33, "strided", 0),  # fixed order, 12 pair iterations
    "affine_d4_shared": (AFFINE, 0, 0, 4, "shared", 0),
    "rqs4_d8": (RQS, 4, 0, 8, "dense", 0),
    "rqs8_d16": (RQS, 8, 0, 16, "dense", 0),
    "rqs8_d16_off1": (RQS, 8, 0, 16, "dense", 1),
    "rqs8_d16_strided": (RQS, 8, 0, 16, "strided", 0),
    "rqs16_d32": (RQS, 16, 0, 32, "dense", 0),             # the ceil(256 / D) floor: R = 8
    "rqs16_d300": (RQS, 16, 0, 300, "dense", 0),           # R = 1, 57600 B of shared memory
    "rqs16_d300_shared": (RQS, 16, 0, 300, "shared", 0),
    "rqs5_d3": (RQS, 5, 0, 3, "dense", 0),                 # runtime K, fixed order over 2 pair iterations
    "rqs101_d40": (RQS, 101, 0, 40, "dense", 0),           # 96 KB cap: R = 2
    "rqs1024_d16": (RQS, 1024, 0, 16, "dense", 0),         # R = 1, 192 KB
    "rqs8_d64_strided": (RQS, 8, 0, 64, "strided", 0),
    "gauss8_d4": (GAUSS, 8, 0, 4, "dense", 0),
    "gauss16_d2_strided": (GAUSS, 16, 0, 2, "strided", 0),
    "gauss3_d3": (GAUSS, 3, 0, 3, "dense", 0),             # R row_bytes % 16 != 0
    "gauss8_d33_shared": (GAUSS, 8, 0, 33, "shared", 0),
    "sosp_d4": (SOSP, 3, 4, 4, "dense", 0),
    "sosp_d8_strided": (SOSP, 3, 4, 8, "strided", 0),
    "sosp23_d3_off3": (SOSP, 2, 3, 3, "dense", 3),
    "sosp_d16_shared": (SOSP, 3, 4, 16, "shared", 0),
    "bern16_d4": (BERN, 0, 16, 4, "dense", 0),
    "bern16_d3_strided": (BERN, 0, 16, 3, "strided", 0),
    "bern7_d8": (BERN, 0, 7, 8, "dense", 0),
    "bern7_d2_shared": (BERN, 0, 7, 2, "shared", 0),
}  # fmt: skip
PAD = 5


def phi_ld_of(case):
    kind, K, deg, D, layout, _ = CASES[case]
    P = n_params(kind, K, deg)
    return {"dense": D * P, "strided": D * P + PAD, "shared": 0}[layout]


def plan_of(case, B=1 << 20):
    kind, K, deg, D, layout, off = CASES[case]
    return uni_plan_of(kind, B, D, K, deg, phi_ld_of(case), 4 * off)


def batches_of(R):
    return sorted({0, 1, max(R - 1, 1), R, R + 1, 2 * R - 1, 3 * R + 77})


# refusals of the plan: (kind, B, D, K, degree, phi_ld) -> reason
REFUSALS = {
    "row_over_200k": ((RQS, 10, 17, 1024, 0, 17 * 3071), "row"),
    "phi_ld_short": ((RQS, 10, 4, 8, 0, 4 * 23 - 1), "phi_ld"),
    "phi_ld_one": ((AFFINE, 10, 4, 0, 0, 1), "phi_ld"),
    "rqs_k0": ((RQS, 10, 4, 0, 0, 0), "K"),
    "rqs_k1025": ((RQS, 10, 4, 1025, 0, 0), "K"),
    "gauss_k0": ((GAUSS, 10, 4, 0, 0, 0), "K"),
    "sosp_degree16": ((SOSP, 10, 4, 3, 16, 0), "degree"),
    "sosp_too_many": ((SOSP, 10, 4, 512, 1, 0), "degree"),
    "bern_degree60": ((BERN, 10, 4, 0, 60, 0), "degree"),
    "kind_crqs": ((E.ZK_UNI_CRQS, 10, 4, 8, 0, 0), "kind"),
    "d0": ((RQS, 10, 0, 8, 0, 0), "shape"),
}


def test_plan_table_reaches_every_cell():
    """The case table reaches every tile-row rule, staging path, reduction, instantiation and refusal (no GPU)."""
    rules, staging, shuffle_d, fixed_d, inst = set(), set(), set(), set(), set()
    multi_iter_fixed = capped = big_r1 = False
    for name, (kind, K, deg, D, layout, off) in CASES.items():
        p = plan_of(name)
        assert p["ok"], name
        rules.add(p["rule"])
        for B in batches_of(p["rows"]):
            if B == 0:
                continue
            pb = uni_plan_of(kind, B, D, K, deg, phi_ld_of(name), 4 * off)
            capped |= pb["capped"]
            staging |= staging_of(pb, B, layout, off)
        (shuffle_d if p["shuffle"] else fixed_d).add(D)
        multi_iter_fixed |= not p["shuffle"] and p["rows"] * D > THREADS
        big_r1 |= p["rows"] == 1 and p["smem"] > 48 * 1024
        inst.add((kind, p["bins"]))
    assert rules == {"24k", "floor", "cap96"}, rules
    assert capped and big_r1 and multi_iter_fixed
    assert staging == {"bulk", "bulk_partial", "misaligned", "tile_bytes", "strided", "shared"}, staging
    assert shuffle_d == {1, 2, 4, 8, 16, 32} and {3, 33, 64, 300} <= fixed_d, (shuffle_d, fixed_d)
    assert inst == {(AFFINE, 0), (RQS, 4), (RQS, 8), (RQS, 16), (RQS, 0), (GAUSS, 8), (GAUSS, 16), (GAUSS, 0), (SOSP, 3),
                    (SOSP, 0), (BERN, 17), (BERN, 0)}, inst  # fmt: skip
    # the cells the issue names by value
    assert plan_of("affine_d1")["rows"] == 3072 and -(-3072 // THREADS) == 12
    assert plan_of("rqs16_d32")["rows"] == 8 and plan_of("rqs16_d32")["rule"] == "floor"
    assert plan_of("rqs101_d40")["rows"] == 2 and plan_of("rqs101_d40")["rule"] == "cap96"
    assert plan_of("rqs1024_d16")["rows"] == 1 and plan_of("rqs1024_d16")["smem"] == 192 * 1024
    assert plan_of("rqs16_d300")["rows"] == 1 and plan_of("rqs16_d300")["smem"] > 48 * 1024
    for name, (args, why) in REFUSALS.items():
        assert uni_plan_of(*args) == {"ok": False, "why": why}, name
    assert uni_plan_of(RQS, 10, 16, 1024, 0, 16 * 3071)["ok"]  # the largest RQS row that fits


# --------------------------------------------------------------------------- #
# GPU helpers
# --------------------------------------------------------------------------- #


@pytest.fixture
def math_mode():
    prev = E.lib().zk_set_fast_math(1)
    yield lambda fast: E.lib().zk_set_fast_math(int(fast))
    E.lib().zk_set_fast_math(prev)


def cpu(t):
    return t.detach().cpu().numpy().astype(np.float64)


def query(kind, B, D, K, deg, phi_ld, addr):
    R, smem, bulk, shfl, bins = ctypes.c_int(-1), ctypes.c_size_t(0), ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_int(-1)
    st = E.lib().zk_univariate_plan(kind, B, D, K, deg, phi_ld, ctypes.c_void_p(addr or None), ctypes.byref(R),
                                    ctypes.byref(smem), ctypes.byref(bulk), ctypes.byref(shfl), ctypes.byref(bins))  # fmt: skip
    return st, (R.value, smem.value, bulk.value, shfl.value, bins.value)


def want(p):
    return p["rows"], p["smem"], p["bulk"], p["shuffle"], p["bins"]


def forward_abi(kind, K, deg, x, ldx, phi, phi_ld, B, D, y, ldy, ladj, acc, device):
    L, st = E.lib(), E.stream_ptr(device)
    p = lambda t: None if t is None else (t if isinstance(t, int) else t.data_ptr())  # noqa: E731
    x, phi, y, ladj = p(x), p(phi), p(y), p(ladj)
    if kind == RQS:
        return L.zk_rqs_forward(x, ldx, phi, phi_ld, B, D, K, RQS_BOUND, SLOPE, y, ldy, ladj, acc, st)
    if kind == AFFINE:
        return L.zk_affine_forward(x, ldx, phi, phi_ld, B, D, SLOPE, y, ldy, ladj, acc, st)
    if kind == GAUSS:
        return L.zk_gaussianization_forward(x, ldx, phi, phi_ld, B, D, K, y, ldy, ladj, acc, st)
    if kind == SOSP:
        return L.zk_sosp_forward(x, ldx, phi, phi_ld, B, D, K, deg, BISECT_BOUND, SLOPE, y, ldy, ladj, acc, st)
    return L.zk_bernstein_forward(x, ldx, phi, phi_ld, B, D, deg, BERN_BOUND, BERN_EPS, y, ldy, ladj, acc, st)


def inverse_abi(kind, K, deg, y, ldy, phi, phi_ld, B, D, x, ldx, device, iterations=STEPS_10):
    L, st = E.lib(), E.stream_ptr(device)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    y, phi, x = p(y), p(phi), p(x)
    if kind == RQS:
        return L.zk_rqs_inverse(y, ldy, phi, phi_ld, B, D, K, RQS_BOUND, SLOPE, x, ldx, st)
    if kind == AFFINE:
        return L.zk_affine_inverse(y, ldy, phi, phi_ld, B, D, SLOPE, x, ldx, st)
    if kind == GAUSS:
        return L.zk_gaussianization_inverse(y, ldy, phi, phi_ld, B, D, K, BISECT_BOUND, iterations, x, ldx, st)
    if kind == SOSP:
        return L.zk_sosp_inverse(y, ldy, phi, phi_ld, B, D, K, deg, BISECT_BOUND, SLOPE, iterations, x, ldx, st)
    return L.zk_bernstein_inverse(y, ldy, phi, phi_ld, B, D, deg, BERN_BOUND, BERN_EPS, x, ldx, st)


def bound_of(kind):
    return {RQS: RQS_BOUND, AFFINE: RQS_BOUND, GAUSS: BISECT_BOUND, SOSP: BISECT_BOUND, BERN: BERN_BOUND}[kind]


def edges_of(kind):
    b = np.float32(bound_of(kind))
    e = [b, -b, np.nextafter(b, np.float32(np.inf)), np.nextafter(-b, np.float32(-np.inf)), np.nextafter(b, np.float32(0)),
         np.nextafter(-b, np.float32(0)), b + 1, -b - 1]  # fmt: skip
    if kind in (RQS, AFFINE, BERN):  # the polynomial and mixture maps overflow float32 there
        e += [1e30, -1e30]
    if kind == BERN:  # t = eps and t = 1 - eps, and their float32 neighbours
        for v in (np.float32(2 * BERN_BOUND * BERN_EPS - BERN_BOUND), np.float32(BERN_BOUND - 2 * BERN_BOUND * BERN_EPS)):
            e += [v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))]
    return np.array(e, np.float32)


def params_of(kind, K, deg, n_rows, D, g):
    """Per-sample parameters (n_rows, D, P), float32, seeded; rows do not depend on n_rows beyond their index."""
    P = n_params(kind, K, deg)
    r = g.standard_normal((n_rows, D, P))
    if kind == RQS:
        # beyond 256 bins the float32 knot sums alone carry ~1e-5 of rounding (the runtime-K kernel and the oracle's
        # float32 sum in different orders): those cases draw uniform bins, whose knots are exact, so that they test
        # the tile (R = 1, 192 KB at K = 1024) rather than the spline's conditioning
        r *= 0.1 if K <= 256 else 0.0
    elif kind == GAUSS:
        r[..., K:] *= 0.3
    elif kind == SOSP:
        r[..., :-1] *= 0.3
    return r.astype(np.float32)


def inputs_of(kind, K, phi, n_rows, D, g):
    """x (n_rows, D) float32: randn * bound / 2 (randn for Gaussianization) with every fourth element an edge and, for RQS, every fourth (offset by 2)
    a knot of its own spline."""
    b = bound_of(kind)
    spread = 1.0 if kind == GAUSS else b / 2  # the Gaussianization map saturates beyond a few units
    x = (g.standard_normal((n_rows, D)) * spread).astype(np.float32)
    flat = x.reshape(-1)
    e = edges_of(kind)
    idx = np.arange(1, flat.size, 4)
    if kind == GAUSS:  # edges on every third row only: the others keep a well-conditioned ladj sum
        idx = idx[(idx // D) % 3 == 0]
    flat[idx] = e[np.arange(idx.size) % e.size]
    if kind == RQS:
        X = O.rqs_knots(phi.astype(np.float64), K, RQS_BOUND, SLOPE)[0].reshape(-1, K + 1)
        idx = np.arange(2, flat.size, 4)
        flat[idx] = X[idx, idx % (K + 1)].astype(np.float32)
    return x


def split(kind, K, deg, phi):
    """The fp64 references' parameter arguments from (..., P)."""
    phi = np.asarray(phi, np.float64)
    if kind == GAUSS:
        return phi[..., :K], phi[..., K:]
    if kind == SOSP:
        return phi[..., :-1].reshape(*phi.shape[:-1], K, deg + 1), phi[..., -1]
    return (phi,)


def reference(kind, K, deg, x, phi):
    """fp64 forward: (y, per-element ladj, well-conditioned mask) and, for RQS, the float32 oracle (y32, l32)."""
    x64 = x.astype(np.float64)
    ok = np.ones(x.shape, bool)
    extra = None
    if kind == RQS:
        y, l = O.rqs_forward(x64, phi, K, RQS_BOUND, SLOPE)
        extra = O.rqs_forward(x, phi.astype(np.float32), K, RQS_BOUND, SLOPE, dtype=np.float32)
    elif kind == AFFINE:
        y, l = O.affine_forward(x64, phi, SLOPE)
    elif kind == GAUSS:
        shift, scale = split(kind, K, deg, phi)
        y, l = GR.forward(x64, shift, scale)
        ok = gauss_ok(x64, shift, scale)
    elif kind == SOSP:
        a, c = split(kind, K, deg, phi)
        y, l = SR.forward(x64, a, c, SLOPE, BISECT_BOUND)
    else:
        y, l = BR.forward(x64, np.asarray(phi, np.float64), BERN_BOUND, BERN_EPS)
    return y, l, ok, extra


def gauss_ok(x64, shift, scale):
    u = x64[..., None] * np.exp(scale) + shift
    return np.abs(GR.C * np.mean(erf(u / math.sqrt(2)), -1)) <= 0.99


def inverse_reference(kind, K, deg, y, phi):
    y64 = y.astype(np.float64)
    if kind == RQS:
        return O.rqs_inverse(y64, phi, K, RQS_BOUND, SLOPE), O.rqs_inverse(y, phi.astype(np.float32), K, RQS_BOUND, SLOPE, dtype=np.float32)
    if kind == AFFINE:
        return O.affine_inverse(y64, phi, SLOPE), None
    if kind == GAUSS:
        return GR.inverse(y64, *split(kind, K, deg, phi), BISECT_BOUND, 1e-6), None
    if kind == SOSP:
        a, c = split(kind, K, deg, phi)
        return SR.inverse(y64, a, c, SLOPE, BISECT_BOUND, 1e-6), None
    return BR.inverse(y64, np.asarray(phi, np.float64), BERN_BOUND, BERN_EPS), None


def interval(kind):
    b = BERN_BOUND if kind == BERN else BISECT_BOUND
    return 2 * b / 2 ** math.ceil(math.log2(2 * b / 1e-6))


def _fail(what, bad, ours, ref):
    i = tuple(int(v) for v in np.argwhere(bad)[0])
    raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} off the reference; first at {i}: ours {ours[i]!r} ref {ref[i]!r}")


def check_forward(kind, what, y, ladj, x, y64, l64, ok, extra):
    """y per element and the summed ladj per row against the family's bar (module docstring)."""
    huge = np.abs(y64) > F32_MAX
    if kind == RQS:
        y32, l32 = (np.asarray(v, np.float64) for v in extra)
        ty = np.maximum(5e-6 * np.maximum(np.abs(y64), 1.0), 3 * np.abs(y32 - y64))
        tl = np.maximum(2e-5, 3 * np.abs(l32 - l64))
    elif kind == AFFINE:
        ty = 5e-6 * np.maximum(np.abs(y64), 1.0)
        tl = np.full(l64.shape, 5e-6)
    else:
        ty = 1e-5 * np.maximum(np.abs(y64), 1.0)
        tl = 1e-5 * np.maximum(np.abs(l64), 1.0)
    with np.errstate(invalid="ignore"):
        bad = ok & ~huge & ~(np.abs(y - y64) <= ty)
    if bad.any():
        _fail(what + " y", bad, y, y64)
    assert np.all(np.isinf(y[huge]) & (np.sign(y[huge]) == np.sign(y64[huge]))), what + " y beyond float32"
    if ladj is None:
        return
    lok = ok.copy()
    if kind == BERN:
        lok &= same_branch(x, BERN_BOUND, BERN_EPS)
    rows = lok.all(-1)
    s64, bar = l64.sum(-1), tl.sum(-1)
    with np.errstate(invalid="ignore"):
        bad = rows & ~(np.abs(ladj - s64) <= bar)
    if bad.any():
        _fail(what + " summed ladj", bad, ladj, s64)


def check_inverse(kind, what, x, x64, extra, ok):
    if kind == RQS:
        tol = np.maximum(2e-5 * np.maximum(np.abs(x64), 1.0), 3 * np.abs(np.asarray(extra, np.float64) - x64))
    elif kind == AFFINE:
        tol = 5e-6 * np.maximum(np.abs(x64), 1.0)
    else:
        tol = np.maximum(1e-5 * np.maximum(np.abs(x64), 1.0), 2 * interval(kind))
    with np.errstate(invalid="ignore"):
        bad = ok & ~(np.abs(x - x64) <= tol)
    if bad.any():
        _fail(what + " inverse", bad, x, x64)


def inverse_ok(kind, K, deg, x64, yin, phi):
    """Well-conditioned elements of a bisection inverse (module docstring); every element for RQS and affine.
    Bernstein's linear branches (|y| >= bound) are exact and always compared."""
    if kind in (RQS, AFFINE):
        return np.ones(x64.shape, bool)
    if kind == GAUSS:
        _, l = GR.forward(x64, *split(kind, K, deg, phi))
    elif kind == SOSP:
        _, l = SR.forward(x64, *split(kind, K, deg, phi), SLOPE, BISECT_BOUND)
    else:
        _, l = BR.forward(x64, np.asarray(phi, np.float64), BERN_BOUND, BERN_EPS)
    b = BERN_BOUND if kind == BERN else BISECT_BOUND
    with np.errstate(invalid="ignore", over="ignore"):
        good = (np.exp(l) >= 0.5) & (np.abs(x64) <= b - 2 * interval(kind))
    if kind == GAUSS:
        good &= gauss_ok(x64, *split(kind, K, deg, phi))
    if kind == BERN:
        good |= np.abs(yin) >= b
    return good


class Data:
    """Seeded parameters and inputs of one case at its largest batch, with the fp64 references (rows are independent,
    so every batch is a prefix)."""

    def __init__(self, name):
        kind, K, deg, D, layout, off = CASES[name]
        self.kind, self.K, self.deg, self.D, self.layout, self.off = kind, K, deg, D, layout, off
        self.plan = plan_of(name)
        self.n = 3 * self.plan["rows"] + 77
        g = np.random.default_rng(zlib.crc32(name.encode()))
        n_phi = 1 if layout == "shared" else self.n
        self.phi = params_of(kind, K, deg, n_phi, D, g)
        full = np.broadcast_to(self.phi, (self.n, *self.phi.shape[1:])) if layout == "shared" else self.phi
        self.x = inputs_of(kind, K, full, self.n, D, g)
        ref_phi = self.phi[0] if layout == "shared" else self.phi
        self.y64, self.l64, self.ok, self.extra = reference(kind, K, deg, self.x, ref_phi)
        # the inverse runs on the forward's fp64 image, rounded to float32 (and the edges themselves)
        yin = np.where(np.abs(self.y64) < F32_MAX, self.y64, self.x).astype(np.float32)
        yin.reshape(-1)[3::4] = self.x.reshape(-1)[3::4]
        self.yin = yin
        self.x64, self.xextra = inverse_reference(kind, K, deg, yin, ref_phi)
        self.iok = inverse_ok(kind, K, deg, self.x64, yin, ref_phi)

    def device_phi(self, device, B):
        """phi of the first B rows laid out as the case asks, NaN in every pad: (tensor, phi_ld)."""
        D, P = self.D, self.phi.shape[-1]
        if self.layout == "shared":
            return torch.from_numpy(self.phi.reshape(-1).copy()).to(device), 0
        rows = torch.from_numpy(self.phi[:B].reshape(B, D * P).copy()).to(device)
        if self.layout == "strided":
            buf = torch.full((max(B, 1), D * P + PAD), float("nan"), device=device)
            buf[:B, : D * P] = rows
            return buf, D * P + PAD
        buf = torch.full((max(B, 1) * D * P + 8,), float("nan"), device=device)
        view = buf[self.off : self.off + max(B, 1) * D * P]
        view[: B * D * P].copy_(rows.reshape(-1))
        return view, D * P


_DATA = {}


def data(name):
    if name not in _DATA:
        _DATA.clear()
        _DATA[name] = Data(name)
    return _DATA[name]


# --------------------------------------------------------------------------- #
# plan query and oracle parity
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
def test_plan_query_matches_restatement(device):
    buf = torch.zeros(1 << 16, device=device)
    base = buf.data_ptr()
    for name, (kind, K, deg, D, layout, off) in CASES.items():
        R = plan_of(name)["rows"]
        for B in batches_of(R):
            p = uni_plan_of(kind, B, D, K, deg, phi_ld_of(name), base + 4 * off)
            st, got = query(kind, B, D, K, deg, phi_ld_of(name), base + 4 * off)
            assert st == E.ZK_OK and got == want(p), (name, B, got, want(p))
    for name, (args, _) in REFUSALS.items():
        st, _ = query(*args, base)
        assert st == E.ZK_EINVAL, name


MATRIX = [(n, f) for n in CASES for f in (1, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,fast", MATRIX, ids=[f"{n}-{'fast' if f else 'ieee'}" for n, f in MATRIX])
def test_oracle_parity_matrix(device, math_mode, name, fast):
    math_mode(fast)
    d = data(name)
    kind, K, deg, D = d.kind, d.K, d.deg, d.D
    for B in batches_of(d.plan["rows"]):
        what = f"{name} B={B} {'fast' if fast else 'ieee'}"
        phi, phi_ld = d.device_phi(device, B)
        st, got = query(kind, B, D, K, deg, phi_ld, phi.data_ptr())
        assert st == E.ZK_OK and got == want(uni_plan_of(kind, B, D, K, deg, phi_ld, phi.data_ptr())), what
        x = torch.from_numpy(d.x[:B].copy()).to(device)
        y = torch.full((max(B, 1), D), float("nan"), device=device)
        ladj = torch.full((max(B, 1),), float("nan"), device=device)
        E.check(forward_abi(kind, K, deg, x, D, phi, phi_ld, B, D, y, D, ladj, 0, device))
        yi = torch.from_numpy(d.yin[:B].copy()).to(device)
        xi = torch.full((max(B, 1), D), float("nan"), device=device)
        E.check(inverse_abi(kind, K, deg, yi, D, phi, phi_ld, B, D, xi, D, device))
        torch.cuda.synchronize(device)
        if B == 0:
            assert torch.isnan(y).all() and torch.isnan(ladj).all() and torch.isnan(xi).all(), what + ": B = 0 wrote"
            continue
        extra = None if d.extra is None else tuple(v[:B] for v in d.extra)
        check_forward(kind, what, cpu(y), cpu(ladj), d.x[:B], d.y64[:B], d.l64[:B], d.ok[:B], extra)
        check_inverse(kind, what, cpu(xi), d.x64[:B], None if d.xextra is None else d.xextra[:B], d.iok[:B])


@pytest.mark.gpu
def test_refusals_of_the_entry_points(device):
    """What the plan refuses, the launch refuses; and the arguments the plan does not see."""
    L, st = E.lib(), E.stream_ptr(device)
    x = torch.zeros(64 * 32, device=device)
    phi = torch.zeros(17 * 3071 + 64, device=device)
    y, ladj = torch.zeros_like(x), torch.zeros(64, device=device)
    p = lambda t: t.data_ptr()  # noqa: E731
    assert L.zk_rqs_forward(p(x), 17, p(phi), 0, 1, 17, 1024, 5.0, SLOPE, p(y), 17, None, 0, st) == E.ZK_EINVAL
    assert L.zk_rqs_forward(p(x), 16, p(phi), 0, 1, 16, 1024, 5.0, SLOPE, p(y), 16, None, 0, st) == E.ZK_OK
    assert L.zk_rqs_forward(p(x), 4, p(phi), 4 * 23 - 1, 2, 4, 8, 5.0, SLOPE, p(y), 4, None, 0, st) == E.ZK_EINVAL
    assert L.zk_rqs_forward(p(x), 4, p(phi), 0, 2, 4, 1025, 5.0, SLOPE, p(y), 4, None, 0, st) == E.ZK_EINVAL
    assert L.zk_sosp_forward(p(x), 4, p(phi), 0, 2, 4, 3, 16, 10.0, SLOPE, p(y), 4, None, 0, st) == E.ZK_EINVAL
    assert L.zk_bernstein_forward(p(x), 4, p(phi), 0, 2, 4, 60, 5.0, 1e-6, p(y), 4, None, 0, st) == E.ZK_EINVAL
    for it in (0, 65):
        assert L.zk_gaussianization_inverse(p(x), 4, p(phi), 0, 2, 4, 8, 10.0, it, p(y), 4, st) == E.ZK_EINVAL
        assert L.zk_sosp_inverse(p(x), 4, p(phi), 0, 2, 4, 3, 4, 10.0, SLOPE, it, p(y), 4, st) == E.ZK_EINVAL
    assert L.zk_affine_forward(p(x), 4, p(phi), 0, 2, 4, SLOPE, p(y), 4, None, 1, st) == E.ZK_EINVAL  # accumulate, no ladj
    torch.cuda.synchronize(device)


# --------------------------------------------------------------------------- #
# C ABI
# --------------------------------------------------------------------------- #

ABI_CASES = ["rqs8_d16", "rqs5_d3", "affine_d2_off2", "gauss8_d4", "sosp_d4", "sosp23_d3_off3", "bern16_d4", "bern7_d8"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ABI_CASES)
def test_padded_rows_of_x_y_and_phi(device, name):
    """ldx = D + 3, ldy = D + 5 and phi_ld = D P + 5 with NaN pads: the pads are never read (the results equal the
    dense call bit for bit) and never written.  Tiles of several rows read every row's own parameters."""
    d = data(name)
    kind, K, deg, D = d.kind, d.K, d.deg, d.D
    P = d.phi.shape[-1]
    B = 2 * d.plan["rows"] + 7
    assert d.layout == "dense" and d.plan["rows"] > 1
    nan = float("nan")
    phi = torch.from_numpy(d.phi[:B].reshape(B, D * P).copy()).to(device)
    x = torch.from_numpy(d.x[:B].copy()).to(device)
    y0, l0 = torch.empty(B, D, device=device), torch.empty(B, device=device)
    E.check(forward_abi(kind, K, deg, x, D, phi, D * P, B, D, y0, D, l0, 0, device))
    xi0 = torch.empty(B, D, device=device)
    E.check(inverse_abi(kind, K, deg, y0, D, phi, D * P, B, D, xi0, D, device))
    phis = torch.full((B, D * P + PAD), nan, device=device)
    phis[:, : D * P] = phi
    xs = torch.full((B, D + 3), nan, device=device)
    xs[:, :D] = x
    ys, ls = torch.full((B, D + 5), nan, device=device), torch.full((B,), nan, device=device)
    E.check(forward_abi(kind, K, deg, xs, D + 3, phis, D * P + PAD, B, D, ys, D + 5, ls, 0, device))
    yi = torch.full((B, D + 3), nan, device=device)
    yi[:, :D] = y0
    xis = torch.full((B, D + 5), nan, device=device)
    E.check(inverse_abi(kind, K, deg, yi, D + 3, phis, D * P + PAD, B, D, xis, D + 5, device))
    torch.cuda.synchronize(device)
    assert torch.isnan(ys[:, D:]).all() and torch.isnan(xis[:, D:]).all(), f"{name}: the row padding was written"
    assert torch.equal(ys[:, :D], y0) and torch.equal(ls, l0), f"{name}: padded rows change the forward"
    assert torch.equal(xis[:, :D], xi0), f"{name}: padded rows change the inverse"
    check_forward(kind, name, cpu(y0), cpu(l0), d.x[:B], d.y64[:B], d.l64[:B], d.ok[:B],
                  None if d.extra is None else tuple(v[:B] for v in d.extra))  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rqs8_d16", "affine_d33_strided", "gauss3_d3", "sosp_d4", "bern7_d8"])
def test_aliasing_null_outputs_and_accumulate(device, name):
    d = data(name)
    kind, K, deg, D = d.kind, d.K, d.deg, d.D
    B = d.plan["rows"] + 3
    phi, phi_ld = d.device_phi(device, B)
    x = torch.from_numpy(d.x[:B].copy()).to(device)
    y, ladj = torch.empty(B, D, device=device), torch.empty(B, device=device)
    E.check(forward_abi(kind, K, deg, x, D, phi, phi_ld, B, D, y, D, ladj, 0, device))
    xi = torch.empty(B, D, device=device)
    E.check(inverse_abi(kind, K, deg, y, D, phi, phi_ld, B, D, xi, D, device))
    # y aliasing x, forward and inverse
    xa = x.clone()
    la = torch.empty(B, device=device)
    E.check(forward_abi(kind, K, deg, xa, D, phi, phi_ld, B, D, xa, D, la, 0, device))
    ya = y.clone()
    E.check(inverse_abi(kind, K, deg, ya, D, phi, phi_ld, B, D, ya, D, device))
    # y = NULL with ladj; ladj = NULL with y
    ln = torch.full((B,), float("nan"), device=device)
    E.check(forward_abi(kind, K, deg, x, D, phi, phi_ld, B, D, None, D, ln, 0, device))
    yn = torch.full((B, D), float("nan"), device=device)
    E.check(forward_abi(kind, K, deg, x, D, phi, phi_ld, B, D, yn, D, None, 0, device))
    # accumulate onto a non-zero buffer
    base = torch.randn(B, generator=torch.Generator().manual_seed(3)).to(device)
    lacc = base.clone()
    E.check(forward_abi(kind, K, deg, x, D, phi, phi_ld, B, D, torch.empty(B, D, device=device), D, lacc, 1, device))
    torch.cuda.synchronize(device)
    assert torch.equal(xa, y) and torch.equal(la, ladj), f"{name}: y aliasing x differs"
    assert torch.equal(ya, xi), f"{name}: the inverse in place differs"
    assert torch.equal(ln, ladj) and torch.equal(yn, y), f"{name}: a NULL output changes the other"
    assert torch.equal(lacc, base + ladj), f"{name}: accumulate = 1 is not buffer + ladj"


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2, 4, 8, 16, 32, 3, 33, 64, 300])
def test_shared_table_at_each_reduction(device, D):
    """phi_ld = 0 equals the table expanded to every row, on both ladj reductions."""
    K, B = 8, 600
    g = np.random.default_rng(D)
    tab = params_of(RQS, K, 0, 1, D, g)
    x = inputs_of(RQS, K, np.broadcast_to(tab, (B, D, 3 * K - 1)), B, D, g)
    t = torch.from_numpy(tab.reshape(-1).copy()).to(device)
    full = t.reshape(1, -1).expand(B, -1).contiguous()
    xd = torch.from_numpy(x).to(device)
    ys, ls, ye, le = (torch.empty(B, D, device=device), torch.empty(B, device=device), torch.empty(B, D, device=device),
                      torch.empty(B, device=device))  # fmt: skip
    E.check(forward_abi(RQS, K, 0, xd, D, t, 0, B, D, ys, D, ls, 0, device))
    E.check(forward_abi(RQS, K, 0, xd, D, full, D * (3 * K - 1), B, D, ye, D, le, 0, device))
    torch.cuda.synchronize(device)
    assert uni_plan_of(RQS, B, D, K, 0, 0)["shuffle"] == int(D in (1, 2, 4, 8, 16, 32))
    assert torch.equal(ys, ye) and torch.equal(ls, le), D
    y64, l64 = O.rqs_forward(x.astype(np.float64), tab[0], K, RQS_BOUND, SLOPE)
    extra = O.rqs_forward(x, tab[0], K, RQS_BOUND, SLOPE, dtype=np.float32)
    check_forward(RQS, f"shared D={D}", cpu(ys), cpu(ls), x, y64, l64, np.ones(x.shape, bool), extra)


# --------------------------------------------------------------------------- #
# bitwise properties
# --------------------------------------------------------------------------- #

BIT_CASES = ["affine_d1", "rqs8_d16", "rqs5_d3", "gauss3_d3", "sosp_d4", "bern16_d4", "rqs16_d32"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIT_CASES)
def test_bitwise_tile_staging_stride_and_runs(device, name):
    """A row's y and ladj do not depend on its tile, on bulk or coalesced staging, on dense or padded phi rows, or on
    the run: every reduction is fixed-order."""
    d = data(name)
    kind, K, deg, D = d.kind, d.K, d.deg, d.D
    P = d.phi.shape[-1]
    R = d.plan["rows"]
    B = d.n
    phi = torch.from_numpy(d.phi.reshape(B, D * P).copy()).to(device)
    x = torch.from_numpy(d.x.copy()).to(device)

    def fwd(xv, ph, ld, n):
        y, l = torch.empty(n, D, device=device), torch.empty(n, device=device)
        E.check(forward_abi(kind, K, deg, xv, D, ph, ld, n, D, y, D, l, 0, device))
        return y, l

    y0, l0 = fwd(x, phi, D * P, B)
    y1, l1 = fwd(x, phi, D * P, B)
    assert torch.equal(y0, y1) and torch.equal(l0, l1), f"{name}: two runs differ"
    for off, n in ((1, R), (R // 2 + 1, R + 3), (R - 1, 2), (B - 77, 77)):
        n = min(n, B - off)
        ys, ls = fwd(x[off : off + n], phi[off : off + n], D * P, n)
        assert torch.equal(ys, y0[off : off + n]) and torch.equal(ls, l0[off : off + n]), f"{name}: rows {off}+{n} differ"
    # the same parameters at a 16-byte aligned and at a misaligned address
    buf = torch.empty(B * D * P + 4, device=device)
    mis = buf[1 : 1 + B * D * P].view(B, D * P)
    mis.copy_(phi)
    _, bulk_aligned = query(kind, B, D, K, deg, D * P, phi.data_ptr())
    _, bulk_mis = query(kind, B, D, K, deg, D * P, mis.data_ptr())
    assert bulk_mis[2] == 0
    ym, lm = fwd(x, mis, D * P, B)
    assert torch.equal(ym, y0) and torch.equal(lm, l0), f"{name}: misaligned staging differs (bulk {bulk_aligned[2]})"
    pad = torch.full((B, D * P + 3), float("nan"), device=device)
    pad[:, : D * P] = phi
    yp, lp = fwd(x, pad, D * P + 3, B)
    assert torch.equal(yp, y0) and torch.equal(lp, l0), f"{name}: padded phi rows differ"


# --------------------------------------------------------------------------- #
# layer paths that run the kernel
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
@pytest.mark.parametrize("features,passthrough", [(12, 4), (10, 3)])
def test_coupling_layer(device, math_mode, features, passthrough, fast):
    """Transformed halves of 8 / 4 (power-of-two, shuffle sum) and 7 / 3 (fixed order) through dim_map."""
    from zuko_b200.distributions import DiagNormal
    from zuko_b200.flows import GeneralCouplingTransform
    from zuko_b200.lazy import Flow, UnconditionalDistribution
    from zuko_b200.transforms import MonotonicRQSTransform

    math_mode(fast)
    torch.manual_seed(SEED)
    C = 3
    mask = torch.arange(features) < passthrough
    t = GeneralCouplingTransform(features, C, mask=mask, univariate=MonotonicRQSTransform, shapes=[(8,), (8,), (7,)],
                                 hidden_features=[64, 64])  # fmt: skip
    flow = Flow([t, GeneralCouplingTransform(features, C, mask=~mask, univariate=MonotonicRQSTransform,
                                             shapes=[(8,), (8,), (7,)], hidden_features=[64, 64])],
                UnconditionalDistribution(DiagNormal, torch.zeros(features), torch.ones(features), buffer=True)).eval()  # fmt: skip
    spec = O.flowspec_from_module(flow)
    g = torch.Generator().manual_seed(features)
    B = 777
    x, c = torch.randn(B, features, generator=g) * 2, torch.randn(B, C, generator=g)
    ref = spec.log_prob(x.numpy().astype(np.float64), c.numpy().astype(np.float64))
    flow = flow.to(device)
    with torch.no_grad():
        lp = cpu(flow(c.to(device)).log_prob(x.to(device)))
    err = np.abs(lp - ref) / np.maximum(np.abs(ref), 1.0)
    assert err.max() <= 1e-5, (features, passthrough, float(err.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
def test_elementwise_gf_broadcast_context(device, math_mode, fast):
    """An element-wise GF layer whose context is one row for the whole batch (ldc = 0, so phi_ld = 0)."""
    from zuko_b200.flows import GF

    math_mode(fast)
    torch.manual_seed(SEED)
    D, C, K = 5, 3, 8
    flow = GF(D, C, transforms=1, components=K, hidden_features=[32, 32]).eval()
    sd = {k: v.detach().numpy() for k, v in flow.state_dict().items()}
    ref_flow = GR.Flow(sd, D, C, K)
    g = torch.Generator().manual_seed(1)
    B = 1000
    x, c = torch.randn(B, D, generator=g), torch.randn(C, generator=g)
    ref = ref_flow.log_prob(x.numpy().astype(np.float64), c.numpy().astype(np.float64))
    flow = flow.to(device)
    with torch.no_grad():
        lp = cpu(flow(c.to(device)).log_prob(x.to(device)))
        lp_e = cpu(flow(c.to(device).expand(B, C).contiguous()).log_prob(x.to(device)))
    # GF bar: test_gpu_gf.py's 1e-5 relative on rows where the map is well-conditioned (module docstring)
    sh, sc = ref_flow._params("mlp", ref_flow.layers[0][1], c.numpy(), B)
    ok = gauss_ok(x.numpy().astype(np.float64), sh, sc).all(-1)
    assert ok.mean() > 0.9
    err = np.abs(lp - ref) / np.maximum(np.abs(ref), 1.0)
    assert err[ok].max() <= 1e-5, float(err[ok].max())
    np.testing.assert_allclose(lp, lp_e, rtol=1e-6, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "ieee"])
def test_unfused_last_layer_with_diag_normal(device, math_mode, fast):
    """zk_set_fused_layers(0): the last autoregressive layer runs the stand-alone kernel with the DiagNormal(loc, scale)
    term fused (scale != 1)."""
    from zuko_b200.distributions import DiagNormal
    from zuko_b200.flows import MaskedAutoregressiveTransform
    from zuko_b200.lazy import Flow, UnconditionalDistribution
    from zuko_b200.transforms import MonotonicRQSTransform

    math_mode(fast)
    torch.manual_seed(SEED)
    D, C = 6, 2
    g = torch.Generator().manual_seed(2)
    base = UnconditionalDistribution(DiagNormal, torch.randn(D, generator=g), torch.randn(D, generator=g).exp() + 0.2, buffer=True)
    layers = [MaskedAutoregressiveTransform(D, C, univariate=MonotonicRQSTransform, shapes=[(8,), (8,), (7,)],
                                            hidden_features=[64, 64]) for _ in range(2)]  # fmt: skip
    flow = Flow(layers, base).eval()
    spec = O.flowspec_from_module(flow)
    B = 999
    x, c = torch.randn(B, D, generator=g), torch.randn(B, C, generator=g)
    ref = spec.log_prob(x.numpy().astype(np.float64), c.numpy().astype(np.float64))
    flow = flow.to(device)
    prev = E.lib().zk_set_fused_layers(0)
    try:
        with torch.no_grad():
            lp = cpu(flow(c.to(device)).log_prob(x.to(device)))
    finally:
        E.lib().zk_set_fused_layers(prev)
    err = np.abs(lp - ref) / np.maximum(np.abs(ref), 1.0)
    assert err.max() <= 1e-5, float(err.max())


# --------------------------------------------------------------------------- #
# small element-wise kernels
# --------------------------------------------------------------------------- #


def _padded(a, extra, device):
    a = torch.as_tensor(a, dtype=torch.float32)
    out = torch.full((a.shape[0], a.shape[1] + extra), float("nan"), device=device)
    out[:, : a.shape[1]] = a.to(device)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("bound", [1.0, 11.0])
def test_softclip(device, bound):
    L, st = E.lib(), E.stream_ptr(device)
    B, D = 1000, 7
    x = (np.random.default_rng(1).standard_normal((B, D)) * 4 * bound).astype(np.float32)
    x[0, :4] = [0.0, bound, -bound, 1e30]
    xs = _padded(x, 3, device)
    y, ladj = torch.full((B, D + 2), float("nan"), device=device), torch.full((B,), float("nan"), device=device)
    E.check(L.zk_softclip_forward(xs.data_ptr(), D + 3, B, D, bound, y.data_ptr(), D + 2, ladj.data_ptr(), 0, st))
    y64, l64 = O.softclip_forward(x.astype(np.float64), bound)
    acc = torch.full((B,), 2.0, device=device)
    E.check(L.zk_softclip_forward(xs.data_ptr(), D + 3, B, D, bound, None, D, acc.data_ptr(), 1, st))
    yn = torch.full((B, D), float("nan"), device=device)
    E.check(L.zk_softclip_forward(xs.data_ptr(), D + 3, B, D, bound, yn.data_ptr(), D, None, 0, st))
    yi = _padded(cpu(y[:, :D]), 1, device)
    xi = torch.full((B, D + 4), float("nan"), device=device)
    E.check(L.zk_softclip_inverse(yi.data_ptr(), D + 1, B, D, bound, xi.data_ptr(), D + 4, st))
    z = torch.full((B, D), float("nan"), device=device)
    E.check(L.zk_softclip_forward(xs.data_ptr(), D + 3, 0, D, bound, z.data_ptr(), D, None, 0, st))
    torch.cuda.synchronize(device)
    # bars of test_gpu_parity.py::test_softclip: 2e-6 relative on y and absolute on the ladj, 2e-5 on the inverse
    fin = np.abs(x) < 1e29
    assert np.all(np.abs(cpu(y[:, :D]) - y64) <= 2e-6 * np.maximum(np.abs(y64), 1.0))
    assert np.all(np.abs(cpu(ladj) - l64.sum(-1))[fin.all(-1)] <= 2e-6 * D)
    assert torch.isnan(y[:, D:]).all() and torch.isnan(xi[:, D:]).all() and torch.isnan(z).all()
    assert torch.equal(acc, 2.0 + ladj) and torch.equal(yn, y[:, :D])
    x64 = O.softclip_inverse(cpu(y[:, :D]), bound)
    ok = np.abs(x64) < 1e6
    assert np.all((np.abs(cpu(xi[:, :D]) - x64) <= 2e-5 * np.maximum(np.abs(x64), 1.0))[ok])


@pytest.mark.gpu
def test_permute(device):
    L, st = E.lib(), E.stream_ptr(device)
    B, D = 513, 9
    x = np.random.default_rng(2).standard_normal((B, D)).astype(np.float32)
    order = np.random.default_rng(3).permutation(D)
    od = torch.from_numpy(order).to(device)
    xs = _padded(x, 2, device)
    y = torch.full((B, D + 3), float("nan"), device=device)
    E.check(L.zk_permute(xs.data_ptr(), D + 2, od.data_ptr(), B, D, y.data_ptr(), D + 3, st))
    E.check(L.zk_permute(xs.data_ptr(), D + 2, od.data_ptr(), 0, D, y.data_ptr(), D + 3, st))
    torch.cuda.synchronize(device)
    assert np.array_equal(y[:, :D].cpu().numpy(), O.permute(x, order)) and torch.isnan(y[:, D:]).all()
    assert L.zk_permute(xs.data_ptr(), D + 2, od.data_ptr(), B, D, xs.data_ptr(), D + 2, st) == E.ZK_EINVAL


@pytest.mark.gpu
@pytest.mark.parametrize("transpose", [0, 1])
def test_rotate(device, transpose):
    L, st = E.lib(), E.stream_ptr(device)
    B, D = 300, 110  # D D 4 = 48400 bytes: the largest R the kernel stages
    g = np.random.default_rng(4)
    R = np.linalg.qr(g.standard_normal((D, D)))[0].astype(np.float32)
    x = g.standard_normal((B, D)).astype(np.float32)
    Rd = torch.from_numpy(R).to(device)
    xs = _padded(x, 1, device)
    y = torch.full((B, D + 2), float("nan"), device=device)
    E.check(L.zk_rotate(xs.data_ptr(), D + 1, Rd.data_ptr(), transpose, B, D, y.data_ptr(), D + 2, st))
    E.check(L.zk_rotate(xs.data_ptr(), D + 1, Rd.data_ptr(), transpose, 0, D, y.data_ptr(), D + 2, st))
    torch.cuda.synchronize(device)
    ref = O.rotate(x.astype(np.float64), R.astype(np.float64), bool(transpose))
    # test_gpu_parity.py::test_rotation: 1e-5 relative
    assert np.max(np.abs(cpu(y[:, :D]) - ref) / np.maximum(np.abs(ref), 1.0)) < 1e-5
    assert torch.isnan(y[:, D:]).all()
    R111 = torch.zeros(111, 111, device=device)
    x111 = torch.zeros(2, 111, device=device)
    y111 = torch.zeros(2, 111, device=device)
    assert L.zk_rotate(x111.data_ptr(), 111, R111.data_ptr(), transpose, 2, 111, y111.data_ptr(), 111, st) == E.ZK_EINVAL


@pytest.mark.gpu
@pytest.mark.parametrize("bound", [1.0, math.pi])
def test_circular_shift(device, bound):
    L, st = E.lib(), E.stream_ptr(device)
    b = np.float32(bound)
    special = np.array([0, b, -b, 2 * b, -2 * b, 4 * b, -6 * b, np.nextafter(b, np.float32(0)), -0.5, -7.25, 3 * b], np.float32)
    x = np.concatenate([special, np.random.default_rng(5).standard_normal(499).astype(np.float32) * 10]).reshape(-1, 5)
    B, D = x.shape
    xs = _padded(x, 3, device)
    y = torch.full((B, D + 1), float("nan"), device=device)
    E.check(L.zk_circular_shift(xs.data_ptr(), D + 3, B, D, bound, y.data_ptr(), D + 1, st))
    E.check(L.zk_circular_shift(xs.data_ptr(), D + 3, 0, D, bound, y.data_ptr(), D + 1, st))
    torch.cuda.synchronize(device)
    # torch.remainder semantics in float32, bit for bit (test_gpu_parity.py::test_circular_shift_and_box_uniform)
    ref = torch.remainder(torch.from_numpy(x), torch.tensor(2 * b)) - torch.tensor(b)
    assert torch.equal(y[:, :D].cpu(), ref) and torch.isnan(y[:, D:]).all()


@pytest.mark.gpu
def test_box_uniform(device):
    L, st = E.lib(), E.stream_ptr(device)
    D = 3
    lo, hi = np.array([-1.0, 0.0, 2.0], np.float32), np.array([1.0, 0.5, 5.0], np.float32)
    rows = [lo, hi, (lo + hi) / 2, np.nextafter(hi, np.float32(-np.inf)), np.nextafter(lo, np.float32(-np.inf)), [0.0, 0.25, 10.0]]
    z = np.concatenate([np.array(rows, np.float32), np.random.default_rng(6).uniform(-2, 6, (300, D)).astype(np.float32)])
    B = z.shape[0]
    ladj = np.random.default_rng(7).standard_normal(B).astype(np.float32)
    zs, lod, hid, ld = _padded(z, 2, device), torch.from_numpy(lo).to(device), torch.from_numpy(hi).to(device), torch.from_numpy(ladj).to(device)
    out, out0 = torch.empty(B, device=device), torch.empty(B, device=device)
    E.check(L.zk_box_uniform_log_prob(zs.data_ptr(), D + 2, lod.data_ptr(), hid.data_ptr(), ld.data_ptr(), B, D, out.data_ptr(), st))
    E.check(L.zk_box_uniform_log_prob(zs.data_ptr(), D + 2, lod.data_ptr(), hid.data_ptr(), None, B, D, out0.data_ptr(), st))
    E.check(L.zk_box_uniform_log_prob(zs.data_ptr(), D + 2, lod.data_ptr(), hid.data_ptr(), None, 0, D, out0.data_ptr(), st))
    torch.cuda.synchronize(device)
    for got, la in ((cpu(out), ladj), (cpu(out0), None)):
        ref = O.box_uniform_log_prob(z, lo, hi, la)
        assert np.array_equal(np.isneginf(got), np.isneginf(ref))
        fin = np.isfinite(ref)
        assert np.all(np.abs(got[fin] - ref[fin]) <= 1e-6 * np.maximum(np.abs(ref[fin]), 1.0))
    assert np.isfinite(cpu(out0)[[0, 2, 3]]).all() and np.isneginf(cpu(out0)[[1, 4, 5]]).all()  # z = lower in, z = upper out


@pytest.mark.gpu
def test_diag_normal(device):
    L, st = E.lib(), E.stream_ptr(device)
    B, D = 700, 6
    g = np.random.default_rng(8)
    z = g.standard_normal((B, D)).astype(np.float32) * 3
    loc, scale = g.standard_normal(D).astype(np.float32), (np.exp(g.standard_normal(D)) + 0.1).astype(np.float32)
    ladj = g.standard_normal(B).astype(np.float32)
    zs = _padded(z, 1, device)
    locd, scd, ld = (torch.from_numpy(v).to(device) for v in (loc, scale, ladj))
    out, out0 = torch.empty(B, device=device), torch.empty(B, device=device)
    E.check(L.zk_diag_normal_log_prob(zs.data_ptr(), D + 1, locd.data_ptr(), scd.data_ptr(), ld.data_ptr(), B, D, out.data_ptr(), st))
    E.check(L.zk_diag_normal_log_prob(zs.data_ptr(), D + 1, None, None, None, B, D, out0.data_ptr(), st))
    E.check(L.zk_diag_normal_log_prob(zs.data_ptr(), D + 1, None, None, None, 0, D, out0.data_ptr(), st))
    torch.cuda.synchronize(device)
    # test_gpu_parity.py::test_diag_normal: 2e-6 relative
    for got, lc, sc, la in ((cpu(out), loc, scale, ladj), (cpu(out0), np.zeros(D), np.ones(D), None)):
        ref = O.diag_normal_log_prob(z.astype(np.float64), lc, sc, la)
        assert np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1.0)) < 2e-6
    assert L.zk_diag_normal_log_prob(zs.data_ptr(), D + 1, locd.data_ptr(), None, None, B, D, out.data_ptr(), st) == E.ZK_EINVAL
    assert L.zk_diag_normal_log_prob(zs.data_ptr(), D + 1, None, scd.data_ptr(), None, B, D, out.data_ptr(), st) == E.ZK_EINVAL
