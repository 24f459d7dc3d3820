"""GPU tests of the flow-level calls of the C ABI (api.cu: zk_flow_forward, zk_flow_log_prob, zk_flow_inverse and
zk_flow_log_prob_host) at their composition, base, lazy-inverse, row-chunk, stride and broadcast edges, against the
fp64 oracle (oracle/oracle.py).  The descriptor of each flow (`flow(c)._flow_call()[0].desc`) is driven directly, so
strides, pads, workspace sizes and NULLs are under the test's control.

* Composition table (CASES): which layer closes the forward (and so whether the DiagNormal term rides in its
  kernel or `base_log_prob` runs after it), inverted (LazyInverse) members first, in the middle and last, a
  BoxUniform base, a sweep-fallback layer that the inverse meets first, permutation / rotation only and no layer at
  all.  Every case runs forward, log_prob with and without the device sum, inverse and inverse + log_prob, at batches
  around the 128-row tiles and the 1024-row granule, with NaN-filled odd pads on every strided buffer and NaN-filled
  outputs, with a per-row and a broadcast context (ldc = 0), and with zk_set_fused_layers on and off where that
  changes the path.  tests/test_flow_edges_host.py checks without a GPU that the table reaches every branch.
* Row chunks: the planner (flow_ws_for per direction + largest_fitting_rows) restated, anchored to
  zk_flow_workspace_bytes, and workspaces that give 1-row, 100-row, 2048-row (rounded to the granule) and minimum
  chunks; the chunk count from zk_launch_count, the outputs bit-identical to one chunk.
* The host-buffer call against zk_flow_log_prob, bit for bit, and its sum against the per-chunk sums.
* Refusals: each returns a status, launches nothing and leaves its outputs untouched.

Bars (the existing ones): z per element max(rtol max(|ref64|, 1), 3 |ref32 - ref64|), rtol 1e-5 with fp32 conditioner
GEMMs and 4e-5 with tensor-core ones (test_gpu_parity.py); x of the inverse SEQ_BAR / SWEEP_BAR
(test_gpu_inverse_edges.py); log_prob and ladj 1e-5 of max(|log_prob64|, 1) per row
(test_gpu_fused_edges.check_row)."""

import ctypes
import math
from functools import partial

import numpy as np
import pytest
import torch

from oracle import oracle as O
from zuko_b200 import _engine as E
from zuko_b200.distributions import BoxUniform, DiagNormal
from zuko_b200.flows import ElementWiseTransform, GeneralCouplingTransform, MaskedAutoregressiveTransform
from zuko_b200.lazy import Flow, LazyInverse, UnconditionalDistribution, UnconditionalTransform
from zuko_b200.transforms import (CircularRQSTransform, MonotonicRQSTransform, PermutationTransform, RotationTransform,
                                  SoftclipTransform)  # fmt: skip

pytestmark = pytest.mark.gpu

SEED = 0
D, C = 8, 3
SEQ_BAR, SWEEP_BAR = 1e-5, 5e-5  # test_gpu_inverse_edges.py
LP_BAR = 1e-5
GRANULE = 1024
REDUCE_SCRATCH = 256 * 8  # reduce_scratch_bytes (bijectors.cu): kRedBlocks doubles
BATCHES = [0, 1, 127, 128, 129, 1023, 1024, 1025, 4099]
NMAX = max(BATCHES)
PAD_X, PAD_Z, PAD_C = 3, 5, 2  # odd row pads of the inputs, the outputs and the context

# --------------------------------------------------------------------------- #
# the case table
# --------------------------------------------------------------------------- #

# token -> what the engine must report for its layer: (kind, fused forward, dimension-sequential inverse, fp32 GEMMs)
LAYERS = {
    "ar": ("ar", True, True, False),  # RQS, hidden [64, 64]: the fused forward kernel
    "ar_aff": ("ar", True, True, False),
    "ar32": ("ar", False, True, True),  # fp32 conditioner GEMMs: the unfused forward
    "sweep": ("ar", False, False, False),  # 4 bins: neither the fused forward nor the sequential inverse
    "circ": ("ar", False, True, False),  # circular spline: never fused in the forward
    "cpl": ("cpl", False, False, False),
    "cpl_aff": ("cpl", False, False, False),
    "ew": ("ew", False, False, False),  # one shared (D, P) table
    "ewc": ("ewc", False, False, False),  # phi = MLP(c)
    "clip": ("clip", False, False, False),
    "perm": ("perm", False, False, False),
    "rot": ("rot", False, False, False),
}

# name -> (members, base); "inv:<token>" is LazyInverse of that layer
CASES = {
    "ar_last": (["rot", "cpl", "ar"], "normal"),
    "ar32_last": (["perm", "ar_aff", "ar32"], "normal"),
    "ew_last": (["ar", "ew"], "normal"),
    "ewc_last": (["cpl", "ewc"], "normal"),
    "cpl_last": (["ar_aff", "cpl"], "normal"),
    "clip_last": (["ar", "clip"], "normal"),
    "perm_last": (["cpl_aff", "perm"], "normal"),
    "rot_last": (["ewc", "rot"], "normal"),
    "box_circ_cpl": (["circ", "cpl_aff"], "box"),
    "box_cpl_circ": (["cpl", "rot", "circ"], "box"),
    "iaf": (["inv:ar", "inv:ar_aff"], "normal"),
    "inv_only": (["inv:ar"], "normal"),
    "inv_first": (["inv:ar", "perm", "cpl"], "normal"),
    "inv_mid_last": (["cpl", "inv:ar", "perm", "inv:ar_aff"], "normal"),
    "inv_circ_box": (["inv:circ", "circ"], "box"),
    "inv_last_box": (["perm", "inv:circ"], "box"),
    "inv_fp32": (["cpl", "inv:ar32"], "normal"),
    "sweep_last": (["cpl", "sweep"], "normal"),
    "perm_rot": (["perm", "rot"], "normal"),
    "rot_perm_box": (["rot", "perm"], "box"),
    "empty": ([], "normal"),
    "empty_box": ([], "box"),
}


def token(m):
    """(layer token, inverted) of a member name."""
    return (m[4:], True) if m.startswith("inv:") else (m, False)


def has_context(name):
    return any(LAYERS[token(m)[0]][0] in ("ar", "cpl", "ewc") for m in CASES[name][0])


def fused_matters(name):
    """zk_set_fused_layers changes the path: an autoregressive layer with the fused forward or the sequential inverse."""
    return any(LAYERS[token(m)[0]][1] or LAYERS[token(m)[0]][2] for m in CASES[name][0])


def inverted_any(name):
    return any(token(m)[1] for m in CASES[name][0])


def case_params():
    """(name, context mode, fused) of every run: per-row and broadcast contexts where the flow has one, both fused
    settings where they change the path."""
    out = []
    for name in CASES:
        for ctx in (("rows", "bcast") if has_context(name) else ("none",)):
            for fused in ((1, 0) if fused_matters(name) else (1,)):
                out.append((name, ctx, fused))
    return out


# --------------------------------------------------------------------------- #
# modules and the oracle
# --------------------------------------------------------------------------- #


def _rqs(K=8, circular=False):
    f = CircularRQSTransform if circular else MonotonicRQSTransform
    return dict(univariate=partial(f, slope=1e-3), shapes=[(K,), (K,), (K - 1,)])


def make_layer(tok):
    h = dict(hidden_features=[64, 64])
    if tok in ("ar", "ar32"):
        t = MaskedAutoregressiveTransform(D, C, **h, **_rqs())
        if tok == "ar32":
            t.hyper.gemm_mode = "fp32"
        return t
    ctors = {
        "ar_aff": lambda: MaskedAutoregressiveTransform(D, C, **h),
        "sweep": lambda: MaskedAutoregressiveTransform(D, C, **h, **_rqs(4)),
        "circ": lambda: MaskedAutoregressiveTransform(D, C, **h, **_rqs(8, circular=True)),
        "cpl": lambda: GeneralCouplingTransform(D, C, **h, **_rqs()),
        "cpl_aff": lambda: GeneralCouplingTransform(D, C, mask=torch.arange(D) < 3, **h),  # n_a = 3, n_b = 5
        "ew": lambda: ElementWiseTransform(D, 0, **_rqs()),
        "ewc": lambda: ElementWiseTransform(D, C, **h, **_rqs()),
        "clip": lambda: UnconditionalTransform(SoftclipTransform, bound=6.0),
        "perm": lambda: UnconditionalTransform(PermutationTransform, torch.randperm(D), buffer=True),
        "rot": lambda: UnconditionalTransform(RotationTransform, torch.randn(D, D), buffer=True),
    }
    return ctors[tok]()


BOX_LO, BOX_HI = -math.pi - 1e-5, math.pi + 1e-5


def make_base(base):
    if base == "box":
        return UnconditionalDistribution(BoxUniform, torch.full((D,), BOX_LO), torch.full((D,), BOX_HI), buffer=True)
    return UnconditionalDistribution(DiagNormal, torch.linspace(-0.3, 0.3, D), torch.linspace(0.8, 1.5, D), buffer=True)


def make_flow(name):
    torch.manual_seed(SEED)
    members, base = CASES[name]
    layers = []
    for m in members:
        tok, inv = token(m)
        t = make_layer(tok)
        layers.append(LazyInverse(t) if inv else t)
    return Flow(layers, make_base(base)).eval()


class Inverted:
    """Oracle of a LazyInverse member (lazy.py:81-98): its forward is the layer's inverse, with ladj = minus the
    layer's ladj at the solution; its inverse is the layer's forward."""

    def __init__(self, layer):
        self.layer = layer

    def forward(self, x, c, dtype=np.float64):
        y = self.layer.inverse(x, c, dtype)
        return y, -self.layer.forward(y, c, dtype)[1]

    def inverse(self, y, c, dtype=np.float64):
        return self.layer.forward(y, c, dtype)[0]


def make_spec(flow):
    plain = [t.transform if isinstance(t, LazyInverse) else t for t in flow.transform.transforms]
    spec = O.flowspec_from_module(Flow(plain, flow.base))
    spec.layers = [Inverted(s) if isinstance(t, LazyInverse) else s for s, t in zip(spec.layers, flow.transform.transforms)]
    return spec


def case_inputs(name):
    """Seeded (x, z, c) of NMAX rows: x for the forward, z for the inverse.  On a BoxUniform base z has rows exactly on
    the lower bound (inside), exactly on the upper bound and at 4 (outside), and so has x where no inverted circular
    member reads it (the circular spline is a bijection of [-pi, pi] only: see check_inverse_lp)."""
    g = torch.Generator().manual_seed(1234)
    box = CASES[name][1] == "box"
    if box:
        x = ((torch.rand(NMAX, D, generator=g) * 2 - 1) * 3.1).numpy()
        z = ((torch.rand(NMAX, D, generator=g) * 2 - 1) * 3.1).numpy()
        lo, hi = np.float32(BOX_LO), np.float32(BOX_HI)
        z[0::5, 0] = lo
        z[1::5, 1] = hi
        z[2::5, 2] = 4.0
        z[3::5, 3] = lo
        if not inverted_any(name):
            x[4::7, 4] = 4.0
            x[5::7, 5] = lo
            x[6::7, 6] = hi
    else:
        x = (torch.randn(NMAX, D, generator=g) * 1.5).numpy()
        z = torch.randn(NMAX, D, generator=g).numpy()
    c = torch.randn(NMAX, C, generator=g).numpy()
    return x.astype(np.float32), z.astype(np.float32), c.astype(np.float32)


class Setup:
    """One case and context mode: modules, oracle on all NMAX rows (64 and 32 bit), the device flow and its call."""

    _cache = {}

    @classmethod
    def get(cls, name, ctx, device):
        key = (name, ctx)
        if key not in cls._cache:
            cls._cache.clear()
            cls._cache[key] = cls(name, ctx, device)
        return cls._cache[key]

    def __init__(self, name, ctx, device):
        self.name, self.ctx = name, ctx
        cpu_flow = make_flow(name)
        self.spec = make_spec(cpu_flow)
        self.x, self.z, c = case_inputs(name)
        self.c = None if ctx == "none" else (c[0] if ctx == "bcast" else c)
        oc = None if ctx == "none" else np.broadcast_to(c[0], (NMAX, C)) if ctx == "bcast" else c
        s = self.spec
        self.z64, self.ladj64 = s.forward(self.x.astype(np.float64), oc)
        self.lp64 = s._base_log_prob(self.z64, self.ladj64, np.float64)
        self.z32 = s.forward(self.x, None if oc is None else np.ascontiguousarray(oc), np.float32)[0]
        self.x64, self.ilp64 = s.inverse_and_log_prob(self.z.astype(np.float64), oc)
        self.x32, self.ilp32 = s.inverse_and_log_prob(self.z, None if oc is None else np.ascontiguousarray(oc), np.float32)
        # the log-density scale a row's ladj is held to; outside the box, the one it would have inside
        inside = -np.log(s.scale - s.loc).sum() + self.ladj64 if s.base == "uniform" else self.lp64
        self.lp_scale = np.where(np.isneginf(self.lp64), inside, self.lp64)
        # rows on which the oracle's forward returns z from the inverse's x (see check_inverse_lp)
        zz = s.forward(self.x64, oc)[0]
        self.bijective = (np.abs(zz - self.z) <= 1e-6 * np.maximum(np.abs(self.z), 1.0)).all(-1)
        self.flow = make_flow(name).to(device)
        self.flow.load_state_dict(cpu_flow.state_dict())
        cd = None if self.c is None else torch.from_numpy(self.c).to(device)
        if CASES[name][0]:
            with torch.no_grad():
                self.fc = self.flow(cd)._flow_call()[0]
            self.desc = self.fc.desc
            self.handles = list(self.fc._handles)
        else:  # no layer: a hand-built descriptor over the base alone
            dist = self.flow.base()
            box = CASES[name][1] == "box"
            self._base = [(dist.lower if box else dist.loc).contiguous(), (dist.upper if box else dist.scale).contiguous()]
            kind = E.ZK_BASE_BOX_UNIFORM if box else E.ZK_BASE_DIAG_NORMAL
            self.desc = E.FlowDesc(0, None, D, 0, self._base[0].data_ptr(), self._base[1].data_ptr(), kind, None)
            self.handles = []
        self.members = [token(m) for m in CASES[name][0]]


# --------------------------------------------------------------------------- #
# buffers and calls
# --------------------------------------------------------------------------- #

F32 = dict(dtype=torch.float32)


def padded(a, pad, device):
    """(B, n + pad) NaN-filled device buffer holding a (B, n) in its first n columns."""
    out = torch.full((a.shape[0], a.shape[1] + pad), float("nan"), device=device, **F32)
    out[:, : a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a))
    return out


def nan(shape, device):
    return torch.full(shape, float("nan"), device=device, **F32)


def ptr(t):
    return None if t is None else t.data_ptr()


def ctx_buf(st, B, device):
    """(device context, ldc): rows with an odd pad, or the broadcast row with ldc = 0."""
    if st.c is None:
        return None, 0
    if st.ctx == "bcast":
        return torch.from_numpy(st.c).to(device), 0
    return padded(st.c[: max(B, 1)], PAD_C, device), C + PAD_C


def cpu(t):
    return t.detach().cpu().numpy().astype(np.float64)


class Call:
    """The four entry points on one descriptor; each returns the status and the launches it made."""

    def __init__(self, desc, device):
        self.desc, self.device, self.L = desc, device, E.lib()

    def _run(self, fn, *args):
        n0 = self.L.zk_launch_count()
        st = fn(ctypes.byref(self.desc), *args, E.stream_ptr(self.device))
        torch.cuda.synchronize(self.device)
        return st, self.L.zk_launch_count() - n0

    def ws(self, nbytes):
        return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device), nbytes

    def forward(self, x, ldx, c, ldc, B, z, ldz, ladj, ws):
        return self._run(self.L.zk_flow_forward, ptr(x), ldx, ptr(c), ldc, B, ptr(z), ldz, ptr(ladj), ptr(ws[0]), ws[1])

    def log_prob(self, x, ldx, c, ldc, B, lp, total, ws):
        return self._run(self.L.zk_flow_log_prob, ptr(x), ldx, ptr(c), ldc, B, ptr(lp), ptr(total), ptr(ws[0]), ws[1])

    def inverse(self, z, ldz, c, ldc, B, x, ldx, lp, ws):
        return self._run(self.L.zk_flow_inverse, ptr(z), ldz, ptr(c), ldc, B, ptr(x), ldx, ptr(lp), ptr(ws[0]), ws[1])


# --------------------------------------------------------------------------- #
# checks
# --------------------------------------------------------------------------- #


def elem_err(ours, ref64, ref32, rtol):
    """max over elements of |ours - ref64| / max(rtol max(|ref64|, 1), 3 |ref32 - ref64|): <= 1 passes."""
    ours, ref64, ref32 = (np.asarray(a, np.float64) for a in (ours, ref64, ref32))
    tol = np.maximum(rtol * np.maximum(np.abs(ref64), 1.0), 3.0 * np.abs(ref32 - ref64))
    with np.errstate(invalid="ignore"):
        r = np.abs(ours - ref64) / tol
    return np.where(np.isnan(r), np.inf, r)


def check_elems(ours, ref64, ref32, rtol, what):
    r = elem_err(ours, ref64, ref32, rtol)
    if r.size and not (r <= 1).all():
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        raise AssertionError(f"{what}: {int((r > 1).sum())} of {r.size} entries off the oracle; worst at {i}: "
                             f"ours {ours[i]!r} ref64 {ref64[i]!r} ref32 {ref32[i]!r}")  # fmt: skip
    return float(np.max(np.abs(np.asarray(ours) - ref64) / np.maximum(np.abs(ref64), 1.0))) if r.size else 0.0


def check_lp(ours, ref64, what, scale=None):
    """check_row of test_gpu_fused_edges on the finite rows; the -inf rows (BoxUniform) must match exactly.
    Returns the largest error relative to max(|ref64|, 1, |scale|)."""
    ours, ref64 = np.asarray(ours, np.float64), np.asarray(ref64, np.float64)
    inf = np.isneginf(ref64)
    assert np.array_equal(np.isneginf(ours), inf), (f"{what}: -inf rows differ from the oracle: ours "
                                                    f"{np.nonzero(np.isneginf(ours) != inf)[0][:8]}")  # fmt: skip
    fin = ~inf
    if not fin.any():
        return 0.0
    sc = np.maximum(np.abs(ref64[fin]), 1.0) if scale is None else np.maximum(np.maximum(np.abs(ref64[fin]), 1.0), np.abs(scale[fin]))
    with np.errstate(invalid="ignore"):
        err = np.abs(ours[fin] - ref64[fin]) / sc
    err = np.where(np.isnan(err), np.inf, err)
    if not (err <= LP_BAR).all():
        i = int(np.argmax(err))
        raise AssertionError(f"{what}: {int((err > LP_BAR).sum())} rows off the oracle; worst row {np.nonzero(fin)[0][i]}: "
                             f"ours {ours[fin][i]!r} ref64 {ref64[fin][i]!r}")  # fmt: skip
    return float(err.max())


def check_inverse_lp(st, ours, rows, bar, what):
    """The log-density of the inverse: the -inf rows match the oracle on every row; the values, at the inverse bar,
    on the rows where the oracle's forward of the returned x gives z back.  A circular spline is a bijection of
    [-pi, pi] only (the BoxUniform of NCSF reaches 1e-5 beyond it, and a coupling layer after it can leave it): where
    a circular layer's input lies outside, its inverse followed by its forward does not return that input, so the
    engine's base(z) + ladj at the solution and the oracle's log p(x) of the returned x are different quantities."""
    ref64, ref32 = st.ilp64[rows], st.ilp32[rows]
    inf = np.isneginf(ref64)
    assert np.array_equal(np.isneginf(ours), inf), f"{what}: -inf rows of the inverse's log_prob differ"
    sel = ~inf & st.bijective[rows]
    if not sel.any():
        return 0.0
    r = elem_err(ours[sel], ref64[sel], ref32[sel], bar)
    assert (r <= 1).all(), f"{what}: inverse log_prob off the oracle at rows {np.nonzero(sel)[0][r > 1][:8]}"
    return float((np.abs(ours[sel] - ref64[sel]) / np.maximum(np.abs(ref64[sel]), 1.0)).max())


def z_rtol(st):
    """1e-5 when every conditioner runs fp32 GEMMs, 4e-5 when one runs on the tensor cores."""
    tc = [LAYERS[t][3] is False for t, _ in st.members if LAYERS[t][0] in ("ar", "cpl", "ewc")]
    return 4e-5 if any(tc) else 1e-5


def inverse_bar(st, fused):
    """SEQ_BAR when the inverse runs only sequential-inverse layers and parameter-free or table layers; SWEEP_BAR
    when it re-rounds a conditioner (sweeps, coupling, element-wise with context, the forward of an inverted member)."""
    for t, inv in st.members:
        kind, _, seq, _ = LAYERS[t]
        if inv or kind in ("cpl", "ewc") or (kind == "ar" and not (seq and fused)):
            return SWEEP_BAR
    return SEQ_BAR


def pads_nan(buf, n):
    return bool(torch.isnan(buf[:, n:]).all())


# --------------------------------------------------------------------------- #
# 1-3. the composition table
# --------------------------------------------------------------------------- #

PARAMS = case_params()


@pytest.mark.parametrize("name,ctx,fused", PARAMS, ids=[f"{n}-{c}-{'fused' if f else 'unfused'}" for n, c, f in PARAMS])
def test_composition_vs_oracle(device, name, ctx, fused, record_property):
    st = Setup.get(name, ctx, device)
    L = E.lib()
    # the engine agrees with the table on every member's paths
    for (t, _), h in zip(st.members, st.handles):
        kind, fwd_fused, seq, _ = LAYERS[t]
        info = (ctypes.c_double * 4)()
        assert (L.zk_layer_fused_info(h, info) == 1) == fwd_fused, f"{name}: {t} fused forward"
        assert bool(L.zk_layer_sequential_inverse(h)) == (kind == "ar" and seq), f"{name}: {t} sequential inverse"
    call = Call(st.desc, device)
    inv_any = inverted_any(name)
    refused_fwd = inv_any and not fused  # an inverted member's sequential inverse does not run unfused
    rt, ibar = z_rtol(st), inverse_bar(st, fused)
    worst = dict(z=0.0, ladj=0.0, lp=0.0, x=0.0, ilp=0.0)
    prev = L.zk_set_fused_layers(fused)
    try:
        for B in BATCHES:
            what = f"{name} ctx={ctx} fused={fused} B={B}"
            rows = slice(0, B)
            ws = call.ws(L.zk_flow_workspace_bytes(ctypes.byref(st.desc), max(B, 1)))
            c, ldc = ctx_buf(st, B, device)
            c_before = None if c is None else c.clone()
            # forward
            x = padded(st.x[rows] if B else st.x[:1], PAD_X, device)
            x_before = x.clone()
            z, ladj = nan((max(B, 1), D + PAD_Z), device), nan((max(B, 1),), device)
            s, n = call.forward(x, D + PAD_X, c, ldc, B, z, D + PAD_Z, ladj, ws)
            if refused_fwd:
                assert s == E.ZK_EUNSUPPORTED and n == 0, f"{what}: forward status {s}, {n} launches"
                assert torch.isnan(z).all() and torch.isnan(ladj).all(), f"{what}: a refused forward wrote its outputs"
            else:
                E.check(s)
                assert pads_nan(z, D), f"{what}: the pad of z was written"
                if B == 0:
                    assert n == 0 and torch.isnan(z).all() and torch.isnan(ladj).all(), f"{what}: B = 0 wrote or launched"
                else:
                    worst["z"] = max(worst["z"], check_elems(cpu(z[:, :D]), st.z64[rows], st.z32[rows], rt, what + " z"))
                    scale = st.lp_scale[rows]
                    worst["ladj"] = max(worst["ladj"], check_lp(cpu(ladj), st.ladj64[rows], what + " ladj", scale=scale))
            # log_prob, with and without the device sum
            for with_sum in (False, True):
                lp = nan((max(B, 1),), device)
                total = torch.full((1,), float("nan"), device=device, dtype=torch.float64) if with_sum else None
                s, n = call.log_prob(x, D + PAD_X, c, ldc, B, lp, total, ws)
                if refused_fwd:
                    assert s == E.ZK_EUNSUPPORTED and n == 0 and torch.isnan(lp).all(), f"{what}: log_prob not refused cleanly"
                    continue
                E.check(s)
                if B == 0:
                    assert torch.isnan(lp).all() and n == (2 if with_sum else 0), f"{what}: B = 0 log_prob"
                    if with_sum:
                        assert total.item() == 0.0, f"{what}: the sum of no rows is {total.item()}"
                    continue
                got = cpu(lp)
                worst["lp"] = max(worst["lp"], check_lp(got, st.lp64[rows], what + f" log_prob sum={with_sum}"))
                if with_sum:
                    ref = got.sum()
                    t = total.item()
                    assert t == ref or abs(t - ref) <= 1e-9 * max(abs(ref), 1.0), f"{what}: sum {t} vs {ref}"
            # inverse, and inverse + log_prob where the flow has no inverted member
            zin = padded(st.z[rows] if B else st.z[:1], PAD_X, device)
            z_before = zin.clone()
            for with_lp in (False, True):
                xo = nan((max(B, 1), D + PAD_Z), device)
                lp = nan((max(B, 1),), device) if with_lp else None
                s, n = call.inverse(zin, D + PAD_X, c, ldc, B, xo, D + PAD_Z, lp, ws)
                if with_lp and inv_any:
                    assert s == E.ZK_EINVAL and n == 0, f"{what}: inverse + log_prob with inverted members: status {s}, {n} launches"
                    assert torch.isnan(xo).all() and torch.isnan(lp).all(), f"{what}: the refused inverse wrote its outputs"
                    continue
                E.check(s)
                assert pads_nan(xo, D), f"{what}: the pad of x was written"
                if B == 0:
                    assert n == 0 and torch.isnan(xo).all() and (lp is None or torch.isnan(lp).all()), f"{what}: B = 0 inverse"
                    continue
                worst["x"] = max(worst["x"], check_elems(cpu(xo[:, :D]), st.x64[rows], st.x32[rows], ibar, what + f" inverse x lp={with_lp}"))
                if with_lp:
                    worst["ilp"] = max(worst["ilp"], check_inverse_lp(st, cpu(lp), rows, ibar, what))
            # the inputs and their pads are untouched
            assert torch.equal(x.isnan(), x_before.isnan()) and torch.equal(x.nan_to_num(), x_before.nan_to_num())
            assert torch.equal(zin.isnan(), z_before.isnan()) and torch.equal(zin.nan_to_num(), z_before.nan_to_num())
            if c is not None:
                assert torch.equal(c.isnan(), c_before.isnan()) and torch.equal(c.nan_to_num(), c_before.nan_to_num())
    finally:
        L.zk_set_fused_layers(prev)
    for k, v in worst.items():
        record_property(k, v)
    print(f"MAXIMA {name} ctx={ctx} fused={fused}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


# --------------------------------------------------------------------------- #
# 4. row chunks
# --------------------------------------------------------------------------- #


def a256(n):
    return (n + 255) // 256 * 256


def largest_fitting_rows(B, ws, need, granule):
    """largest_fitting_rows (api_internal.cuh) restated."""
    if B <= 0:
        return 0
    if need(B) <= ws:
        return B
    if need(1) > ws:
        return 0
    lo, hi = 1, B
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        if need(mid) <= ws:
            lo = mid
        else:
            hi = mid - 1
    if granule > 1 and lo >= 2 * granule and need(lo // granule * granule) <= ws:
        lo = lo // granule * granule
    return lo


class Planner:
    """flow_ws_for / flow_chunk_rows (api.cu) restated from the layer queries of the C ABI: the scratch of each member
    in the direction it runs (an inverted member runs its layer's inverse in the forward direction and its forward
    in the inverse one); dir 0 is the public figure, 1 forward, 2 inverse."""

    def __init__(self, st, fused=True):
        L = E.lib()
        self.D, self.fused = D, fused
        self.layers = []
        for (t, inv), h in zip(st.members, st.handles):
            info = (ctypes.c_double * 4)()
            self.layers.append((LAYERS[t][0] == "ar", L.zk_layer_fused_info(h, info) == 1, bool(L.zk_layer_sequential_inverse(h)),
                                inv, (lambda n, h=h: L.zk_layer_workspace_bytes(h, n))))  # fmt: skip

    def layer_ws(self, layer, n, d):
        ar, fwd_fused, seq, _, ws = layer
        if d and ar and self.fused:
            if d == 1 and fwd_fused:
                return 0
            if d == 2 and seq:
                return 0
        return ws(n)

    def need(self, n, d):
        m = 0
        for layer in self.layers:
            run = 3 - d if (d and layer[3]) else d
            w = self.layer_ws(layer, n, run)
            if run == 2 and w:
                w = max(w, self.layer_ws(layer, n, 1))
            m = max(m, w)
        return 2 * a256(n * self.D * 4) + a256(n * 4) + a256(n * self.D * 4) + a256(REDUCE_SCRATCH) + m + 1024

    def rows(self, B, ws, d):
        return largest_fitting_rows(B, ws, lambda n: self.need(n, d), GRANULE)


def workspace_for(plan, desc, d, target):
    """(workspace bytes, the chunk rows the planner takes with it, batch) for a target chunk."""
    if target == "one":
        ws = plan.need(1, d)
        assert plan.need(2, d) > ws, "one row is not the largest chunk that fits this workspace"
        return ws, 1, 300
    if target == "hundred":
        ws = plan.need(100, d)
        assert plan.need(101, d) > ws
        return ws, 100, 1037
    if target == "granule":  # the search finds 2048 + k rows, which round down to 2048
        ws = plan.need(2048 + 333, d)
        B = 5000
        lo = largest_fitting_rows(B, ws, lambda n: plan.need(n, d), 1)
        assert 2 * GRANULE < lo < 3 * GRANULE and lo % GRANULE, lo
        return ws, 2048, B
    ws = E.lib().zk_flow_min_workspace_bytes(ctypes.byref(desc))
    B = 3001
    return ws, plan.rows(B, ws, d), B


CHUNK_CALLS = [("cpl_last", "log_prob"), ("cpl_last", "forward"), ("inv_mid_last", "log_prob"), ("sweep_last", "inverse_lp"),
               ("inv_fp32", "inverse"), ("inv_fp32", "log_prob"), ("inv_circ_box", "inverse"), ("ewc_last", "inverse_lp")]  # fmt: skip
CHUNK_TARGETS = ["one", "hundred", "granule", "min"]


@pytest.mark.parametrize("target", CHUNK_TARGETS)
@pytest.mark.parametrize("name,what", CHUNK_CALLS, ids=[f"{n}-{w}" for n, w in CHUNK_CALLS])
def test_row_chunks(device, name, what, target):
    st = Setup.get(name, "rows", device)
    L = E.lib()
    plan = Planner(st)
    for n in (1, 2, 3, 100, 101, 1024, 2048, 2381, 3001, 5000):  # the dir-0 restatement is the public figure
        assert plan.need(n, 0) == L.zk_flow_workspace_bytes(ctypes.byref(st.desc), n), n
    assert plan.need(1, 0) == L.zk_flow_min_workspace_bytes(ctypes.byref(st.desc))
    d = 2 if what.startswith("inverse") else 1
    ws_bytes, rows, B = workspace_for(plan, st.desc, d, target)
    assert plan.rows(B, ws_bytes, d) == rows, (plan.rows(B, ws_bytes, d), rows)
    assert rows < B, f"{target}: one chunk"
    chunks = -(-B // rows)
    call = Call(st.desc, device)
    g = torch.Generator().manual_seed(B)
    inp = padded(torch.randn(B, D, generator=g).numpy(), PAD_X, device)
    c = padded(torch.randn(B, C, generator=g).numpy(), PAD_C, device)
    full = call.ws(L.zk_flow_workspace_bytes(ctypes.byref(st.desc), B))
    small = call.ws(ws_bytes)

    def run(ws):
        if what == "log_prob":
            lp, total = nan((B,), device), torch.zeros(1, device=device, dtype=torch.float64)
            s, n = call.log_prob(inp, D + PAD_X, c, C + PAD_C, B, lp, total, ws)
            outs = [lp, total]
        elif what == "forward":
            z, ladj = nan((B, D + PAD_Z), device), nan((B,), device)
            s, n = call.forward(inp, D + PAD_X, c, C + PAD_C, B, z, D + PAD_Z, ladj, ws)
            outs = [z, ladj]
        else:
            xo = nan((B, D + PAD_Z), device)
            lp = nan((B,), device) if what == "inverse_lp" else None
            s, n = call.inverse(inp, D + PAD_X, c, C + PAD_C, B, xo, D + PAD_Z, lp, ws)
            outs = [xo] + ([lp] if lp is not None else [])
        E.check(s)
        return [cpu(o) for o in outs], n

    ref, n1 = run(full)
    got, n = run(small)
    extra = 2 if what == "log_prob" else 0  # the two reduction launches
    assert n == chunks * (n1 - extra) + extra, f"{name} {what} {target}: {n} launches, {chunks} chunks of {n1 - extra}"
    for a, b in zip(got, ref):
        assert np.array_equal(a, b, equal_nan=True), f"{name} {what} {target}: {rows}-row chunks differ from one chunk"
    assert np.isfinite(got[0][:, :D] if got[0].ndim == 2 else got[0]).all()


# --------------------------------------------------------------------------- #
# 5. the host-buffer call
# --------------------------------------------------------------------------- #


def sm_count():
    n, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    E.check(E.lib().zk_device_info(ctypes.byref(n), ctypes.byref(major), ctypes.byref(minor)))
    return n.value


def host_plan(st, B, ws_bytes):
    """host_chunk_plan with the cap zk_flow_log_prob_host derives from the workspace (api.cu), restated."""
    L = E.lib()
    wave = sm_count() * max([64] + [L.zk_layer_fused_tile_rows(h) for h in st.handles])

    def need(n):
        return (2 * (a256(n * D * 4) + a256(n * C * 4) + a256(n * 4)) + a256(C * 4) + a256(4096 * 8)
                + L.zk_flow_workspace_bytes(ctypes.byref(st.desc), n))  # fmt: skip

    Bmax = B
    while Bmax > 1 and need(Bmax) > ws_bytes:
        Bmax = max(wave, Bmax // 2 // wave * wave) if Bmax > wave else (Bmax + 1) // 2
    out = (ctypes.c_int64 * 4096)()
    k = L.zk_debug_host_chunk_plan(B, wave, Bmax, out, 4096)
    return list(out[:k]), wave


HOST = ["small", "growing", "capped", "strided", "bcast", "no_sum", "empty"]


@pytest.mark.parametrize("mode", HOST)
def test_host_buffer_call(device, mode):
    """A mixed flow on a BoxUniform base (coupling, rotation, circular autoregressive, all inside the box)."""
    ctx = "bcast" if mode == "bcast" else "rows"
    st = Setup.get("box_cpl_circ", ctx, device)
    L = E.lib()
    wave = host_plan(st, 1, 1 << 40)[1]
    B = {"growing": 4 * wave + wave // 2 + 77, "empty": 0}.get(mode, 20011)
    g = torch.Generator().manual_seed(B + 1)
    ldx = D + (PAD_X if mode == "strided" else 0)
    ldc = 0 if mode == "bcast" else C + (PAD_C if mode == "strided" else 0)
    xh = torch.full((max(B, 1), ldx), float("nan"), **F32)
    xh[:B, :D] = (torch.rand(B, D, generator=g) * 2 - 1) * 3.1
    ch = torch.randn(C, generator=g) if ldc == 0 else torch.full((max(B, 1), ldc), float("nan"), **F32)
    if ldc:
        ch[:B, :C] = torch.randn(B, C, generator=g)
    want = L.zk_flow_host_workspace_bytes(ctypes.byref(st.desc), B)
    ws_bytes = L.zk_flow_host_workspace_bytes(ctypes.byref(st.desc), 1000) if mode == "capped" else want
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
    lph = torch.full((max(B, 1),), float("nan"), **F32)
    total = ctypes.c_double(float("nan"))
    with torch.cuda.device(device):
        E.check(L.zk_flow_log_prob_host(ctypes.byref(st.desc), xh.data_ptr(), ldx, ch.data_ptr(), ldc, B, lph.data_ptr(),
                                        None if mode == "no_sum" else ctypes.byref(total), ws.data_ptr(), ws_bytes,
                                        E.stream_ptr(device)))  # fmt: skip
    if mode == "empty":
        assert total.value == 0.0 and torch.isnan(lph).all()
        return
    plan, wave = host_plan(st, B, ws_bytes)
    assert sum(plan) == B
    if mode == "small":
        assert B <= 4 * wave and len(plan) > 1 and len(set(plan[:-1])) == 1, plan
    if mode == "growing":
        assert B > 4 * wave and plan[0] == wave and plan[1] == 2 * wave, plan
    if mode == "capped":
        assert ws_bytes < want and max(plan) < max(host_plan(st, B, want)[0]), plan
    # the device call on the same rows, bit for bit
    call = Call(st.desc, device)
    xd = xh[:B, :D].contiguous().to(device)
    cd = ch.to(device) if ldc == 0 else ch[:B, :C].contiguous().to(device)
    lpd = nan((B,), device)
    E.check(call.log_prob(xd, D, cd, 0 if ldc == 0 else C, B, lpd, None, call.ws(L.zk_flow_workspace_bytes(ctypes.byref(st.desc), B)))[0])
    assert torch.equal(lph, lpd.cpu()), f"{mode}: the host-buffer call differs from the device call"
    assert torch.isfinite(lph).all()
    if mode == "no_sum":
        assert math.isnan(total.value)
        return
    # the sum: the fixed-order sum of the per-chunk device sums
    acc, i0 = 0.0, 0
    tot = torch.zeros(1, device=device, dtype=torch.float64)
    for n in plan:
        E.check(call.log_prob(xd[i0 : i0 + n], D, cd if ldc == 0 else cd[i0 : i0 + n], 0 if ldc == 0 else C, n, lpd[i0 : i0 + n], tot,
                              call.ws(L.zk_flow_workspace_bytes(ctypes.byref(st.desc), n)))[0])  # fmt: skip
        acc += tot.item()
        i0 += n
    assert total.value == acc, f"{mode}: sum {total.value!r} vs per-chunk sums {acc!r}"


# --------------------------------------------------------------------------- #
# 6. refusals
# --------------------------------------------------------------------------- #

REFUSALS = ["alias_forward", "alias_inverse", "ws_forward", "ws_log_prob", "ws_inverse", "inverse_lp_inverted",
            "no_context_forward", "no_context_log_prob", "no_context_inverse", "no_context_host", "unfused_inverted_forward",
            "unfused_inverted_log_prob", "unfused_inverted_host"]  # fmt: skip


@pytest.mark.parametrize("kind", REFUSALS)
def test_refusals(device, kind):
    """Each refused call returns a status before it launches anything, and its outputs keep their NaN fill."""
    name = {"inverse_lp_inverted": "inv_first"}.get(kind, "inv_fp32" if kind.startswith("unfused") else "cpl_last")
    st = Setup.get(name, "rows", device)
    L = E.lib()
    call = Call(st.desc, device)
    B = 300
    plan = Planner(st)
    x = padded(st.x[:B], PAD_X, device)
    c, ldc = ctx_buf(st, B, device)
    if kind.startswith("no_context"):
        c = None
    full = call.ws(L.zk_flow_workspace_bytes(ctypes.byref(st.desc), B))
    ws = full
    if kind.startswith("ws_"):
        d = 2 if kind == "ws_inverse" else 1
        below = plan.need(1, d) - 1
        assert below < L.zk_flow_min_workspace_bytes(ctypes.byref(st.desc))
        ws = call.ws(below)
    z, ladj, lp = nan((B, D + PAD_Z), device), nan((B,), device), nan((B,), device)
    total = torch.full((1,), float("nan"), device=device, dtype=torch.float64)
    prev = L.zk_set_fused_layers(0 if kind.startswith("unfused") else 1)
    try:
        if kind.endswith("host"):
            xh, lph, tot = torch.from_numpy(st.x[:B].copy()), torch.full((B,), float("nan"), **F32), ctypes.c_double(float("nan"))
            chh = torch.from_numpy(st.c[:B].copy())
            n0 = L.zk_launch_count()
            s = L.zk_flow_log_prob_host(ctypes.byref(st.desc), xh.data_ptr(), D, None if kind.startswith("no_context") else chh.data_ptr(),
                                        C, B, lph.data_ptr(), ctypes.byref(tot), full[0].data_ptr(), full[1], E.stream_ptr(device))  # fmt: skip
            torch.cuda.synchronize(device)
            n = L.zk_launch_count() - n0
            assert torch.isnan(lph).all(), f"{kind}: the refused host call wrote its output"
        elif kind.endswith("forward"):
            s, n = call.forward(x, D + PAD_X, c, ldc, B, x if kind.startswith("alias") else z, D + PAD_X if kind.startswith("alias") else D + PAD_Z, ladj, ws)  # fmt: skip
        elif kind.endswith("log_prob"):
            s, n = call.log_prob(x, D + PAD_X, c, ldc, B, lp, total, ws)
        else:  # inverse
            zin = x
            s, n = call.inverse(zin, D + PAD_X, c, ldc, B, zin if kind.startswith("alias") else z,
                                D + PAD_X if kind.startswith("alias") else D + PAD_Z, lp if kind == "inverse_lp_inverted" else None, ws)  # fmt: skip
    finally:
        L.zk_set_fused_layers(prev)
    assert s != E.ZK_OK, f"{kind}: accepted"
    assert s == (E.ZK_EUNSUPPORTED if kind.startswith("unfused") else E.ZK_EINVAL), (kind, s, L.zk_last_error())
    assert n == 0, f"{kind}: {n} launches before the refusal ({L.zk_last_error().decode()})"
    assert torch.isnan(z).all() and torch.isnan(ladj).all() and torch.isnan(lp).all(), f"{kind}: outputs written"
    assert torch.isnan(total).all()
    ref = padded(st.x[:B], PAD_X, device)
    assert torch.equal(x.nan_to_num(), ref.nan_to_num()) and torch.equal(x.isnan(), ref.isnan()), f"{kind}: input written"


def test_inverted_member_workspace_in_both_directions(device):
    """Any workspace >= zk_flow_min_workspace_bytes is accepted, so the planner must count an inverted member at the
    direction it runs: its layer's forward (unfused for fp32 GEMMs or a circular spline) in the inverse, its
    sequential inverse (no scratch) in the forward."""
    L = E.lib()
    for name in ("inv_fp32", "inv_circ_box", "inv_last_box"):
        st = Setup.get(name, "rows", device)
        call = Call(st.desc, device)
        plan = Planner(st)
        B = 4099
        mn = L.zk_flow_min_workspace_bytes(ctypes.byref(st.desc))
        zin = padded(st.z[:B], PAD_X, device)
        c, ldc = ctx_buf(st, B, device)
        outs = []
        for ws in (call.ws(L.zk_flow_workspace_bytes(ctypes.byref(st.desc), B)), call.ws(mn), call.ws(mn + 12345)):
            xo = nan((B, D + PAD_Z), device)
            E.check(call.inverse(zin, D + PAD_X, c, ldc, B, xo, D + PAD_Z, None, ws)[0])
            outs.append(cpu(xo))
        for o in outs[1:]:
            assert np.array_equal(o, outs[0], equal_nan=True), f"{name}: capped inverse differs"
        # the forward direction plans with no scratch for the inverted member: taller chunks at the same workspace
        assert plan.rows(B, mn, 1) >= plan.rows(B, mn, 2)
