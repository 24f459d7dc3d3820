"""Tests of the CNF backward (zk_cnf_backward: cnf_replay_kernel, cnf_adjoint_kernel, cnf_grad_reduce_kernel and
cnf_context_sum_kernel in cnf.cu, and the _CNFAdjoint node of transforms.py) at its launch-plan, multi-block, chunk,
MLP-shape, NULL-output, step-log, time-interval and Python-layer edges, against the fp64 restatement of the adjoint
(tests/cnf_adjoint_reference.py) replaying the engine's own step log.

* Plan: `back_plan` (test_cnf_grad_host.py) restates cnf_back_geometry; the case table reaches 256, 128, 64 and 32
  threads with and without a trace, and holds the widest two-layer hidden width of CNF(3, 2) at 32 threads next to
  the next multiple of 8, which is refused.  The chunk rows of zk_cnf_backward_plan follow whole blocks of threads
  over a range of workspace sizes, and the Python layer refuses at the forward call what the plan refuses.
* Rows: batches tiled from one base block, at sizes around one block and around one and two blocks per CTA, give
  the base rows' gradients bit for bit (a row's arithmetic depends only on the row and the step log) and n times
  the base block's parameter gradients up to fp32 reassociation; chunked calls with padded strides give the
  one-chunk call's bits.
* Shapes and contracts: 16 linear layers, freqs 0 and 32, D = 1, D = 64, C = 0, C = 130 (two blocks of the context
  sum), NULL outputs, rejected rows anywhere in the log, a log of 100+ accepted steps and every time interval of the
  forward's edge tests; the Python layer against direct C-ABI calls.

Bars: BAR = 1e-4 of each gradient tensor's largest entry against the restatement, as in test_gpu_cnf_grad.py.
Parameter gradients of a tiled batch meet n times the base block's within SUM_BAR = 2e-5 of the largest entry: the
CTA partials sum different rows in fp32 (measured 1.3e-6 on an NVIDIA H100 80GB HBM3 at a 700 W power limit).
grad_ladj = 0 meets the trace-free call within 1e-6, and a broadcast context's gradient the sum of its per-row one
within 1e-6: both only reorder fp32 additions.  Everything else is bitwise."""

import ctypes

import numpy as np
import pytest
import torch

import cnf_adjoint_reference as A
import cnf_reference as R
from test_cnf_grad_host import back_plan, relmax
from test_gpu_cnf_edges import INTERVALS, TRACES, make, padded, raw, times_of
from test_gpu_cnf_grad import BAR, WORST, _field, _random_case, as_np, backward, check_against_restatement
from zuko_b200 import _engine as E
from zuko_b200.flows import CNF

NAN = float("nan")
SENT = 7.0  # bytes an output must leave alone
SUM_BAR = 2e-5
FAMILIES = (R.TRACE_NONE, R.TRACE_EXACT)


# --------------------------------------------------------------------------- #
# helpers
# --------------------------------------------------------------------------- #


def ptr(t):
    return t if t is None or isinstance(t, int) else t.data_ptr()


def ld(t, n):
    return n if t is None or t.dim() < 2 else t.stride(0)


def on(device):
    """numpy -> fp32 tensors on `device`, None kept."""
    return lambda a: None if a is None else torch.as_tensor(np.asarray(a), dtype=torch.float32, device=device)


def last_error():
    return E.lib().zk_last_error().decode()


def bplan_call(h, B, trace, accepted, ws_bytes=1 << 40):
    out = [ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_int64(-1), ctypes.c_size_t(0)]
    st = E.lib().zk_cnf_backward_plan(h, B, trace, accepted, ws_bytes, *map(ctypes.byref, out))
    return st, tuple(v.value for v in out)


def call(eng, B, lg, counts, trace, *, x, c=None, ldc=None, eps=None, gy=None, gl=None, gx=None, gc=None, ldgc=None,
         gW=None, gb=None, grads=True, ws=None, ws_bytes=None):  # fmt: skip
    """One zk_cnf_backward call with every pointer and stride in the caller's hands (device tensors or views, None
    for NULL; a None entry of gW / gb is a NULL layer); returns the status after a device synchronise."""
    lib = E.lib()
    h = eng.t._cnf_handle()
    n = len(eng.t.ode._linears())
    lgs = None
    if grads:
        lgs = E.LayerGrads()
        if gW is not None:
            lgs.grad_weight = (ctypes.c_void_p * n)(*map(ptr, gW))
        if gb is not None:
            lgs.grad_bias = (ctypes.c_void_p * n)(*map(ptr, gb))
    log = torch.as_tensor(np.asarray(lg, np.float32).reshape(-1, 4), device=eng.dev)
    if ws_bytes is None:
        ws_bytes = lib.zk_cnf_backward_workspace_bytes(h, B, trace, counts[1])
    if ws is None:
        ws = torch.empty(max(ws_bytes, 256), dtype=torch.uint8, device=eng.dev)
    if ldc is None:
        ldc = 0 if c is None or c.dim() < 2 else c.stride(0)
    st = lib.zk_cnf_backward(
        h, ptr(x), ld(x, eng.D), ptr(c), ldc, B, log.data_ptr(), counts[0], counts[1], trace, ptr(eps), ld(eps, eng.D),
        ptr(gy), ld(gy, eng.D), ptr(gl), ptr(gx), ld(gx, eng.D), ptr(gc), ld(gc, eng.C) if ldgc is None else ldgc,
        None if lgs is None else ctypes.byref(lgs), ptr(ws), ws_bytes, E.stream_ptr(eng.dev))  # fmt: skip
    torch.cuda.synchronize()
    return st


def flat(out):
    gx, gc, gW, gb = out
    return [gx, gc, *gW, *gb]


def assert_same(a, b, what=""):
    for i, (u, v) in enumerate(zip(flat(a), flat(b), strict=True)):
        assert (u is None) == (v is None), (what, i)
        assert u is None or torch.equal(u, v), (what, i)


def out_view(shape, device, pad=2):
    """A NaN-filled output view inside a buffer whose pads hold SENT: (buffer, view)."""
    big, view = padded(np.full(shape, NAN), device, pad=pad, fill=SENT)
    return big, view


def pads_untouched(big, pad, n):
    return bool(torch.all(big[:, :pad] == SENT) and torch.all(big[:, pad + n :] == SENT))


# --------------------------------------------------------------------------- #
# A. the launch plan
# --------------------------------------------------------------------------- #

# name -> (D, C, F, hidden); the comments give the threads without / with a trace
BACK_PLAN_CASES = {
    "d1_f0": (1, 0, 0, ()),           # 256 / 256
    "d2_h16": (2, 1, 3, (16, 16)),    # 128 / 256
    "h24": (3, 2, 3, (24, 24)),       # 256 / 128
    "h48": (3, 2, 3, (48, 48)),       # 128 / 64
    "cnf168": (16, 8, 3, (64, 64)),   # 64 / 32
    "h96": (3, 2, 3, (96, 96)),       # 64 / 32: the widest (h, h) of CNF(3, 2) with a trace
    "h104": (3, 2, 3, (104, 104)),    # 64 / refused
    "h128": (3, 2, 3, (128, 128)),    # 32 / refused
    "h144": (3, 2, 3, (144, 144)),    # 32 / refused: the widest (h, h) of CNF(3, 2)
    "h152": (3, 2, 3, (152, 152)),    # refused / refused
}  # fmt: skip


def bplan(name, trace):
    D, C, F, hidden = BACK_PLAN_CASES[name]
    return back_plan(D, C, F, [D + C + 2 * F, *hidden, D], trace)


def test_back_plan_table_reaches_every_cell():
    for trace in FAMILIES:
        threads = {(bplan(n, trace) or (None,))[0] for n in BACK_PLAN_CASES}
        assert threads >= {256, 128, 64, 32, None}, (trace, threads)
    for trace, widest in ((R.TRACE_NONE, "h144"), (R.TRACE_EXACT, "h96")):
        assert bplan(widest, trace)[0] == 32
        D, C, F, (h, _) = BACK_PLAN_CASES[widest]
        assert back_plan(D, C, F, [D + C + 2 * F, h + 8, h + 8, D], trace) is None
    assert bplan("h128", R.TRACE_NONE)[0] == 32 and bplan("h128", R.TRACE_EXACT) is None
    assert bplan("h152", R.TRACE_NONE) is None
    # the Hutchinson trace keeps the exact trace's per-row state
    assert all(bplan(n, R.TRACE_HUTCHINSON) == bplan(n, R.TRACE_EXACT) for n in BACK_PLAN_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BACK_PLAN_CASES))
def test_back_plan_matches_restatement(device, name):
    eng = make(device, *BACK_PLAN_CASES[name])
    h = eng.t._cnf_handle()
    lib = E.lib()
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    for trace in TRACES.values():
        want = bplan(name, trace)
        st, (ctas, nt, rows, smem) = bplan_call(h, 1000, trace, 10)
        if want is None:
            assert st == E.ZK_EUNSUPPORTED and "backward state" in last_error()
            assert lib.zk_cnf_backward_min_workspace_bytes(h, trace, 10) == 0
            assert lib.zk_cnf_backward_workspace_bytes(h, 1000, trace, 10) == 0
            continue
        assert st == E.ZK_OK and (nt, smem) == want, (trace, nt, smem, want)
        assert ctas >= sms and ctas % sms == 0 and rows == 1000


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d2_h16", "cnf168"])
def test_chunk_rows_follow_whole_blocks(device, name):
    eng = make(device, *BACK_PLAN_CASES[name])
    h = eng.t._cnf_handle()
    lib = E.lib()
    for trace in TRACES.values():
        for acc in (0, 9):
            nt = bplan_call(h, 1, trace, acc)[1][1]
            fixed = lib.zk_cnf_backward_workspace_bytes(h, 0, trace, acc)
            row = lib.zk_cnf_backward_workspace_bytes(h, 1, trace, acc) - fixed
            # accepted + 1 replayed states, the 7 stage values of f, the 6 of da/dt, a; and the context row
            assert row == ((acc + 15) * eng.D + eng.C) * 4
            least = lib.zk_cnf_backward_min_workspace_bytes(h, trace, acc)
            assert least == fixed + nt * row
            for B in (1, nt - 1, nt, nt + 1, 5 * nt + 3, 100000):
                full = lib.zk_cnf_backward_workspace_bytes(h, B, trace, acc)
                sizes = {least - 1, least, full - 1, full, full + 1}
                sizes |= {least + k * row + e for k in (1, nt - 1, nt, nt + 1, 2 * nt - 1, 2 * nt, 3 * nt + 1) for e in (-1, 0)}
                for ws in sorted(sizes):
                    st, (_, _, rows, _) = bplan_call(h, B, trace, acc, ws)
                    if ws < fixed + min(B, nt) * row:
                        assert st == E.ZK_EINVAL and "workspace" in last_error(), (B, ws)
                        continue
                    fit = (ws - fixed) // row
                    assert st == E.ZK_OK and rows == (B if fit >= B else fit // nt * nt), (B, ws, rows)
                    assert rows == B or (0 < rows < B and rows % nt == 0)
        st, (_, _, rows, _) = bplan_call(h, 0, trace, 9, 0)  # B = 0 needs no workspace
        assert st == E.ZK_OK and rows == 0


@pytest.mark.gpu
def test_misaligned_and_null_workspace(device):
    eng = make(device, 3, 2, 3, (24, 24))
    B = 40
    x, c, eps, gy, gl = _random_case(eng, B, seed=4)
    _, _, counts, lg = eng.run(x, c)
    T = on(device)
    ws = torch.empty(E.lib().zk_cnf_backward_workspace_bytes(eng.t._cnf_handle(), B, R.TRACE_EXACT, counts[1]) + 512,
                     dtype=torch.uint8, device=device)  # fmt: skip
    gx = torch.full((B, 3), NAN, device=device)
    st = call(eng, B, lg, counts, R.TRACE_EXACT, x=T(x), c=T(c), gy=T(gy), gl=T(gl), gx=gx, ws=ws.data_ptr() + 128,
              ws_bytes=ws.numel() - 128)  # fmt: skip
    assert st == E.ZK_EINVAL and "aligned" in last_error() and torch.isnan(gx).all()
    # B = 0: no workspace is needed; the summed context row is still written
    gc = torch.full((2,), NAN, device=device)
    st = call(eng, 0, lg, counts, R.TRACE_EXACT, x=None, c=T(c[0]), gl=T(gl), gc=gc, ws=0, ws_bytes=0)
    assert st == E.ZK_OK and torch.equal(gc, torch.zeros(2, device=device))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["h128", "h152"])
def test_python_layer_refuses_what_the_plan_refuses(device, name):
    D, C, F, hidden = BACK_PLAN_CASES[name]
    torch.manual_seed(0)
    flow = CNF(D, C, freqs=F, hidden_features=list(hidden), adjoint=True).to(device).train()
    c = torch.randn(16, C, device=device)
    x = torch.randn(16, D, device=device)
    if bplan(name, R.TRACE_NONE) is not None:  # sampling integrates x alone: its backward fits without a trace
        flow(c).rsample().square().sum().backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in flow.parameters())
    else:
        with pytest.raises(NotImplementedError, match="backward state"):
            flow(c).rsample()
    with pytest.raises(NotImplementedError, match="backward state"):
        flow(c).log_prob(x)
    with torch.no_grad():
        assert torch.isfinite(flow(c).log_prob(x)).all() and flow(c).sample().shape == (16, D)
    flow.eval()
    with pytest.raises(NotImplementedError, match="backward state"):
        flow(c).log_prob(x.clone().requires_grad_())


# --------------------------------------------------------------------------- #
# B. many blocks per CTA, and chunks
# --------------------------------------------------------------------------- #

B0 = 29


def _sub(a, idx):
    return None if a is None else a[idx]


@pytest.mark.gpu
@pytest.mark.parametrize("name,trace", [("d2_h16", "exact"), ("cnf168", "hut"), ("cnf168", "exact")])
def test_tiled_batches_reproduce_the_base_block(device, name, trace):
    tr = TRACES[trace]
    eng = make(device, *BACK_PLAN_CASES[name])
    h = eng.t._cnf_handle()
    x, c, eps, gy, gl = _random_case(eng, B0, seed=11, trace=tr)
    _, _, counts, lg = eng.run(x, c, tr, eps=eps)
    st, (ctas, nt, _, _) = bplan_call(h, 1, tr, counts[1])
    assert st == E.ZK_OK and nt == (256 if name == "d2_h16" else 32)
    base = backward(eng, x, c, lg, counts, tr, eps, gy, gl)
    sizes = [B0, nt - 1, nt + 1, ctas * nt - 1, ctas * nt + 1, 2 * ctas * nt + 77]
    worst = 0.0
    for B in sizes:
        idx = np.arange(B) % B0
        out = backward(eng, x[idx], c[idx], lg, counts, tr, _sub(eps, idx), gy[idx], gl[idx])
        assert torch.equal(out[0], base[0][idx]) and torch.equal(out[1], base[1][idx]), B
        # parameter gradients: q copies of the base block and its first r rows
        q, r = divmod(B, B0)
        part = backward(eng, x[:r], c[:r], lg, counts, tr, _sub(eps, np.arange(r)), gy[:r], gl[:r]) if r else None
        for i, (a, g) in enumerate(zip(out[2] + out[3], base[2] + base[3], strict=True)):
            want = q * as_np(g) + (as_np((part[2] + part[3])[i]) if r else 0.0)
            worst = max(worst, relmax(as_np(a), want))
    print(f"{name}-{trace}: ctas {ctas} x {nt} threads, tiled parameter gradients vs n x base: {worst:.2e} (bar {SUM_BAR:.0e})")
    assert worst <= SUM_BAR
    # rows at the first block, block and pass boundaries and the end of the largest batch, against the restatement
    B = sizes[-1]
    rows = np.unique(np.concatenate([np.arange(3), nt + np.arange(-1, 2), ctas * nt + np.arange(-2, 3),
                                     2 * ctas * nt + np.arange(-2, 3), B - np.arange(1, 4)]))  # fmt: skip
    idx = rows % B0
    field = _field(eng)
    check_against_restatement(eng, field, x[idx].astype(np.float64), c[idx], lg, tr, _sub(eps, idx), gy[idx], gl[idx],
                              (out[0][rows], out[1][rows], [], []), f"edge-tiled-{name}-{trace}-rows")  # fmt: skip
    if name == "d2_h16":  # the small field: the whole batch's parameter gradients too
        idx = np.arange(B) % B0
        check_against_restatement(eng, field, x[idx].astype(np.float64), c[idx], lg, tr, None, gy[idx], gl[idx], out,
                                  f"edge-tiled-{name}-{trace}-all")  # fmt: skip


CHUNK_SHAPE = (3, 2, 3, (48, 48))  # 128 threads without a trace, 64 with one


@pytest.mark.gpu
@pytest.mark.parametrize("trace", list(TRACES))
@pytest.mark.parametrize("ctx", ["rows", "broadcast"])
def test_chunks_with_padded_strides_give_the_one_chunk_bits(device, trace, ctx):
    tr = TRACES[trace]
    eng = make(device, *CHUNK_SHAPE)
    D, C = eng.D, eng.C
    h = eng.t._cnf_handle()
    lib = E.lib()
    _, nt, _, _ = bplan_call(h, 1, tr, 1)[1]
    B = 7 * nt + 5
    x, c, eps, gy, gl = _random_case(eng, B, seed=21, trace=tr)
    if ctx == "broadcast":
        c = c[0]
    _, _, counts, lg = eng.run(x, c, tr, eps=eps, ldc=0 if ctx == "broadcast" else None)
    T = on(device)
    lins = eng.t.ode._linears()

    def grads():
        return [torch.zeros_like(m.weight) for m in lins], [torch.zeros_like(m.bias) for m in lins]

    gW, gb = grads()
    one = (torch.full((B, D), NAN, device=device), torch.full(np.shape(c) if ctx == "broadcast" else (B, C), NAN, device=device), gW, gb)
    E.check(call(eng, B, lg, counts, tr, x=T(x), c=T(c), eps=T(eps), gy=T(gy), gl=T(gl), gx=one[0], gc=one[1], gW=gW, gb=gb))
    fixed = lib.zk_cnf_backward_workspace_bytes(h, 0, tr, counts[1])
    row = lib.zk_cnf_backward_workspace_bytes(h, 1, tr, counts[1]) - fixed
    _, xv = padded(x, device, pad=1)
    _, cv = padded(c, device, pad=2) if ctx == "rows" else (None, T(c))
    ev = None if eps is None else padded(eps, device, pad=3)[1]
    _, gyv = padded(gy, device, pad=4)
    for blocks in (1, 2, 3, 2.5):
        ws = fixed + int(blocks * nt) * row
        assert bplan_call(h, B, tr, counts[1], ws)[1][2] == int(blocks) * nt
        gxb, gxv = out_view((B, D), device, pad=2)
        gcb, gcv = out_view((B, C), device, pad=3) if ctx == "rows" else (None, torch.full((C,), NAN, device=device))
        gW, gb = grads()
        E.check(call(eng, B, lg, counts, tr, x=xv, c=cv, eps=ev, gy=gyv, gl=T(gl), gx=gxv, gc=gcv, gW=gW, gb=gb, ws_bytes=ws))
        assert_same((gxv, gcv, gW, gb), one, (trace, ctx, blocks))
        assert pads_untouched(gxb, 2, D) and (gcb is None or pads_untouched(gcb, 3, C))


# --------------------------------------------------------------------------- #
# C. MLP shapes
# --------------------------------------------------------------------------- #

# name -> (D, C, F, hidden, B)
SHAPES = {
    "sixteen_layers": (4, 2, 2, (16,) * 15, 32),
    "f0": (3, 2, 0, (32, 32), 32),
    "f32": (3, 2, 32, (32, 32), 32),
    "d1": (1, 2, 3, (16, 16), 32),
    "d64": (64, 0, 3, (64, 64), 6),
    "c0": (3, 0, 3, (32, 32), 32),
    "c130": (3, 130, 3, (32, 32), 24),
    "w64_w65": (16, 8, 3, (64, 65), 24),  # 32 threads with a trace
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("trace", list(TRACES))
def test_shapes_against_restatement(device, name, trace):
    D, C, F, hidden, B = SHAPES[name]
    tr = TRACES[trace]
    eng = make(device, D, C, F, hidden)
    if name == "w64_w65" and tr:
        assert bplan_call(eng.t._cnf_handle(), 1, tr, 1)[1][1] == 32
    field = _field(eng)
    # D = 64 with the exact trace: 64 tangents per stage, and the restatement's D autograd calls: one direction
    directions = (+1,) if name == "d64" and tr == R.TRACE_EXACT else (+1, -1)
    for direction in directions:
        x, c, eps, gy, gl = _random_case(eng, B, seed=len(name) + direction, trace=tr)
        forms = [c, c[0]] if name == "c130" else [c]  # per row and broadcast: two blocks of the context sum
        for cc in forms:
            _, _, counts, lg = eng.run(x, cc, tr, direction, eps, ldc=0 if cc is not None and cc.ndim == 1 else None)
            out = backward(eng, x, cc, lg, counts, tr, eps, gy, gl)
            check_against_restatement(eng, field, x.astype(np.float64), cc, lg, tr, eps, gy, gl, out,
                                      f"edge-{name}-{trace}-{direction}-{np.ndim(cc)}")  # fmt: skip


# --------------------------------------------------------------------------- #
# D. NULL outputs and grad_ladj
# --------------------------------------------------------------------------- #


@pytest.mark.gpu
@pytest.mark.parametrize("trace", ["exact", "hut"])
def test_null_outputs_leave_the_rest_unchanged(device, trace):
    tr = TRACES[trace]
    eng = make(device, 3, 2, 3, (24, 24))
    B = 70
    x, c, eps, gy, gl = _random_case(eng, B, seed=5, trace=tr)
    _, _, counts, lg = eng.run(x, c, tr, eps=eps)
    T = on(device)
    xt, ct, et, gyt, glt = map(T, (x, c, eps, gy, gl))
    lins = eng.t.ode._linears()

    def run(gx=True, gc=True, grads=True, gW=True, gb=True, skip=None, gy=gyt, gl=glt, trace=tr):
        ox = torch.full((B, 3), NAN, device=device) if gx else None
        oc = torch.full((B, 2), NAN, device=device) if gc else None
        W = [torch.full_like(m.weight, SENT) if i == skip else torch.zeros_like(m.weight) for i, m in enumerate(lins)]
        b = [torch.full_like(m.bias, SENT) if i == skip else torch.zeros_like(m.bias) for i, m in enumerate(lins)]
        pw = [None if i == skip else w for i, w in enumerate(W)] if gW else None
        pb = [None if i == skip else v for i, v in enumerate(b)] if gb else None
        E.check(call(eng, B, lg, counts, trace, x=xt, c=ct, eps=et if trace == R.TRACE_HUTCHINSON else None, gy=gy,
                     gl=gl, gx=ox, gc=oc, gW=pw, gb=pb, grads=grads))  # fmt: skip
        return ox, oc, W, b

    full = run()
    zero_W = [torch.zeros_like(m.weight) for m in lins]
    zero_b = [torch.zeros_like(m.bias) for m in lins]
    assert_same(run(gx=False), (None, *full[1:]), "grad_x NULL")
    assert_same(run(gc=False), (full[0], None, *full[2:]), "grad_c NULL")
    assert_same(run(grads=False), (*full[:2], zero_W, zero_b), "grads NULL")
    assert_same(run(gW=False), (*full[:2], zero_W, full[3]), "grad_weight NULL")
    assert_same(run(gb=False), (*full[:3], zero_b), "grad_bias NULL")
    for skip in range(len(lins)):
        gx, gc, W, b = run(skip=skip)
        assert torch.all(W[skip] == SENT) and torch.all(b[skip] == SENT), skip
        W[skip], b[skip] = full[2][skip], full[3][skip]
        assert_same((gx, gc, W, b), full, f"layer {skip} NULL")
    assert_same(run(gy=None), run(gy=torch.zeros_like(gyt)), "grad_y NULL")
    # grad_ladj = 0: the trace's terms vanish, leaving what grad_y contributes
    with_trace = run(gl=torch.zeros_like(glt))
    without = run(gl=None, trace=R.TRACE_NONE)
    for u, v in zip(flat(with_trace), flat(without), strict=True):
        assert relmax(as_np(u), as_np(v)) <= 1e-6


# --------------------------------------------------------------------------- #
# E. step logs and time intervals
# --------------------------------------------------------------------------- #


def with_rejections(lg):
    """lg with rejected rows (NaN t, dt and error) at the front, after the first accepted row, three in a row after
    the third, and at the end."""
    rej = np.array([[NAN, NAN, NAN, 0.0]])
    rows = [rej, rej]
    for i, r in enumerate(lg):
        rows.append(r[None])
        if i == 0:
            rows.append(rej)
        if i == 2:
            rows += [rej] * 3
    rows.append(rej)
    return np.concatenate(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("trace", ["exact", "hut"])
def test_rejected_rows_anywhere_in_the_log(device, trace):
    tr = TRACES[trace]
    eng = make(device, 3, 2, 3, (24, 24))
    x, c, eps, gy, gl = _random_case(eng, 50, seed=6, trace=tr)
    _, _, counts, lg = eng.run(x, c, tr, eps=eps)
    assert counts[1] >= 3
    ref = backward(eng, x, c, lg, counts, tr, eps, gy, gl)
    lg2 = with_rejections(lg)
    out = backward(eng, x, c, lg2, (len(lg2), counts[1]), tr, eps, gy, gl)
    assert_same(out, ref)


@pytest.mark.gpu
def test_only_rejected_trials_is_the_identity(device):
    eng = make(device, 3, 2, 3, (24, 24))
    x, c, eps, gy, gl = _random_case(eng, 40, seed=7)
    lg = np.tile([[NAN, NAN, NAN, 0.0]], (5, 1))
    for cc in (c, c[0]):
        gx, gc, gW, gb = backward(eng, x, cc, lg, (5, 0), R.TRACE_EXACT, None, gy, gl)
        assert torch.equal(gx, on(device)(gy))
        assert torch.all(gc == 0) and all(torch.all(g == 0) for g in gW + gb)


@pytest.mark.gpu
def test_long_log_against_restatement(device):
    """100+ accepted steps: the workspace holds one replayed state per accepted step."""
    eng = make(device, 3, 2, 3, (32, 32), scale=2.0)
    B = 24
    x, c, eps, gy, gl = _random_case(eng, B, seed=8)
    xt, ct = on(device)(x), on(device)(c)
    y = torch.empty(B, 3, device=device)
    ladj = torch.empty(B, device=device)
    cn = torch.zeros(2, dtype=torch.int32, device=device)
    log = torch.full((1000, 4), NAN, device=device)
    E.check(raw(eng, xt, B, c=ct, ldc=2, times=times_of(0.0, 4.0, device), y=y, ladj=ladj, counts=cn, log=log,
                atol=1e-7, rtol=1e-6))  # fmt: skip
    counts = tuple(cn.tolist())
    lg = log[: counts[0]].double().cpu().numpy()
    assert counts[1] >= 100 and counts[0] > counts[1], counts
    out = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl)
    check_against_restatement(eng, _field(eng), x.astype(np.float64), c, lg, R.TRACE_EXACT, None, gy, gl, out, "edge-long-log")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(INTERVALS))
def test_time_intervals_against_restatement(device, name):
    t0, t1, F = INTERVALS[name]
    eng = make(device, 3, 2, F, (32, 32))
    x, c, eps, gy, gl = _random_case(eng, 48, seed=9)
    _, _, counts, lg = eng.run(x, c, R.TRACE_EXACT, times=times_of(t0, t1, device))
    assert counts[1] >= 1
    out = backward(eng, x, c, lg, counts, R.TRACE_EXACT, None, gy, gl)
    check_against_restatement(eng, _field(eng), x.astype(np.float64), c, lg, R.TRACE_EXACT, None, gy, gl, out,
                              f"edge-interval-{name}")  # fmt: skip


# --------------------------------------------------------------------------- #
# F. the Python layer against direct C-ABI calls
# --------------------------------------------------------------------------- #


def training(device, D=3, C=2, seed=0):
    eng = make(device, D, C, 3, (24, 24), seed=seed)
    eng.t.adjoint = True
    eng.flow.train()
    return eng


def param_grads(eng):
    lins = eng.t.ode._linears()
    return [m.weight.grad for m in lins], [m.bias.grad for m in lins]


@pytest.mark.gpu
def test_empty_batch_gives_zero_gradients(device):
    eng = training(device)
    # in deterministic mode torch.empty fills floats with NaN: a gradient never written cannot read as 0 by chance
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        _empty_batch_gradients(eng, device)
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn_only)
        eng.t.exact = True


def _empty_batch_gradients(eng, device):
    for c in (torch.randn(2, device=device), torch.randn(1, 2, device=device), torch.randn(0, 2, device=device)):
        for exact in (True, False):
            eng.t.exact = exact
            eng.flow.zero_grad()
            c.grad = None
            cg = c.requires_grad_()
            x = torch.randn(0, 3, device=device, requires_grad=True)
            y, ladj = eng.t(cg).call_and_ladj(x)
            (y.sum() + ladj.sum()).backward()
            assert torch.equal(cg.grad, torch.zeros_like(cg)), (tuple(c.shape), exact, cg.grad)
            assert x.grad.shape == (0, 3)
            assert all(torch.equal(p.grad, torch.zeros_like(p)) for p in eng.flow.parameters())
            assert eng.t(cg).inv(x).shape == (0, 3)


def abi_grads(eng, x, c, gy, gl, trace=R.TRACE_EXACT, eps=None, direction=+1):
    """The forward by zk_cnf_integrate (it reproduces the Python layer's step log), then zk_cnf_backward."""
    _, _, counts, lg = eng.run(x, c, trace, direction, eps)
    return backward(eng, x, c, lg, counts, trace, eps, gy, gl)


@pytest.mark.gpu
def test_frozen_layer_and_x_without_grad(device):
    eng = training(device)
    x, c, _, gy, gl = _random_case(eng, 40, seed=10)
    ref = abi_grads(eng, x, c, gy, gl)
    T = on(device)
    lins = eng.t.ode._linears()

    def py(x_grad):
        eng.flow.zero_grad()
        xt, ct = T(x).requires_grad_(x_grad), T(c).requires_grad_()
        y, ladj = eng.t(ct).call_and_ladj(xt)
        ((y * T(gy)).sum() + (ladj * T(gl)).sum()).backward()
        return xt.grad, ct.grad, *param_grads(eng)

    assert_same(py(True), ref)
    gx, gc, gW, gb = py(False)
    assert gx is None
    assert_same((None, gc, gW, gb), (None, *ref[1:]))
    lins[0].weight.requires_grad_(False)
    try:
        gx, gc, gW, gb = py(True)
    finally:
        lins[0].weight.requires_grad_(True)
    assert gW[0] is None
    gW[0] = ref[2][0]
    assert_same((gx, gc, gW, gb), ref)


@pytest.mark.gpu
def test_leading_dimensions_and_context_shapes(device):
    eng = training(device)
    g = torch.Generator().manual_seed(12)
    x, gy, gl = torch.randn(4, 5, 3, generator=g), torch.randn(4, 5, 3, generator=g), torch.randn(4, 5, generator=g)
    rows = torch.randn(4, 5, 2, generator=g)
    x2, gy2, gl2 = x.reshape(20, 3).numpy(), gy.reshape(20, 3).numpy(), gl.reshape(20).numpy()
    field = _field(eng)
    for c in (rows[0], rows[:, :1], rows[0, :1], rows[0, 0]):  # (5, C), (4, 1, C), (1, C), (C,)
        cr = c.expand(4, 5, 2).reshape(20, 2).numpy()
        _, _, counts, lg = eng.run(x2, cr)
        ref = backward(eng, x2, cr, lg, counts, R.TRACE_EXACT, None, gy2, gl2)
        eng.flow.zero_grad()
        xt, ct = x.to(device).requires_grad_(), c.to(device).requires_grad_()
        y, ladj = eng.t(ct).call_and_ladj(xt)
        ((y * gy.to(device)).sum() + (ladj * gl.to(device)).sum()).backward()
        assert xt.grad.shape == x.shape and ct.grad.shape == c.shape
        assert_same((xt.grad.reshape(20, 3), None, *param_grads(eng)), (ref[0], None, *ref[2:]), tuple(c.shape))
        summed = ref[1].reshape(4, 5, 2).sum_to_size(c.shape)
        if c.dim() == 1 or c.shape[0] == 1:  # one broadcast row: the engine sums the rows, in row order
            bc = backward(eng, x2, c.reshape(2).numpy(), lg, counts, R.TRACE_EXACT, None, gy2, gl2)
            assert torch.equal(ct.grad.reshape(2), bc[1])
            assert relmax(as_np(ct.grad), as_np(summed)) <= 1e-6
        else:  # the Python layer sums the per-row gradient to c's shape
            assert torch.equal(ct.grad, summed)
        rc = A.adjoint(field, x2.astype(np.float64), cr, lg, R.TRACE_EXACT, None, gy2, gl2)["c"]
        err = relmax(as_np(ct.grad), torch.as_tensor(rc).reshape(4, 5, 2).sum_to_size(c.shape).numpy())
        WORST[f"edge-python-c{tuple(c.shape)}"] = err
        assert err <= BAR, (tuple(c.shape), err)


@pytest.mark.gpu
def test_loss_on_y_only_or_ladj_only(device):
    eng = training(device)
    x, c, _, gy, gl = _random_case(eng, 40, seed=13)
    T = on(device)
    for use_y, use_l in ((True, False), (False, True)):
        ref = abi_grads(eng, x, c, gy if use_y else None, gl if use_l else np.zeros_like(gl))
        eng.flow.zero_grad()
        xt, ct = T(x).requires_grad_(), T(c).requires_grad_()
        y, ladj = eng.t(ct).call_and_ladj(xt)
        ((y * T(gy)).sum() if use_y else (ladj * T(gl)).sum()).backward()
        assert_same((xt.grad, ct.grad, *param_grads(eng)), ref, (use_y, use_l))


@pytest.mark.gpu
def test_hutchinson_training_redraws_eps(device):
    eng = training(device)
    eng.t.exact = False
    x, c, _, gy, gl = _random_case(eng, 40, seed=14)
    T = on(device)
    xt, ct = T(x).requires_grad_(), T(c).requires_grad_()
    torch.manual_seed(1234)
    y, ladj = eng.t(ct).call_and_ladj(xt)
    ((y * T(gy)).sum() + (ladj * T(gl)).sum()).backward()
    torch.manual_seed(1234)
    eps = torch.randn_like(xt.detach())
    ref = abi_grads(eng, x, c, gy, gl, trace=R.TRACE_HUTCHINSON, eps=eps)
    assert_same((xt.grad, ct.grad, *param_grads(eng)), ref)
    eng.t.exact = True


@pytest.mark.gpu
def test_inverse_and_rsample_gradients(device):
    eng = training(device)
    z, c, _, gy, gl = _random_case(eng, 40, seed=15)
    T = on(device)
    # .inv integrates from t1 to t0; its call_and_ladj carries the trace
    for with_ladj in (False, True):
        eng.flow.zero_grad()
        zt, ct = T(z).requires_grad_(), T(c).requires_grad_()
        inv = eng.t(ct).inv
        if with_ladj:
            y, ladj = inv.call_and_ladj(zt)
            ((y * T(gy)).sum() + (ladj * T(gl)).sum()).backward()
            ref = abi_grads(eng, z, c, gy, gl, direction=-1)
        else:
            (inv(zt) * T(gy)).sum().backward()
            ref = abi_grads(eng, z, c, gy, None, trace=R.TRACE_NONE, direction=-1)
        assert_same((zt.grad, ct.grad, *param_grads(eng)), ref, with_ladj)
    # rsample: the base draw, then .inv
    eng.flow.zero_grad()
    ct = T(c).requires_grad_()
    dist = eng.flow(ct)
    torch.manual_seed(99)
    (dist.rsample() * T(gy)).sum().backward()
    torch.manual_seed(99)
    z0 = dist.base.rsample().detach().cpu().numpy()
    ref = abi_grads(eng, z0, c, gy, None, trace=R.TRACE_NONE, direction=-1)
    assert_same((None, ct.grad, *param_grads(eng)), (None, *ref[1:]))


def test_report_worst():
    """Prints the worst gradient error of this file against the restatement."""
    errs = {k: v for k, v in WORST.items() if k.startswith("edge-")}  # the dict is shared with test_gpu_cnf_grad.py
    if errs:
        k = max(errs, key=errs.get)
        print(f"worst gradient error vs the fp64 restatement: {errs[k]:.2e} ({k}) over {len(errs)} checks")
