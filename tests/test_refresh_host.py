"""CPU tests of the decisions in front of the in-place weight refresh: which change of a layer's tensors refreshes
its handle (zk_layer_update_weights), which one builds a new handle and which one hits the cache
(PackedLayerMixin._zk_layer_ref / _weights_only_change), and the same for the GMM handle key (GMM.handle).  The
layer signatures are built by hand, one field changed at a time; the GMM handle runs against a recording stand-in
for the library.  Also replays the edits of the GPU refresh sequences (tests/test_gpu_refresh_edges.py) on CPU copies
of its cases: which rows they reach and which branch they take."""

from __future__ import annotations

import contextlib

import pytest
import torch

import test_gpu_refresh_edges as G
import zuko_b200 as zuko
from zuko_b200 import _engine as E
from zuko_b200.flows import GeneralCouplingTransform, MaskedAutoregressiveTransform

CUDA0, CUDA1 = torch.device("cuda", 0), torch.device("cuda", 1)
F32 = torch.float32


def ar_layer(bias=True):
    torch.manual_seed(0)
    t = MaskedAutoregressiveTransform(4, 2, hidden_features=[16, 16])
    if not bias:
        for m in t.hyper._linears():
            m.bias = None
    return t


def coupling_layer():
    torch.manual_seed(0)
    return GeneralCouplingTransform(5, 2, hidden_features=[16])


def signature(t, **change):
    """A hand-built signature of `t` in the layout of _layer_signature: gemm mode, activation code, then
    (ptr, version, device, dtype) of weight / bias / mask per linear layer, phi, the order and (coupling) the mask.
    `change` names one field: ("weight", i), ("bias", i), ("mask", i), "order", "coupling_mask", "gemm_mode",
    "activation", ("ptr", i) or "device"."""
    ptr = iter(range(0x1000, 0x100000, 0x100))
    dev = change.get("device", CUDA0)

    def ent(tensor, bump=0, new_ptr=False):
        if tensor is None:
            return None
        p = next(ptr)
        return (p + (0x80 if new_ptr else 0), 3 + bump, dev, F32)

    sig = [change.get("gemm_mode", "auto"), change.get("activation", E.ZK_ACT_RELU)]
    for i, m in enumerate(t.hyper._linears()):
        sig.append(ent(m.weight, change.get("weight") == i, change.get("ptr") == i))
        sig.append(ent(m.bias, change.get("bias") == i))
        sig.append(ent(getattr(m, "mask", None), change.get("mask") == i))
    if torch.is_tensor(getattr(t, "order", None)):
        sig.append(ent(t.order, "order" in change))
    if isinstance(t, GeneralCouplingTransform):
        sig.append(ent(t.mask, "coupling_mask" in change))
    return tuple(sig)


def decide(t, old, new) -> str:
    """_zk_layer_ref's branch for a handle on a CUDA device: the cache, an in-place refresh, or a new handle."""
    if old == new:
        return "cache"
    return "refresh" if t._weights_only_change(old, new) else "rebuild"


# (row, layer, change, expected)
LAYER_ROWS = [
    ("unchanged", "ar", {}, "cache"),
    ("weight_version", "ar", {"weight": 0}, "refresh"),
    ("last_weight_version", "ar", {"weight": 2}, "refresh"),
    ("bias_version", "ar", {"bias": 1}, "refresh"),
    ("no_bias_weight_version", "ar_nobias", {"weight": 1}, "refresh"),
    ("mask_version", "ar", {"mask": 0}, "rebuild"),
    ("last_mask_version", "ar", {"mask": 2}, "rebuild"),
    ("order", "ar", {"order": True}, "rebuild"),
    ("coupling_weight_version", "coupling", {"weight": 0}, "refresh"),
    ("coupling_mask", "coupling", {"coupling_mask": True}, "rebuild"),
    ("gemm_mode", "ar", {"gemm_mode": "fp32"}, "rebuild"),
    ("activation", "ar", {"activation": E.ZK_ACT_ELU}, "rebuild"),
    ("data_ptr", "ar", {"ptr": 0}, "rebuild"),
    ("device", "ar", {"device": CUDA1}, "rebuild"),
]
LAYERS = {"ar": ar_layer, "ar_nobias": lambda: ar_layer(bias=False), "coupling": coupling_layer}


@pytest.mark.parametrize("row,layer,change,want", LAYER_ROWS, ids=[r[0] for r in LAYER_ROWS])
def test_layer_decision_table(row, layer, change, want):
    t = LAYERS[layer]()
    assert decide(t, signature(t), signature(t, **change)) == want


def test_signature_layout_matches_the_module():
    """The hand-built signatures have the layout _layer_signature produces, field by field."""
    for make in LAYERS.values():
        t = make()
        real = t._layer_signature()
        hand = signature(t)
        assert len(real) == len(hand)
        for a, b in zip(real, hand):
            assert (a is None) == (b is None) and (type(a) is tuple) == (type(b) is tuple)


def test_module_edits_take_the_expected_branch():
    """The same rows from real in-place edits of a CPU module (versions move, pointers stay)."""
    t = ar_layer()
    lin = t.hyper._linears()
    s0 = t._layer_signature()
    with torch.no_grad():
        lin[0].weight.add_(1.0)
    s1 = t._layer_signature()
    assert decide(t, s0, s1) == "refresh"
    with torch.no_grad():
        lin[1].bias.mul_(2.0)
    s2 = t._layer_signature()
    assert decide(t, s1, s2) == "refresh"
    with torch.no_grad():
        lin[0].mask.logical_not_().logical_not_()
    assert decide(t, s2, t._layer_signature()) == "rebuild"
    s3 = t._layer_signature()
    t.order.add_(0)
    assert decide(t, s3, t._layer_signature()) == "rebuild"
    s4 = t._layer_signature()
    t.hyper.gemm_mode = "fp32"
    assert decide(t, s4, t._layer_signature()) == "rebuild"
    s5 = t._layer_signature()
    t.load_state_dict(ar_layer().state_dict())  # copies the mask and order buffers in place as well
    assert decide(t, s5, t._layer_signature()) == "rebuild"


class RecordingLib:
    """Stands in for the library in GMM.handle: records create / update / destroy."""

    def __init__(self):
        self.calls = []
        self.next = 100

    def zk_gmm_create(self, desc, out):
        self.next += 1
        out._obj.value = self.next
        self.calls.append("create")
        return E.ZK_OK

    def zk_gmm_update_weights(self, h, W, Bv, stream):
        self.calls.append("refresh")
        return E.ZK_OK

    def zk_gmm_destroy(self, h):
        self.calls.append("destroy")
        return E.ZK_OK

    def zk_set_pack_stream(self, s):
        pass


@pytest.fixture
def gmm_handle(monkeypatch):
    gmm = zuko.mixtures.GMM(3, 5, components=4, hidden_features=[16, 16])
    rec = RecordingLib()
    monkeypatch.setattr(E, "lib", lambda: rec)
    monkeypatch.setattr(E, "stream_ptr", lambda device: None)
    monkeypatch.setattr(E, "require_cuda", lambda t, what: None)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())

    def decide_gmm(edit):
        gmm.handle(gmm.params())
        n = len(rec.calls)
        edit(gmm)
        h = gmm.handle(gmm.params())
        new = rec.calls[n:]
        gmm.__dict__.pop("_zk_cache", None)
        return "cache" if not new else ("refresh" if new == ["refresh"] else ("rebuild" if "create" in new else new)), h

    return decide_gmm


def _weight_version(g):
    with torch.no_grad():
        g.hyper[0].weight.add_(1.0)


def _bias_version(g):
    with torch.no_grad():
        g.hyper[-1].bias.mul_(2.0)


def _data_ptr(g):
    g.hyper[0].weight = torch.nn.Parameter(g.hyper[0].weight.detach().clone())


def _gemm_mode(g):
    g.hyper.gemm_mode = "fp32" if g.hyper.gemm_mode != "fp32" else "bf16x3"


def _activation(g):
    for i, m in enumerate(g.hyper):
        if isinstance(m, torch.nn.ReLU):
            g.hyper[i] = torch.nn.ELU()


def _device(g):
    real = g._structure
    g._structure = lambda params: (*real(params)[:-1], ("moved",))


GMM_ROWS = [
    ("unchanged", lambda g: None, "cache"),
    ("weight_version", _weight_version, "refresh"),
    ("bias_version", _bias_version, "refresh"),
    ("data_ptr", _data_ptr, "refresh"),  # a new tensor of the same structure (a posterior draw) is copied in
    ("gemm_mode", _gemm_mode, "rebuild"),
    ("activation", _activation, "rebuild"),
    ("device", _device, "rebuild"),
]


@pytest.mark.parametrize("row,edit,want", GMM_ROWS, ids=[r[0] for r in GMM_ROWS])
def test_gmm_handle_decision_table(gmm_handle, row, edit, want):
    got, _ = gmm_handle(edit)
    assert got == want


def labels(t) -> list[str]:
    """Row name of every field of t._layer_signature(), in its order."""
    out = ["gemm_mode", "activation"]
    for _ in t.hyper._linears():
        out += ["weight_version", "bias_version", "mask_version"]
    out += ["phi"] * len(getattr(t, "phi", []) or [])
    if torch.is_tensor(getattr(t, "order", None)):
        out.append("order")
    if isinstance(t, GeneralCouplingTransform):
        out.append("coupling_mask")
    return out


def apply_sequence(case, seq, flow):
    """The parameter and buffer edits of a GPU sequence (test_gpu_refresh_edges.run_sequence), on a CPU module."""
    if seq == "c_twice":
        G.step(flow, seed=1)
        G.step(flow, seed=2)
    elif seq == "d_biases_adam":
        G.adam_biases(flow)
    elif seq == "e_weights_only":
        G.step(flow, "weights")
    elif seq == "f_masked_entries":
        G.mask_noise(flow)
    elif seq == "i_load_state_dict":
        flow.load_state_dict(G.other_checkpoint(case, flow))
    else:
        G.step(flow)


def test_gpu_sequences_reach_the_parameter_and_buffer_rows():
    """The edits each GPU sequence makes, replayed on CPU copies of its case: the signature fields they move (the rows
    of the decision table they reach), and the branch _zk_layer_ref then takes, which must be the one the GPU test
    asserts from generation and OwnedLayer identity (rebuild after load_state_dict of a layer holding mask or order
    buffers, refresh otherwise).  The structural rows (gemm mode, activation, data_ptr, device) and the no-bias row
    are reached by the CPU decision table above only: no refresh sequence changes them."""
    reached = set()
    for name, seq in G.FLOW_MATRIX:
        case = G.CASES[name]
        flow = case.build()
        layers = G.conditioned(flow)
        before = [t._layer_signature() for t in layers]
        apply_sequence(case, seq, flow)
        for t, old in zip(layers, before, strict=True):
            new = t._layer_signature()
            moved = {lab for lab, a, b in zip(labels(t), old, new, strict=True) if a != b}
            assert moved, (name, seq)
            want = "rebuild" if seq == "i_load_state_dict" and G.rebuilds_on_load(t) else "refresh"
            assert decide(t, old, new) == want, (name, seq, sorted(moved))
            reached |= moved
    # (j): MAF(randperm=True) checkpoints of another seed move the order and the masks
    torch.manual_seed(7)
    flow = G._maf_randperm()
    torch.manual_seed(8)
    other = G._maf_randperm()
    old = [t._layer_signature() for t in G.conditioned(flow)]
    flow.load_state_dict(other.state_dict())
    for t, o in zip(G.conditioned(flow), old, strict=True):
        assert decide(t, o, t._layer_signature()) == "rebuild"
        reached |= {lab for lab, a, b in zip(labels(t), o, t._layer_signature(), strict=True) if a != b}
    assert {"weight_version", "bias_version", "mask_version", "order", "coupling_mask"} <= reached, sorted(reached)
    # every tile plan, the sequential inverse and the sweeps, every conditioned member kind, both GMM sources and modes
    cases = G.CASES.values()
    assert {c.rows for c in cases} == {0, 64, 128}
    assert {c.seq_inverse for c in cases if c.kind == "ar"} == {0, 1}
    assert {c.kind for c in cases} == {"ar", "coupling", "elementwise"}
    assert {c.mode for c in cases} == {"fp32", "bf16x3", "bf16x1"}
    assert any(c.folded for c in cases)
    assert {v for v in G.GMM.values()} == {(s, m) for s in ("full_untied", "bcast") for m in ("fp32", "bf16x3")}
    for s in G.SEQUENCES:
        assert any(seq == s for _, seq in G.FLOW_MATRIX), s
