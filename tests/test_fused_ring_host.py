"""CPU tests of the weight-ring protocol of the fused layer kernel (zuko_b200/csrc/fused_layer.cu): g++ compiles
tests/native/fused_ring_host.cpp, a replay of the kernel's producer and consumer tile sequences for 64- and 128-row
tiles under random interleavings with mbarrier parity semantics.  A protocol error would hang the kernel, so every
ring depth, hidden width and output-layer chunk count the launcher can pick is replayed here first."""

import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
MAX_LINEAR = 6


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libfused_ring_host.so"
    src = ROOT / "tests" / "native" / "fused_ring_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so)], check=True)
    return ctypes.CDLL(str(so))


def replay(harness, kbmask, KB0, nch, n_last, rows, n_stages, n_tiles=3, seeds=range(4)):
    kb = np.zeros((MAX_LINEAR, 128), np.uint8)
    kb[: kbmask.shape[0], : kbmask.shape[1]] = kbmask
    msg = ctypes.create_string_buffer(256)
    for seed in seeds:
        rc = harness.ring_replay(kb.ctypes.data_as(ctypes.c_void_p), kbmask.shape[0], KB0, nch, n_last, rows, n_stages,
                                 n_tiles, seed, msg, 256)  # fmt: skip
        if rc:
            return rc, msg.value.decode()
    return 0, ""


def random_masks(rng, L, KB0, nch, n_last):
    """[L][128] table of non-zero K blocks: hidden layers over nch chunks, the output layer over n_last (some empty)."""
    kb = np.zeros((L, 128), np.uint8)
    for layer in range(L - 1):
        width = KB0 if layer == 0 else nch
        kb[layer, :nch] = rng.integers(0, 1 << width, nch)
    kb[L - 1, :n_last] = rng.integers(0, 1 << nch, n_last)
    return kb


def flagship_masks():
    """The zero-tile table of NSF(16, 8, transforms=4, bins=8, hidden_features=[256] * 3), computed with the
    degree sort and zero-tile rule of fused_layer_prepare."""
    import torch

    import zuko_b200 as zuko
    from zuko_b200.nn import MaskedLinear

    torch.manual_seed(0)
    flow = zuko.flows.NSF(16, 8, transforms=4, bins=8, hidden_features=[256] * 3)
    masks = [m.mask.numpy().astype(bool) for m in flow.transform.transforms[0].hyper.modules() if isinstance(m, MaskedLinear)]
    D, P, DPC = 16, 23, 2
    L = len(masks)
    perms, dep = [], None
    for layer in range(L - 1):
        m = masks[layer]
        dep = m.copy() if layer == 0 else (m.astype(np.int64) @ dep.astype(np.int64)) > 0  # inputs each unit can see
        perms.append(np.argsort(dep.sum(1), kind="stable"))
    n_last = (D + DPC - 1) // DPC
    kb = np.zeros((L, 128), np.uint8)
    for layer in range(L):
        m = masks[layer]
        if layer > 0:
            m = m[:, perms[layer - 1]]
        if layer < L - 1:
            rows = [perms[layer][ch * 64 : ch * 64 + 64] for ch in range(m.shape[0] // 64)]
        else:
            rows = [[d * P + j % P for j in range(DPC * P) if (d := ch * DPC + j // P) < D] for ch in range(n_last)]
        for ch, r in enumerate(rows):
            cols = np.flatnonzero(m[r].any(0))
            kb[layer, ch] = np.bitwise_or.reduce(1 << (cols // 64)) if cols.size else 0
    return kb, n_last


def test_flagship_table_has_44_tiles():
    kb, n_last = flagship_masks()
    assert kb.shape[0] == 4 and n_last == 8
    assert sum(bin(v).count("1") for v in kb.ravel()) == 44


@pytest.mark.parametrize("rows,n_stages", [(128, s) for s in range(4, 9)] + [(64, s) for s in (4, 6, 8)])
def test_flagship_ring(harness, rows, n_stages):
    kb, n_last = flagship_masks()
    assert replay(harness, kb, KB0=1, nch=4, n_last=n_last, rows=rows, n_stages=n_stages) == (0, "")


@pytest.mark.parametrize("n_stages", range(3, 9))
@pytest.mark.parametrize("nch", [1, 2, 3, 4])
def test_wide_ring_random_masks(harness, n_stages, nch):
    if nch > n_stages:
        pytest.skip("an output chunk holds up to nch slots: the launcher never pairs such a ring with 128-row tiles")
    rng = np.random.default_rng(100 * n_stages + nch)
    for n_last in (1, 2, 3, 7, 128):
        for L in (2, 4):
            KB0 = int(rng.integers(1, 5))
            kb = random_masks(rng, L, KB0, nch, n_last)
            assert replay(harness, kb, KB0, nch, n_last, 128, n_stages, seeds=range(2)) == (0, ""), (n_last, L)


@pytest.mark.parametrize("n_stages", [4, 6, 8])
@pytest.mark.parametrize("nch", [1, 2, 3, 4, 6, 8])
def test_narrow_ring_random_masks(harness, n_stages, nch):
    rng = np.random.default_rng(100 * n_stages + nch)
    for n_last in (1, 2, 5, 128):
        KB0 = int(rng.integers(1, 9))
        kb = random_masks(rng, 3, KB0, nch, n_last)
        assert replay(harness, kb, KB0, nch, n_last, 64, n_stages, seeds=range(2)) == (0, ""), n_last


def test_wide_ring_shallower_than_a_chunk_deadlocks(harness):
    """An output chunk's slots stay held until its MMAs are done: a ring with fewer slots than a chunk has tiles
    cannot make progress, which is why 128-row tiles need n_stages >= 4 >= nch.  The replay must see it."""
    kb = np.zeros((2, 128), np.uint8)
    kb[0, :4] = 1
    kb[1, :2] = 0b1111
    rc, msg = replay(harness, kb, KB0=1, nch=4, n_last=2, rows=128, n_stages=3, seeds=[0])
    assert rc == 1 and "deadlock" in msg
