"""CPU tests of the weight-ring protocol of the fused layer kernel on 128-row tiles with the output layer's chunks
multiplied in pairs (zuko_b200/csrc/fused_layer.cu): g++ compiles tests/native/fused_pair_ring_host.cpp, a replay of the
kernel's producer and consumer tile sequences under random interleavings with mbarrier parity semantics.  A pair's
tiles are one stream of asynchronous MMAs that releases each slot one tile late, so a consumer holds at most two slots
and a pair of 4 + 4 tiles runs on the four-slot ring of the flagship shape."""

import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest

from test_fused_ring_host import MAX_LINEAR, flagship_masks, random_masks

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libfused_pair_ring_host.so"
    src = ROOT / "tests" / "native" / "fused_pair_ring_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so)], check=True)
    return ctypes.CDLL(str(so))


def replay(harness, kbmask, KB0, nch, n_last, n_stages, n_tiles=3, seeds=range(4)):
    """(return code, message, most slots one consumer held) of the first failing seed, or of the last one."""
    kb = np.zeros((MAX_LINEAR, 128), np.uint8)
    kb[: kbmask.shape[0], : kbmask.shape[1]] = kbmask
    msg = ctypes.create_string_buffer(256)
    held = ctypes.c_int(-1)
    for seed in seeds:
        rc = harness.pair_ring_replay(kb.ctypes.data_as(ctypes.c_void_p), kbmask.shape[0], KB0, nch, n_last, n_stages,
                                      n_tiles, seed, msg, 256, ctypes.byref(held))  # fmt: skip
        if rc:
            return rc, msg.value.decode(), None
    return 0, "", held.value


@pytest.mark.parametrize("n_stages", range(4, 9))
def test_flagship_ring(harness, n_stages):
    kb, n_last = flagship_masks()
    assert replay(harness, kb, KB0=1, nch=4, n_last=n_last, n_stages=n_stages) == (0, "", 2)


def full_pairs(L, n_last, nch=4):
    """Output chunks of nch tiles each: pairs of nch + nch tiles, and (n_last odd) a last pair of nch + 0."""
    kb = np.zeros((L, 128), np.uint8)
    kb[: L - 1, :nch] = 1
    kb[L - 1, :n_last] = (1 << nch) - 1
    return kb


@pytest.mark.parametrize("n_stages", range(4, 9))
@pytest.mark.parametrize("n_last", [1, 2, 3, 8, 9])
def test_four_plus_four_pairs(harness, n_stages, n_last):
    """4 + 4 tiles per pair: more than a four-slot ring holds, so slots roll over inside a pair and across pair
    boundaries; an odd n_last leaves a last pair with an empty chunk B."""
    kb = full_pairs(3, n_last)
    assert replay(harness, kb, KB0=1, nch=4, n_last=n_last, n_stages=n_stages) == (0, "", 2)


@pytest.mark.parametrize("n_stages", range(4, 9))
def test_one_and_four_tile_neighbours(harness, n_stages):
    """Adjacent chunks of 1 and 4 non-zero tiles in both orders, and all-zero chunks, with an odd n_last."""
    kb = np.zeros((3, 128), np.uint8)
    kb[:2, :4] = 0b1111
    last = [0b0001, 0b1111, 0b1111, 0b1000, 0b0000, 0b1111, 0b0100, 0b0000, 0b0010]
    kb[2, : len(last)] = last
    assert replay(harness, kb, KB0=4, nch=4, n_last=len(last), n_stages=n_stages)[:2] == (0, "")


@pytest.mark.parametrize("n_stages", range(4, 9))
@pytest.mark.parametrize("nch", [1, 2, 3, 4])
def test_random_masks(harness, n_stages, nch):
    rng = np.random.default_rng(1000 + 100 * n_stages + nch)
    for n_last in (1, 2, 3, 7, 128):
        for L in (2, 4):
            KB0 = int(rng.integers(1, 5))
            kb = random_masks(rng, L, KB0, nch, n_last)
            assert replay(harness, kb, KB0, nch, n_last, n_stages, seeds=range(2))[:2] == (0, ""), (n_last, L)


def test_a_pair_never_holds_more_than_two_slots(harness):
    """The one-tile-late release bounds what a consumer holds at two slots, whatever a chunk's tile count: even a
    two-slot ring, which the launcher never picks, runs 4 + 4 pairs.  (Waiting for a whole chunk's batch before its
    release needed as many slots as the chunk has tiles.)"""
    kb = full_pairs(2, 5)
    assert replay(harness, kb, KB0=1, nch=4, n_last=5, n_stages=2) == (0, "", 2)
