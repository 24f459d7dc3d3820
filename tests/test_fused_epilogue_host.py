"""CPU tests of the fused layer kernel's output chunks (zuko_b200/csrc/fused_layer.cu): g++ compiles
tests/native/fused_out_chunk_host.cpp against zuko_b200/csrc/fused_out_chunk.cuh, the column order the pack gives an
output chunk and the register exchange through which each consumer thread gathers the parameters it evaluates from
the wgmma accumulators.  For RQS with 8 and 16 bins and affine layers, with full and partial last chunks, every thread
must end up with the staging-order parameters of its (row, slot), no pad column or absent dim may be read, every
(row, dim) must be evaluated exactly once, and the pack must keep each chunk's rows inside the chunk."""

import ctypes
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

SHAPES = {"rqs8": (23, 2), "rqs16": (47, 1), "affine": (2, 32)}
DIMS = {
    "rqs8": [1, 2, 5, 16, 17, 64, 255],
    "rqs16": [1, 3, 16, 64],
    "affine": [1, 16, 31, 32, 40, 70, 128],
}


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = tmp_path_factory.mktemp("native") / "libfused_out_chunk_host.so"
    src = ROOT / "tests" / "native" / "fused_out_chunk_host.cpp"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so)], check=True)
    return ctypes.CDLL(str(so))


@pytest.mark.parametrize("kind,D", [(k, d) for k, ds in DIMS.items() for d in ds])
def test_out_chunk_exchange(harness, kind, D):
    P, DPC = SHAPES[kind]
    msg = ctypes.create_string_buffer(256)
    rc = harness.out_chunk_check(P, DPC, D, msg, 256)
    assert rc == 0, msg.value.decode()

