"""ctypes binding of ``libzuko_b200.so`` (C ABI in ``include/zuko_b200.h``).

PyTorch is used for device memory, streams and ``torch.distributed`` only: every
compute call goes through the C ABI with raw device pointers and the current CUDA
stream.  There is no CPU or eager fallback — if the library is missing or there is
no CUDA device the calls raise.
"""

from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint8, c_void_p
from pathlib import Path

import torch

__all__ = ["lib", "EngineError", "check", "stream_ptr", "Workspace", "LIB_PATH"]

LIB_PATH = Path(__file__).resolve().parent / "lib" / "libzuko_b200.so"

# status codes (include/zuko_b200.h)
ZK_OK, ZK_EINVAL, ZK_EUNSUPPORTED, ZK_ECUDA, ZK_ENOMEM = range(5)
ZK_UNI_AFFINE, ZK_UNI_RQS, ZK_UNI_CRQS, ZK_UNI_GAUSS, ZK_UNI_SOSP, ZK_UNI_BERNSTEIN = 1, 2, 3, 4, 5, 6
ZK_BASE_DIAG_NORMAL, ZK_BASE_BOX_UNIFORM = 0, 1
(
    ZK_LAYER_AUTOREGRESSIVE,
    ZK_LAYER_COUPLING,
    ZK_LAYER_ELEMENTWISE,
    ZK_LAYER_SOFTCLIP,
    ZK_LAYER_PERMUTATION,
    ZK_LAYER_ROTATION,
) = range(1, 7)
ZK_GEMM_AUTO, ZK_GEMM_FP32, ZK_GEMM_BF16X3, ZK_GEMM_BF16X1 = range(4)
(ZK_ACT_RELU, ZK_ACT_ELU, ZK_ACT_TANH, ZK_ACT_SILU, ZK_ACT_GELU, ZK_ACT_LEAKY_RELU, ZK_ACT_SOFTPLUS,
 ZK_ACT_SIGMOID) = (0, 2, 3, 4, 5, 6, 7, 8)  # fmt: skip
ZK_CNF_TRACE_NONE, ZK_CNF_TRACE_EXACT, ZK_CNF_TRACE_HUTCHINSON = range(3)
GEMM_MODES = {"auto": ZK_GEMM_AUTO, "fp32": ZK_GEMM_FP32, "bf16x3": ZK_GEMM_BF16X3, "bf16x1": ZK_GEMM_BF16X1}


class EngineError(RuntimeError):
    """Raised when a C-ABI call returns a non-zero ``zk_status``."""


class MlpDesc(ctypes.Structure):
    _fields_ = [
        ("n_linear", c_int),
        ("dims", POINTER(c_int)),
        ("weight", POINTER(c_void_p)),
        ("bias", POINTER(c_void_p)),
        ("mask", POINTER(c_void_p)),
        ("gemm_mode", c_int),
        ("activation", c_int),
        ("layer_act", POINTER(c_int)),
        ("layer_res", POINTER(c_int)),
    ]


class LayerDesc(ctypes.Structure):
    _fields_ = [
        ("kind", c_int),
        ("features", c_int),
        ("context", c_int),
        ("univariate", c_int),
        ("bins", c_int),
        ("bound", c_float),
        ("slope", c_float),
        ("passes", c_int),
        ("order", POINTER(c_int64)),
        ("coupling_mask", POINTER(c_uint8)),
        ("hyper", POINTER(MlpDesc)),
        ("phi", c_void_p),
        ("rotation", c_void_p),
        ("iterations", c_int),
        ("degree", c_int),
    ]


class LayerGrads(ctypes.Structure):
    """``zk_layer_grads``: where one layer's parameter gradients are accumulated."""

    _fields_ = [
        ("grad_weight", POINTER(c_void_p)),
        ("grad_bias", POINTER(c_void_p)),
        ("grad_phi", c_void_p),
        ("grad_rotation", c_void_p),
    ]


class FlowDesc(ctypes.Structure):
    _fields_ = [
        ("n_layers", c_int),
        ("layers", POINTER(c_void_p)),
        ("features", c_int),
        ("context", c_int),
        ("base_loc", c_void_p),
        ("base_scale", c_void_p),
        ("base_kind", c_int),
        ("inverted", POINTER(c_int)),
    ]


_P = c_void_p
_SIGNATURES = {
    # name: (restype, argtypes)
    "zk_version": (c_int, []),
    "zk_last_error": (c_char_p, []),
    "zk_launch_count": (c_int64, []),
    "zk_set_fast_math": (c_int, [c_int]),
    "zk_set_fused_layers": (c_int, [c_int]),
    "zk_set_tc_backward": (c_int, [c_int]),
    "zk_device_info": (c_int, [POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "zk_rqs_forward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_float, c_float, _P, c_int64, _P, c_int, _P]),
    "zk_rqs_inverse": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_float, c_float, _P, c_int64, _P]),
    "zk_affine_forward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_float, _P, c_int64, _P, c_int, _P]),
    "zk_affine_inverse": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_float, _P, c_int64, _P]),
    "zk_gaussianization_forward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, _P, c_int64, _P, c_int, _P]),
    "zk_gaussianization_inverse": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_float, c_int, _P, c_int64, _P]),
    "zk_sosp_forward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_int, c_float, c_float, _P, c_int64, _P, c_int, _P]),
    "zk_sosp_inverse": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_int, c_float, c_float, c_int, _P, c_int64, _P]),
    "zk_bernstein_forward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_float, c_float, _P, c_int64, _P, c_int, _P]),
    "zk_bernstein_inverse": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_float, c_float, _P, c_int64, _P]),
    "zk_univariate_plan": (c_int, [c_int, c_int64, c_int, c_int, c_int, c_int64, _P, POINTER(c_int), POINTER(c_size_t), POINTER(c_int),
                                   POINTER(c_int), POINTER(c_int)]),
    "zk_softclip_forward": (c_int, [_P, c_int64, c_int64, c_int, c_float, _P, c_int64, _P, c_int, _P]),
    "zk_softclip_inverse": (c_int, [_P, c_int64, c_int64, c_int, c_float, _P, c_int64, _P]),
    "zk_permute": (c_int, [_P, c_int64, _P, c_int64, c_int, _P, c_int64, _P]),
    "zk_rotate": (c_int, [_P, c_int64, _P, c_int, c_int64, c_int, _P, c_int64, _P]),
    "zk_circular_shift": (c_int, [_P, c_int64, c_int64, c_int, c_float, _P, c_int64, _P]),
    "zk_box_uniform_log_prob": (c_int, [_P, c_int64, _P, _P, _P, c_int64, c_int, _P, _P]),
    "zk_diag_normal_log_prob": (c_int, [_P, c_int64, _P, _P, _P, c_int64, c_int, _P, _P]),
    "zk_mlp_create": (c_int, [POINTER(MlpDesc), POINTER(c_void_p)]),
    "zk_mlp_destroy": (c_int, [_P]),
    "zk_mlp_workspace_bytes": (c_size_t, [_P, c_int64]),
    "zk_mlp_forward": (c_int, [_P, _P, c_int64, c_int, _P, c_int64, c_int, c_int64, _P, c_int64, _P, c_size_t, _P]),
    "zk_mlp_gemm_mode": (c_int, [_P]),
    "zk_layer_create": (c_int, [POINTER(LayerDesc), POINTER(c_void_p)]),
    "zk_layer_destroy": (c_int, [_P]),
    "zk_layer_workspace_bytes": (c_size_t, [_P, c_int64]),
    "zk_layer_fused_info": (c_int, [_P, c_void_p]),
    "zk_layer_fused_tile_rows": (c_int, [_P]),
    "zk_layer_fused_stream_bytes": (c_size_t, [_P]),
    "zk_layer_fused_plan": (c_int, [_P, POINTER(c_int), POINTER(c_size_t)]),
    "zk_layer_inverse_geometry": (c_int, [_P, POINTER(c_int), POINTER(c_int), POINTER(c_size_t)]),
    "zk_layer_sequential_inverse": (c_int, [_P]),
    "zk_comm_init_all": (c_int, [c_int, POINTER(c_void_p)]),
    "zk_comm_destroy": (c_int, [_P]),
    "zk_comm_size": (c_int, [_P]),
    "zk_comm_group_begin": (c_int, [_P]),
    "zk_comm_group_end": (c_int, [_P]),
    "zk_allreduce_sum": (c_int, [_P, c_int, _P, c_int, _P]),
    "zk_layer_update_weights": (c_int, [_P, c_void_p, c_void_p, _P]),
    "zk_set_pack_stream": (None, [_P]),
    "zk_layer_forward": (c_int, [_P, _P, c_int64, _P, c_int64, c_int64, _P, c_int64, _P, c_int, _P, c_size_t, _P]),
    "zk_layer_inverse": (c_int, [_P, _P, c_int64, _P, c_int64, c_int64, _P, c_int64, _P, c_size_t, _P]),
    "zk_flow_workspace_bytes": (c_size_t, [POINTER(FlowDesc), c_int64]),
    "zk_flow_host_workspace_bytes": (c_size_t, [POINTER(FlowDesc), c_int64]),
    "zk_debug_host_chunk_plan": (c_int64, [c_int64, c_int64, c_int64, c_void_p, c_int64]),
    "zk_flow_min_workspace_bytes": (c_size_t, [POINTER(FlowDesc)]),
    "zk_flow_forward": (c_int, [POINTER(FlowDesc), _P, c_int64, _P, c_int64, c_int64, _P, c_int64, _P, _P, c_size_t, _P]),
    "zk_flow_log_prob": (c_int, [POINTER(FlowDesc), _P, c_int64, _P, c_int64, c_int64, _P, _P, _P, c_size_t, _P]),
    "zk_flow_inverse": (c_int, [POINTER(FlowDesc), _P, c_int64, _P, c_int64, c_int64, _P, c_int64, _P, _P, c_size_t, _P]),
    "zk_univariate_backward_workspace_bytes": (c_size_t, [c_int64, c_int, c_int, c_int64]),
    "zk_univariate_backward_plan": (c_int, [c_int, c_int64, c_int, c_int, c_int, c_int64, POINTER(c_int), POINTER(c_size_t),
                                            POINTER(c_int)]),
    "zk_rqs_backward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_float, c_float, _P, c_int64, _P, _P, c_int64, _P, _P, c_size_t, _P]),
    "zk_affine_backward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_float, _P, c_int64, _P, _P, c_int64, _P, _P, c_size_t, _P]),
    "zk_gaussianization_backward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, _P, c_int64, _P, _P, c_int64, _P, _P, c_size_t, _P]),
    "zk_sosp_backward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_int, c_float, c_float, _P, c_int64, _P, _P, c_int64, _P, _P, c_size_t, _P]),
    "zk_bernstein_backward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int, c_int, c_float, c_float, _P, c_int64, _P, _P, c_int64, _P, _P, c_size_t, _P]),
    "zk_softclip_backward": (c_int, [_P, c_int64, c_int64, c_int, c_float, _P, c_int64, _P, _P, c_int64, _P]),
    "zk_layer_backward_workspace_bytes": (c_size_t, [_P, c_int64]),
    "zk_layer_backward": (c_int, [_P, _P, c_int64, _P, c_int64, c_int64, _P, c_int64, _P, _P, c_int64, _P, c_int64, POINTER(LayerGrads), _P, c_size_t, _P]),
    "zk_flow_backward_workspace_bytes": (c_size_t, [POINTER(FlowDesc), c_int64]),
    "zk_flow_backward_min_workspace_bytes": (c_size_t, [POINTER(FlowDesc)]),
    "zk_flow_backward": (c_int, [POINTER(FlowDesc), _P, c_int64, _P, c_int64, c_int64, _P, c_int64, _P, _P, _P, c_int64, _P, c_int64,
                                 POINTER(POINTER(LayerGrads)), _P, c_size_t, _P]),
    "zk_flow_inverse_backward_workspace_bytes": (c_size_t, [POINTER(FlowDesc), c_int64]),
    "zk_flow_inverse_backward_min_workspace_bytes": (c_size_t, [POINTER(FlowDesc)]),
    "zk_flow_inverse_backward": (c_int, [POINTER(FlowDesc), _P, c_int64, _P, c_int64, c_int64, _P, c_int64, _P, _P, c_int64, _P, c_int64,
                                         _P, c_int64, POINTER(POINTER(LayerGrads)), _P, c_size_t, _P]),
    "zk_cnf_create": (c_int, [POINTER(MlpDesc), c_int, c_int, c_int, _P, POINTER(c_void_p)]),
    "zk_cnf_destroy": (c_int, [_P]),
    "zk_cnf_workspace_bytes": (c_size_t, [_P, c_int64, c_int]),
    "zk_cnf_plan": (c_int, [_P, c_int64, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_size_t)]),
    "zk_cnf_integrate": (c_int, [_P, _P, c_int64, _P, c_int64, c_int64, _P, c_float, c_float, c_int, _P, c_int64, c_int, _P, c_int64,
                                 _P, _P, _P, _P, c_size_t, _P]),
    "zk_cnf_backward_workspace_bytes": (c_size_t, [_P, c_int64, c_int, c_int]),
    "zk_cnf_backward_min_workspace_bytes": (c_size_t, [_P, c_int, c_int]),
    "zk_cnf_backward_plan": (c_int, [_P, c_int64, c_int, c_int, c_size_t, POINTER(c_int), POINTER(c_int), POINTER(c_int64),
                                     POINTER(c_size_t)]),
    "zk_cnf_backward": (c_int, [_P, _P, c_int64, _P, c_int64, c_int64, _P, c_int, c_int, c_int, _P, c_int64, _P, c_int64, _P, _P,
                                c_int64, _P, c_int64, POINTER(LayerGrads), _P, c_size_t, _P]),
    "zk_flow_log_prob_host": (c_int, [POINTER(FlowDesc), _P, c_int64, _P, c_int64, c_int64, _P, POINTER(c_double), _P, c_size_t, _P]),
}  # fmt: skip

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


def lib() -> ctypes.CDLL:
    """Loads the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise EngineError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). zuko_b200 has no CPU / eager fallback."
            )
        handle = ctypes.CDLL(os.fspath(LIB_PATH))
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(status: int) -> None:
    if status != ZK_OK:
        msg = lib().zk_last_error()
        msg = msg.decode("utf-8", "replace") if msg else ""
        kind = {ZK_EINVAL: "invalid argument", ZK_EUNSUPPORTED: "unsupported", ZK_ECUDA: "CUDA error", ZK_ENOMEM: "out of memory"}.get(status, f"status {status}")  # fmt: skip
        if status == ZK_EUNSUPPORTED:
            raise NotImplementedError(f"zuko_b200: {kind}: {msg}")
        if status == ZK_EINVAL:
            raise ValueError(f"zuko_b200: {kind}: {msg}")
        raise EngineError(f"zuko_b200: {kind}: {msg}")


def stream_ptr(device: torch.device) -> c_void_p:
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def hold_storage(tensors) -> list:
    """Detached aliases of the tensors a cache entry keyed on ``data_ptr`` was built from.  Kept with the entry,
    they keep the storage alive, so that no other tensor can be allocated at the same address while the entry
    exists: a fresh tensor (``_version`` 0) reusing the freed address of an earlier one — a new posterior draw
    swapped in by ``torch.nn.utils.stateless``, say — would otherwise match the entry and be served stale.

    Cost: each entry keeps one copy of the weights it was packed from alive until it is replaced — one per layer
    handle, per stand-alone conditioner and per CNF, and up to 9 per autoregressive layer in its cache of
    permutation-folded handles; for tensors a module still owns this is no extra memory."""
    return [t.detach() for t in tensors if torch.is_tensor(t)]


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise EngineError(
            f"zuko_b200: {what} lives on {t.device}; the engine only runs on CUDA (sm_90a) and has no "
            "CPU fallback. Move the flow and its inputs to an H100 with .cuda()."
        )
    if t.dtype != torch.float32:
        raise TypeError(f"zuko_b200: {what} has dtype {t.dtype}; the engine computes in float32 only")


class Workspace:
    """Grow-only scratch tensor handed to the C ABI (the caller owns all memory), one per (device, CUDA
    stream): engine calls issued on different torch streams never share scratch, and a buffer that is
    outgrown is handed back to the caching allocator with ``record_stream`` so that it cannot be reused
    while kernels queued on its stream still run."""

    _cache: dict = {}
    # workspace ceiling: the flow calls chunk the batch to fit whatever they are given
    max_bytes = 8 << 30

    @classmethod
    def get(cls, device: torch.device, want: int, minimum: int) -> torch.Tensor:
        want = max(minimum, min(want, cls.max_bytes))
        index = device.index if device.index is not None else torch.cuda.current_device()
        stream = torch.cuda.current_stream(device)
        key = (device.type, index, stream.cuda_stream)
        buf = cls._cache.get(key)
        if buf is None or buf.numel() < want:
            old = cls._cache.pop(key, None)
            if old is not None:
                old.record_stream(stream)
            del old
            buf = torch.empty(want, dtype=torch.uint8, device=device)
            cls._cache[key] = buf
        return buf

    @classmethod
    def clear(cls) -> None:
        cls._cache.clear()
