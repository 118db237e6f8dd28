"""ctypes binding of libdistegnn_b200.so (the C ABI declared in include/distegnn_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libdistegnn_b200.so")

# field ids of the per-layer parameter block — must match the enum in include/distegnn_b200.h
P_FIELDS = [
    "E_W1A", "E_W1B", "E_W1R", "E_W1E", "E_B1", "E_W2", "E_B2", "E_WC", "E_BC", "E_W3",
    "V_W1H", "V_W1V", "V_W1R", "V_W1M", "V_B1", "V_W2", "V_B2", "V_WXV", "V_BXV", "V_W3XV",
    "V_WX", "V_BX", "V_W3X", "L_W", "L_B", "L_W3", "L_B3", "N_W1", "N_B1", "N_W2", "N_B2",
    "M_W1", "M_B1", "M_W2", "M_B2",
]
FLAG_NORMALIZE, FLAG_LAST, FLAG_INIT, FLAG_ZERO_VSUM, FLAG_ZERO_AGG, FLAG_INIT_CENTROID = 1, 2, 4, 8, 16, 32
MAX_CHANNELS, MAX_EDGE_ATTR, MAX_NODE_ATTR, MAX_NODE_FEAT, HIDDEN = 16, 8, 8, 16, 64

_i64, _i32, _u32, _vp = C.c_int64, C.c_int, C.c_uint, C.c_void_p

# name -> argtypes (restype is int for all but last_error)
SIGNATURES = {
    "distegnn_abi_version": [],
    "distegnn_param_layout": [_i32, _i32, _i32, C.POINTER(_i64), C.POINTER(_i64)],
    "distegnn_csr_workspace_bytes": [_i64, _i64, C.POINTER(_i64)],
    "distegnn_build_csr": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp],
    "distegnn_gather_rows": [_vp, _vp, _i64, _i32, _vp, _vp],
    "distegnn_scatter_rows": [_vp, _vp, _i64, _i32, _vp, _vp],
    "distegnn_embed_fwd": [_i64, _i32, _i32, _i32, _i32, _i32] + [_vp] * 15,
    "distegnn_edge_layer_fwd": [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 11,
    "distegnn_edge_layer_bwd": [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 15,
    "distegnn_edge_layer_bwd_inputs": [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 16,
    "distegnn_radius_csr_workspace_bytes": [_i64, _i64, C.POINTER(_i64)],
    "distegnn_radius_graph_csr": [_i64, _i32, _vp, _vp, C.c_float, _i32, _i32, _i64, _i64] + [_vp] * 6 + [_i64, _vp],
    "distegnn_rollout_advance": [_i64, _i32, _i32, C.c_float, _i32] + [_vp] * 10,
    "distegnn_edge_lengths_csr": [_i64, _i32] + [_vp] * 6,
    "distegnn_rollout_centroid": [_i64, _i32] + [_vp] * 4,
    "distegnn_edge_lengths_bwd": [_i64, _i32] + [_vp] * 7,
    "distegnn_rollout_advance_bwd": [_i64, _i32, _i32, C.c_float] + [_vp] * 9,
    "distegnn_cutoff_csr_workspace_bytes": [_i64, _i32, _i64, C.POINTER(_i64)],
    "distegnn_cutoff_csr": [_i64, _i32, _vp, _vp, C.c_double, _i32, _vp, _vp, _vp, _vp, _i64] + [_vp] * 7 + [_i64, _vp],
    "distegnn_kmeans_lloyd": [_i64, _i32, _vp, _vp, _vp, _vp, _vp, C.c_float, _i32, _vp],
    "distegnn_virtual_layer_bwd": [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 16,
    "distegnn_virtual_bwd_prepare": [_i32, _i32, _i32, _vp, _vp, _vp],
    "distegnn_virtual_layer_fwd": [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 10,
    "distegnn_node_layer_fwd": [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 20,
    "distegnn_virtual_update_fwd": [_i32, _i32, _i32, _i32, _u32] + [_vp] * 10,
    "distegnn_virtual_update_bwd": [_i32, _i32, _i32, _i32, _u32] + [_vp] * 14,
    "distegnn_node_layer_bwd": [_i64, _i32, _i32, _i32, _u32] + [_vp] * 24,
    "distegnn_embed_bwd": [_i64, _i32, _i32, _i32, _i32] + [_vp] * 11,
    "distegnn_node_layer_bwd_inputs": [_i64, _i32, _i32, _i32, _u32] + [_vp] * 26,
    "distegnn_embed_bwd_inputs": [_i64, _i32, _i32, _i32, _i32] + [_vp] * 17,
    "distegnn_comm_handle_bytes": [],
    "distegnn_comm_init": [_i32, _i32, _i32, _i32, C.POINTER(_vp), _vp],
    "distegnn_comm_connect": [_vp, _vp],
    "distegnn_comm_set_timeout_ms": [_vp, _i64],
    "distegnn_comm_status": [_vp, C.POINTER(_i32)],
    "distegnn_comm_disconnect": [_vp],
    "distegnn_comm_destroy": [_vp],
    "distegnn_allreduce_packed": [_vp, _vp, _i64, _vp],
    "distegnn_loss_packed_floats": [_i32, _i32],
    "distegnn_loss_partials": [_i64, _i32, _i32, _i32, _i32, _i32, C.c_float] + [_vp] * 10,
    "distegnn_loss_finalize": [_i64, _i32, _i32, _i32, _i32, _i32, C.c_float, C.c_float, _i32] + [_vp] * 10,
    "distegnn_deterministic_workspace_bytes": [_i64, _i64, _i32, C.POINTER(_i64)],
    "distegnn_edge_layer_fwd_det": [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 11 + [_i64, _vp],
    "distegnn_edge_combine_det": [_i64, _i64, _i32] + [_vp] * 5 + [_i64, _vp],
    "distegnn_virtual_layer_fwd_det": [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 10 + [_i64, _vp],
    "distegnn_vsum_combine_det": [_i64, _i32, _i32, _u32] + [_vp] * 4 + [_i64, _vp],
    "distegnn_rollout_centroid_det": [_i64, _i32] + [_vp] * 4,
    "distegnn_frames_assemble": [_i32, _i32, _i64, _i64] + [_vp] * 14,
    "distegnn_frames_targets": [_i32, _i64, _i64, _i32] + [_vp] * 6,
    "distegnn_rollout_sq_err_workspace_bytes": [_i64, C.POINTER(_i64)],
    "distegnn_rollout_sq_err": [_i64, _i32, _i32] + [_vp] * 6 + [_i64, _vp],
    "distegnn_rollout_chamfer_workspace_bytes": [_i64, _i32, C.POINTER(_i64)],
    "distegnn_rollout_chamfer": [_i64, _i32, _i32] + [_vp] * 6 + [_i64, _vp],
}
FRAMES_NBODY, FRAMES_WATER3D, FRAMES_LARGEFLUID = 0, 1, 2
ABI_VERSION = 3

_lib: Optional[C.CDLL] = None


class DistEGNNError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the shared library (once).  Raises with build instructions if it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DistEGNNError(
            f"{LIB_PATH} not found — build it with `python -m distegnn_b200.build` "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU/eager fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.distegnn_last_error.argtypes = []
    lib.distegnn_last_error.restype = C.c_char_p
    if lib.distegnn_abi_version() != ABI_VERSION:
        raise DistEGNNError(f"{LIB_PATH} has ABI version {lib.distegnn_abi_version()}, this package needs {ABI_VERSION} — "
                            "rebuild it with `python -m distegnn_b200.build --force`")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().distegnn_last_error().decode("utf-8", "replace")
        exc = ValueError if rc == -1 else DistEGNNError
        raise exc(f"{what} failed (code {rc}): {msg}")


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """Device pointer of a contiguous tensor (None -> NULL)."""
    if t is None:
        return None
    assert t.is_contiguous(), "non-contiguous tensor at the C-ABI boundary"
    return t.data_ptr()


def stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def deterministic_workspace_bytes(N: int, E: int, Cn: int) -> int:
    """Bytes of the deterministic mode's workspace for N nodes, an edge capacity E and Cn virtual channels."""
    nbytes = _i64(0)
    check(load().distegnn_deterministic_workspace_bytes(N, E, Cn, C.byref(nbytes)), "deterministic_workspace_bytes")
    return int(nbytes.value)


def param_layout(A: int, Cn: int, Na: int):
    """(dict field -> offset in floats, total floats) from the library itself."""
    offs = (_i64 * len(P_FIELDS))()
    total = _i64(0)
    check(load().distegnn_param_layout(A, Cn, Na, offs, C.byref(total)), "distegnn_param_layout")
    return {name: int(offs[i]) for i, name in enumerate(P_FIELDS)}, int(total.value)
