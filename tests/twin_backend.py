"""Cross-check twins of the production kernels (libdistegnn_b200_testing.so, include/distegnn_b200_testing.h).

Test infrastructure: earlier implementations of the same stages (fp32 FMA on the CUDA cores) behind their own C symbols,
used to cross-check the production kernels at sizes the CPU oracle cannot reach.  `TwinBackend` has the production backend's methods plus the twins'; nothing in
the package imports this module.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from distegnn_b200 import _lib
from distegnn_b200._lib import ptr
from distegnn_b200.backend import CudaBackend

_i64, _i32, _u32, _vp = C.c_int64, C.c_int, C.c_uint, C.c_void_p
TESTING_LIB_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), "libdistegnn_b200_testing.so")

TWIN_SIGNATURES = {
    "distegnn_embed_fwd_simt": [_i64, _i32, _i32, _i32, _i32, _i32] + [_vp] * 14,
    "distegnn_edge_layer_bwd_simt": [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 14,
    "distegnn_virtual_layer_bwd_simt": [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 16,
    "distegnn_edge_layer_fwd_simt": [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 10,
    "distegnn_virtual_layer_fwd_simt": [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 10,
    "distegnn_node_layer_fwd_simt": [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 20,
}

_tlib = None


def load_testing() -> C.CDLL:
    global _tlib
    if _tlib is None:
        lib = C.CDLL(TESTING_LIB_PATH)
        for name, argtypes in TWIN_SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = argtypes
            fn.restype = C.c_int
        lib.distegnn_last_error.argtypes = []
        lib.distegnn_last_error.restype = C.c_char_p
        _tlib = lib
    return _tlib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load_testing().distegnn_last_error().decode("utf-8", "replace")
        raise (ValueError if rc == -1 else _lib.DistEGNNError)(f"{what} failed (code {rc}): {msg}")


class TwinBackend(CudaBackend):
    """Production backend + the cross-check twins (`self.lib` stays the production library)."""

    def __init__(self) -> None:
        super().__init__()
        self.tlib = load_testing()

    def embed_simt(self, dims, node_feat, node_loc, data_batch, emb_wt, emb_b, layer0, h, x4, batch32, P, Q,
                   Hn, vsum) -> None:
        """fp32-FMA twin of embed (cross-check only)."""
        N, B, F, A, Cn, Na = dims
        check(self.tlib.distegnn_embed_fwd_simt(N, B, F, A, Cn, Na, ptr(node_feat), ptr(node_loc),
                                               ptr(data_batch), ptr(emb_wt), ptr(emb_b), ptr(layer0), ptr(h),
                                               ptr(x4), ptr(batch32), ptr(P), ptr(Q), ptr(Hn), ptr(vsum),
                                               self._s(h)), "embed_fwd_simt")

    def edge_layer_bwd_simt(self, dims, flags, row, col, ea, x4, P, Q, lp, g_agg_m, g_agg_x, g_P, g_Q, g_x4, g_lp) -> None:
        """fp32-FMA twin of edge_layer_bwd (cross-check only)."""
        N, E, A, Cn, Na = dims
        check(self.tlib.distegnn_edge_layer_bwd_simt(N, E, A, Cn, Na, flags, ptr(row), ptr(col), ptr(ea), ptr(x4),
                                                    ptr(P), ptr(Q), ptr(lp), ptr(g_agg_m), ptr(g_agg_x), ptr(g_P),
                                                    ptr(g_Q), ptr(g_x4), ptr(g_lp), self._s(x4)), "edge_layer_bwd_simt")

    def edge_layer_simt(self, dims, flags, row, col, ea, x4, P, Q, lp, agg_m, agg_x) -> None:
        """fp32-FMA twin of edge_layer (cross-check only; FastEGNN.forward never calls it)."""
        N, E, A, Cn, Na = dims
        check(self.tlib.distegnn_edge_layer_fwd_simt(N, E, A, Cn, Na, flags, ptr(row), ptr(col), ptr(ea),
                                                    ptr(x4), ptr(P), ptr(Q), ptr(lp), ptr(agg_m),
                                                    ptr(agg_x), self._s(x4)), "edge_layer_fwd_simt")

    def virtual_layer_simt(self, dims, flags, batch32, x4, Hn, Xv, G, lp, agg_v, trans_v, vsum) -> None:
        """fp32-FMA twin of virtual_layer (cross-check only)."""
        N, B, A, Cn, Na = dims
        check(self.tlib.distegnn_virtual_layer_fwd_simt(N, B, A, Cn, Na, flags, ptr(batch32), ptr(x4), ptr(Hn),
                                                       ptr(Xv), ptr(G), ptr(lp), ptr(agg_v), ptr(trans_v),
                                                       ptr(vsum), self._s(x4)), "virtual_layer_fwd_simt")

    def node_layer_simt(self, dims, flags, rowptr, batch32, h, x4, vel, attr, agg_m, agg_x, agg_v, trans_v,
                        lp, lp_next, h_out, x4_out, P, Q, Hn, loc_out, vsum) -> None:
        """fp32-FMA twin of node_layer (cross-check only)."""
        N, B, A, Cn, Na = dims
        check(self.tlib.distegnn_node_layer_fwd_simt(N, B, A, Cn, Na, flags, ptr(rowptr), ptr(batch32), ptr(h),
                                                    ptr(x4), ptr(vel), ptr(attr), ptr(agg_m), ptr(agg_x),
                                                    ptr(agg_v), ptr(trans_v), ptr(lp), ptr(lp_next),
                                                    ptr(h_out), ptr(x4_out), ptr(P), ptr(Q), ptr(Hn),
                                                    ptr(loc_out), ptr(vsum), self._s(x4)), "node_layer_fwd_simt")

    def virtual_layer_bwd_simt(self, dims, flags, batch32, x4, Hn, Xv, G, lp, wT, g_agg_v, g_trans_v, g_vsum, g_Hn, g_xv,
                               g_G, g_Xv, g_lp) -> None:
        """fp32-FMA twin of virtual_layer_bwd (cross-check only); wT = the three matrices transposed, fp32."""
        N, B, A, Cn, Na = dims
        check(self.tlib.distegnn_virtual_layer_bwd_simt(N, B, A, Cn, Na, flags, ptr(batch32), ptr(x4), ptr(Hn), ptr(Xv),
                                                       ptr(G), ptr(lp), ptr(wT), ptr(g_agg_v), ptr(g_trans_v), ptr(g_vsum),
                                                       ptr(g_Hn), ptr(g_xv), ptr(g_G), ptr(g_Xv), ptr(g_lp), self._s(x4)),
              "virtual_layer_bwd_simt")


_twin = None


def twin_backend() -> TwinBackend:
    global _twin
    if _twin is None:
        _twin = TwinBackend()
    return _twin
