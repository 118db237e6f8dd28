"""The edge kernel counts tiles and edges in int32, so both edge-stage entry points reject an edge count (or, with a
device-side count, a capacity) of 2^31 - 63 or more before anything is launched.  The device count here is 0, so even a
launch would read no edge: the test fails on the return code, never by touching memory past the small tensors."""
import ctypes

import pytest
import torch

from distegnn_b200 import _lib
from distegnn_b200._lib import ptr

pytestmark = pytest.mark.gpu

INT32_MAX = 2 ** 31 - 1


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("n_edges", [INT32_MAX - 62, INT32_MAX, 2 ** 40])
def test_edge_count_past_int32_tiles_is_rejected(det, n_edges):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    dev = torch.device("cuda:0")
    lib = _lib.load()
    A, C, Na, N = 2, 3, 0, 8
    _, total = _lib.param_layout(A, C, Na)
    row = torch.zeros(64, dtype=torch.int32, device=dev)
    col = torch.zeros(64, dtype=torch.int32, device=dev)
    ea = torch.zeros(64, A, device=dev)
    x4 = torch.zeros(N, 4, device=dev)
    P, Q = torch.zeros(N, 64, device=dev), torch.zeros(N, 64, device=dev)
    lp = torch.zeros(total, device=dev)
    agg_m, agg_x = torch.zeros(N, 64, device=dev), torch.zeros(N, 4, device=dev)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=dev)
    args = [N, n_edges, A, C, Na, 0, ptr(row), ptr(col), ptr(ea), ptr(x4), ptr(P), ptr(Q), ptr(lp), ptr(agg_m),
            ptr(agg_x), ptr(n_dev)]
    stream = torch.cuda.current_stream().cuda_stream
    if det:
        rc = lib.distegnn_edge_layer_fwd_det(*args, ptr(ws), ws.numel(), stream)
    else:
        rc = lib.distegnn_edge_layer_fwd(*args, stream)
    torch.cuda.synchronize()
    assert rc == -1   # DISTEGNN_EINVAL
    assert b"2^31 - 64" in lib.distegnn_last_error()
    assert not agg_m.any() and not agg_x.any()
