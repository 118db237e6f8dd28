"""On-device graph construction (SURVEY §8 f-2): `radius_graph` with the call shape of
`torch_geometric.nn.radius_graph` as the reference's partitioners use it (datasets/distribute_graphs.py:43-44:
`radius_graph(pos_i, r=radius, max_num_neighbors=pos_i.size(0))` followed by `edge_attr = ‖Δx‖` repeated twice).

The cell keys are sorted with torch (library radix sort); the neighbour search, the degree count and the edge fill are
hand-written kernels behind the C ABI (csrc/radius_graph.cu).  Edges come out grouped by destination row in ascending
order, so `distegnn_build_csr`'s sort finds them already ordered.  CUDA only — there is no CPU path.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib

Tensor = torch.Tensor
_MAX_DIM = 1024            # cells per axis
_MAX_TABLE = 1 << 27       # entries of the dense cell table (graphs x cells)
_FLT_MAX = float(torch.finfo(torch.float32).max)


def radius_graph(pos: Tensor, r: float, batch: Optional[Tensor] = None, loop: bool = False,
                 max_num_neighbors: Optional[int] = None, edge_attr_nf: int = 2) -> Tuple[Tensor, Tensor]:
    """All ordered pairs (i, j), i != j unless `loop`, of the same graph with ‖pos_i − pos_j‖ < r (strict, as torch_cluster).

    Returns (edge_index [2,E] int64 with edge_index[0] = i ascending, edge_attr [E, edge_attr_nf] fp32 = the edge length
    in every column — what distribute_graphs.py:44 builds).  `max_num_neighbors` is accepted for signature compatibility;
    the reference always passes the node count (no cap), a smaller cap raises.
    """
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.radius_graph runs only on CUDA tensors (no CPU path)")
    N = int(pos.shape[0])
    if max_num_neighbors is not None and max_num_neighbors < N - 1:
        raise NotImplementedError("max_num_neighbors below the node count is not supported (the reference never caps)")
    dev = pos.device
    if N == 0:
        return torch.zeros(2, 0, dtype=torch.int64, device=dev), torch.zeros(0, edge_attr_nf, device=dev)
    from .backend import cuda_backend
    be = cuda_backend()
    x4 = torch.zeros(N, 4, dtype=torch.float32, device=dev)
    x4[:, :3] = pos.detach().to(torch.float32)
    if not bool(torch.isfinite(x4[:, :3]).all()):
        raise ValueError("radius_graph: positions must be finite (partition.radius_graph_csr gives nodes with an inf or "
                         "NaN coordinate no edges instead)")
    batch32 = None if batch is None else batch.to(torch.int32).contiguous()
    B = 1 if batch is None else int(batch.max().item()) + 1
    if B + 1 > _MAX_TABLE:
        raise ValueError(f"radius_graph: {B} graphs exceed the cell table ({_MAX_TABLE} entries)")
    lo, hi = x4[:, :3].amin(0), x4[:, :3].amax(0)
    lo_h = [float(v) for v in lo.tolist()]
    ext = [h - l for h, l in zip(hi.tolist(), lo_h)]          # float64: finite even where the fp32 difference overflows
    # first cell r·(1 + 2^-10) in fp32, the margin that keeps pairs closer than r within adjacent cells despite the
    # rounding of the fp32 cell index (csrc/radius_grid.cuh)
    cell = float(torch.tensor(float(r), dtype=torch.float32) * (1.0 + 2.0 ** -10))
    while True:                                               # grow the cell until the dense table fits
        dims = [min(int(e / cell) + 1, 1 << 30) for e in ext]
        if max(dims) <= _MAX_DIM and B * dims[0] * dims[1] * dims[2] + 1 <= _MAX_TABLE:
            break
        if cell * 1.5 > _FLT_MAX:                             # r tiny against an extent near FLT_MAX: one cell per graph
            dims = [1, 1, 1]
            break
        cell *= 1.5
    inv_cell = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(cell, dtype=torch.float32)   # the kernel's 1/cell
    dims_t = torch.tensor(dims, dtype=torch.int32, device=dev)
    idx = ((x4[:, :3] - lo) * inv_cell.to(dev)).to(torch.int32)                  # same fp32 expression as the kernel
    idx = torch.minimum(idx.clamp(min=0), dims_t - 1).to(torch.int64)
    ncell = dims[0] * dims[1] * dims[2]
    key = (idx[:, 0] * dims[1] + idx[:, 1]) * dims[2] + idx[:, 2]
    if batch is not None:
        key = key + batch.to(torch.int64) * ncell
    skey, order = torch.sort(key)
    cell_start = torch.searchsorted(skey, torch.arange(B * ncell + 1, dtype=torch.int64, device=dev))
    order32 = order.to(torch.int32)
    deg = torch.empty(N, dtype=torch.int32, device=dev)
    grid = (lo_h, cell, dims)
    be.radius_count(N, x4, batch32, order32, cell_start, grid, float(r), loop, deg)
    rowptr = torch.zeros(N + 1, dtype=torch.int64, device=dev)
    torch.cumsum(deg, 0, out=rowptr[1:])
    E = int(rowptr[-1].item())
    row = torch.empty(E, dtype=torch.int32, device=dev)
    col = torch.empty(E, dtype=torch.int32, device=dev)
    dist = torch.empty(E, dtype=torch.float32, device=dev)
    if E:
        be.radius_fill(N, x4, batch32, order32, cell_start, grid, float(r), loop, rowptr, row, col, dist)
    edge_index = torch.stack([row, col]).to(torch.int64)
    edge_attr = dist.unsqueeze(1).repeat(1, edge_attr_nf) if edge_attr_nf > 0 else dist.new_zeros(E, 0)
    return edge_index, edge_attr


def split_large_graph_random(pos: Tensor, x: Tensor, target: Tensor, vel: Tensor, attr: Optional[Tensor], radius: float,
                             world_size: int, special_nodes: Optional[Tensor] = None, generator=None):
    """Device-side form of the reference's random partitioner (datasets/distribute_graphs.py:17-51): one host `randperm`
    (same chunking: P−1 chunks of ⌊N/P⌋, remainder to the last), every chunk gets its own radius graph — built here with
    the on-device `radius_graph` instead of PyG on the host — and `edge_attr` = the edge length in two columns (:44); every
    partition carries the GLOBAL `loc_mean` (:32).  Returns a list of dicts with the reference's `Data` field names
    (`x, pos, vel, attr, target, loc_mean, edge_index, edge_attr, special_nodes`); tensors stay on `pos.device`.
    Pass `generator=torch.Generator().manual_seed(s)` to reproduce `torch.manual_seed(s)` + the reference's `randperm`."""
    n = int(pos.shape[0])
    idx = torch.randperm(n, generator=generator)                      # on the host, as the reference (device == 'cpu')
    sizes = [n // world_size] * (world_size - 1)
    sizes.append(n - sum(sizes))
    chunks = torch.split(idx, sizes)
    loc_mean = pos.mean(dim=0, keepdim=True)
    if special_nodes is None:
        special_nodes = torch.ones(n, dtype=torch.bool, device=pos.device)
    out = []
    for ch in chunks:
        ch = ch.to(pos.device)
        pos_i = pos[ch]
        ei, ea = radius_graph(pos_i, radius, max_num_neighbors=int(pos_i.shape[0]))
        out.append(dict(x=x[ch], pos=pos_i, vel=vel[ch], attr=None if attr is None else attr[ch], target=target[ch],
                        loc_mean=loc_mean, edge_index=ei, edge_attr=ea, special_nodes=special_nodes[ch]))
    return out
