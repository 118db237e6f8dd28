"""On-device graph partitioning and construction (SURVEY §8 f-2) — the device form of datasets/distribute_graphs.py.

    graph, edge_attr = radius_graph_csr(pos, r, batch=None)        # CSR by destination, int32, no int64 edge_index
    labels = kmeans_labels(pos, world_size)                          # == sklearn KMeans(random_state=0).fit_predict
    parts = split_large_graph(pos, x, target, vel, attr, r, P, split_mode="random" | "kmeans")

`radius_graph_csr` is one C-ABI call (csrc/radius_csr.cu): bounding box, grid sizing, cell keys, sort, counts, prefix sums
and the fill all run on the device, so it never synchronises when the caller passes a `capacity` (rollouts: reuse the
previous step's edge count plus slack); without one it reads the edge count back once to allocate exactly.  The result is
a `CSRGraph` that `FastEGNN.forward` takes as is — no COO->CSR sort, no edge_attr permutation.

`kmeans_labels` keeps sklearn's own k-means++ seeding (`sklearn.cluster.kmeans_plusplus`, host — it reproduces the
reference's `random_state=0`) and runs the Lloyd iterations with sklearn's stopping rules on the device (csrc/kmeans.cu).
CUDA only; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib
from ._lib import check, ptr
from .shards import CSRGraph

Tensor = torch.Tensor
_TABLE_CELLS = 1 << 22          # dense cell table (graphs x cells), int32: 16 MiB of workspace


class RadiusGraphBuffers:
    """Preallocated outputs of `radius_graph_csr` for `capacity` edges: rowptr, row, col, edge_attr, info and the build
    workspace live at fixed addresses, so repeated builds (a rollout rebuilds the graph every step) allocate nothing and
    can be captured in a CUDA graph.  `graph` is the CSRGraph over them (capacity-sized, count on the device)."""

    def __init__(self, n_nodes: int, capacity: int, edge_attr_nf: int, device, table_cells: int = _TABLE_CELLS):
        lib = _lib.load()
        nbytes = C.c_int64(0)
        check(lib.distegnn_radius_csr_workspace_bytes(n_nodes, table_cells, C.byref(nbytes)), "radius_csr_workspace_bytes")
        self.n_nodes, self.capacity, self.edge_attr_nf, self.table_cells = int(n_nodes), int(capacity), edge_attr_nf, table_cells
        self.ws = torch.empty(int(nbytes.value), dtype=torch.uint8, device=device)
        self.rowptr = torch.empty(n_nodes + 1, dtype=torch.int32, device=device)
        self.info = torch.zeros(4, dtype=torch.int32, device=device)
        self.row = torch.empty(self.capacity, dtype=torch.int32, device=device)
        self.col = torch.empty(self.capacity, dtype=torch.int32, device=device)
        self.edge_attr = (torch.empty(self.capacity, edge_attr_nf, dtype=torch.float32, device=device)
                          if edge_attr_nf > 0 else None)
        self.graph = CSRGraph(self.rowptr, self.col, self.row)
        self.graph.n_edges_dev, self.graph.info = self.info[0:1], self.info


def _build_into(buf: RadiusGraphBuffers, pos: Tensor, r: float, batch: Optional[Tensor], n_graphs: int, loop: bool,
                capacity: int) -> None:
    """One C-ABI call; `pos` float32 contiguous, `batch` int64 contiguous or None."""
    with torch.cuda.device(pos.device):
        check(_lib.load().distegnn_radius_graph_csr(
            buf.n_nodes, n_graphs, ptr(pos), ptr(batch), float(r), int(loop), buf.edge_attr_nf, capacity, buf.table_cells,
            ptr(buf.rowptr), ptr(buf.row if capacity else None), ptr(buf.col if capacity else None),
            ptr(buf.edge_attr if capacity else None), ptr(buf.info), ptr(buf.ws), buf.ws.numel(),
            _lib.stream_ptr(pos.device)), "radius_graph_csr")


def radius_graph_csr(pos: Tensor, r: float, batch: Optional[Tensor] = None, loop: bool = False, edge_attr_nf: int = 2,
                     capacity: Optional[int] = None, n_graphs: Optional[int] = None, table_cells: int = _TABLE_CELLS,
                     out: Optional[RadiusGraphBuffers] = None) -> Tuple[CSRGraph, Optional[Tensor]]:
    """All ordered pairs (i, j) of the same graph with ‖pos_i − pos_j‖ < r (j != i unless `loop`) as a CSRGraph grouped
    by destination i, plus edge_attr [E, edge_attr_nf] = the edge length in every column (distribute_graphs.py:43-44).

    capacity=None: exact allocation (one host read of the edge count).  capacity=K: no host synchronisation at all — the
    buffers hold K entries, `graph.n_edges_dev` (int32 [1] on the device) says how many are valid, the kernels read it
    there, and `graph.overflowed()` (a sync) tells whether K was too small.  out=RadiusGraphBuffers: capacity mode into
    those buffers (capacity = out.capacity); returns `(out.graph, out.edge_attr)`.  `batch` int64, sorted (PyG
    convention)."""
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.radius_graph_csr runs only on CUDA tensors (no CPU path)")
    dev = pos.device
    N = int(pos.shape[0])
    B = 1 if batch is None else (int(n_graphs) if n_graphs is not None else int(batch[-1].item()) + 1)
    p = pos.detach().to(torch.float32).contiguous()
    b = None if batch is None else batch.to(torch.int64).contiguous()
    if out is not None:
        if out.n_nodes != N or out.edge_attr_nf != edge_attr_nf or out.ws.device != dev:
            raise ValueError(f"RadiusGraphBuffers are for {out.n_nodes} nodes, edge_attr_nf={out.edge_attr_nf} on "
                             f"{out.ws.device}; got {N}, {edge_attr_nf} on {dev}")
        if N:
            _build_into(out, p, r, b, B, loop, out.capacity)
        return out.graph, out.edge_attr
    if N == 0:
        z = torch.zeros(0, dtype=torch.int32, device=dev)
        return CSRGraph(torch.zeros(1, dtype=torch.int32, device=dev), z, z.clone()), torch.zeros(0, edge_attr_nf, device=dev)
    if capacity is None:
        buf = RadiusGraphBuffers(N, 0, edge_attr_nf, dev, table_cells)
        _build_into(buf, p, r, b, B, loop, 0)                    # count only
        E = int(buf.info[0].item())
        buf = _resized(buf, E)
        _build_into(buf, p, r, b, B, loop, E)
        return CSRGraph(buf.rowptr, buf.col, buf.row), buf.edge_attr
    buf = RadiusGraphBuffers(N, int(capacity), edge_attr_nf, dev, table_cells)
    _build_into(buf, p, r, b, B, loop, buf.capacity)
    return buf.graph, buf.edge_attr


def _resized(buf: RadiusGraphBuffers, capacity: int) -> RadiusGraphBuffers:
    """The same rowptr / info / workspace with edge buffers for `capacity` edges."""
    new = RadiusGraphBuffers.__new__(RadiusGraphBuffers)
    new.__dict__.update(buf.__dict__)
    dev = buf.ws.device
    new.capacity = int(capacity)
    new.row = torch.empty(new.capacity, dtype=torch.int32, device=dev)
    new.col = torch.empty(new.capacity, dtype=torch.int32, device=dev)
    new.edge_attr = (torch.empty(new.capacity, buf.edge_attr_nf, dtype=torch.float32, device=dev)
                     if buf.edge_attr_nf > 0 else None)
    new.graph = CSRGraph(new.rowptr, new.col, new.row)
    new.graph.n_edges_dev, new.graph.info = new.info[0:1], new.info
    return new


def kmeans_labels(pos: Tensor, n_clusters: int, random_state: int = 0, max_iter: int = 300, tol: float = 1e-4,
                  chunk: int = 16) -> Tensor:
    """`sklearn.cluster.KMeans(n_clusters, random_state=random_state, n_init="auto").fit_predict(pos)` with the Lloyd
    iterations on the device: int64 labels [N] on `pos.device` (distribute_graphs.py:188-198).  The seeding is sklearn's
    own k-means++ on the host (on the mean-centred float32 positions, exactly as `KMeans.fit` does); iterations are
    enqueued `chunk` at a time and the device-side convergence state is read once per chunk."""
    import numpy as np
    from sklearn.cluster import kmeans_plusplus
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.kmeans_labels runs only on CUDA tensors (no CPU path)")
    lib = _lib.load()
    dev = pos.device
    p = pos.detach().to(torch.float32).contiguous()
    N = int(p.shape[0])
    X = p.cpu().numpy()
    mean = X.mean(axis=0)
    Xc = X - mean                                                # KMeans.fit centres the data first
    c0, _ = kmeans_plusplus(Xc, n_clusters, random_state=np.random.RandomState(random_state))
    tol_abs = float(tol * np.mean(np.var(Xc, axis=0)))           # sklearn's _tolerance
    centers = torch.from_numpy((c0 + mean).astype(np.float32)).to(dev).contiguous()
    labels = torch.full((N,), -1, dtype=torch.int32, device=dev)
    sums = torch.zeros(n_clusters, 4, dtype=torch.float64, device=dev)
    state = torch.zeros(4, dtype=torch.int32, device=dev)
    done = 0
    with torch.cuda.device(dev):
        while done < max_iter + 1:
            n = min(chunk, max_iter + 1 - done)
            check(lib.distegnn_kmeans_lloyd(N, n_clusters, ptr(p), ptr(centers), ptr(labels), ptr(sums), ptr(state),
                                            tol_abs, n, _lib.stream_ptr(dev)), "kmeans_lloyd")
            done += n
            if int(state[0].item()) == 2:
                break
    return labels.to(torch.int64)


def split_large_graph(pos: Tensor, x: Tensor, target: Tensor, vel: Tensor, attr: Optional[Tensor], radius: float,
                      world_size: int, split_mode: str = "random", special_nodes: Optional[Tensor] = None, generator=None,
                      edge_attr_nf: int = 2) -> List[Dict[str, Tensor]]:
    """Device-side form of the reference's partitioners (datasets/distribute_graphs.py:17-51 random, :118-143 k-means):
    node chunks by a host `randperm` (P−1 chunks of ⌊N/P⌋ + remainder) or by k-means cluster (`pos[cluster == i]`, nodes in
    index order), every chunk with its own radius graph built on the device as CSR, `edge_attr` = the edge length in
    `edge_attr_nf` columns (:44) and the GLOBAL `loc_mean` (:32).  Returns dicts with the reference's `Data` field names,
    `edge_index` being a `CSRGraph` (what `FastEGNN.forward` consumes directly)."""
    n = int(pos.shape[0])
    if split_mode == "random":
        idx = torch.randperm(n, generator=generator)             # on the host, as the reference (device == 'cpu')
        sizes = [n // world_size] * (world_size - 1)
        sizes.append(n - sum(sizes))
        chunks = [c.to(pos.device) for c in torch.split(idx, sizes)]
    elif split_mode == "kmeans":
        labels = kmeans_labels(pos, world_size)
        chunks = [torch.nonzero(labels == i, as_tuple=False).flatten() for i in range(world_size)]
    else:
        raise ValueError(f"unsupported split_mode {split_mode!r} (random|kmeans)")
    loc_mean = pos.mean(dim=0, keepdim=True)
    if special_nodes is None:
        special_nodes = torch.ones(n, dtype=torch.bool, device=pos.device)
    out = []
    for ch in chunks:
        pos_i = pos[ch]
        g, ea = radius_graph_csr(pos_i, radius, edge_attr_nf=edge_attr_nf)
        out.append(dict(x=x[ch], pos=pos_i, vel=vel[ch], attr=None if attr is None else attr[ch], target=target[ch],
                        loc_mean=loc_mean, edge_index=g, edge_attr=ea, special_nodes=special_nodes[ch]))
    return out
