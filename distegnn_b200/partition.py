"""On-device graph partitioning and construction (SURVEY §8 f-2) — the device form of datasets/distribute_graphs.py.

    graph, edge_attr = radius_graph_csr(pos, r, batch=None)        # CSR by destination, int32, no int64 edge_index
    edge_index, edge_attr = radius_graph(pos, r, batch=None)         # the same graph as PyG's int64 edge_index
    graph, edge_attr = cutoff_edges_csr(graph, pos, 0.5, batch)      # FastEGNN's cutoff: the shortest half of each graph
    labels = kmeans_labels(pos, world_size)                          # == sklearn KMeans(random_state=0).fit_predict
    labels = spectral_labels(pos, world_size)                        # the reference's SpectralClustering (spectral.py)
    labels = metis_labels(pos, world_size, outer_radius)             # the reference's METIS on the outer-radius graph
    parts = split_large_graph(pos, x, target, vel, attr, r, P, split_mode="random" | "kmeans" | "spectral" | "metis")

`radius_graph_csr` is one C-ABI call (csrc/radius_csr.cu): bounding box, grid sizing, cell keys, sort, counts, prefix sums
and the fill all run on the device, so it never synchronises when the caller passes a `capacity` (rollouts: reuse the
previous step's edge count plus slack); without one it reads the edge count back once to allocate exactly.  The result is
a `CSRGraph` that `FastEGNN.forward` takes as is — no COO->CSR sort, no edge_attr permutation.

`kmeans_labels` keeps sklearn's own k-means++ seeding (`sklearn.cluster.kmeans_plusplus`, host — it reproduces the
reference's `random_state=0`) and runs the Lloyd iterations with sklearn's stopping rules on the device (csrc/kmeans.cu).
CUDA only; there is no CPU path.

`metis_labels` builds the outer-radius graph and sorts its rows on the device (csrc/metis.cu), then runs the CUDA
toolkit's METIS (`METIS_PartGraphRecursive`, linked into the library) on the host, as the reference does.
"""
from __future__ import annotations

import ctypes as C
import numbers
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib
from ._lib import check, ptr
from .shards import CSRGraph
from .spectral import spectral_labels

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
                     out: Optional[RadiusGraphBuffers] = None,
                     cutoff_rate: float = 0.0) -> Tuple[CSRGraph, Optional[Tensor]]:
    """All ordered pairs (i, j) of the same graph with ‖pos_i − pos_j‖ < r (j != i unless `loop`) as a CSRGraph grouped
    by destination i, plus edge_attr [E, edge_attr_nf] = the edge length in every column (distribute_graphs.py:43-44).

    capacity=None: exact allocation (one host read of the edge count).  capacity=K: no host synchronisation at all — the
    buffers hold K entries, `graph.n_edges_dev` (int32 [1] on the device) says how many are valid, the kernels read it
    there, and `graph.overflowed()` (a sync) tells whether K was too small.  out=RadiusGraphBuffers: capacity mode into
    those buffers (capacity = out.capacity); returns `(out.graph, out.edge_attr)`.  `batch` int64, sorted (PyG
    convention).

    cutoff_rate > 0 (FastEGNN's cutoff_edges mode): the radius graph is the candidate set and `cutoff_edges_csr` keeps
    the int(E_b * (1 - cutoff_rate)) shortest edges of every graph.  `capacity` / `out.capacity` count the CANDIDATES;
    the returned graph holds the kept edges (count in `graph.n_edges_dev` in capacity mode).  0 runs no cutoff at all."""
    _check_rate(cutoff_rate)
    if cutoff_rate > 0:
        return _radius_then_cut(pos, r, batch, loop, edge_attr_nf, capacity, n_graphs, table_cells, out,
                                float(cutoff_rate))
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


def radius_graph(pos: Tensor, r: float, batch: Optional[Tensor] = None, loop: bool = False,
                 max_num_neighbors: Optional[int] = None, edge_attr_nf: int = 2) -> Tuple[Tensor, Tensor]:
    """`radius_graph_csr` in the call shape of `torch_geometric.nn.radius_graph` as the reference's partitioners use it
    (datasets/distribute_graphs.py:43-44: `radius_graph(pos_i, r=radius, max_num_neighbors=pos_i.size(0))` followed by
    `edge_attr = ‖Δx‖` repeated twice).

    Returns (edge_index [2,E] int64 with edge_index[0] = i ascending, edge_attr [E, edge_attr_nf] fp32 = the edge length
    in every column).  `max_num_neighbors` is accepted for signature compatibility; the reference always passes the node
    count (no cap), a smaller cap raises.  Non-finite positions raise.  Counts in int32 as `radius_graph_csr` does, so
    E < 2^31."""
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.radius_graph runs only on CUDA tensors (no CPU path)")
    N = int(pos.shape[0])
    if max_num_neighbors is not None and max_num_neighbors < N - 1:
        raise NotImplementedError("max_num_neighbors below the node count is not supported (the reference never caps)")
    if N == 0:
        return (torch.zeros(2, 0, dtype=torch.int64, device=pos.device),
                torch.zeros(0, edge_attr_nf, device=pos.device))
    p = pos.detach().to(torch.float32).contiguous()
    if not bool(torch.isfinite(p).all()):
        raise ValueError("radius_graph: positions must be finite (radius_graph_csr gives nodes with an inf or NaN "
                         "coordinate no edges instead)")
    B = 1 if batch is None else int(batch.max().item()) + 1
    g, ea = radius_graph_csr(p, r, batch, loop=loop, edge_attr_nf=min(edge_attr_nf, 1), n_graphs=B,
                             table_cells=max(_TABLE_CELLS, B + 1))
    edge_index = torch.stack([g.row, g.col]).to(torch.int64)
    edge_attr = ea.repeat(1, edge_attr_nf) if edge_attr_nf > 0 else p.new_zeros(g.num_edges, 0)
    return edge_index, edge_attr


# ---- edge cutoff (FastEGNN's cutoff_edges mode; csrc/cutoff_csr.cu) ----------------------------------------------------
def _check_rate(rate) -> None:
    if isinstance(rate, bool) or not isinstance(rate, numbers.Real):
        raise ValueError(f"cutoff_rate must be a real number in [0, 1] (got {rate!r})")
    if not 0.0 <= float(rate) <= 1.0:                          # NaN fails too
        raise ValueError(f"cutoff_rate must lie in [0, 1] (got {rate!r})")


def _cut_workspace(out: RadiusGraphBuffers, n_graphs: int, capacity: int) -> Tensor:
    """The cutoff's workspace, kept on the output buffers (allocated on first use, reused at a fixed address after)."""
    key = (int(n_graphs), int(capacity))
    if getattr(out, "cut_key", None) != key:
        nbytes = C.c_int64(0)
        check(_lib.load().distegnn_cutoff_csr_workspace_bytes(out.n_nodes, key[0], key[1], C.byref(nbytes)),
              "cutoff_csr_workspace_bytes")
        out.cut_ws = torch.empty(int(nbytes.value), dtype=torch.uint8, device=out.ws.device)
        out.cut_key = key
    return out.cut_ws


def _cut_into(out: RadiusGraphBuffers, graph: CSRGraph, pos: Tensor, rate: float, batch: Optional[Tensor],
              n_graphs: int) -> None:
    """One C-ABI call: the kept edges of `graph` into `out` (no host synchronisation).  `pos` float32 contiguous,
    `batch` int64 contiguous or None."""
    cap = graph.num_edges
    ws = _cut_workspace(out, n_graphs, cap)
    overflow = graph.info[1:2] if graph.info is not None else None
    rows = graph.rows().contiguous() if cap else None
    with torch.cuda.device(pos.device):
        check(_lib.load().distegnn_cutoff_csr(
            out.n_nodes, n_graphs, ptr(pos), ptr(batch), float(rate), out.edge_attr_nf, ptr(graph.rowptr.contiguous()),
            ptr(rows), ptr(graph.col.contiguous() if cap else None), ptr(graph.n_edges_dev), cap, ptr(overflow),
            ptr(out.rowptr), ptr(out.row if cap else None), ptr(out.col if cap else None),
            ptr(out.edge_attr if cap else None), ptr(out.info), ptr(ws), ws.numel(), _lib.stream_ptr(pos.device)),
            "cutoff_csr")


def cutoff_edges_csr(graph: CSRGraph, pos: Tensor, cutoff_rate: float, batch: Optional[Tensor] = None,
                     n_graphs: Optional[int] = None, edge_attr_nf: int = 2, capacity: Optional[int] = None,
                     out: Optional[RadiusGraphBuffers] = None) -> Tuple[CSRGraph, Optional[Tensor]]:
    """FastEGNN's edge cutoff on the device (datasets/process_dataset.py:300-305, once per sample): of every graph of the
    batch keep the int(E_b * (1 - cutoff_rate)) shortest edges of `graph` and drop the rest.

    `graph` is any CSRGraph (built on the device, read from a shard, or `CSRGraph.from_edge_index`); its edges below
    `graph.n_edges_dev` are the candidates.  The length is the fp32 ‖pos_i − pos_j‖ of the radius build; ties are broken by
    CSR position (a stable selection), NaN sorts last.  Returns the kept edges as a CSRGraph in the candidates' order plus
    edge_attr [E, edge_attr_nf] = the length in every column (:104).

    capacity=None: exact (one host read of the kept count).  capacity=K (>= graph.num_edges): no host synchronisation —
    buffers of K entries, the kept count in `graph.n_edges_dev` on the device.  out=RadiusGraphBuffers: into those
    buffers (out.capacity >= graph.num_edges).  `batch` int64, sorted; pass `n_graphs` to avoid reading its last entry."""
    _check_rate(cutoff_rate)
    if not isinstance(graph, CSRGraph):
        raise ValueError("graph must be a distegnn_b200.shards.CSRGraph")
    if pos.device.type != "cuda" or graph.rowptr.device != pos.device:
        raise _lib.DistEGNNError("distegnn_b200.cutoff_edges_csr runs only on CUDA tensors, graph and pos on one device "
                                 "(no CPU path)")
    dev = pos.device
    N = int(pos.shape[0])
    if graph.num_nodes != N:
        raise ValueError(f"graph has {graph.num_nodes} nodes, pos has {N}")
    E = graph.num_edges
    B = 1 if batch is None else (int(n_graphs) if n_graphs is not None else int(batch[-1].item()) + 1)
    p = pos.detach().to(torch.float32).contiguous()
    b = None if batch is None else batch.to(torch.int64).contiguous()
    if out is not None:
        if out.n_nodes != N or out.edge_attr_nf != edge_attr_nf or out.ws.device != dev or out.capacity < E:
            raise ValueError(f"RadiusGraphBuffers are for {out.n_nodes} nodes, {out.capacity} edges, edge_attr_nf="
                             f"{out.edge_attr_nf} on {out.ws.device}; got {N}, {E} candidates, {edge_attr_nf} on {dev}")
        if N:
            _cut_into(out, graph, p, float(cutoff_rate), b, B)
        return out.graph, out.edge_attr
    if N == 0:
        z = torch.zeros(0, dtype=torch.int32, device=dev)
        return CSRGraph(torch.zeros(1, dtype=torch.int32, device=dev), z, z.clone()), torch.zeros(0, edge_attr_nf, device=dev)
    if capacity is not None:
        if int(capacity) < E:
            raise ValueError(f"capacity {capacity} is below the candidate buffers' {E} entries")
        buf = RadiusGraphBuffers(N, int(capacity), edge_attr_nf, dev, table_cells=27)
        _cut_into(buf, graph, p, float(cutoff_rate), b, B)
        return buf.graph, buf.edge_attr
    buf = RadiusGraphBuffers(N, E, edge_attr_nf, dev, table_cells=27)
    _cut_into(buf, graph, p, float(cutoff_rate), b, B)
    kept, overflowed = buf.info[0:2].tolist()
    if overflowed:
        raise ValueError(f"the candidate graph overflowed its capacity {E} (its true edge count is "
                         f"{int(buf.info[2].item())}): the candidates are incomplete")
    ea = buf.edge_attr[:kept] if buf.edge_attr is not None else None
    return CSRGraph(buf.rowptr, buf.col[:kept], buf.row[:kept]), ea


def _radius_then_cut(pos, r, batch, loop, edge_attr_nf, capacity, n_graphs, table_cells, out, rate):
    """radius_graph_csr(cutoff_rate > 0): the candidates (no edge_attr: the cutoff recomputes the lengths), then the cut."""
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.radius_graph_csr runs only on CUDA tensors (no CPU path)")
    N = int(pos.shape[0])
    B = 1 if batch is None else (int(n_graphs) if n_graphs is not None else int(batch[-1].item()) + 1)
    if out is None and capacity is None:
        g, _ = radius_graph_csr(pos, r, batch, loop=loop, edge_attr_nf=0, n_graphs=B, table_cells=table_cells)
        return cutoff_edges_csr(g, pos, rate, batch, B, edge_attr_nf)
    if out is None:
        out = RadiusGraphBuffers(N, int(capacity), edge_attr_nf, pos.device, table_cells)
    if getattr(out, "candidates", None) is None:
        out.candidates = RadiusGraphBuffers(out.n_nodes, out.capacity, 0, out.ws.device, out.table_cells)
    cg, _ = radius_graph_csr(pos, r, batch, loop=loop, edge_attr_nf=0, n_graphs=B, table_cells=table_cells,
                             out=out.candidates)
    return cutoff_edges_csr(cg, pos, rate, batch, B, edge_attr_nf, out=out)


def kmeans_labels(pos: Tensor, n_clusters: int, random_state: int = 0, max_iter: int = 300, tol: float = 1e-4,
                  chunk: int = 16) -> Tensor:
    """`sklearn.cluster.KMeans(n_clusters, random_state=random_state, n_init="auto").fit_predict(pos)` with the Lloyd
    iterations on the device: int64 labels [N] on `pos.device` (distribute_graphs.py:188-198).  The seeding is sklearn's
    own k-means++ on the host; the seeding and the iterations both run on the mean-centred float32 positions, exactly as
    `KMeans.fit` does (fp32 distances and centres far from the origin would lose their digits to the offset).  Iterations
    are enqueued `chunk` at a time and the device-side convergence state is read once per chunk; a run that reaches
    `max_iter` ends with sklearn's closing assignment (the header's state[0] = 1 call)."""
    import numpy as np
    from sklearn.cluster import kmeans_plusplus
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.kmeans_labels runs only on CUDA tensors (no CPU path)")
    lib = _lib.load()
    dev = pos.device
    X = pos.detach().to(torch.float32).cpu().numpy()
    N = int(X.shape[0])
    Xc = X - X.mean(axis=0)                                      # KMeans.fit centres the data first
    c0, _ = kmeans_plusplus(Xc, n_clusters, random_state=np.random.RandomState(random_state))
    tol_abs = float(tol * np.mean(np.var(Xc, axis=0)))           # sklearn's _tolerance
    p = torch.from_numpy(np.ascontiguousarray(Xc)).to(dev)
    centers = torch.from_numpy(np.ascontiguousarray(c0, dtype=np.float32)).to(dev)
    labels = torch.full((N,), -1, dtype=torch.int32, device=dev)
    sums = torch.zeros(n_clusters, 4, dtype=torch.float64, device=dev)
    state = torch.zeros(4, dtype=torch.int32, device=dev)

    def lloyd(n):
        check(lib.distegnn_kmeans_lloyd(N, n_clusters, ptr(p), ptr(centers), ptr(labels), ptr(sums), ptr(state),
                                        tol_abs, n, _lib.stream_ptr(dev)), "kmeans_lloyd")
    done = 0
    with torch.cuda.device(dev):
        while done < max_iter and int(state[0].item()) != 2:
            n = min(chunk, max_iter - done)
            lloyd(n)
            done += n
        if int(state[0].item()) != 2:
            state[0] = 1                                         # max_iter passes: sklearn's closing E-step
            lloyd(1)
    return labels.to(torch.int64)


def csr_sorted_i64(graph: CSRGraph) -> Tuple[Tensor, Tensor]:
    """(xadj int64 [N+1], adjncy int64 [capacity]) of a device-built id-order CSR graph with every row's neighbours
    ascending: `index2ptr(sort_edge_index(edge_index))` as the reference hands it to METIS (distribute_graphs.py:155-157).
    One launch (csrc/metis.cu), no host synchronisation; the edge count on the device is honoured (`graph.n_edges_dev`),
    entries of adjncy at and past it are left unwritten."""
    if graph.rowptr.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.csr_sorted_i64 runs only on CUDA tensors (no CPU path)")
    dev = graph.rowptr.device
    N, cap = graph.num_nodes, int(graph.col.numel())
    xadj = torch.empty(N + 1, dtype=torch.int64, device=dev)
    adjncy = torch.empty(cap, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().distegnn_csr_sorted_i64(
            N, cap, ptr(graph.rowptr.contiguous()), ptr(graph.col.contiguous() if cap else None),
            ptr(graph.n_edges_dev), ptr(xadj), ptr(adjncy if cap else None), _lib.stream_ptr(dev)), "csr_sorted_i64")
    return xadj, adjncy


def metis_recursive(xadj, adjncy, n_parts: int) -> Tuple["np.ndarray", int]:
    """(labels int64 [N], edge cut) of `METIS_PartGraphRecursive` on the host CSR (numpy int64 xadj [N+1], adjncy), with
    the reference's arguments (distribute_graphs.py:151-185: no weights, default options) and its `num_parts <= 1` rule
    (zeros, no METIS call).  Malformed input or n_parts outside [1, N] raises ValueError before METIS runs."""
    import numpy as np
    xadj = np.ascontiguousarray(xadj, dtype=np.int64)
    adjncy = np.ascontiguousarray(adjncy, dtype=np.int64)
    n = int(xadj.shape[0]) - 1
    if n < 1:
        raise ValueError("metis_recursive: the graph needs at least one node")
    if int(xadj[-1]) > adjncy.shape[0]:
        raise ValueError(f"metis_recursive: xadj[-1] = {int(xadj[-1])} past adjncy's {adjncy.shape[0]} entries")
    part = np.empty(n, dtype=np.int64)
    cut = C.c_int64(0)
    check(_lib.load().distegnn_metis_recursive(n, xadj.ctypes.data, adjncy.ctypes.data if adjncy.size else None,
                                                int(n_parts), part.ctypes.data, C.byref(cut)), "metis_recursive")
    return part, int(cut.value)


def metis_labels(pos: Tensor, n_parts: int, outer_radius: float) -> Tensor:
    """The reference's METIS split (distribute_graphs.py:54-87, 151-185) as int64 labels [N] on `pos.device`: the
    outer-radius graph `radius_graph(pos, outer_radius)` (symmetric, no self loops, no neighbour cap) built on the device,
    its CSR sorted by (row, col) on the device (`csr_sorted_i64`), one copy to pinned host buffers,
    `METIS_PartGraphRecursive` of the CUDA toolkit's METIS 5 on the host (`metis_recursive`), and one copy back.  The same
    graph and the same call as the reference's, so the same labels wherever its METIS is the same version.  ValueError for
    non-finite positions, outer_radius <= 0 or n_parts outside [1, N]."""
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.metis_labels runs only on CUDA tensors (no CPU path)")
    import math
    N = int(pos.shape[0])
    if isinstance(n_parts, bool) or not isinstance(n_parts, numbers.Integral) or not 1 <= int(n_parts) <= N:
        raise ValueError(f"metis_labels: n_parts must be an int in [1, N = {N}] (got {n_parts!r})")
    if isinstance(outer_radius, bool) or not isinstance(outer_radius, numbers.Real) or \
            not (math.isfinite(float(outer_radius)) and float(outer_radius) > 0):
        raise ValueError(f"metis_labels: outer_radius must be finite and > 0 (got {outer_radius!r})")
    dev = pos.device
    p = pos.detach().to(torch.float32).contiguous()
    if not bool(torch.isfinite(p).all()):
        raise ValueError("metis_labels: positions must be finite (the radius graph gives a node with an inf or NaN "
                         "coordinate no edges)")
    if int(n_parts) == 1:                                        # the reference's metis(): zeros, no METIS call
        return torch.zeros(N, dtype=torch.int64, device=dev)
    g, _ = radius_graph_csr(p, float(outer_radius), edge_attr_nf=0)
    xadj, adjncy = csr_sorted_i64(g)
    xadj_h = torch.empty(N + 1, dtype=torch.int64, pin_memory=True)
    adj_h = torch.empty(adjncy.numel(), dtype=torch.int64, pin_memory=True)
    with torch.cuda.device(dev):
        xadj_h.copy_(xadj, non_blocking=True)
        adj_h.copy_(adjncy, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
    part, _ = metis_recursive(xadj_h.numpy(), adj_h.numpy(), int(n_parts))
    part_h = torch.from_numpy(part).pin_memory()
    return part_h.to(dev, non_blocking=True)


def node_chunks(n_nodes: int, world_size: int, split_mode: str = "random", pos: Optional[Tensor] = None,
                generator=None, outer_radius: Optional[float] = None) -> List[Tensor]:
    """The node sets of the reference's partitioners, one int64 index tensor per rank: "random" = a host `randperm(n)` cut
    into P−1 chunks of ⌊n/P⌋ plus the remainder, in permutation order (distribute_graphs.py:26-30; host tensors);
    "kmeans" = `nonzero(kmeans_labels(pos) == i)`, nodes in index order (:188-198; on `pos.device`, needs `pos`);
    "spectral" = the same with `spectral_labels(pos)` (:201-223; world_size <= 16); "metis" = the same with
    `metis_labels(pos, world_size, outer_radius)` (:54-87; needs `outer_radius`)."""
    n = int(n_nodes)
    if split_mode == "random":
        idx = torch.randperm(n, generator=generator)             # on the host, as the reference (device == 'cpu')
        sizes = [n // world_size] * (world_size - 1)
        sizes.append(n - sum(sizes))
        return list(torch.split(idx, sizes))
    if split_mode in ("kmeans", "spectral", "metis"):
        if pos is None:
            raise ValueError(f"split_mode={split_mode!r} needs the positions")
        if split_mode == "metis":
            if outer_radius is None:
                raise ValueError("split_mode='metis' needs outer_radius (the radius of the graph METIS partitions)")
            labels = metis_labels(pos, world_size, outer_radius)
        else:
            labels = kmeans_labels(pos, world_size) if split_mode == "kmeans" else spectral_labels(pos, world_size)
        return [torch.nonzero(labels == i, as_tuple=False).flatten() for i in range(world_size)]
    raise ValueError(f"unsupported split_mode {split_mode!r} (random|kmeans|spectral|metis)")


def split_large_graph(pos: Tensor, x: Tensor, target: Tensor, vel: Tensor, attr: Optional[Tensor], radius: float,
                      world_size: int, split_mode: str = "random", special_nodes: Optional[Tensor] = None, generator=None,
                      edge_attr_nf: int = 2, outer_radius: Optional[float] = None) -> List[Dict[str, Tensor]]:
    """Device-side form of the reference's partitioners (datasets/distribute_graphs.py:17-51 random, :54-87 METIS,
    :118-143 k-means, :90-115 spectral): node chunks by a host `randperm` (P−1 chunks of ⌊N/P⌋ + remainder) or by METIS
    part (of the `outer_radius` graph), k-means or spectral cluster (`pos[cluster == i]`, nodes in index order), every
    chunk with its own radius graph (`radius`, the reference's inner_radius) built on the device as CSR, `edge_attr` =
    the edge length in `edge_attr_nf` columns (:44) and the GLOBAL `loc_mean` (:32).  Returns dicts with the reference's
    `Data` field names, `edge_index` being a `CSRGraph` (what `FastEGNN.forward` consumes directly)."""
    n = int(pos.shape[0])
    chunks = [c.to(pos.device) for c in node_chunks(n, world_size, split_mode, pos=pos, generator=generator,
                                                    outer_radius=outer_radius)]
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
