"""Synthetic particle graphs and partitioners for tests and ``bench.py``.

The datasets of the reference are not redistributable/offline, so every workload here is a seeded
synthetic restatement of what the reference's data pipeline hands to ``FastEGNN.forward``:

* point clouds sized like BASELINE.json's configs (SURVEY §8d),
* ``radius_graph(pos, r, loop=False, max_num_neighbors=N)`` as used at
  ``datasets/distribute_graphs.py:43`` (all ordered pairs with ‖Δx‖ < r, both directions),
* ``edge_attr`` = the edge length duplicated into two columns (``distribute_graphs.py:44``),
* ``loc_mean`` = centroid of the *whole* graph, shared by all partitions (``distribute_graphs.py:32``),
* ``split_mode=random`` (``distribute_graphs.py:26-30``), ``split_mode=kmeans``
  (``distribute_graphs.py:118-143,188-198``), ``split_mode=spectral`` (``:90-115,201-223``) and
  ``split_mode=metis`` (``:54-87,151-185``) node partitioning with per-partition radius graphs
  (cross-partition edges are dropped, as in the reference).

CPU/numpy only — this is input preparation, not part of the measured path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch


@dataclass
class Workload:
    """Model dims + graph recipe of one BASELINE.json config."""
    name: str
    n_nodes: int
    radius: Optional[float]      # None = fully connected
    degree: float                # expected degree used to size the box
    node_feat_nf: int
    node_attr_nf: int
    edge_attr_nf: int
    virtual_channels: int
    normalize: bool


# BASELINE.json configs (SURVEY §8 table)
WORKLOADS: Dict[str, Workload] = {
    "nbody100": Workload("nbody100", 100, None, 99.0, 2, 0, 2, 3, True),
    "water3d_10k": Workload("water3d_10k", 10_000, 0.035, 12.2, 2, 0, 2, 3, False),
    "fluid113k": Workload("fluid113k", 113_140, 0.075, 15.1, 3, 2, 2, 5, False),
    "synth1m": Workload("synth1m", 1_000_000, 0.075, 21.0, 3, 2, 2, 8, False),
}


def box_side(n: int, r: float, degree: float) -> float:
    """Side L of the cube such that uniform points have the expected degree: n·(4/3)πr³/L³ = d."""
    return (n * (4.0 / 3.0) * math.pi * r ** 3 / degree) ** (1.0 / 3.0)


def radius_graph_np(pos: np.ndarray, r: float) -> np.ndarray:
    """All ordered pairs (i,j), i≠j, ‖x_i−x_j‖<r → int64 [2,E].  Ordered like PyG's radius_graph
    output is *not* required by FastEGNN (it scatters by edge_index[0]); we emit pairs grouped by
    the second row (the 'col'/source), mimicking radius_graph's sort-by-target convention so that
    edge_index[0] is unsorted — the CSR build must not assume sortedness."""
    from scipy.spatial import cKDTree
    if pos.shape[0] == 0:
        return np.zeros((2, 0), dtype=np.int64)
    tree = cKDTree(pos)
    pairs = tree.query_pairs(r, output_type="ndarray")          # i<j, unique
    if pairs.size == 0:
        return np.zeros((2, 0), dtype=np.int64)
    src = np.concatenate([pairs[:, 0], pairs[:, 1]])
    dst = np.concatenate([pairs[:, 1], pairs[:, 0]])
    order = np.argsort(dst, kind="stable")                       # group by edge_index[1]
    return np.stack([src[order], dst[order]]).astype(np.int64)


def fully_connected_np(n: int) -> np.ndarray:
    """[(i,j) for i for j if i≠j] as the N-body pipeline builds it (process_dataset.py:98-99)."""
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    m = i != j
    return np.stack([i[m], j[m]]).astype(np.int64)


def make_points(w: Workload, seed: int = 0, n_nodes: Optional[int] = None) -> Dict[str, np.ndarray]:
    """Seeded node arrays of one whole (un-partitioned) graph."""
    n = w.n_nodes if n_nodes is None else n_nodes
    rng = np.random.default_rng(seed)
    if w.radius is None:                                         # N-body-like
        pos = rng.normal(0.0, 2.8, size=(n, 3))
        vel = rng.normal(size=(n, 3))
        vel *= 0.5 / np.linalg.norm(vel, axis=1, keepdims=True)
    else:
        side = box_side(n, w.radius, w.degree)
        pos = rng.uniform(0.0, side, size=(n, 3))
        vel = rng.normal(0.0, 0.01, size=(n, 3))
    feat = rng.normal(size=(n, w.node_feat_nf))
    attr = rng.normal(size=(n, w.node_attr_nf))
    return dict(pos=pos.astype(np.float32), vel=vel.astype(np.float32),
                feat=feat.astype(np.float32), attr=attr.astype(np.float32))


def _graph_inputs(pos, vel, feat, attr, loc_mean, radius, edge_attr_nf) -> Dict[str, torch.Tensor]:
    ei = fully_connected_np(pos.shape[0]) if radius is None else radius_graph_np(pos, radius)
    d = np.sqrt(((pos[ei[0]] - pos[ei[1]]) ** 2).sum(-1, dtype=np.float32)).astype(np.float32)
    ea = np.repeat(d[:, None], edge_attr_nf, axis=1)
    n = pos.shape[0]
    return dict(
        node_feat=torch.from_numpy(feat), node_loc=torch.from_numpy(pos),
        node_vel=torch.from_numpy(vel), loc_mean=torch.from_numpy(loc_mean),
        edge_index=torch.from_numpy(ei), data_batch=torch.zeros(n, dtype=torch.long),
        edge_attr=torch.from_numpy(np.ascontiguousarray(ea)),
        node_attr=torch.from_numpy(attr) if attr.shape[1] > 0 else None)


def random_partition(n: int, world_size: int, seed: int = 0) -> List[np.ndarray]:
    """distribute_graphs.py:26-30 — randperm, P−1 chunks of ⌊N/P⌋, remainder to the last."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(n, generator=g).numpy()
    sizes = [n // world_size] * (world_size - 1)
    sizes.append(n - sum(sizes))
    out, o = [], 0
    for s in sizes:
        out.append(idx[o:o + s])
        o += s
    return out


def kmeans_partition(pos: np.ndarray, world_size: int) -> List[np.ndarray]:
    """distribute_graphs.py:188-198 — sklearn KMeans(n_clusters=P, random_state=0, n_init='auto')
    on float32 positions; partition i = nodes with label i, in index order (``pos[cluster == i]``)."""
    from sklearn.cluster import KMeans
    labels = KMeans(n_clusters=world_size, random_state=0, n_init="auto").fit_predict(
        pos.astype(np.float32))
    return [np.nonzero(labels == i)[0] for i in range(world_size)]


def spectral_partition(pos: np.ndarray, world_size: int) -> List[np.ndarray]:
    """distribute_graphs.py:201-223 — sklearn SpectralClustering(n_clusters=P, affinity='rbf', gamma=1/(2σ²),
    assign_labels='kmeans', random_state=0, eigen_solver='arpack') on float32 positions, σ the median nonzero distance
    among min(N, 2000) nodes drawn by RandomState(0), plus 1e-12; partition i = nodes with label i, in index order.
    Forms the dense N×N affinity (51 GB at 113,140 nodes): a host restatement for tests and small
    benchmarks; ``make_partitions(..., device=...)`` uses the device partitioner instead."""
    from sklearn.cluster import SpectralClustering
    X = pos.astype(np.float32)
    n = X.shape[0]
    idx = np.random.RandomState(0).choice(n, size=min(n, 2000), replace=False)
    D = np.linalg.norm(X[idx, None, :] - X[None, idx, :], axis=2)
    sigma = np.median(D[D > 0]) + 1e-12
    sc = SpectralClustering(n_clusters=world_size, affinity="rbf", gamma=1.0 / (2.0 * (sigma ** 2)),
                            assign_labels="kmeans", random_state=0, eigen_solver="arpack")
    labels = sc.fit_predict(X)
    return [np.nonzero(labels == i)[0] for i in range(world_size)]


def metis_csr_np(pos: np.ndarray, outer_radius: float):
    """(xadj, adjncy) int64 of the reference's METIS input (distribute_graphs.py:66-67, 155-157): the pairs of
    ``radius_graph_np(pos, outer_radius)`` lexsorted by (row, col), the row counts as a pointer array."""
    n = pos.shape[0]
    ei = radius_graph_np(pos, outer_radius)
    order = np.lexsort((ei[1], ei[0]))
    xadj = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(ei[0], minlength=n), out=xadj[1:])
    return xadj, np.ascontiguousarray(ei[1][order], dtype=np.int64)


def metis_partition(pos: np.ndarray, world_size: int, outer_radius: float) -> List[np.ndarray]:
    """distribute_graphs.py:54-87, 151-185 — ``METIS_PartGraphRecursive`` (the library's
    ``distegnn_metis_recursive``, the toolkit's METIS) on the cKDTree outer-radius graph ``metis_csr_np``;
    partition i = nodes with label i, in index order (``pos[cluster == i]``).  The host restatement of
    ``distegnn_b200.metis_labels``: the same C call on a graph built without the device."""
    from .partition import metis_recursive
    xadj, adjncy = metis_csr_np(pos, outer_radius)
    labels, _ = metis_recursive(xadj, adjncy, world_size)
    return [np.nonzero(labels == i)[0] for i in range(world_size)]


def make_partitions(w: Workload, world_size: int = 1, split_mode: str = "random", seed: int = 0,
                    n_nodes: Optional[int] = None, only_rank: Optional[int] = None, device=None,
                    outer_radius: Optional[float] = None) -> List[Optional[Dict[str, torch.Tensor]]]:
    """One input dict per partition (= per rank), each with the forward() argument names.

    ``only_rank`` builds the (expensive) radius graph for that rank only and leaves ``None``
    elsewhere — every rank of a torchrun job calls this with its own rank and the same seed.
    ``device`` (a CUDA device) takes the spectral split's labels from the device partitioner
    (``distegnn_b200.spectral_labels``, O(N) memory) instead of the dense host restatement,
    which only suits small clouds; the other modes ignore it.  ``outer_radius`` is the radius of the
    graph the metis split partitions (default: the workload's radius).
    """
    pts = make_points(w, seed, n_nodes)
    n = pts["pos"].shape[0]
    loc_mean = pts["pos"].mean(axis=0, keepdims=True, dtype=np.float64).astype(np.float32)
    if world_size == 1:
        chunks = [np.arange(n)]
    elif split_mode == "random":
        chunks = random_partition(n, world_size, seed)
    elif split_mode == "kmeans":
        chunks = kmeans_partition(pts["pos"], world_size)
    elif split_mode == "spectral" and device is not None:
        from .partition import node_chunks
        pos = torch.from_numpy(pts["pos"]).to(device)
        chunks = [c.cpu().numpy() for c in node_chunks(n, world_size, "spectral", pos=pos)]
    elif split_mode == "spectral":
        chunks = spectral_partition(pts["pos"], world_size)
    elif split_mode == "metis":
        chunks = metis_partition(pts["pos"], world_size, w.radius if outer_radius is None else outer_radius)
    else:
        raise ValueError(f"unsupported split_mode {split_mode!r} (random|kmeans|spectral|metis)")
    out: List[Optional[Dict[str, torch.Tensor]]] = []
    for r, idx in enumerate(chunks):
        if only_rank is not None and r != only_rank:
            out.append(None)
            continue
        out.append(_graph_inputs(pts["pos"][idx], pts["vel"][idx], pts["feat"][idx], pts["attr"][idx],
                                 loc_mean, w.radius, w.edge_attr_nf))
    return out
