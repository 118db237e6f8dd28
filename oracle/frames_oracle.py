"""Oracle of distegnn_b200.frames: the reference's per-sample lines (datasets/process_dataset.py, distribute_graphs.py),
applied verbatim in torch on the CPU.

Three substitutions, none of them in the arithmetic of the node fields:
  * `torch_geometric.nn.radius_graph` -> `radius_edges`, a brute-force float64 pair test (< r) grouped by destination;
  * the random split's `torch.randperm(n)` takes a `generator` (the loader seeds one per sample);
  * the k-means split is the reference's `kmeans_clustering` (sklearn KMeans, random_state=0) itself.

`sample(...)` returns one dict per rank with the reference's `Data` field names.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

Tensor = torch.Tensor


def radius_edges(pos: Tensor, r: float) -> Tensor:
    """All (i, j), i != j, ‖pos_i − pos_j‖ < r (float64), row-major: int64 [2,E] with edge_index[0] = i ascending."""
    p = pos.double()
    ok = torch.cdist(p, p) < r
    ok &= ~torch.eye(pos.shape[0], dtype=torch.bool)
    i, j = ok.nonzero(as_tuple=True)
    return torch.stack([i, j])


def complete_edges(num_nodes: int) -> Tensor:
    edge_index = [[i, j] for i in range(num_nodes) for j in range(num_nodes) if i != j]     # process_dataset.py:98
    return torch.tensor(edge_index, dtype=torch.long).reshape(-1, 2).T


def cutoff_edge(edge_index, pos, cutoff_rate):                                               # process_dataset.py:300-305
    edge_dist = torch.norm(pos[edge_index[0]] - pos[edge_index[1]], p=2, dim=1)
    _, id_chosen = torch.sort(edge_dist)
    id_chosen = id_chosen[:int(id_chosen.size(0) * (1 - cutoff_rate))]
    edge_index = edge_index[:, id_chosen]
    return edge_index


def kmeans_clustering(pos, num_parts):                                                     # distribute_graphs.py:188-198
    from sklearn.cluster import KMeans
    X = pos.detach().cpu().numpy().astype(np.float32)
    kmeans = KMeans(n_clusters=num_parts, random_state=0, n_init="auto")
    labels = kmeans.fit_predict(X)
    return torch.from_numpy(labels).to(torch.long)


def node_fields(recipe: str, position: Tensor, velocity: Optional[Tensor], static: Dict[str, Tensor], frame: int,
                delta_t: int):
    """(pos, x, vel, attr, target, loc_mean) of one sample over the whole scene."""
    if recipe == "nbody":                                                                    # :82-84, :107-112
        loc_0, loc_t, vel_0 = position[frame], position[frame + delta_t], velocity[frame]
        charges = static["charges"].reshape(-1, 1).float()
        feat_node_velocity = torch.sqrt(torch.sum(vel_0 ** 2, dim=1)).unsqueeze(1)
        node_feat = torch.cat([feat_node_velocity, charges / charges.max()], dim=1)
        return loc_0, node_feat, vel_0, charges, loc_t, torch.mean(loc_0, dim=0).unsqueeze(0)
    if recipe == "water3d":                                                                  # :251-274, :345-346
        particle_type = static["particle_type"].float().reshape(-1).unsqueeze(-1)
        loc_0, loc_t = position[frame, :, :], position[frame + delta_t, :, :]
        vel_frame = position[frame + 1, :, :] - position[frame, :, :]
        node_feat = torch.cat([torch.sqrt(torch.sum(vel_frame ** 2, dim=-1)).unsqueeze(-1),
                               particle_type / particle_type.max()], dim=-1)
        return loc_0, node_feat, vel_frame, particle_type, loc_t, torch.mean(loc_0, dim=0).unsqueeze(0)
    if recipe == "largefluid":                                                               # :504-505
        viscosity, mass = static["viscosity"].float().reshape(-1), static["mass"].float().reshape(-1)
        node_attr = torch.stack([viscosity, mass], dim=-1)
        node_feat = torch.cat([node_attr, torch.sqrt(torch.sum(velocity[frame] ** 2, dim=-1)).unsqueeze(-1)], dim=-1)
        loc_0 = position[frame, :, :]
        return (loc_0, node_feat, velocity[frame], node_attr, position[frame + delta_t, :, :],
                torch.mean(loc_0, dim=0).unsqueeze(0))
    raise ValueError(recipe)


def sample(recipe: str, position: Tensor, velocity: Optional[Tensor], static: Dict[str, Tensor], frame: int,
           delta_t: int, radius: Optional[float], cutoff_rate: float = 0.0, world_size: int = 1,
           split_mode: str = "random", generator=None) -> List[Dict[str, Tensor]]:
    pos, x, vel, attr, target, loc_mean = node_fields(recipe, position, velocity, static, frame, delta_t)
    node_cnt = pos.size(0)
    if world_size == 1:
        chunks = [torch.arange(node_cnt)]
    elif split_mode == "random":                                                             # distribute_graphs.py:26-30
        indices = torch.randperm(node_cnt, generator=generator)
        chunk_sizes = [node_cnt // world_size for _ in range(world_size - 1)]
        chunk_sizes.append(node_cnt - sum(chunk_sizes))
        chunks = list(torch.split(indices, chunk_sizes))
    elif split_mode == "kmeans":                                                             # :123-133
        cluster = kmeans_clustering(pos, world_size)
        chunks = [torch.nonzero(cluster == i).flatten() for i in range(world_size)]
    else:
        raise ValueError(split_mode)
    out = []
    for ch in chunks:
        pos_i = pos[ch]
        n_i = pos_i.size(0)
        edge_index = complete_edges(n_i) if radius is None else radius_edges(pos_i, radius)
        if cutoff_rate > 0:
            edge_index = cutoff_edge(edge_index, pos_i, cutoff_rate)
        edge_attr = torch.norm(pos_i[edge_index[0], :] - pos_i[edge_index[1], :], p=2, dim=1).unsqueeze(-1).repeat(1, 2)
        out.append(dict(x=x[ch], pos=pos_i, vel=vel[ch], attr=attr[ch], target=target[ch], loc_mean=loc_mean,
                        edge_index=edge_index, edge_attr=edge_attr, index=ch))
    return out
