"""Oracle of the protein recipe (distegnn_b200.frames / distegnn_b200.protein): the reference's per-sample lines
(datasets/process_dataset.py:142-198) applied in torch on the CPU to a trajectory already in memory.

Two substitutions, none of them in the arithmetic of the node fields:
  * `MDAnalysis.Universe` -> the arrays themselves: `positions` [T, N, 3] float32 (every atom), `charges` [N] and the
    selection `ix` (what `select_atoms('backbone').ix` or `atoms.ix` give);
  * `distances.contact_matrix(loc_0, cutoff=r, returntype="sparse")` -> `contact_edges`, a `scipy.spatial.cKDTree`
    pair search with the distance recomputed in float64 and kept when strictly below r (contact_matrix's test), the
    diagonal left out (:178-179), in the sparse matrix's row-major order.

The test-time rotation and translation are not restated (FrameLoader's rotate / translate are tested on their own).
"""
from __future__ import annotations

import numpy as np
import torch
from scipy.spatial import cKDTree

from oracle.frames_oracle import cutoff_edge


def contact_edges(loc: np.ndarray, r: float) -> torch.Tensor:
    """All (i, j), i != j, ‖loc_i − loc_j‖ < r in float64: int64 [2, E], rows ascending, then columns."""
    p = np.asarray(loc, dtype=np.float64)
    pairs = cKDTree(p).query_pairs(r, output_type="ndarray")
    d = np.linalg.norm(p[pairs[:, 0]] - p[pairs[:, 1]], axis=1) if len(pairs) else np.zeros(0)
    pairs = pairs[d < r]
    ij = np.concatenate([pairs, pairs[:, ::-1]]) if len(pairs) else np.zeros((0, 2), dtype=np.int64)
    ij = ij[np.lexsort((ij[:, 1], ij[:, 0]))]
    return torch.from_numpy(np.ascontiguousarray(ij.T)).long()


def sample(positions: np.ndarray, charges: np.ndarray, ix: np.ndarray, t: int, delta_t: int, radius: float,
           cutoff_rate: float = 0.0):
    """One sample (frame t) with the reference's `Data` field names."""
    charges = torch.tensor(charges[ix]).float().unsqueeze(-1)                                     # :147
    frame_0, frame_t = t, t + delta_t                                                             # :149
    loc_0 = torch.tensor(positions[frame_0][ix])                                                  # :157-159
    vel_0 = torch.tensor(positions[frame_0 + 1][ix]) - loc_0
    loc_t = torch.tensor(positions[frame_t][ix])
    edge_index = contact_edges(loc_0.numpy(), radius)                                             # :177-181
    edge_index = cutoff_edge(edge_index, loc_0, cutoff_rate)                                      # :184
    edge_attr = torch.norm(loc_0[edge_index[0], :] - loc_0[edge_index[1], :], p=2, dim=1).unsqueeze(-1).repeat(1, 2)
    feat_node_velocity = torch.sqrt(torch.sum(vel_0 ** 2, dim=1)).unsqueeze(1)                    # :190-192
    node_feat = torch.cat([feat_node_velocity, charges / charges.max()], dim=1)
    loc_mean = torch.mean(loc_0, dim=0).unsqueeze(0)                                              # :195
    return dict(x=node_feat, pos=loc_0, vel=vel_0, attr=charges, target=loc_t, loc_mean=loc_mean,
                edge_index=edge_index, edge_attr=edge_attr)
