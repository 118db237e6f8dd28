"""Oracle of the multi-step targets of distegnn_b200.frames.FrameLoader(horizon=K) and of the per-step error of
rollout(targets=...), in float64 on the CPU.

Every recipe's target is a recorded position (datasets/process_dataset.py: N-body `loc[frame_T]` :84, Water-3D and
Fluid113K `position[frame + delta_t]` :252, :507); a K-step horizon repeats that line for frame + tΔ, t = 1..K.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

Tensor = torch.Tensor


def targets(recipe: str, position: Tensor, frame: int, delta_t: int, horizon: int,
            index: Optional[Tensor] = None) -> Tensor:
    """float64 [horizon, m, 3]: the scene's positions at frame + tΔ, t = 1..horizon, of the nodes `index` (all: None)."""
    if recipe not in ("nbody", "water3d", "largefluid"):
        raise ValueError(recipe)
    T = position.shape[0]
    rows = []
    for t in range(1, horizon + 1):
        f = frame + t * delta_t
        if not 0 <= f < T:
            raise ValueError(f"frame {f} outside the scene's {T} frames")
        p = position[f].double()
        rows.append(p if index is None else p[index])
    return torch.stack(rows)


def sq_err(pred: Tensor, target: Tensor, batch: Optional[Tensor], n_graphs: int) -> Tensor:
    """float64 [n_graphs]: Σ over graph b's rows of ‖pred − target‖², from the float32 differences (the rollout's
    definition), squared in float64 and summed correctly rounded (math.fsum: a sequential float64 sum of millions of
    terms is itself off by ~1e-12)."""
    d = (pred.float() - target.float()).double()
    per = (d * d).sum(1).cpu().numpy()
    b = np.zeros(pred.shape[0], dtype=np.int64) if batch is None else batch.cpu().long().numpy()
    out = torch.zeros(n_graphs, dtype=torch.float64)
    for g in range(n_graphs):
        out[g] = math.fsum(per[b == g].tolist())
    return out
