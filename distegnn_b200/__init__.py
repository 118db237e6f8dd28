"""distegnn_b200 — H100-native (sm_90a) implementation of the DistEGNN hot path.

Public surface mirrors the reference: ``from distegnn_b200 import FastEGNN`` is a drop-in for
``from models.FastEGNN import FastEGNN``.
"""
from .fast_egnn import E_GCL_vel, FastEGNN  # noqa: F401
from .loss import chamfer_distance, train_loss  # noqa: F401  (fused weighted-MSE + MMD loss, SURVEY §8 f-3; DESIGN §21)
from .partition import cutoff_edges_csr, kmeans_labels, metis_labels, radius_graph, radius_graph_csr, split_large_graph  # noqa: F401  (CSR out, no host round trip)
from .spectral import spectral_labels  # noqa: F401  (the spectral partitioner, DESIGN §10)
from .rollout import RolloutResult, differentiable_rollout, rollout  # noqa: F401  (multi-step, on the device)

__all__ = ["FastEGNN", "E_GCL_vel", "radius_graph", "radius_graph_csr", "kmeans_labels", "spectral_labels", "metis_labels", "split_large_graph",
           "train_loss", "chamfer_distance", "rollout", "RolloutResult",
           "differentiable_rollout", "cutoff_edges_csr"]
