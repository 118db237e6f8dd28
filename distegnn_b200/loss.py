"""Loss side of the reference's training step (utils/train.py:98-147), fused (SURVEY §8 f-3).

    loss, info = distegnn_b200.train_loss(loc_pred, loc_target, virtual_node_loc, batch, world_size=..., mmd_samples=50,
                                          mmd_sigma=3, mmd_weight=0.01, accumulation_steps=4, loc_mean=loc_mean)
    loss.backward()

computes what the reference computes between the model call and `loss_loc.backward()`:

  * node-count weighted MSE  `world_size · n_r/Σn · MSE(loc_pred, loc_target)`                        (train.py:98-110)
  * the MMD regulariser between the virtual coordinates and `mmd_samples·C` sampled target positions per graph, kernel
    `exp(−‖x−y‖/(2σ²))`                                                                               (train.py:11-14, 119-147)
  * the per-step collectives — total node count (:104), logged loss (:109), `loc_mean` consistency check (:52-61) —
    folded into ONE packed SUM all-reduce

in two kernel launches + one collective (csrc/loss.cu) instead of a Python loop over the graphs with ~20 ATen launches
each and three collectives; the forward already produces the gradients w.r.t. `loc_pred` and `virtual_node_loc`, the
backward only scales them by the incoming gradient.  Sampling follows the reference exactly — one
`torch.randperm(num_node)[:S]` per graph on the global CPU generator, in graph order — unless `samples` is passed in.
CUDA only (no CPU path); `info` holds device scalars (`logged`, `mmd`, `loc_mean_dev`) — reading them synchronises.
Given [K,N,3] positions and [K,B,3,C] virtual coordinates (a rollout's `trajectory` and `virtual_locs`), it is the mean
of the K one-step losses in the same two launches and one collective (DESIGN §26).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import check, ptr

Tensor = torch.Tensor


def graph_offsets(batch: Tensor, n_graphs: int) -> Tensor:
    """[B+1] int64 first-node offsets of a sorted `batch` vector (device, no host sync)."""
    return torch.searchsorted(batch.contiguous(), torch.arange(n_graphs + 1, device=batch.device, dtype=batch.dtype))


def draw_samples(node_counts: Sequence[int], num_sample: int) -> Tensor:
    """The reference's sampling (train.py:124-129): `torch.randperm(num_node)[:num_sample]` per graph, in graph order, on
    the global CPU generator → int32 [B, num_sample] of graph-local indices, −1 where a graph has fewer nodes."""
    out = torch.full((len(node_counts), num_sample), -1, dtype=torch.int32)
    for i, n in enumerate(node_counts):
        idx = torch.randperm(int(n))[:num_sample]
        out[i, :idx.numel()] = idx.to(torch.int32)
    return out


class _TrainLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, Xv, target, gptr, samples, loc_mean, cfg):
        lib = _lib.load()
        dev = pred.device
        K = cfg["steps"]                                     # None: the one-step [N,3] call
        N, (B, _, Cn) = int(pred.shape[-2]), Xv.shape[-3:]
        S, world, rank = int(samples.shape[-1]), cfg["world"], cfg["rank"]
        stream = _lib.stream_ptr(dev)
        npk = lib.distegnn_loss_packed_floats(B, world) if K is None else lib.distegnn_loss_packed_floats_steps(K, B, world)
        na = 3 * (K or 1)
        scratch = torch.zeros(na + npk, dtype=torch.float32, device=dev)         # acc[3K] | packed[npk]
        acc, packed = scratch[:na], scratch[na:]
        gV_raw = torch.empty(Xv.shape, dtype=torch.float32, device=dev)
        p, t, xv = pred.detach().contiguous(), target.contiguous(), Xv.detach().contiguous()
        with torch.cuda.device(dev):
            args = (N, B, Cn, S, world, rank, cfg["sigma"], ptr(p), ptr(t), ptr(xv), ptr(loc_mean), ptr(gptr),
                    ptr(samples), ptr(acc), ptr(packed), ptr(gV_raw), stream)
            check(lib.distegnn_loss_partials(*args) if K is None else lib.distegnn_loss_partials_steps(K, *args),
                  "loss_partials")
            if world > 1:                                    # the ONE collective of the call (all K steps)
                comm, be = cfg.get("comm"), cfg.get("backend")
                if comm is not None and be is not None and npk <= comm.max_slots * comm.slot_floats:
                    be.allreduce_packed(comm, packed)
                else:
                    import torch.distributed as dist
                    dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=cfg.get("group"))
            g_pred = torch.empty_like(p)
            g_Xv = torch.empty_like(xv)
            out = torch.empty(4 + 2 * (K or 0), dtype=torch.float32, device=dev)
            args = (N, B, Cn, S, world, rank, cfg["sigma"], cfg["weight"], cfg["accum"], ptr(p), ptr(t), ptr(loc_mean),
                    ptr(acc), ptr(packed), ptr(gV_raw), ptr(g_pred), ptr(g_Xv), ptr(out))
            check(lib.distegnn_loss_finalize(*args, stream) if K is None else
                  lib.distegnn_loss_finalize_steps(K, *args, ptr(out[4:]), stream), "loss_finalize")
        ctx.save_for_backward(g_pred, g_Xv)
        ctx.mark_non_differentiable(out)
        return out[0].clone(), out

    @staticmethod
    def backward(ctx, g_loss, _g_out):
        g_pred, g_Xv = ctx.saved_tensors
        return g_loss * g_pred, g_loss * g_Xv, None, None, None, None, None


def train_loss(loc_pred: Tensor, loc_target: Tensor, virtual_node_loc: Tensor, batch: Tensor, *, world_size: int = 1,
               mmd_samples: int = 50, mmd_sigma: float = 3.0, mmd_weight: float = 0.01, accumulation_steps: int = 1,
               loc_mean: Optional[Tensor] = None, samples: Optional[Tensor] = None,
               node_counts: Optional[Sequence[int]] = None, process_group=None, model=None
               ) -> Tuple[Tensor, Dict[str, Tensor]]:
    """See the module docstring.  `node_counts` (host ints per graph, e.g. from the loader's `ptr`) avoids the one host
    sync needed to size the reference's `randperm` draws; `samples` (int32 [B,S], graph-local, −1 padded) overrides the
    draw; `model` (a distegnn_b200.FastEGNN of a multi-partition job) lends its peer-memory communicator to the
    collective.

    Stepped (K steps of a rollout, DESIGN §26): loc_pred, loc_target [K,N,3], virtual_node_loc [K,B,3,C], samples
    [K,B,S].  The loss is (1/K)·Σ_t ℓ_t, ℓ_t the one-step loss of step t (its MSE, and the MMD of virtual_node_loc[t]
    against samples of loc_target[t]), in one partials launch, one packed all-reduce and one finalize launch; the
    gradients are [K,N,3] and [K,B,3,C].  info["logged"] and info["mmd"] are the means over the steps,
    info["logged_steps"] and info["mmd_steps"] float32 [K] the values of every step.  The default samples are
    `draw_samples` once per step, in step order, so K = 1 draws what the one-step call draws and gives its bits.  With
    several ranks the packed vector has 1 + K + world·3B floats; when it is larger than the model's communicator holds
    (max_slots·slot_floats), the exchange goes through torch.distributed as without a communicator."""
    if loc_pred.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.train_loss runs only on CUDA tensors (no CPU path)")
    stepped = loc_pred.dim() == 3
    if stepped:
        if loc_pred.shape != loc_target.shape or loc_pred.shape[2] != 3 or loc_pred.shape[0] < 1:
            raise ValueError("stepped loc_pred / loc_target must both be [K,N,3], K >= 1")
        if virtual_node_loc.dim() != 4 or virtual_node_loc.shape[2] != 3 or \
                virtual_node_loc.shape[0] != loc_pred.shape[0]:
            raise ValueError(f"stepped virtual_node_loc must be [K={loc_pred.shape[0]},B,3,C]")
    else:
        if loc_pred.shape != loc_target.shape or loc_pred.dim() != 2 or loc_pred.shape[1] != 3:
            raise ValueError("loc_pred / loc_target must both be [N,3]")
        if virtual_node_loc.dim() != 3 or virtual_node_loc.shape[1] != 3:
            raise ValueError("virtual_node_loc must be [B,3,C]")
    dev = loc_pred.device
    K = int(loc_pred.shape[0]) if stepped else None
    B, _, Cn = virtual_node_loc.shape[-3:]
    if Cn > _lib.MAX_CHANNELS:
        raise ValueError(f"virtual_channels={Cn} exceeds the compiled limit {_lib.MAX_CHANNELS}")
    S = int(mmd_samples) * Cn                                      # train.py:122
    gptr = graph_offsets(batch, B)
    if samples is None:
        if node_counts is None:
            node_counts = (gptr[1:] - gptr[:-1]).tolist()          # one host sync (the reference has B of them)
        samples = draw_samples(node_counts, S) if not stepped else \
            torch.stack([draw_samples(node_counts, S) for _ in range(K)])
    samples = samples.to(device=dev, dtype=torch.int32).contiguous()
    want = (B, S) if not stepped else (K, B, S)
    if samples.shape != want:
        raise ValueError(f"samples must be [{'K=%d, ' % K if stepped else ''}B={B}, S={S}]")
    rank = 0
    if world_size > 1:
        import torch.distributed as dist
        rank = dist.get_rank(process_group)
    cfg = dict(world=int(world_size), rank=rank, sigma=float(mmd_sigma), weight=float(mmd_weight),
               accum=int(accumulation_steps), group=process_group, steps=K)
    if model is not None and getattr(model, "_comm", None):
        from .backend import cuda_backend
        cfg["comm"], cfg["backend"] = model._comm, cuda_backend()
    lm = None if loc_mean is None else loc_mean.detach().to(torch.float32).contiguous()
    loss, out = _TrainLoss.apply(loc_pred.to(torch.float32), virtual_node_loc.to(torch.float32),
                                 loc_target.detach().to(torch.float32), gptr, samples, lm, cfg)
    info = {"logged": out[1], "mmd": out[2], "loc_mean_dev": out[3], "samples": samples}
    if stepped:
        info["logged_steps"], info["mmd_steps"] = out[4:4 + K], out[4 + K:]
    return loss, info


class _ChamferDistance(torch.autograd.Function):
    """Forward: distegnn_chamfer_distance (the sums and each minimum's nearest id); backward: distegnn_chamfer_distance_bwd
    on those ids.  See DESIGN §21."""

    @staticmethod
    def forward(ctx, pred, target, batch, B):
        from .backend import cuda_backend
        be = cuda_backend()
        dev, N = pred.device, int(pred.shape[0])
        p, t = pred.detach(), target.detach()
        out = torch.empty(B, 2, dtype=torch.float64, device=dev)
        nearest = torch.empty(2 * N, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            be.chamfer_distance(p, t, batch, out, nearest, be.rollout_chamfer_workspace(N, B, dev))
        ctx.save_for_backward(p, t, nearest, batch)
        return out

    @staticmethod
    def backward(ctx, g):
        from .backend import cuda_backend
        be = cuda_backend()
        p, t, nearest, batch = ctx.saved_tensors
        g_pred = torch.empty_like(p) if ctx.needs_input_grad[0] else None
        g_target = torch.empty_like(t) if ctx.needs_input_grad[1] else None
        if g_pred is not None or g_target is not None:
            with torch.cuda.device(p.device):
                be.chamfer_distance_bwd(p, t, batch, nearest, g.to(torch.float64).contiguous(), g_pred, g_target,
                                        be.chamfer_distance_bwd_workspace(int(p.shape[0]), p.device))
        return g_pred, g_target, None, None


def chamfer_distance(pred: Tensor, target: Tensor, data_batch: Optional[Tensor] = None,
                     n_graphs: Optional[int] = None) -> Tensor:
    """Differentiable per-graph Chamfer distance of two clouds with the same rows (DESIGN §21) -> float64 [B, 2]:

        out[b, 0] = Σ_{i in graph b} min_{j in graph b} d(pred_i, target_j)      (prediction -> record)
        out[b, 1] = Σ_{j in graph b} min_{i in graph b} d(target_j, pred_i)      (record -> prediction)

    with d the rollout's per-node squared error (fp32 differences, fp64 squares and sums), bit for bit one step of
    `rollout(..., chamfer=True)`.  pred, target: contiguous float32 [N,3] CUDA tensors, row i of both node i;
    data_batch: sorted int64 [N] (None: one graph).  A graph without nodes gives 0, a graph with a non-finite coordinate
    NaN (and NaN gradient rows).  The gradient flows to whichever of pred and target requires it, in a fixed order with no
    floating-point atomics, so it is bitwise reproducible.  n_graphs=None reads data_batch.max() + 1 once (a host sync);
    with n_graphs given, neither the forward nor the backward synchronises.  With several ranks the value and the
    gradients are this rank's partition-local ones.  Memory is O(N + B): nothing of N² size."""
    for name, x in (("pred", pred), ("target", target)):
        if not isinstance(x, torch.Tensor):
            raise ValueError(f"{name} must be a tensor")
        if x.dtype != torch.float32:
            raise ValueError(f"{name} must be float32 (got {x.dtype})")
        if x.dim() != 2 or x.shape[1] != 3:
            raise ValueError(f"{name} must be [N,3] (got {list(x.shape)})")
        if not x.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    if pred.shape[0] != target.shape[0]:
        raise ValueError(f"pred and target must have the same rows (got {pred.shape[0]} and {target.shape[0]})")
    N = int(pred.shape[0])
    if data_batch is not None:
        if not isinstance(data_batch, torch.Tensor) or data_batch.dtype != torch.int64 or data_batch.shape != (N,):
            raise ValueError(f"data_batch must be an int64 [N={N}] tensor")
        if not data_batch.is_contiguous():
            raise ValueError("data_batch must be contiguous")
    if n_graphs is not None and (isinstance(n_graphs, bool) or not isinstance(n_graphs, int) or n_graphs < 1):
        raise ValueError(f"n_graphs must be an int >= 1 (got {n_graphs!r})")
    if data_batch is None and n_graphs is not None and n_graphs > 1:
        raise ValueError("n_graphs > 1 needs data_batch")
    for name, x in (("pred", pred), ("target", target), ("data_batch", data_batch)):
        if x is not None and x.device.type != "cuda":
            raise ValueError(f"{name} must be a CUDA tensor (distegnn_b200 has no CPU path)")
        if x is not None and x.device != pred.device:
            raise ValueError(f"{name} is on {x.device}, pred on {pred.device}")
    if n_graphs is None:
        n_graphs = 1 if data_batch is None or N == 0 else int(data_batch.max()) + 1
    return _ChamferDistance.apply(pred, target, data_batch, int(n_graphs))
