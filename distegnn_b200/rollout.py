"""Multi-step inference: feed the model's prediction back in, rebuild the graph, repeat — on the device.

    res = rollout(model, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr=None, *,
                  steps, radius=None, graph=None, loop=False, tau=1.0, speed_col=None,
                  capacity=None, check_every=None, return_trajectory=False, targets=None, chamfer=False)

Step t -> t+1 restates the reference's data pipeline on predicted positions (DESIGN §14):
  x_{t+1} = the model's output;  v_{t+1} = (x_{t+1} − x_t) / tau (process_dataset.py:345);  node_feat[:, speed_col] =
  ‖v_{t+1}‖ (the |v| feature of each dataset; other columns and node_attr stay);  loc_mean = per-graph mean of x_{t+1}
  over all partitions (distribute_graphs.py:32);  graph = radius graph of x_{t+1} with edge_attr = length in every column
  (`radius`), or the caller's `graph` kept with only its edge_attr recomputed (`radius=None`, e.g. fully connected N-body).
Step 0 uses the caller's loc_mean; later steps take the centroid from the statistics the forward's first exchange already
sums (FLAG_INIT_CENTROID), so a step costs L+1 exchanges like a forward.  Nodes stay on their rank.

Per step: radius graph into fixed buffers with a capacity (no host read), the inference forward on a persistent
workspace, `distegnn_rollout_advance` (one launch).  The graph build's overflow flag is kept on the device; it is read
once per chunk of `check_every` steps (an OR over the ranks: every rank takes the same branch) and an overflowed chunk is
rerun from its saved start with the capacity grown to 1.25x the largest true edge count.  `check_every=0` defers the
check to `RolloutResult.check()`: the whole rollout is then enqueued without any host synchronisation.  With
`model.cuda_graph = True` the step is captured once (after the eager step 0) and replayed.

`cutoff_rate > 0` (FastEGNN's cutoff_edges mode, one device): each step's graph is the int(E_b·(1 − cutoff_rate))
shortest edges of every graph of the candidates above (process_dataset.py:103, `partition.cutoff_edges_csr`), re-selected
from the current lengths; the capacity and its regrowth count the candidates, `n_edges` the kept edges (DESIGN §16).

`targets` [steps,N,3] (recorded positions, e.g. from `FrameLoader(horizon=steps)`) adds the per-step, per-graph squared
error against them, computed inside the step (DESIGN §19): `sq_err`, `graph_nodes` and `mse` of the result.
`chamfer=True` adds the per-step, per-graph Chamfer distance to them, which does not pair node i with node i (DESIGN
§20): `chamfer` and `chamfer_mse` of the result.

`differentiable_rollout` (same arguments, without `targets`) runs the same steps and attaches `trajectory` and `virtual_locs` to autograd;
its backward recomputes one step at a time in reverse (DESIGN §15).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional

import torch

from . import _lib
from .fast_egnn import FastEGNN
from .partition import _check_rate
from .shards import CSRGraph

Tensor = torch.Tensor
GROWTH = 1.25              # capacity = GROWTH x edge count (initial build and every regrowth)
MAX_REGROWTHS = 4          # per chunk; then the rollout raises
_bwd_timing: Optional[list] = None   # benchmarks: a list receives (step, part, CUDA event) at each part of the backward


@dataclass
class RolloutResult:
    node_loc: Tensor                   # [N,3] state after `steps` steps
    node_vel: Tensor                   # [N,3]
    node_feat: Tensor                  # [N,F] (speed column updated)
    loc_mean: Tensor                   # [B,3] per-graph mean of node_loc over all partitions
    virtual_loc: Tensor                # [B,3,C] of the last step
    trajectory: Optional[Tensor]       # [steps,N,3] positions after each step, or None
    n_edges: Tensor                    # int32 [steps] on the device: edges of each step's graph
    capacity: Optional[int] = None     # final edge capacity of the rebuilt graph (radius mode)
    regrowths: List[int] = field(default_factory=list)   # capacities the graph buffers were grown to
    replays: int = 0                   # CUDA-graph replays (model.cuda_graph)
    status: Optional[Tensor] = None    # int32 device counter: [1] overflow flag, [2] first overflowing step, [3] max count

    graph: Optional[CSRGraph] = None   # the last step's graph (radius mode: capacity-sized, count in graph.n_edges_dev)
    edge_attr: Optional[Tensor] = None  # its edge_attr, in CSR order
    virtual_locs: Optional[Tensor] = None   # [steps,B,3,C] each step's virtual_loc (differentiable_rollout only)
    # with `targets` (rollout only), on the device:
    sq_err: Optional[Tensor] = None    # float64 [steps,B]: Σ over graph b's nodes of ‖x_{t+1} − targets[t]‖², all ranks
    graph_nodes: Optional[Tensor] = None   # int64 [B]: node counts over all ranks
    mse: Optional[Tensor] = None       # float64 [steps]: Σ_b sq_err[t] / (3 Σ_b graph_nodes), the training loss's MSE
    # with `targets` and chamfer=True: [t, b, 0] prediction -> record, [t, b, 1] record -> prediction
    chamfer: Optional[Tensor] = None   # float64 [steps,B,2]: Σ of nearest-neighbour d per graph, partition-local, all ranks
    chamfer_mse: Optional[Tensor] = None   # float64 [steps,2]: Σ_b chamfer[t,b,k] / (3 Σ_b graph_nodes) <= mse

    def check(self) -> None:
        """Raise if a graph build overflowed its capacity, or if the backward of a differentiable rollout rebuilt a graph
        that differs from the forward's (one host read).  Only needed with `check_every=0`, or after a backward."""
        s = self.status.tolist()
        if s[1]:
            raise RuntimeError(f"rollout: the radius graph first outgrew the capacity {self.capacity} at step {s[2]} (the "
                               f"largest edge count of any step was {max(s[3], s[6])}); the results from that step on are wrong — "
                               "pass a larger capacity or let rollout check (check_every > 0)")
        if s[5]:
            raise RuntimeError(f"differentiable_rollout: the backward rebuilt {s[5]} step graph(s) with another edge count "
                               "than the forward had; the gradients are wrong")


def _unwrap(model) -> FastEGNN:
    m = getattr(model, "module", model)
    if not isinstance(m, FastEGNN):
        raise TypeError(f"rollout needs a distegnn_b200.FastEGNN (or a DDP-wrapped one), got {type(model).__name__}")
    return m


def _validate(m: FastEGNN, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius, graph, tau,
              speed_col, capacity, check_every, cutoff_rate=0.0) -> None:
    is_int = lambda v: isinstance(v, int) and not isinstance(v, bool)
    _check_rate(cutoff_rate)
    if cutoff_rate > 0 and m.world_size > 1:
        raise ValueError("cutoff_rate > 0 is a single-device mode (the reference's cutoff_edges); with several ranks the "
                         "partitions already drop their cross edges")
    if not is_int(steps) or steps < 1:
        raise ValueError(f"steps must be an int >= 1 (got {steps!r})")
    if not tau > 0:
        raise ValueError(f"tau must be > 0 (got {tau!r})")
    if (radius is None) == (graph is None):
        raise ValueError("give exactly one of `radius` (rebuild the radius graph every step) and `graph` (keep it)")
    if radius is not None and not radius > 0:
        raise ValueError(f"radius must be > 0 (got {radius!r})")
    if graph is not None and not isinstance(graph, CSRGraph):
        raise ValueError("graph must be a distegnn_b200.shards.CSRGraph (e.g. from radius_graph_csr or "
                         "CSRGraph.from_edge_index)")
    if m.n_layers < 1:
        raise ValueError("rollout needs a model with at least one layer")
    F = m.node_feat_nf
    if speed_col is not None and not (is_int(speed_col) and 0 <= speed_col < F):
        raise ValueError(f"speed_col must be an int in [0, {F}) (got {speed_col!r})")
    if capacity is not None and not (is_int(capacity) and capacity > 0):
        raise ValueError(f"capacity must be a positive int (got {capacity!r})")
    if check_every is not None and not (is_int(check_every) and check_every >= 0):
        raise ValueError(f"check_every must be an int >= 0 (got {check_every!r})")
    N = int(node_loc.shape[0]) if node_loc.dim() == 2 else -1
    B = int(loc_mean.shape[0]) if loc_mean.dim() == 2 else -1
    if node_loc.shape != (N, 3) or node_vel.shape != (N, 3) or node_feat.shape != (N, F):
        raise ValueError(f"bad node tensor shapes: feat {tuple(node_feat.shape)}, loc {tuple(node_loc.shape)}, vel "
                         f"{tuple(node_vel.shape)}; expected N={N}, F={F}")
    if loc_mean.shape != (B, 3) or B < 1:
        raise ValueError("loc_mean must be [B,3], B >= 1")
    if data_batch.shape != (N,) or data_batch.dtype != torch.int64:
        raise ValueError("data_batch must be int64 [N]")
    if m.node_attr_nf > 0 and (node_attr is None or node_attr.shape != (N, m.node_attr_nf)):
        raise ValueError(f"node_attr must be [N,{m.node_attr_nf}]")
    if graph is not None and graph.num_nodes != N:
        raise ValueError(f"graph has {graph.num_nodes} nodes, node_loc has {N}")
    dev = node_loc.device
    for name, t in (("node_feat", node_feat), ("node_vel", node_vel), ("loc_mean", loc_mean), ("data_batch", data_batch),
                    ("node_attr", node_attr)):
        if t is not None and t.device != dev:
            raise ValueError(f"{name} is on {t.device}, node_loc on {dev}")
    if graph is not None and graph.rowptr.device != dev:
        raise ValueError(f"graph is on {graph.rowptr.device}, node_loc on {dev}")
    for name, t in (("node_feat", node_feat), ("node_loc", node_loc), ("node_vel", node_vel), ("loc_mean", loc_mean)):
        if not t.is_floating_point():
            raise ValueError(f"{name} must be a floating tensor")


def _check_targets(targets, steps: int, node_loc: Tensor, chamfer: bool = False) -> None:
    if not isinstance(chamfer, bool):
        raise ValueError(f"chamfer must be a bool (got {type(chamfer).__name__})")
    if targets is None:
        if chamfer:
            raise ValueError("chamfer=True needs targets: the Chamfer distance is taken against the recorded frames")
        return
    N = int(node_loc.shape[0])
    if not isinstance(targets, torch.Tensor):
        raise ValueError(f"targets must be a tensor (got {type(targets).__name__})")
    if targets.dtype != torch.float32:
        raise ValueError(f"targets must be float32 (got {targets.dtype})")
    if tuple(targets.shape) != (steps, N, 3):
        raise ValueError(f"targets must be [steps, N, 3] = [{steps}, {N}, 3] (got {list(targets.shape)})")
    if targets.device != node_loc.device:
        raise ValueError(f"targets is on {targets.device}, node_loc on {node_loc.device}")


class _Rollout:
    """State buffers at fixed addresses + the per-step enqueue (eager or CUDA-graph replay)."""

    def __init__(self, m: FastEGNN, be, dev, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius,
                 graph, loop, tau, speed_col, return_trajectory, cutoff_rate=0.0, targets=None, chamfer=False):
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).clone().contiguous()
        self.m, self.be, self.dev = m, be, dev
        self.N, self.B = int(node_loc.shape[0]), int(loc_mean.shape[0])
        Cn, self.A = m.virtual_channels, m.edge_attr_nf
        self.K = 4 + 3 * Cn + _lib.HIDDEN * Cn
        self.steps, self.radius, self.loop, self.tau, self.speed_col = steps, radius, loop, tau, speed_col
        # the state: private copies (the caller's tensors are never written)
        self.loc, self.vel, self.feat = f32(node_loc), f32(node_vel), f32(node_feat)
        self.loc_mean0 = f32(loc_mean)
        self.attr = f32(node_attr) if m.node_attr_nf > 0 else None
        self.batch = data_batch.contiguous()
        self.counter = torch.zeros(8, dtype=torch.int32, device=dev)
        self.counter[2:3].fill_(-1)
        self.traj = torch.empty(steps, self.N, 3, dtype=torch.float32, device=dev) if return_trajectory else None
        self.n_edges = torch.zeros(steps, dtype=torch.int32, device=dev)
        self.targets = self.sq_err = self.sq_ws = None
        if targets is not None:                                # per-step error: row counter[0] of sq_err, every step
            self.targets = targets.detach().contiguous()
            self.sq_err = torch.zeros(steps, self.B, dtype=torch.float64, device=dev)
            self.sq_ws = be.rollout_sq_err_workspace(self.N, dev)
        self.chamfer = self.ch_ws = None
        if chamfer:                                            # and row counter[0] of chamfer, after sq_err
            self.chamfer = torch.zeros(steps, self.B, 2, dtype=torch.float64, device=dev)
            self.ch_ws = be.rollout_chamfer_workspace(self.N, self.B, dev)
        self.pk = m._packed_params(dev)
        self.ws = m._workspace(dev, self.N, self.B, self.K)
        self.comm = m._get_comm(be, dev, self.B, self.K)       # collective on first use
        self.graphed = (m.cuda_graph and (m.world_size == 1 or self.comm is not None) and m._backend is None
                        and dev.type == "cuda" and m._timing is None)
        self.cuda_graph, self.graph_launches, self.replays = None, 0, 0
        self.bufs, self.capacity = None, None
        self.keep = None                                       # differentiable_rollout: per-step state for the backward
        self.rate = float(cutoff_rate)
        self.cut, self.cand = None, None                       # cutoff: kept-edge buffers, the candidate graph
        if graph is not None:                                  # fixed graph: only edge_attr changes
            graph.validate(dev)
            self.rowptr, self.row, self.col = graph.rowptr.contiguous(), graph.rows().contiguous(), graph.col.contiguous()
            self.E = graph.num_edges
            self.nE = graph.n_edges_dev
            self.edge_count = self.nE if self.nE is not None else \
                torch.full((1,), self.E, dtype=torch.int32, device=dev)
            self.overflow = None
            self.ea = torch.empty(self.E, self.A, dtype=torch.float32, device=dev) if self.A > 0 and not self.rate else None
            if self.rate > 0:                                  # the caller's graph is the candidate set
                self.cand = graph
                self._cut_buffers()

    # ---- graph buffers (radius mode) ----------------------------------------------------------------------------------
    def exact_capacity(self) -> int:
        """Count the edges of step 0's graph (one host read): the initial capacity is GROWTH x that."""
        probe = self.be.graph_buffers(self.N, 0, self.A, self.dev)
        self.be.radius_graph_into(probe, self.loc, self.radius, self._gbatch(), self.B, self.loop)
        return max(1, math.ceil(GROWTH * int(probe.info[0].item())))

    def set_capacity(self, cap: int) -> None:
        self.capacity = int(cap)
        # with a cutoff the radius graph is only the candidate set: no edge_attr (the cutoff writes the kept lengths)
        self.bufs = self.be.graph_buffers(self.N, self.capacity, 0 if self.rate > 0 else self.A, self.dev)
        g = self.bufs.graph
        self.rowptr, self.row, self.col, self.ea = g.rowptr, g.row, g.col, self.bufs.edge_attr
        self.E, self.nE = self.capacity, g.n_edges_dev
        self.edge_count, self.overflow = self.bufs.info[0:1], self.bufs.info[1:2]
        if self.rate > 0:
            self.cand = g
            self._cut_buffers()
        if self.m.deterministic:                               # sized here: the next step may be captured straight away
            self.m._det_workspace(self.ws, self.dev, self.N, self.E)
        self.cuda_graph = None                                 # captured addresses are stale

    def _cut_buffers(self) -> None:
        """Buffers of the kept edges (as many entries as the candidates): the model runs on them, and the advance records
        their count."""
        self.cut = self.be.graph_buffers(self.N, self.E, self.A, self.dev)
        g = self.cut.graph
        self.rowptr, self.row, self.col, self.ea, self.nE = g.rowptr, g.row, g.col, self.cut.edge_attr, g.n_edges_dev
        self.edge_count = self.cut.info[0:1]

    def cut_graph(self, x: Tensor) -> None:
        """The kept edges of the candidates at positions x; counter[6] keeps the largest candidate count (regrowth)."""
        self.be.cutoff_into(self.cut, self.cand, x, self.rate, self._gbatch(), self.B)
        torch.maximum(self.counter[6:7], self.cut.info[2:3], out=self.counter[6:7])

    def _gbatch(self) -> Optional[Tensor]:
        return self.batch if self.B > 1 else None

    def keep_steps(self) -> None:
        """Also keep, per step, what the backward's recompute needs besides the trajectory: the step's input velocity and
        speed column and its virtual_loc ([steps,·] buffers written at the device step index: capturable), plus x_0."""
        K, N, B, Cn = self.steps, self.N, self.B, self.m.virtual_channels
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.dev)
        self.keep = dict(x0=self.loc.clone(), feat0=self.feat.clone(), vel=new(K, N, 3), Xv=new(K, B, 3, Cn),
                         speed=new(K, N) if self.speed_col is not None else None)

    # ---- one step -----------------------------------------------------------------------------------------------------
    def _enqueue(self, init_centroid: bool) -> None:
        m, be = self.m, self.be
        if self.keep is not None:
            idx = self.counter[0:1].long()                     # this step's index, on the device
            self.keep["vel"].index_copy_(0, idx, self.vel.unsqueeze(0))
            if self.keep["speed"] is not None:
                self.keep["speed"].index_copy_(0, idx, self.feat[:, self.speed_col].unsqueeze(0))
        if self.bufs is not None:
            be.radius_graph_into(self.bufs, self.loc, self.radius, self._gbatch(), self.B, self.loop)
        elif self.ea is not None and self.cut is None:
            be.edge_lengths(self.row, self.col, self.loc, self.nE, self.ea)
        if self.cut is not None:
            self.cut_graph(self.loc)
        args = dict(node_feat=self.feat, node_loc=self.loc, node_vel=self.vel, loc_mean=self.loc_mean0, attr=self.attr,
                    data_batch=self.batch, rowptr=self.rowptr, row=self.row, col=self.col, ea=self.ea, nE=self.nE)
        m._run(be, self.pk, (self.N, self.E, self.B, self.K), args, self.ws, self.comm, init_centroid=init_centroid)
        if self.keep is not None:
            self.keep["Xv"].index_copy_(0, idx, self.ws["Xv"].unsqueeze(0))
        if self.targets is not None:                           # reads the step counter before the advance moves it
            be.rollout_sq_err(self.ws["out"], self.targets, self._gbatch(), self.counter, self.sq_err, self.sq_ws)
        if self.chamfer is not None:
            be.rollout_chamfer(self.ws["out"], self.targets, self._gbatch(), self.counter, self.chamfer, self.ch_ws)
        be.rollout_advance(self.speed_col, self.tau, self.ws["out"], self.loc, self.vel,
                           self.feat if self.speed_col is not None else None, self.traj, self.edge_count, self.overflow,
                           self.n_edges, self.counter)

    def step(self, t: int) -> None:
        if t == 0 or not self.graphed:                         # step 0 reads the caller's loc_mean (and warms up)
            self._enqueue(init_centroid=t > 0)
            return
        if self.cuda_graph is None:
            g = torch.cuda.CUDAGraph()
            n0 = self.be.launches
            with torch.cuda.graph(g):
                self._enqueue(init_centroid=True)
            self.cuda_graph, self.graph_launches = g, self.be.launches - n0
            self.graph_det_ws = self.ws.get("det")              # baked into the graph: keep it alive with it
            self.be.launches = n0
        self.cuda_graph.replay()
        self.be.launches += self.graph_launches
        self.replays += 1

    # ---- chunk bookkeeping --------------------------------------------------------------------------------------------
    def snapshot(self):
        return tuple(t.clone() for t in (self.loc, self.vel, self.feat, self.counter))

    def restore(self, saved) -> None:
        for dst, src in zip((self.loc, self.vel, self.feat, self.counter), saved):
            dst.copy_(src)

    def overflowed_anywhere(self):
        """(any rank overflowed, this rank overflowed, this rank's largest true edge count): one host read, plus one
        MAX all-reduce of the flag with several ranks."""
        st = self.counter[1:4].clone()                         # [own flag, first step, largest count]
        if self.cut is not None:                               # regrow from the candidates, not the kept edges
            st[2:3] = self.counter[6:7]
        flag = st[0:1].clone()
        if self.m.world_size > 1:
            import torch.distributed as dist
            dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=self.m.process_group)
        v = torch.cat([flag, st]).tolist()
        return bool(v[0]), bool(v[1]), int(v[3])

    def finish(self) -> Tensor:
        """Per-graph centroid of the final positions over all partitions: one kernel (fp64 sums: exact count, no fp32
        rounding of Σx), one [B,4] fp64 all-reduce.  With targets the [steps,B] error sums (and the [steps,B,2]
        partition-local Chamfer sums) ride in the same all-reduce, and `graph_nodes` takes the node counts from the
        centroid sums."""
        sums = torch.zeros(self.B, 4, dtype=torch.float64, device=self.dev)
        self.be.rollout_centroid(self.loc, self._gbatch(), sums, **(dict(deterministic=True) if self.m.deterministic else {}))
        if self.m.world_size > 1:                              # one fp64 SUM all-reduce (the peer exchange sums fp32)
            import torch.distributed as dist
            if self.sq_err is None:
                dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=self.m.process_group)
            else:
                parts = [sums, self.sq_err] + ([self.chamfer] if self.chamfer is not None else [])
                packed = torch.cat([p.reshape(-1) for p in parts])
                dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=self.m.process_group)
                sums, self.sq_err, *rest = packed.split([p.numel() for p in parts])
                sums = sums.view(self.B, 4)
                self.sq_err = self.sq_err.view(self.steps, self.B)
                if rest:
                    self.chamfer = rest[0].view(self.steps, self.B, 2)
        if self.sq_err is not None:
            self.graph_nodes = sums[:, 3].round().long()
        return (sums[:, :3] / sums[:, 3:4].clamp(min=1.0)).float()

    def errors(self) -> dict:
        """sq_err, graph_nodes and mse of RolloutResult (all None without targets), and chamfer and chamfer_mse (None
        without chamfer=True)."""
        if self.sq_err is None:
            return {}
        denom = (3.0 * self.graph_nodes.sum().double()).clamp(min=1.0)
        out = dict(sq_err=self.sq_err, graph_nodes=self.graph_nodes, mse=self.sq_err.sum(1) / denom)
        if self.chamfer is not None:
            out.update(chamfer=self.chamfer, chamfer_mse=self.chamfer.sum(1) / denom)
        return out


def rollout(model, node_feat: Tensor, node_loc: Tensor, node_vel: Tensor, loc_mean: Tensor, data_batch: Tensor,
            node_attr: Optional[Tensor] = None, *, steps: int, radius: Optional[float] = None,
            graph: Optional[CSRGraph] = None, loop: bool = False, tau: float = 1.0, speed_col: Optional[int] = None,
            capacity: Optional[int] = None, check_every: Optional[int] = None,
            return_trajectory: bool = False, cutoff_rate: float = 0.0,
            targets: Optional[Tensor] = None, chamfer: bool = False) -> RolloutResult:
    """Roll `model` (a FastEGNN, or one wrapped in DistributedDataParallel) out for `steps` steps from the given state;
    see the module docstring for the update rules.  With several ranks every rank calls it with its own partition.

    capacity: edge capacity of the rebuilt graph (radius mode); None = count step 0's graph (one host sync) and take
    1.25x that.  check_every: steps per overflow check (default: all steps, one check at the end); 0 = no check inside
    (call `RolloutResult.check()`).  Runs under no_grad; the caller's tensors are not modified.

    cutoff_rate > 0 (FastEGNN's cutoff_edges mode, single device): every step keeps the int(E_b·(1 − cutoff_rate))
    shortest edges of each graph's candidates (the rebuilt radius graph, or the caller's `graph`), re-selected from the
    current lengths (`cutoff_edges_csr`).  `n_edges` then counts the kept edges; `capacity` and its regrowth count the
    candidates.  0 runs no cutoff at all.

    targets: float32 [steps,N,3] on node_loc's device, this rank's rows of the recorded positions after each step (e.g.
    `FrameLoader(horizon=steps)`'s extras["targets"]).  Each step then adds one launch, between the forward and the
    advance, that stores sq_err[t, b] = Σ_{i in graph b} ‖x_{t+1,i} − targets[t,i]‖² (fp32 differences, fp64 sums in a
    fixed order: bitwise reproducible in deterministic mode); the result's `sq_err`, `graph_nodes` and `mse` hold it,
    summed over the ranks in the end-of-rollout all-reduce (DESIGN §19).

    chamfer=True (needs `targets`): each step also stores, after the sq_err launch and before the advance,
    chamfer[t, b, 0] = Σ_{i in graph b} min_j d(x_{t+1,i}, targets[t,j]) and chamfer[t, b, 1] = Σ_j min_i d(targets[t,j],
    x_{t+1,i}) over graph b's nodes of this rank, d the sq_err term: exact nearest neighbours on a device cell grid, a
    fixed number of launches per step, no host read (DESIGN §20).  The result's `chamfer` [steps,B,2] and `chamfer_mse`
    [steps,2] (normalised like `mse`, and never above it) hold it.  With several ranks each rank's partition-local sums
    are added in the end-of-rollout all-reduce: the result lies between the whole-cloud Chamfer sum and sq_err.  The
    trajectory, sq_err and mse do not change with it."""
    m = _unwrap(model)
    _validate(m, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius, graph, tau, speed_col,
              capacity, check_every, cutoff_rate)
    _check_targets(targets, steps, node_loc, chamfer)
    dev = node_loc.device
    be = m._get_backend(dev)                                    # raises on a CPU tensor (no CPU path)
    import contextlib
    guard = torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()
    with guard, torch.no_grad():
        r = _Rollout(m, be, dev, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius, graph,
                     loop, tau, speed_col, return_trajectory, cutoff_rate, targets, chamfer)
        grown = _drive(r, capacity, check_every)
        loc_mean_out = r.finish()
        return RolloutResult(node_loc=r.loc, node_vel=r.vel, node_feat=r.feat, loc_mean=loc_mean_out,
                             virtual_loc=r.ws["Xv"].clone(), trajectory=r.traj, n_edges=r.n_edges, capacity=r.capacity,
                             regrowths=grown, replays=r.replays, status=r.counter,
                             graph=_result_graph(r), edge_attr=r.ea, **r.errors())


def _result_graph(r: _Rollout) -> CSRGraph:
    if r.cut is not None:
        return r.cut.graph
    return r.bufs.graph if r.bufs is not None else CSRGraph(r.rowptr, r.col, r.row)


def _drive(r: _Rollout, capacity: Optional[int], check_every: Optional[int]) -> List[int]:
    """Run every step of `r` with the overflow policy of the module docstring; returns the capacities grown to."""
    steps = r.steps
    grown: List[int] = []
    if r.radius is not None:
        r.set_capacity(capacity if capacity is not None else r.exact_capacity())
    cap0 = r.capacity
    chunk = steps if check_every is None else (check_every or steps)
    check = check_every != 0
    t = 0
    while t < steps:
        n = min(chunk, steps - t)
        saved = r.snapshot() if (check and r.bufs is not None) else None
        for attempt in range(MAX_REGROWTHS + 1):
            for s in range(t, t + n):
                r.step(s)
            if saved is None:
                break
            anywhere, mine, count = r.overflowed_anywhere()
            if not anywhere:
                break
            if attempt == MAX_REGROWTHS:
                raise RuntimeError(f"rollout: steps {t}..{t + n - 1} still overflow the radius graph after "
                                   f"{MAX_REGROWTHS} regrowths (capacities {[cap0] + grown}, largest edge count "
                                   f"on this rank {count})")
            r.restore(saved)                                   # every rank reruns the chunk
            if mine:
                r.set_capacity(max(r.capacity + 1, math.ceil(GROWTH * count)))
                grown.append(r.capacity)
        t += n
    return grown


# ---- training through a rollout ---------------------------------------------------------------------------------------
def differentiable_rollout(model, node_feat: Tensor, node_loc: Tensor, node_vel: Tensor, loc_mean: Tensor,
                           data_batch: Tensor, node_attr: Optional[Tensor] = None, *, steps: int,
                           radius: Optional[float] = None, graph: Optional[CSRGraph] = None, loop: bool = False,
                           tau: float = 1.0, speed_col: Optional[int] = None, capacity: Optional[int] = None,
                           check_every: Optional[int] = None, cutoff_rate: float = 0.0) -> RolloutResult:
    """`rollout()` with a backward: `trajectory` [steps,N,3] and `virtual_locs` [steps,B,3,C] are attached to autograd, so
    a loss on any steps back-propagates into the model's parameters (summed over the steps) and into each of node_feat,
    node_loc, node_vel, loc_mean and node_attr that requires grad.  Same arguments, checks, update rules and overflow
    policy as `rollout()`; every other field of the result is detached and means what it means there.

    The forward is `rollout()`'s step loop; per step it keeps only O(N) state (the velocity, the speed column, the virtual
    coordinates; the positions are the trajectory).  The backward runs the steps in reverse, one at a time: it rebuilds
    step t's graph from x_t (radius mode; the build is deterministic, so the same positions give the same graph, and a
    differing edge count is recorded for `RolloutResult.check()`), recomputes step t's forward with its activations, and
    runs the backward kernels, the edge-length backward and the advance backward.  Peak memory is one step's training
    peak plus O(steps·N).  The graph is piecewise constant and gets no gradient; the edge lengths do.  loc_mean is read at
    step 0 only (later steps use the centroid of x_t, as in `rollout()`).  `model.input_grads` is not used or changed.
    The backward reuses the rollout's graph buffers: after it, `graph` / `edge_attr` hold step 0's graph.  With
    `cutoff_rate` the backward re-selects each step's kept edges from x_t (deterministic: the forward's); the selection
    is piecewise constant and gets no gradient, the kept edges' lengths do.

    With several ranks (the model may be wrapped in DistributedDataParallel: its module is used) every rank calls this
    and then backward on its own partition.  The state gradients are exact on every rank (every cross-rank term goes
    through the model's packed exchanges).  The parameter gradients are this rank's contribution only — DDP's reducer does
    not see this call — so sum them over the ranks yourself, e.g. `dist.all_reduce(p.grad)` for every parameter."""
    m = _unwrap(model)
    _validate(m, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius, graph, tau, speed_col,
              capacity, check_every, cutoff_rate)
    dev = node_loc.device
    be = m._get_backend(dev)
    import contextlib
    guard = torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()
    with guard:
        emb_wt, emb_b, hv0, lps = m._differentiable_params(dev)
        out = {}
        opts = dict(data_batch=data_batch, steps=steps, radius=radius, graph=graph, loop=loop, tau=tau,
                    speed_col=speed_col, capacity=capacity, check_every=check_every, cutoff_rate=cutoff_rate)
        traj, vlocs = _RolloutFunction.apply(out, m, be, opts, emb_wt, emb_b, hv0, *lps, node_feat, node_loc, node_vel,
                                             loc_mean, node_attr)
    r = out["r"]
    return RolloutResult(node_loc=r.loc, node_vel=r.vel, node_feat=r.feat, loc_mean=out["loc_mean"],
                         virtual_loc=r.ws["Xv"].clone(), trajectory=traj, n_edges=r.n_edges, capacity=r.capacity,
                         regrowths=out["grown"], replays=r.replays, status=r.counter,
                         graph=_result_graph(r), edge_attr=r.ea, virtual_locs=vlocs)


class _RolloutFunction(torch.autograd.Function):
    """Autograd node of `differentiable_rollout`: inputs (packed parameters, then node_feat, node_loc, node_vel,
    loc_mean, node_attr), outputs (trajectory, virtual_locs).  See DESIGN §15."""

    @staticmethod
    def forward(ctx, out, m, be, opts, emb_wt, emb_b, hv0, *rest):
        L = m.n_layers
        node_feat, node_loc, node_vel, loc_mean, node_attr = rest[L:]
        o = opts
        r = _Rollout(m, be, node_loc.device, node_feat, node_loc, node_vel, loc_mean, o["data_batch"], node_attr,
                     o["steps"], o["radius"], o["graph"], o["loop"], o["tau"], o["speed_col"], True, o["cutoff_rate"])
        r.keep_steps()
        out["grown"] = _drive(r, o["capacity"], o["check_every"])
        out["loc_mean"], out["r"] = r.finish(), r
        ctx.r = r
        ctx.params = (emb_wt.detach().contiguous(), emb_b.detach().contiguous(), hv0.detach().contiguous(),
                      [lp.detach().contiguous() for lp in rest[:L]])
        ctx.inputs = [None if t is None else t.dtype for t in rest[L:]]
        ctx.save_for_backward(r.traj)                          # an in-place change of the trajectory is caught
        return r.traj, r.keep["Xv"]

    @staticmethod
    def backward(ctx, g_traj, g_vlocs):
        from .fast_egnn import _backward_saved
        r = ctx.r
        (traj,) = ctx.saved_tensors
        m, be, dev = r.m, r.be, r.dev
        emb_wt, emb_b, hv0, layers = ctx.params
        L, N, B, Cn, Na, A = len(layers), r.N, r.B, m.virtual_channels, m.node_attr_nf, r.A
        w_feat, w_loc, w_vel, w_lm, w_attr = ctx.needs_input_grad[7 + L:7 + L + 5]
        sc = r.speed_col
        zeros = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        g_traj = g_traj.contiguous().float() if g_traj is not None else zeros(r.steps, N, 3)
        g_vlocs = g_vlocs.contiguous().float() if g_vlocs is not None else zeros(r.steps, B, 3, Cn)
        g_emb_wt, g_emb_b, g_hv0 = torch.zeros_like(emb_wt), torch.zeros_like(emb_b), torch.zeros_like(hv0)
        g_lps = [torch.zeros_like(lp) for lp in layers]
        g_attr_sum = zeros(N, Na) if (w_attr and Na > 0) else None
        g_x_next = g_v_next = g_f_next = g_lm = None
        feat_t = r.keep["feat0"].clone()
        import contextlib
        guard = torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()
        with guard, torch.no_grad():
            for t in reversed(range(r.steps)):
                mark = _marker(t)
                mark("rebuild")
                x_t = r.keep["x0"] if t == 0 else traj[t - 1]
                # 1. step t's graph from x_t: rebuilt (deterministic: the forward's graph) or the kept one's lengths
                if r.bufs is not None:
                    be.radius_graph_into(r.bufs, x_t, r.radius, r._gbatch(), r.B, r.loop)
                elif r.ea is not None and r.cut is None:
                    be.edge_lengths(r.row, r.col, x_t, r.nE, r.ea)
                if r.cut is not None:                          # the kept edges, re-selected from x_t
                    r.cut_graph(x_t)
                if r.bufs is not None or r.cut is not None:    # the edge count the model ran on, against the forward's
                    r.counter[5:6] += (r.edge_count != r.n_edges[t:t + 1]).to(torch.int32)
                # 2. step t's forward again, with its activations
                if sc is not None:
                    feat_t[:, sc] = r.keep["speed"][t]
                a = dict(node_feat=feat_t, node_loc=x_t, node_vel=r.keep["vel"][t], loc_mean=r.loc_mean0, attr=r.attr,
                         data_batch=r.batch, rowptr=r.rowptr, row=r.row, col=r.col, ea=r.ea, nE=r.nE)
                dims = (N, r.E, B, r.K)
                mark("recompute")
                _, _, st = m._run_saving(be, dims, a, emb_wt, emb_b, hv0, layers, init_centroid=t > 0)
                # 3. the advance: upstream of the prediction x_{t+1}, and its −g_v/tau share of g_x_t
                mark("advance_bwd")
                g_pred, g_x = torch.empty(N, 3, device=dev), torch.empty(N, 3, device=dev)
                be.rollout_advance_bwd(sc, r.tau, traj[t], x_t, g_traj[t], g_x_next, g_v_next,
                                       g_f_next if sc is not None else None, g_pred, g_x)
                # 4. the model's backward (t >= 1: the state feeds back, so positions, velocities and the speed column
                #    always need their gradient; at t = 0 only the inputs that require grad)
                mark("model_bwd")
                first = t == 0
                want = (w_feat or (not first and sc is not None), w_loc or not first, w_vel or not first,
                        first and w_lm, A > 0 and (w_loc or not first), w_attr)
                ge, gb, gh, glps, g_in = _backward_saved(m, be, dims, a, st, ctx.params, g_pred, g_vlocs[t], want,
                                                         init_centroid=not first)
                del st, a
                g_emb_wt += ge
                g_emb_b += gb
                g_hv0 += gh
                for acc, g in zip(g_lps, glps):
                    acc += g
                g_feat, g_loc, g_vel, g_lm_t, g_ea, g_attr = g_in
                if g_attr_sum is not None and g_attr is not None:
                    g_attr_sum += g_attr
                # 5. g_x_t = the advance's part + the model's (centroid included) + the edge lengths'
                if g_loc is not None:
                    g_x += g_loc
                mark("edge_lengths_bwd")
                if g_ea is not None:
                    be.edge_lengths_bwd(r.row, r.col, x_t, r.nE, g_ea, g_x)
                del g_ea
                mark("end")
                if g_feat is not None and g_f_next is not None:
                    g_feat += g_f_next                         # columns other than speed_col pass straight through
                elif g_feat is None:
                    g_feat = g_f_next
                g_x_next, g_v_next, g_f_next, g_lm = g_x, g_vel, g_feat, g_lm_t
        g_in = (g_f_next if w_feat else None, g_x_next if w_loc else None, g_v_next if w_vel else None,
                g_lm if w_lm else None, g_attr_sum if w_attr else None)
        shapes = (N, m.node_feat_nf), (N, 3), (N, 3), (B, 3), (N, Na)
        outs = []
        for want, dtype, g, shape in zip((w_feat, w_loc, w_vel, w_lm, w_attr), ctx.inputs, g_in, shapes):
            if not want:
                outs.append(None)
            else:
                outs.append(torch.zeros(shape, dtype=dtype, device=dev) if g is None else g.to(dtype))
        return (None, None, None, None, g_emb_wt, g_emb_b, g_hv0, *g_lps, *outs)


def _marker(step: int):
    if _bwd_timing is None:
        return lambda name: None

    def mark(name: str) -> None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        _bwd_timing.append((step, name, ev))
    return mark
