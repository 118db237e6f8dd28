"""Multi-step inference: feed the model's prediction back in, rebuild the graph, repeat — on the device.

    res = rollout(model, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr=None, *,
                  steps, radius=None, graph=None, loop=False, tau=1.0, speed_col=None,
                  capacity=None, check_every=None, return_trajectory=False)

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
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional

import torch

from . import _lib
from .fast_egnn import FastEGNN
from .shards import CSRGraph

Tensor = torch.Tensor
GROWTH = 1.25              # capacity = GROWTH x edge count (initial build and every regrowth)
MAX_REGROWTHS = 4          # per chunk; then the rollout raises


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

    def check(self) -> None:
        """Raise if a graph build overflowed its capacity (one host read).  Only needed with `check_every=0`."""
        s = self.status.tolist()
        if s[1]:
            raise RuntimeError(f"rollout: the radius graph first outgrew the capacity {self.capacity} at step {s[2]} (the "
                               f"largest edge count of any step was {s[3]}); the results from that step on are wrong — "
                               "pass a larger capacity or let rollout check (check_every > 0)")


def _unwrap(model) -> FastEGNN:
    m = getattr(model, "module", model)
    if not isinstance(m, FastEGNN):
        raise TypeError(f"rollout needs a distegnn_b200.FastEGNN (or a DDP-wrapped one), got {type(model).__name__}")
    return m


def _validate(m: FastEGNN, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius, graph, tau,
              speed_col, capacity, check_every) -> None:
    is_int = lambda v: isinstance(v, int) and not isinstance(v, bool)
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


class _Rollout:
    """State buffers at fixed addresses + the per-step enqueue (eager or CUDA-graph replay)."""

    def __init__(self, m: FastEGNN, be, dev, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius,
                 graph, loop, tau, speed_col, return_trajectory):
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
        self.pk = m._packed_params(dev)
        self.ws = m._workspace(dev, self.N, self.B, self.K)
        self.comm = m._get_comm(be, dev, self.B, self.K)       # collective on first use
        self.graphed = (m.cuda_graph and (m.world_size == 1 or self.comm is not None) and m._backend is None
                        and dev.type == "cuda" and m._timing is None)
        self.cuda_graph, self.graph_launches, self.replays = None, 0, 0
        self.bufs, self.capacity = None, None
        if graph is not None:                                  # fixed graph: only edge_attr changes
            graph.validate(dev)
            self.rowptr, self.row, self.col = graph.rowptr.contiguous(), graph.rows().contiguous(), graph.col.contiguous()
            self.E = graph.num_edges
            self.nE = graph.n_edges_dev
            self.edge_count = self.nE if self.nE is not None else \
                torch.full((1,), self.E, dtype=torch.int32, device=dev)
            self.overflow = None
            self.ea = torch.empty(self.E, self.A, dtype=torch.float32, device=dev) if self.A > 0 else None

    # ---- graph buffers (radius mode) ----------------------------------------------------------------------------------
    def exact_capacity(self) -> int:
        """Count the edges of step 0's graph (one host read): the initial capacity is GROWTH x that."""
        probe = self.be.graph_buffers(self.N, 0, self.A, self.dev)
        self.be.radius_graph_into(probe, self.loc, self.radius, self._gbatch(), self.B, self.loop)
        return max(1, math.ceil(GROWTH * int(probe.info[0].item())))

    def set_capacity(self, cap: int) -> None:
        self.capacity = int(cap)
        self.bufs = self.be.graph_buffers(self.N, self.capacity, self.A, self.dev)
        g = self.bufs.graph
        self.rowptr, self.row, self.col, self.ea = g.rowptr, g.row, g.col, self.bufs.edge_attr
        self.E, self.nE = self.capacity, g.n_edges_dev
        self.edge_count, self.overflow = self.bufs.info[0:1], self.bufs.info[1:2]
        self.cuda_graph = None                                 # captured addresses are stale

    def _gbatch(self) -> Optional[Tensor]:
        return self.batch if self.B > 1 else None

    # ---- one step -----------------------------------------------------------------------------------------------------
    def _enqueue(self, init_centroid: bool) -> None:
        m, be = self.m, self.be
        if self.bufs is not None:
            be.radius_graph_into(self.bufs, self.loc, self.radius, self._gbatch(), self.B, self.loop)
        elif self.ea is not None:
            be.edge_lengths(self.row, self.col, self.loc, self.nE, self.ea)
        args = dict(node_feat=self.feat, node_loc=self.loc, node_vel=self.vel, loc_mean=self.loc_mean0, attr=self.attr,
                    data_batch=self.batch, rowptr=self.rowptr, row=self.row, col=self.col, ea=self.ea, nE=self.nE)
        m._run(be, self.pk, (self.N, self.E, self.B, self.K), args, self.ws, self.comm, init_centroid=init_centroid)
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
        flag = st[0:1].clone()
        if self.m.world_size > 1:
            import torch.distributed as dist
            dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=self.m.process_group)
        v = torch.cat([flag, st]).tolist()
        return bool(v[0]), bool(v[1]), int(v[3])

    def finish(self) -> Tensor:
        """Per-graph centroid of the final positions over all partitions: one kernel (fp64 sums: exact count, no fp32
        rounding of Σx), one [B,4] fp64 all-reduce."""
        sums = torch.zeros(self.B, 4, dtype=torch.float64, device=self.dev)
        self.be.rollout_centroid(self.loc, self._gbatch(), sums)
        if self.m.world_size > 1:                              # one fp64 SUM all-reduce (the peer exchange sums fp32)
            import torch.distributed as dist
            dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=self.m.process_group)
        return (sums[:, :3] / sums[:, 3:4].clamp(min=1.0)).float()


def rollout(model, node_feat: Tensor, node_loc: Tensor, node_vel: Tensor, loc_mean: Tensor, data_batch: Tensor,
            node_attr: Optional[Tensor] = None, *, steps: int, radius: Optional[float] = None,
            graph: Optional[CSRGraph] = None, loop: bool = False, tau: float = 1.0, speed_col: Optional[int] = None,
            capacity: Optional[int] = None, check_every: Optional[int] = None,
            return_trajectory: bool = False) -> RolloutResult:
    """Roll `model` (a FastEGNN, or one wrapped in DistributedDataParallel) out for `steps` steps from the given state;
    see the module docstring for the update rules.  With several ranks every rank calls it with its own partition.

    capacity: edge capacity of the rebuilt graph (radius mode); None = count step 0's graph (one host sync) and take
    1.25x that.  check_every: steps per overflow check (default: all steps, one check at the end); 0 = no check inside
    (call `RolloutResult.check()`).  Runs under no_grad; the caller's tensors are not modified."""
    m = _unwrap(model)
    _validate(m, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius, graph, tau, speed_col,
              capacity, check_every)
    dev = node_loc.device
    be = m._get_backend(dev)                                    # raises on a CPU tensor (no CPU path)
    import contextlib
    guard = torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()
    with guard, torch.no_grad():
        r = _Rollout(m, be, dev, node_feat, node_loc, node_vel, loc_mean, data_batch, node_attr, steps, radius, graph,
                     loop, tau, speed_col, return_trajectory)
        grown: List[int] = []
        if radius is not None:
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
                r.restore(saved)                               # every rank reruns the chunk
                if mine:
                    r.set_capacity(max(r.capacity + 1, math.ceil(GROWTH * count)))
                    grown.append(r.capacity)
            t += n
        loc_mean_out = r.finish()
        return RolloutResult(node_loc=r.loc, node_vel=r.vel, node_feat=r.feat, loc_mean=loc_mean_out,
                             virtual_loc=r.ws["Xv"].clone(), trajectory=r.traj, n_edges=r.n_edges, capacity=r.capacity,
                             regrowths=grown, replays=r.replays, status=r.counter,
                             graph=r.bufs.graph if r.bufs is not None else CSRGraph(r.rowptr, r.col, r.row),
                             edge_attr=r.ea)
