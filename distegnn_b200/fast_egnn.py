"""Host-side mirror of the reference's FastEGNN / DistEGNN model (models/FastEGNN.py).

Same class name, constructor signature, ``forward`` signature, return tuple and ``state_dict`` keys as
the reference (SURVEY §8b), so ``main.py:61-62``, ``utils/train.py:63-71``, DDP wrapping and
checkpoints work unchanged — but ``forward`` runs entirely in the hand-written sm_90a kernels behind
the C ABI (include/distegnn_b200.h).  There is no eager/CPU fallback.

Per forward (L layers) the device work is
    embed → sync+virtual_update(INIT)
    L × { edge_layer, virtual_layer, node_layer → sync+virtual_update }
i.e. 2 + 4L kernel launches and nothing else: ONE exchange of the packed statistics per layer plus one up front
(the reference issues 6 NCCL calls per layer, each behind host syncs: FastEGNN.py:196-197, 226-227, 260-261,
310-319), fused into the virtual-node update kernel as a push over NVLink peer memory (csrc/comm.cuh; when
CUDA IPC between the ranks is not available the exchange is a `torch.distributed` all-reduce instead).  No memset or
copy launches (the consumers clear `vsum` / `agg_*` for the next layer), so the whole forward — collectives
included — replays as one CUDA graph (`model.cuda_graph = True`), for any world size.

In grad mode the same kernels run with per-layer activations kept and the outputs are attached to autograd
(``_FastEGNNFunction``): backward = hand-written kernels for the per-edge and real<->virtual stages, torch
recompute for the dense per-node stages, one packed all-reduce of the statistics' gradient per layer (DESIGN §9).
By default the inputs are constants of that graph, as in the reference's training loop; with `model.input_grads = True`
every floating input that requires grad (node_feat, node_loc, node_vel, loc_mean, edge_attr, node_attr) receives the
gradient the reference module's autograd would give it — multi-step rollout training, edge_attr computed in torch from the
positions, sensitivity analysis.  edge_index / data_batch / CSRGraph are not differentiable, and neither is the edge_attr
that `radius_graph_csr` builds on the device: `rollout.differentiable_rollout` back-propagates through edge lengths.
"""
from __future__ import annotations

import contextlib
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _lib

Tensor = torch.Tensor
H = _lib.HIDDEN


# --------------------------------------------------------------------------------------------------
# parameter containers with the reference's module/parameter names (they hold weights only — the
# compute happens in the fused kernels)
# --------------------------------------------------------------------------------------------------
def _mlp(n_in: int, n_hidden: int, n_out: int, act: nn.Module, last_act: bool) -> nn.Sequential:
    mods = [nn.Linear(n_in, n_hidden), act, nn.Linear(n_hidden, n_out)]
    if last_act:
        mods.append(act)
    return nn.Sequential(*mods)


def _coord_head(n_hidden: int, act: nn.Module) -> nn.Sequential:
    # reference draws the 1-wide projection first, then the hidden layer (FastEGNN.py:96-103); keeping
    # that order keeps `torch.manual_seed(s); FastEGNN(...)` weight-identical to the reference.
    out = nn.Linear(n_hidden, 1, bias=False)
    nn.init.xavier_uniform_(out.weight, gain=0.001)
    return nn.Sequential(nn.Linear(n_hidden, n_hidden), act, out)


class E_GCL_vel(nn.Module):
    """Weights of one equivariant layer (reference E_GCL_vel, FastEGNN.py:46-141).  Not callable on its
    own: the layer is executed by FastEGNN.forward through the fused kernels."""

    def __init__(self, hidden_nf: int, node_attr_nf: int, edge_attr_nf: int, virtual_channels: int,
                 act_fn: nn.Module):
        super().__init__()
        Hh, Cc = hidden_nf, virtual_channels
        self.edge_mlp = _mlp(2 * Hh + 1 + edge_attr_nf, Hh, Hh, act_fn, True)           # φ_e
        self.edge_mlp_virtual = _mlp(2 * Hh + 1 + Cc, Hh, Hh, act_fn, True)             # φ_ev
        self.coord_mlp_r = _coord_head(Hh, act_fn)                                      # φ_x
        self.coord_mlp_r_virtual = _coord_head(Hh, act_fn)                              # φ_xv
        self.coord_mlp_v_virtual = _coord_head(Hh, act_fn)                              # φ_X
        self.coord_mlp_vel = _mlp(Hh, Hh, 1, act_fn, False)                             # φ_v
        self.node_mlp = _mlp(3 * Hh + node_attr_nf, Hh, Hh, act_fn, False)              # φ_h
        self.node_mlp_virtual = _mlp(2 * Hh, Hh, Hh, act_fn, False)                     # φ_hv

    def forward(self, *args, **kwargs):  # pragma: no cover
        raise RuntimeError("E_GCL_vel layers are executed by FastEGNN.forward (fused CUDA path)")


# --------------------------------------------------------------------------------------------------
# packing of one layer's weights into the flat block the kernels read (include/distegnn_b200.h)
# --------------------------------------------------------------------------------------------------
def pack_layer_params(g: nn.Module, A: int, Cn: int, Na: int, device, offs: Dict[str, int], total: int) -> Tensor:
    """Flat parameter block of one layer, built with torch.cat from the live parameters (zeros in the gaps of the
    layout), so that the gradient of the block flows back to the nn.Parameters through autograd."""
    pieces: List[Tuple[int, Tensor]] = []

    def put(name: str, t: Tensor) -> None:
        pieces.append((offs[name], t.to(device=device, dtype=torch.float32).reshape(-1)))

    W1, b1 = g.edge_mlp[0].weight, g.edge_mlp[0].bias            # [64, 2H+1+A]
    put("E_W1A", W1[:, 0:H].t()); put("E_W1B", W1[:, H:2 * H].t()); put("E_W1R", W1[:, 2 * H])
    if A:
        put("E_W1E", W1[:, 2 * H + 1:2 * H + 1 + A].t())
    put("E_B1", b1)
    put("E_W2", g.edge_mlp[2].weight.t()); put("E_B2", g.edge_mlp[2].bias)
    put("E_WC", g.coord_mlp_r[0].weight.t()); put("E_BC", g.coord_mlp_r[0].bias)
    put("E_W3", g.coord_mlp_r[2].weight[0])
    V1, vb1 = g.edge_mlp_virtual[0].weight, g.edge_mlp_virtual[0].bias   # [64, 2H+1+C]
    put("V_W1H", V1[:, 0:H].t()); put("V_W1V", V1[:, H:2 * H].t()); put("V_W1R", V1[:, 2 * H])
    put("V_W1M", V1[:, 2 * H + 1:2 * H + 1 + Cn].t()); put("V_B1", vb1)
    put("V_W2", g.edge_mlp_virtual[2].weight.t()); put("V_B2", g.edge_mlp_virtual[2].bias)
    put("V_WXV", g.coord_mlp_r_virtual[0].weight.t()); put("V_BXV", g.coord_mlp_r_virtual[0].bias)
    put("V_W3XV", g.coord_mlp_r_virtual[2].weight[0])
    put("V_WX", g.coord_mlp_v_virtual[0].weight.t()); put("V_BX", g.coord_mlp_v_virtual[0].bias)
    put("V_W3X", g.coord_mlp_v_virtual[2].weight[0])
    put("L_W", g.coord_mlp_vel[0].weight.t()); put("L_B", g.coord_mlp_vel[0].bias)
    put("L_W3", g.coord_mlp_vel[2].weight[0]); put("L_B3", g.coord_mlp_vel[2].bias)
    put("N_W1", g.node_mlp[0].weight.t()); put("N_B1", g.node_mlp[0].bias)
    put("N_W2", g.node_mlp[2].weight.t()); put("N_B2", g.node_mlp[2].bias)
    put("M_W1", g.node_mlp_virtual[0].weight.t()); put("M_B1", g.node_mlp_virtual[0].bias)
    put("M_W2", g.node_mlp_virtual[2].weight.t()); put("M_B2", g.node_mlp_virtual[2].bias)
    parts, pos = [], 0
    for off, t in sorted(pieces, key=lambda p: p[0]):
        if off > pos:
            parts.append(torch.zeros(off - pos, dtype=torch.float32, device=device))
        parts.append(t)
        pos = off + t.numel()
    if pos < total:
        parts.append(torch.zeros(total - pos, dtype=torch.float32, device=device))
    return torch.cat(parts)


class _GraphCache:
    """CSR form of recent edge_index tensors.  Entries hold a strong reference to the tensor they were built from, so its
    storage cannot be recycled under the same pointer; a hit additionally requires an unchanged in-place version counter.

    With `pos`, the rows are stored in the spatial order of those positions, the ones of the call that builds the entry
    (DESIGN §3); later calls reuse that order whatever their positions, since outside the deterministic mode the order
    only decides which neighbour rows the edge kernels find in L2.  Without `pos` they are in id order, which depends on
    edge_index alone: the deterministic mode's bits depend on where each row starts in the edge list (§17), so it asks
    for id order.  The two orders are cached as separate entries.  The torch stand-in of the CPU tests has no
    `build_csr_cells`; it restates the kernels with order-independent sums, and gets id order."""

    def __init__(self, capacity: int = 4):
        self.capacity = capacity
        self.entries: "OrderedDict[Tuple[int, bool], tuple]" = OrderedDict()
        self.builds = 0
        self.pending = None                # device counter of the last build's out-of-range edge ids (read after embed)

    def get(self, backend, edge_index: Tensor, n_nodes: int, validate: bool = True, pos: Optional[Tensor] = None,
            batch: Optional[Tensor] = None, n_graphs: int = 1):
        spatial = pos is not None and hasattr(backend, "build_csr_cells")
        key = (id(edge_index), spatial)
        hit = self.entries.get(key)
        if hit is not None and hit[0] is edge_index and hit[1] == edge_index._version and hit[2] == n_nodes:   # noqa: E501
            self.entries.move_to_end(key)
            return hit[3]
        ei = edge_index if edge_index.is_contiguous() else edge_index.contiguous()
        mode = "defer" if validate else False
        built = (backend.build_csr_cells(ei, n_nodes, pos, batch, n_graphs, mode) if spatial
                 else backend.build_csr(ei, n_nodes, mode))
        csr, self.pending = tuple(built[:4]), (built[4] if validate else None)     # counter of out-of-range ids, not yet read
        self.builds += 1
        self.entries[key] = (edge_index, edge_index._version, n_nodes, csr)
        while len(self.entries) > self.capacity:
            self.entries.popitem(last=False)
        return csr

    def sorted_edge_attr(self, backend, edge_index: Tensor, edge_attr: Tensor, perm: Tensor) -> Tensor:
        """edge_attr permuted into CSR order, cached next to the CSR of `edge_index` that `perm` belongs to while the SAME
        edge_attr tensor (identity + in-place version) keeps being passed — the steady state of inference / rollouts."""
        key = next((k for k, e in self.entries.items() if e[3][3] is perm), None)
        ent = self.entries.get(key)
        if ent is not None and ent[0] is edge_index and len(ent) == 6 and ent[4][0] is edge_attr \
                and ent[4][1] == edge_attr._version:
            return ent[5]
        ea = backend.gather_rows(edge_attr.detach().to(torch.float32).contiguous(), perm)
        if ent is not None and ent[0] is edge_index:
            self.entries[key] = ent[:4] + ((edge_attr, edge_attr._version), ea)
        return ea


# --------------------------------------------------------------------------------------------------
# the model
# --------------------------------------------------------------------------------------------------
class FastEGNN(nn.Module):
    """Drop-in for the reference ``models.FastEGNN.FastEGNN`` (FastEGNN.py:279-307)."""

    def __init__(self, node_feat_nf, node_attr_nf, edge_attr_nf, hidden_nf, virtual_channels, world_size,
                 act_fn=nn.SiLU(), n_layers=4, residual=True, attention=False, normalize=False, tanh=False,
                 gravity=None):
        super().__init__()
        assert virtual_channels > 0, f'Channels of virtual node must greater than 0 (got {virtual_channels})'
        if hidden_nf != H:
            raise ValueError(f"distegnn_b200 kernels are built for hidden_nf={H} (got {hidden_nf})")
        if not isinstance(act_fn, nn.SiLU):
            raise ValueError("only act_fn=nn.SiLU() is supported (the reference never uses another)")
        if attention or tanh or gravity is not None or not residual:
            raise ValueError("attention/tanh/gravity/residual=False are never enabled by the reference "
                             "(main.py:61-62) and are not implemented")
        for name, v, hi in (("virtual_channels", virtual_channels, _lib.MAX_CHANNELS),
                            ("edge_attr_nf", edge_attr_nf, _lib.MAX_EDGE_ATTR),
                            ("node_attr_nf", node_attr_nf, _lib.MAX_NODE_ATTR),
                            ("node_feat_nf", node_feat_nf, _lib.MAX_NODE_FEAT)):
            if v > hi:
                raise ValueError(f"{name}={v} exceeds the compiled limit {hi}")
        self.hidden_nf = hidden_nf
        self.n_layers = n_layers
        self.node_feat_nf = node_feat_nf
        self.node_attr_nf = node_attr_nf
        self.edge_attr_nf = edge_attr_nf
        self.virtual_channels = virtual_channels
        self.world_size = world_size
        self.normalize = normalize
        # same construction order as the reference ⇒ same RNG stream ⇒ same initial weights
        self.virtual_node_feat = nn.Parameter(data=torch.randn(size=(1, hidden_nf, virtual_channels)),
                                              requires_grad=True)
        self.embedding_in = nn.Linear(node_feat_nf, hidden_nf)
        for i in range(n_layers):
            self.add_module("gcl_%d" % i, E_GCL_vel(hidden_nf, node_attr_nf, edge_attr_nf,
                                                    virtual_channels, act_fn))
        # non-persistent runtime state
        self._backend = None               # tests may inject a stand-in; default = CUDA C-ABI backend
        self._graphs = _GraphCache()
        self._packed = None                # (key, tensors)
        self._timing = None                # bench.py: list collecting (name, start_evt, end_evt)
        self.cuda_graph = False            # opt-in: replay the forward as a CUDA graph (see _forward_graphed)
        self._graph_cache: Dict[tuple, tuple] = {}
        self._graph_max_captures = 8
        self.process_group = None          # torch.distributed group for the virtual-node sync (None = WORLD)
        self.validate_inputs = True        # check edge ids / data_batch once per distinct tensor (one host sync each)
        self.input_grads = False           # opt-in: back-propagate into the floating inputs too (see _FastEGNNFunction)
        self.deterministic = False         # opt-in: bitwise-reproducible forward (see the property)
        self._validated_batch = None       # (tensor, version, N, B) of the last data_batch that passed
        self._workspaces: Dict[tuple, Dict[str, Tensor]] = {}
        self._keep_state = None            # tests: a list that receives the training-path forward's saved state
        self._comm = None                  # backend.Comm | False (peer exchange unavailable: torch.distributed instead)
        self._comm_key = None

    @property
    def deterministic(self) -> bool:
        """Opt-in deterministic mode (default False; DESIGN §17).  While it is on, the inference forward, the forward of the
        training path, `rollout()` and the forward of `differentiable_rollout()` (trajectory and virtual_loc) are bitwise
        reproducible: their bits depend only on the input tensors, N, B, C, A, Na, the layer flags and the library build
        — not on the edge capacity, the grid, the stream, CUDA-graph capture or concurrent work.  Every per-destination
        and per-graph sum is then taken in a fixed order instead of with atomics, at some cost in speed and a workspace
        of about 17 bytes per edge of capacity.  Gradients are not covered: the backward keeps the existing
        run-to-run bound.  Across ranks the per-rank values are deterministic and the peer-memory exchange adds them in
        rank order; the torch.distributed fallback of that exchange is not covered."""
        return self._deterministic

    @deterministic.setter
    def deterministic(self, on: bool) -> None:
        if not isinstance(on, bool):
            raise TypeError(f"deterministic must be a bool (got {type(on).__name__})")
        self._deterministic = on

    # ---- runtime helpers -----------------------------------------------------------------------
    def _get_backend(self, device: torch.device):
        if self._backend is not None:
            return self._backend
        if device.type != "cuda":
            raise _lib.DistEGNNError(
                "distegnn_b200.FastEGNN runs only on CUDA (sm_90a kernels); there is no CPU fallback — "
                "move the model and inputs to a CUDA device")
        from .backend import cuda_backend
        return cuda_backend()

    def _pack_params(self, device: torch.device) -> Dict:
        """The weights as the kernels read them, {layers: [flat block per layer], emb_wt, emb_b, hv0 [C,64]}, packed from
        the live parameters with torch ops, so that the gradients of the packed tensors flow back to the nn.Parameters."""
        A, Cn, Na = self.edge_attr_nf, self.virtual_channels, self.node_attr_nf
        offs, total = _lib.param_layout(A, Cn, Na)
        layers = [pack_layer_params(getattr(self, "gcl_%d" % i), A, Cn, Na, device, offs, total)
                  for i in range(self.n_layers)]
        emb_wt = self.embedding_in.weight.t().contiguous().to(device=device, dtype=torch.float32)
        emb_b = self.embedding_in.bias.to(device=device, dtype=torch.float32)
        hv0 = self.virtual_node_feat[0].t().contiguous().to(device=device, dtype=torch.float32)
        return dict(layers=layers, emb_wt=emb_wt, emb_b=emb_b, hv0=hv0)

    def _packed_params(self, device: torch.device) -> Dict:
        """`_pack_params` detached, cached while no parameter is replaced or changed in place."""
        key = (str(device),) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._packed is not None and self._packed[0] == key:
            return self._packed[1]
        with torch.no_grad():
            pk = self._pack_params(device)
        # detached: emb_b may be the bias Parameter itself (`.to` returns it when nothing changes)
        packed = dict(layers=[t.detach() for t in pk["layers"]], emb_wt=pk["emb_wt"].detach(),
                      emb_b=pk["emb_b"].detach(), hv0=pk["hv0"].detach())
        self._packed = (key, packed)
        return packed

    def _get_comm(self, be, dev: torch.device, B: int, K: int):
        """Communicator of the virtual-node sync for calls of [B,K] floats, or None (single partition / stand-in
        backend / no peer access: then `_sync_virtual` goes through torch.distributed).  Creation is collective."""
        if self.world_size == 1 or self._backend is not None or dev.type != "cuda":
            return None
        import os
        import torch.distributed as dist
        if self._comm is False or os.environ.get("DISTEGNN_B200_COMM", "p2p") == "nccl":
            return None
        if self._comm is not None and self._comm_key[0] >= B and self._comm_key[1] >= K:
            return self._comm
        from .backend import Comm
        if self._comm is not None:                       # capacity grows: all ranks see the same B, K
            torch.cuda.synchronize(dev)
            dist.barrier(group=self.process_group)
            self._comm.destroy()
            self._comm = None
            self._graph_cache.clear()
        try:
            self._comm = Comm(be.lib, dev, self.process_group, max(B, 1), K)
            self._comm_key = (max(B, 1), K)
        except _lib.DistEGNNError as e:
            import warnings
            warnings.warn(f"distegnn_b200: peer-memory exchange unavailable ({e}); the virtual-node sync uses "
                          "torch.distributed all_reduce", RuntimeWarning)
            self._comm = False
            return None
        return self._comm

    def release_comm(self) -> None:
        """Collective teardown of the peer-memory communicator (call on every rank, e.g. before destroying the process
        group); captured CUDA graphs that reference it are dropped.  A later forward creates a new one."""
        if self._comm:
            import torch.distributed as dist
            torch.cuda.synchronize()
            dist.barrier(group=self.process_group)       # nobody unmaps while a peer still has an exchange in flight
            self._comm.destroy()
        self._comm, self._comm_key = None, None
        self._graph_cache.clear()

    def _sync_virtual(self, vsum: Tensor, be=None, comm=None) -> None:
        """weighted_average_reduce (FastEGNN.py:310-319) on the packed statistics: one SUM all-reduce;
        the division by the summed node count happens in virtual_update."""
        if self.world_size > 1:
            if comm is not None:
                be.allreduce_packed(comm, vsum)
                return
            import torch.distributed as dist
            dist.all_reduce(vsum, op=dist.ReduceOp.SUM, group=self.process_group)

    # ---- forward -------------------------------------------------------------------------------
    def forward(self, node_feat, node_loc, node_vel, loc_mean, edge_index, data_batch, edge_attr=None,
                node_attr=None) -> Tuple[Tensor, Tensor]:
        inputs = (node_feat, node_loc, node_vel, loc_mean, edge_attr, node_attr)
        want_inputs = self.input_grads and torch.is_grad_enabled() and \
            any(t is not None and t.requires_grad for t in inputs)
        training_path = want_inputs or (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()))
        dev = node_loc.device
        be = self._get_backend(dev)
        A, Cn, Na, F = self.edge_attr_nf, self.virtual_channels, self.node_attr_nf, self.node_feat_nf
        from .shards import CSRGraph
        pre_csr = isinstance(edge_index, CSRGraph)           # graph already sorted by destination (shards.py, f-4)
        N, B = int(node_loc.shape[0]), int(loc_mean.shape[0])
        E = edge_index.num_edges if pre_csr else int(edge_index.shape[1])
        if pre_csr and edge_index.num_nodes != N:
            raise ValueError(f"CSRGraph has {edge_index.num_nodes} nodes, node_loc has {N}")
        if node_feat.shape != (N, F) or node_vel.shape != (N, 3) or node_loc.shape != (N, 3):
            raise ValueError(f"bad node tensor shapes: feat {tuple(node_feat.shape)}, loc "
                             f"{tuple(node_loc.shape)}, vel {tuple(node_vel.shape)}; expected N={N}, F={F}")
        if not pre_csr and (edge_index.shape[0] != 2 or edge_index.dtype != torch.int64):
            raise ValueError("edge_index must be int64 [2,E] (or a distegnn_b200.shards.CSRGraph)")
        if data_batch.shape != (N,) or data_batch.dtype != torch.int64:
            raise ValueError("data_batch must be int64 [N]")
        if A > 0 and (edge_attr is None or edge_attr.shape != (E, A)):
            raise ValueError(f"edge_attr must be [E,{A}]")
        if Na > 0 and (node_attr is None or node_attr.shape != (N, Na)):
            raise ValueError(f"node_attr must be [N,{Na}]")
        if loc_mean.shape != (B, 3):
            raise ValueError("loc_mean must be [B,3]")
        K = 4 + 3 * Cn + H * Cn
        dims = (N, E, B, K)
        if pre_csr:
            edge_index.validate(dev)
        with device_guard(dev):                               # launches and smem opt-ins happen on the tensors' device
            with torch.no_grad():
                args = self._kernel_args(be, N, node_feat, node_loc, node_vel, loc_mean, edge_index, data_batch,
                                         edge_attr, node_attr)
            if training_path:      # per-layer activations kept (N-sized only), gradients through _FastEGNNFunction
                for name, t in (("node_feat", node_feat), ("node_loc", node_loc), ("node_vel", node_vel),
                                ("edge_attr", edge_attr), ("node_attr", node_attr)):
                    if t is not None and t.requires_grad and not self.input_grads:
                        import warnings
                        warnings.warn(f"distegnn_b200.FastEGNN: `{name}` requires grad, but the fused path treats inputs "
                                      "as constants (the reference trains weights only, utils/train.py:149-158): no "
                                      "gradient will flow to it; set `model.input_grads = True` to back-propagate into "
                                      "the inputs", RuntimeWarning, stacklevel=2)
                pk = self._pack_params(dev)
                ins = inputs if self.input_grads else ()
                return _FastEGNNFunction.apply(self, be, dims, args, pk["emb_wt"], pk["emb_b"], pk["hv0"], *pk["layers"],
                                               *ins)
            with torch.no_grad():
                pk = self._packed_params(dev)
                comm = self._get_comm(be, dev, B, K)
                graph_ok = self.world_size == 1 or comm is not None      # NCCL calls are not captured
                if self.cuda_graph and graph_ok and self._backend is None and dev.type == "cuda" \
                        and self._timing is None and self._batch_checked(args["data_batch"], N, B):
                    return self._forward_graphed(be, pk, dims, args, comm)
                ws = self._workspace(dev, N, B, K)
                # results go straight into fresh tensors (no copy launch); everything else lives in the workspace
                out, Xv, _ = self._forward(be, pk, dims, args, ws, out=torch.empty(N, 3, dtype=torch.float32, device=dev),
                                           Xv=torch.empty(B, 3, Cn, dtype=torch.float32, device=dev))
                return out, Xv

    def _batch_checked(self, data_batch: Tensor, N: int, B: int) -> bool:
        v = self._validated_batch
        return (not self.validate_inputs) or (v is not None and v[0] is data_batch and v[1] == data_batch._version
                                              and v[2] == N and v[3] == B)

    def _check_batch(self, counter: Optional[Tensor], data_batch: Tensor, N: int, B: int) -> None:
        """Read the device-side validation counters — out-of-range edge ids of a CSR build that has just happened, and the
        embed kernel's count of unsorted / out-of-range data_batch entries — in one pipeline drain, and raise like the
        reference's index assert / scatter would.  Only when a new edge_index / data_batch tensor shows up."""
        pend, self._graphs.pending = self._graphs.pending, None
        if pend is not None:
            bad_e = int(pend.item())
            if bad_e:
                self._graphs.entries.clear()
                raise ValueError(f"edge_index has {bad_e} edge(s) with a node id outside [0, {N})")
        if counter is None:
            return
        bad = int(counter.item())
        if bad:
            raise ValueError(f"data_batch has {bad} entr{'y' if bad == 1 else 'ies'} that are not non-decreasing or "
                             f"lie outside [0, {B}) (B = loc_mean.shape[0]); PyG batches are sorted and the fused "
                             "per-graph reductions rely on it")
        self._validated_batch = (data_batch, data_batch._version, N, B)

    def _kernel_args(self, be, N: int, node_feat, node_loc, node_vel, loc_mean, edge_index, data_batch, edge_attr,
                     node_attr) -> Dict[str, Tensor]:
        """The caller's tensors as the kernels read them (float32, contiguous, detached), and the graph as rowptr, row,
        col, edge_attr in CSR order and the device edge count: from the cache / a radix sort for an int64 edge_index
        (then `perm` maps CSR positions to the caller's edges), or straight from a pre-sorted CSRGraph (shards.py) — then
        nothing is sorted or permuted."""
        from .shards import CSRGraph
        A, Na = self.edge_attr_nf, self.node_attr_nf
        f32 = lambda t: t if (t.dtype == torch.float32 and t.is_contiguous() and not t.requires_grad) \
            else t.detach().to(dtype=torch.float32).contiguous()
        a = dict(node_feat=f32(node_feat), node_loc=f32(node_loc), node_vel=f32(node_vel), loc_mean=f32(loc_mean),
                 attr=f32(node_attr) if Na > 0 else None, data_batch=data_batch.contiguous())
        if isinstance(edge_index, CSRGraph):
            a.update(rowptr=edge_index.rowptr.contiguous(), row=edge_index.rows().contiguous(),
                     col=edge_index.col.contiguous(), ea=f32(edge_attr) if A > 0 else None, nE=edge_index.n_edges_dev)
            return a
        B = int(loc_mean.shape[0])
        pos = None if self.deterministic else a["node_loc"]         # the deterministic mode's bits need id order (§17)
        rowptr, row, col, perm = self._graphs.get(be, edge_index, N, self.validate_inputs, pos,
                                                  None if B == 1 else a["data_batch"], B)
        ea = self._graphs.sorted_edge_attr(be, edge_index, edge_attr, perm) if A > 0 else None
        a.update(rowptr=rowptr, row=row, col=col, ea=ea, nE=None, perm=perm)
        return a

    # ---- device work ---------------------------------------------------------------------------
    def _det_workspace(self, ws: Dict[str, Tensor], dev, N: int, E: int) -> Tensor:
        """The deterministic mode's slots (csrc/det.cuh), kept in `ws` and grown to N nodes and E edges of capacity.  Growing
        replaces the tensor: a captured graph that wrote to the old one holds its own reference (`_forward_graphed`,
        `rollout`)."""
        nbytes = max(_lib.deterministic_workspace_bytes(N, E, self.virtual_channels), 1)
        det = ws.get("det")
        if det is None or det.numel() < nbytes:
            det = ws["det"] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        return det

    def _workspace(self, dev, N: int, B: int, K: int) -> Dict[str, Tensor]:
        """Per-shape buffers of the inference path, kept between calls.  `vsum`, `agg_m`, `agg_x` are accumulators: they
        start zeroed and every forward leaves them zeroed again (the consuming kernels clear them), so no memset is
        launched in steady state.  A forward that raised half-way marks the set dirty and it is re-zeroed."""
        key = (str(dev), N, B, K)
        ws = self._workspaces.get(key)
        if ws is None:
            Cn = self.virtual_channels
            new = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=dev)
            zeros = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
            ws = dict(h=new(N, H), P=new(N, H), Q=new(N, H), Hn=new(N, H), agg_m=zeros(N, H), agg_v=new(N, H),
                      x4=new(N, 4), agg_x=zeros(N, 4), trans_v=new(N, 4), batch32=new(N, dt=torch.int32),
                      vsum=zeros(B, K), G=new(B, Cn, H), Xv=new(B, 3, Cn), Hv=new(B, Cn, H), out=new(N, 3),
                      counter=torch.zeros(1, dtype=torch.int32, device=dev), dirty=False)
            while len(self._workspaces) >= 4:
                self._workspaces.pop(next(iter(self._workspaces)))
            self._workspaces[key] = ws
        return ws

    def _forward(self, be, pk, dims, a: Dict[str, Tensor], ws: Optional[Dict[str, Tensor]] = None,
                 out: Optional[Tensor] = None, Xv: Optional[Tensor] = None, init_centroid: bool = False):
        """Enqueue one forward on the current stream: 2 + 4L kernel launches; nothing syncs unless a new data_batch tensor
        has to be validated.  Returns (out, Xv, saved state or None).

        With a workspace `ws` (inference) nothing allocates: every buffer is reused, and the consuming kernels clear the
        accumulators for the next layer and the next call (FLAG_ZERO_AGG / FLAG_ZERO_VSUM).  Results are written to `out` /
        `Xv` (default: the workspace's own buffers, which the next forward overwrites).  Without one (the training path and
        the differentiable rollout's recompute) every layer writes fresh tensors, and the saved state keeps them for
        `_backward_saved`.

        `init_centroid` (rollouts): the initial virtual coordinates are the per-graph centroid of `node_loc` over all
        partitions, taken from the statistics the first exchange already sums, instead of `loc_mean` (which is then not
        read)."""
        A, Cn, Na, F = self.edge_attr_nf, self.virtual_channels, self.node_attr_nf, self.node_feat_nf
        N, E, B, K = dims
        L, layers = self.n_layers, pk["layers"]
        dev = a["node_loc"].device
        save = ws is None
        new = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=dev)
        zeros = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        if save:
            ws = dict(h=new(N, H), P=new(N, H), Q=new(N, H), Hn=new(N, H), x4=new(N, 4), batch32=new(N, dt=torch.int32),
                      vsum=zeros(B, K), G=new(B, Cn, H), Xv=new(B, 3, Cn), Hv=new(B, Cn, H), out=new(N, 3), dirty=False)
        h, P, Q, Hn, x4, batch32 = ws["h"], ws["P"], ws["Q"], ws["Hn"], ws["x4"], ws["batch32"]
        vsum, G, Hv = ws["vsum"], ws["G"], ws["Hv"]
        out = ws["out"] if out is None else out
        Xv = ws["Xv"] if Xv is None else Xv
        if ws["dirty"]:
            vsum.zero_(); ws["agg_m"].zero_(); ws["agg_x"].zero_()
        ws["dirty"] = True
        counter = None
        if not self._batch_checked(a["data_batch"], N, B):
            counter = zeros(1, dt=torch.int32) if save else ws["counter"].zero_()
        comm = self._get_comm(be, dev, B, K)
        det = self._det_workspace(ws, dev, N, E) if self.deterministic and L else None
        dk = {} if det is None else dict(det_ws=det)
        be.embed((N, B, F, A, Cn, Na), a["node_feat"], a["node_loc"], a["data_batch"], pk["emb_wt"], pk["emb_b"],
                 layers[0] if L else None, h, x4, batch32, P, Q, Hn, vsum, counter, **dk)
        self._check_batch(counter, a["data_batch"], N, B)
        st = dict(batch32=batch32, vsum_init=vsum, layers=[], comm=comm) if save else None
        if L == 0:
            vsum.zero_()
            out.copy_(a["node_loc"])
            Xv.copy_(a["loc_mean"].unsqueeze(-1).expand(B, 3, Cn))
            ws["dirty"] = False
            return out, Xv, st
        sync = comm is None and self.world_size > 1              # torch.distributed path (stand-in backend / no P2P)
        if sync:
            self._sync_virtual(vsum)
        # the saved statistics and aggregates of every layer outlive it: only the inference path clears them
        zero_vsum, zero_agg = (0, 0) if save else (_lib.FLAG_ZERO_VSUM, _lib.FLAG_ZERO_AGG)
        # FastEGNN.py:299-300 (initial Hv, Xv) are folded into the INIT update
        init = _lib.FLAG_INIT | zero_vsum | (_lib.FLAG_INIT_CENTROID if init_centroid else 0)
        be.virtual_update((B, A, Cn, Na), init, vsum, Xv, Hv, None, layers[0], G,
                          None if init_centroid else a["loc_mean"], pk["hv0"], comm)
        base = _lib.FLAG_NORMALIZE if self.normalize else 0
        timed = not save and self._timing is not None
        mark = _event if timed else (lambda: None)
        for i in range(L):
            last = i == L - 1
            flags = base | (_lib.FLAG_LAST if last else 0)
            lp, lp_next = layers[i], (None if last else layers[i + 1])
            if save:
                agg_m, agg_v = (None, None) if last else (zeros(N, H), new(N, H))
                agg_x, trans_v, vsum = zeros(N, 4), new(N, 4), zeros(B, K)
                hn, Pn, Qn, Hnn = (None,) * 4 if last else (new(N, H), new(N, H), new(N, H), new(N, H))
                x4n, Gn = new(N, 4), (None if last else new(B, Cn, H))
            else:
                agg_m, agg_v = (None, None) if last else (ws["agg_m"], ws["agg_v"])
                agg_x, trans_v = ws["agg_x"], ws["trans_v"]
                hn, Pn, Qn, Hnn = (None,) * 4 if last else (h, P, Q, Hn)
                x4n, Gn = x4, G
            t0 = mark()
            be.edge_layer((N, E, A, Cn, Na), flags, a["row"], a["col"], a["ea"], x4, P, Q, lp, agg_m, agg_x, a["nE"], **dk)
            t1 = mark()
            be.virtual_layer((N, B, A, Cn, Na), flags, batch32, x4, Hn, Xv, G, lp, agg_v, trans_v, vsum, **dk)
            t2 = mark()
            be.node_layer((N, B, A, Cn, Na), flags | zero_agg, a["rowptr"], batch32, h, x4, a["node_vel"], a["attr"], agg_m,
                          agg_x, agg_v, trans_v, lp, lp_next, hn, x4n, Pn, Qn, Hnn, out if last else None, vsum, **dk)
            t3 = mark()
            if sync:
                self._sync_virtual(vsum)
            if save:
                st["layers"].append(dict(h=h, x4=x4, P=P, Q=Q, Hn=Hn, Xv=Xv, Hv=Hv, G=G, agg_m=agg_m, agg_x=agg_x,
                                         agg_v=agg_v, trans_v=trans_v, vsum=vsum, flags=flags))
                Xv, Hv = Xv.clone(), (Hv if last else Hv.clone())
            # with a communicator the update kernel all-reduces `vsum` first and leaves the summed statistics in it
            be.virtual_update((B, A, Cn, Na), (flags & ~_lib.FLAG_NORMALIZE) | zero_vsum, vsum, Xv, Hv, lp, lp_next, Gn,
                              comm=comm)
            t4 = mark()
            if timed:
                self._timing.append((i, t0, t1, t2, t3, t4))
            h, x4, P, Q, Hn, G = hn, x4n, Pn, Qn, Hnn, Gn
        ws["dirty"] = False
        if save and self._keep_state is not None:
            self._keep_state.append(st)
        return out, Xv, st

    def _forward_graphed(self, be, pk, dims, a: Dict[str, Tensor], comm=None) -> Tuple[Tensor, Tensor]:
        """CUDA-graph replay of `_forward` (opt-in: `model.cuda_graph = True`).  Works for any world size when the
        virtual-node sync is the library's own peer-memory exchange (it is part of the update kernels, so the graph holds
        the collectives too; every rank must replay — same call sequence as eager).  The graph is keyed by the addresses
        and shapes of every tensor it reads, so it is valid for as long as the caller keeps passing the same (possibly
        in-place updated) tensors — inference loops, rollouts, benchmarks.  New tensors trigger a re-capture; after
        `_graph_max_captures` distinct keys the model falls back to eager launches for unseen keys."""
        key = (dims, id(pk), id(comm), self.deterministic) + tuple((k, v.data_ptr(), tuple(v.shape)) for k, v in a.items() if v is not None)
        ent = self._graph_cache.get(key)
        dev = a["node_loc"].device
        if ent is None:
            ws = self._workspace(dev, dims[0], dims[2], dims[3])
            if len(self._graph_cache) >= self._graph_max_captures:
                out, Xv, _ = self._forward(be, pk, dims, a, ws)
                return out.clone(), Xv.clone()
            # warm-up run + capture run: both are real forwards on every rank (the exchange inside stays matched)
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):            # warm-up outside capture: lazy inits (smem opt-ins)
                self._forward(be, pk, dims, a, ws)
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            g = torch.cuda.CUDAGraph()
            n0 = be.launches
            with torch.cuda.graph(g):
                self._forward(be, pk, dims, a, ws)
            # keep the keyed tensors alive: their addresses are baked in.  So is the deterministic workspace, which `ws`
            # swaps for a larger one when a later call brings more edges: the entry keeps the one it captured
            ent = (g, ws, be.launches - n0, a, pk, ws.get("det"))
            self._graph_cache[key] = ent
        ent[0].replay()
        be.launches += ent[2]
        return ent[1]["out"].clone(), ent[1]["Xv"].clone()


def _event():
    ev = torch.cuda.Event(enable_timing=True)
    ev.record()
    return ev


def device_guard(dev: torch.device):
    """Make `dev` current for the launches and shared-memory opt-ins of a call (no-op for the CPU stand-ins' tensors)."""
    return torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()


class _FastEGNNFunction(torch.autograd.Function):
    """Autograd node of the fused path.  forward = the sm_90a kernels (FastEGNN._forward, saving); backward = per layer, in
    reverse: virtual-node update, ONE packed all-reduce of the statistics' gradient (the reference's _AllReduce.backward,
    FastEGNN.py:19-21, issues one per aggregate), per-node stage, real<->virtual stage, per-edge stage, and finally the
    initial virtual state and the embedding prologue — every one a hand-written kernel behind the C ABI (csrc/*bwd*.cu,
    csrc/virtual_update.cu); torch only adds three gradient tensors per layer.

    With `model.input_grads` the six raw inputs (node_feat, node_loc, node_vel, loc_mean, edge_attr, node_attr) follow
    the parameter blocks, and the same kernels also produce the gradients of those that need one (ctx.needs_input_grad):
    edge_attr and node_vel / node_attr accumulate over the layers in the edge and node kernels, node_feat and node_loc
    come out of the embedding backward (node_loc = layer 0's coordinate gradient + the Σx term of the initial centroid,
    summed over the partitions by one more packed exchange), loc_mean is the channel sum of the initial Xv's gradient."""

    @staticmethod
    def forward(ctx, model, be, dims, a, emb_wt, emb_b, hv0, *rest):
        L = model.n_layers
        ctx.pk = _detached(emb_wt, emb_b, hv0, rest[:L])
        out, Xv, st = model._forward(be, ctx.pk, dims, a)
        ctx.model, ctx.be, ctx.dims, ctx.a, ctx.st = model, be, dims, a, st
        ctx.inputs = [None if t is None else (t.dtype, t.shape) for t in rest[L:]]
        return out, Xv

    @staticmethod
    def backward(ctx, g_out, g_Xv_out):
        model = ctx.model
        N, E, B, K = ctx.dims
        emb_wt, emb_b, hv0 = ctx.pk["emb_wt"], ctx.pk["emb_b"], ctx.pk["hv0"]
        L = len(ctx.pk["layers"])
        n_in = len(ctx.inputs)
        want = ctx.needs_input_grad[7 + L:7 + L + n_in] if n_in else (False,) * 6
        if L == 0:                                           # out = node_loc, Xv = loc_mean broadcast
            dev = emb_wt.device
            g_x = g_out.contiguous().to(torch.float32) if g_out is not None else torch.zeros(N, 3, device=dev)
            g_Xv = g_Xv_out.contiguous().to(torch.float32) if g_Xv_out is not None else \
                torch.zeros(B, 3, model.virtual_channels, device=dev)
            g_in = (None, g_x if want[1] else None, None, g_Xv.sum(-1) if want[3] else None, None, None)
            return (None, None, None, None, torch.zeros_like(emb_wt), torch.zeros_like(emb_b),
                    torch.zeros_like(hv0)) + _FastEGNNFunction._input_grads(ctx, g_in)
        g_emb_wt, g_emb_b, g_hv0, g_lps, g_in = _backward_saved(model, ctx.be, ctx.dims, ctx.a, ctx.st, ctx.pk, g_out,
                                                                      g_Xv_out, want)
        grads = (None, None, None, None, g_emb_wt, g_emb_b, g_hv0, *g_lps)
        if not n_in:
            return grads
        g_ea = g_in[4]
        if g_ea is not None and ctx.a.get("perm") is not None:             # CSR order -> the caller's edge order
            g_ea = ctx.be.gather_rows(g_ea, ctx.a["perm"], inverse=True)
        return grads + _FastEGNNFunction._input_grads(ctx, g_in[:4] + (g_ea,) + g_in[5:])

    @staticmethod
    def _input_grads(ctx, g_in):
        """Gradients of the six raw inputs in their own dtype; zeros for a wanted input that has no path to the outputs
        (edge_attr with edge_attr_nf = 0, node_attr with node_attr_nf = 0 or a single layer)."""
        if not ctx.inputs:
            return ()
        out = []
        for want, meta, g in zip(ctx.needs_input_grad[7 + len(ctx.pk["layers"]):], ctx.inputs, g_in):
            if not want:
                out.append(None)
                continue
            dtype, shape = meta
            dev = ctx.pk["emb_wt"].device
            out.append(torch.zeros(shape, dtype=dtype, device=dev) if g is None else g.to(dtype).reshape(shape))
        return tuple(out)


def _detached(emb_wt, emb_b, hv0, layers) -> Dict:
    """The packed parameters that an autograd node received, as `FastEGNN._forward` and `_backward_saved` read them."""
    return dict(layers=[lp.detach().contiguous() for lp in layers], emb_wt=emb_wt.detach().contiguous(),
                emb_b=emb_b.detach().contiguous(), hv0=hv0.detach().contiguous())


def _backward_saved(model: FastEGNN, be, dims, a, st, pk, g_out, g_Xv_out, want, init_centroid: bool = False):
    """The backward kernels of one forward whose activations `FastEGNN._forward` kept (L >= 1), shared by `_FastEGNNFunction` and the
    differentiable rollout.  `want` = which of (node_feat, node_loc, node_vel, loc_mean, edge_attr, node_attr) need a
    gradient.  Returns (g_emb_wt, g_emb_b, g_hv0, [g_layer_params], (g_feat, g_loc, g_vel, g_loc_mean, g_ea in CSR order,
    g_attr)), None for the inputs not wanted.

    `init_centroid`: the forward ran with FLAG_INIT_CENTROID (X_0 = x̄ of node_loc, from the summed initial statistics).
    The INIT update's backward then runs as a plain FLAG_INIT one with X_0 = that x̄, which returns the gradient w.r.t. X_0
    as if it were independent; since X_0 = Σx/n, Σ_c g_X0 / n is folded into the Σx entries of g_vsum0 before its exchange,
    and the embedding backward spreads it onto every node's g_loc.  No loc_mean gradient then."""
    N, E, B, K = dims
    A, Cn, Na = model.edge_attr_nf, model.virtual_channels, model.node_attr_nf
    emb_wt, emb_b, hv0, layers = pk["emb_wt"], pk["emb_b"], pk["hv0"], pk["layers"]
    L = len(layers)
    dev = emb_wt.device
    offs, total = _lib.param_layout(A, Cn, Na)
    zeros = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
    g_lps = [zeros(total) for _ in range(L)]
    g_emb_wt, g_emb_b, g_hv0 = torch.zeros_like(emb_wt), torch.zeros_like(emb_b), torch.zeros_like(hv0)
    w_feat, w_loc, w_vel, w_lm, w_ea, w_attr = want
    g_x = g_out.contiguous().to(torch.float32) if g_out is not None else zeros(N, 3)
    g_Xv = g_Xv_out.contiguous().to(torch.float32) if g_Xv_out is not None else zeros(B, 3, Cn)
    attr = a["attr"]
    # input-gradient accumulators, only for the inputs that need one (the kernels then take the *_inputs entry points)
    g_vel = zeros(N, 3) if w_vel else None
    g_attr = zeros(N, Na) if (w_attr and Na > 0) else None
    g_ea = zeros(E, A) if (w_ea and A > 0 and E > 0) else None          # CSR order
    kw_node = dict(g_vel=g_vel, g_attr=g_attr) if (g_vel is not None or g_attr is not None) else {}
    kw_edge = dict(g_ea=g_ea) if g_ea is not None else {}
    g_Hv = g_G = g_h = g_P = g_Q = g_Hn = None
    for i in reversed(range(L)):
        S = st["layers"][i]
        last = i == L - 1
        lp, lp_next = layers[i], (None if last else layers[i + 1])
        # ---- 1. virtual-node update (CUDA): (g_Xv', g_Hv', g_G') -> g_vsum, g_Xv, g_Hv, parameter gradients -------------
        g_vsum, g_Xv_i = torch.empty(B, K, device=dev), torch.empty(B, 3, Cn, device=dev)
        g_Hv_i = None if last else torch.empty(B, Cn, H, device=dev)
        be.virtual_update_bwd((B, A, Cn, Na), S["flags"] & ~_lib.FLAG_NORMALIZE, S["vsum"], S["Xv"], S["Hv"], lp, lp_next,
                              g_Xv, g_Hv, g_G, g_vsum, g_Xv_i, g_Hv_i, g_lps[i], None if last else g_lps[i + 1])
        if model.world_size > 1:                     # _AllReduce.backward (FastEGNN.py:19-21), one packed call
            model._sync_virtual(g_vsum, be, st.get("comm"))
        # ---- 2. node stage (CUDA): (g_x', g_h', g_P', g_Q', g_Hn') -> g_h, g_x, g_agg_*, g_trans_v, parameter gradients ----
        g_h_i, g_x_i = torch.empty(N, H, device=dev), torch.empty(N, 3, device=dev)
        g_agg_x, g_trans_v = torch.empty(N, 4, device=dev), torch.empty(N, 4, device=dev)
        g_agg_m = None if last else torch.empty(N, H, device=dev)
        g_agg_v = None if last else torch.empty(N, H, device=dev)
        be.node_layer_bwd((N, B, A, Cn, Na), S["flags"], a["rowptr"], st["batch32"], S["h"], a["node_vel"], attr,
                          S["agg_m"], S["agg_v"], lp, lp_next, g_x, g_vsum, g_h, g_P, g_Q, g_Hn, g_h_i, g_x_i,
                          g_agg_x, g_trans_v, g_agg_m, g_agg_v, g_lps[i], None if last else g_lps[i + 1], **kw_node)
        # ---- 3. real<->virtual stage (CUDA) ------------------------------------------------------------------------
        wT = be.virtual_bwd_prepare(A, Cn, Na, lp)           # operand images of the stage's weights for the tensor cores
        g_Hn_i, g_xv = torch.empty(N, H, device=dev), torch.empty(N, 4, device=dev)
        g_G_i, g_Xv_acc = zeros(B, Cn, H), g_Xv_i.contiguous().clone()
        be.virtual_layer_bwd((N, B, A, Cn, Na), S["flags"], st["batch32"], S["x4"], S["Hn"], S["Xv"], S["G"], lp, wT,
                             g_agg_v, g_trans_v, g_vsum, g_Hn_i, g_xv, g_G_i, g_Xv_acc, g_lps[i])
        # ---- 4. per-edge stage (CUDA) --------------------------------------------------------------------------------
        g_P_i, g_Q_i, g_x4e = zeros(N, H), zeros(N, H), zeros(N, 4)
        be.edge_layer_bwd((N, E, A, Cn, Na), S["flags"], a["row"], a["col"], a["ea"], S["x4"], S["P"], S["Q"], lp,
                          g_agg_m, g_agg_x, g_P_i, g_Q_i, g_x4e, g_lps[i], a["nE"], **kw_edge)
        g_x = g_x_i + g_xv[:, :3] + g_x4e[:, :3]
        g_h, g_P, g_Q, g_Hn = g_h_i, g_P_i, g_Q_i, g_Hn_i
        g_Xv, g_Hv, g_G = g_Xv_acc, g_Hv_i, g_G_i
    # ---- initial virtual state (CUDA): G_0 = f(Hv_0 = hv0, X_0 = loc_mean, x̄_0; layer-0 parameters) ---------------------
    # (init_centroid: X_0 = x̄ exactly as the forward's INIT update wrote it, kept as layer 0's Xv)
    Xv0 = st["layers"][0]["Xv"] if init_centroid else a["loc_mean"].unsqueeze(-1).expand(B, 3, Cn).contiguous()
    Hv0 = hv0.unsqueeze(0).expand(B, Cn, H).contiguous()
    g_Hv0 = torch.empty(B, Cn, H, device=dev)
    g_vsum0, g_Xv0 = torch.empty(B, K, device=dev), torch.empty(B, 3, Cn, device=dev)
    # with loc_mean wanted, layer 0's g_Xv goes in as the upstream of X_0, so g_Xv0 is the whole gradient w.r.t. X_0
    be.virtual_update_bwd((B, A, Cn, Na), _lib.FLAG_INIT, st["vsum_init"], Xv0, Hv0, None, layers[0],
                          g_Xv if (w_lm or init_centroid) else None, g_Hv, g_G, g_vsum0, g_Xv0, g_Hv0, None, g_lps[0])
    g_hv0 += g_Hv0.sum(0)                                # virtual_node_feat is shared by the graphs of the batch
    if init_centroid and w_loc:                          # X_0 = Σx / n: fold Σ_c g_X0 / n into the Σx entries
        g_vsum0[:, 0:3] += g_Xv0.sum(-1) / st["vsum_init"][:, 3:4].clamp(min=1.0)
    if w_loc and model.world_size > 1:                   # x̄_0 is all-reduced: its Σx gradient is summed back
        model._sync_virtual(g_vsum0, be, st.get("comm"))
    # ---- embedding + layer-0 projections (CUDA) ----------------------------------------------------------------------------
    g_feat = torch.empty(N, model.node_feat_nf, device=dev) if w_feat else None
    g_loc = torch.empty(N, 3, device=dev) if w_loc else None
    kw_emb = {} if (g_feat is None and g_loc is None) else dict(
        g_feat=g_feat, g_loc=g_loc, emb_wt=emb_wt, batch32=st["batch32"], g_x0=g_x.contiguous() if w_loc else None,
        g_vsum0=g_vsum0 if w_loc else None)
    be.embed_bwd((N, B, model.node_feat_nf, A, Cn, Na), a["node_feat"], st["layers"][0]["h"], layers[0], g_h, g_P, g_Q,
                 g_Hn, g_emb_wt, g_emb_b, g_lps[0], **kw_emb)
    g_lm = g_Xv0.sum(-1) if (w_lm and not init_centroid) else None
    return g_emb_wt, g_emb_b, g_hv0, g_lps, (g_feat, g_loc, g_vel, g_lm, g_ea if w_ea else None,
                                             g_attr if w_attr else None)
