"""The one place where torch tensors become raw device pointers for the C ABI.

`CudaBackend` is the product path.  It has no CPU branch: tensors must live on a CUDA device and the
shared library must load.  (tests/ contains a pure-torch stand-in with the same method names that is
used ONLY to exercise the host-side sequencing and the multi-partition all-reduce logic under gloo on
machines without a GPU; it is never importable from the package.)
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import check, ptr

Tensor = torch.Tensor


class CudaBackend:
    name = "cuda-sm100a"

    def __init__(self) -> None:
        self.lib = _lib.load()
        self.launches = 0          # kernels of ours enqueued (bench.py reports it as gpu_launches)

    # ---- helpers -------------------------------------------------------------------------------
    @staticmethod
    def _s(t: Tensor) -> int:
        if not t.is_cuda:
            raise _lib.DistEGNNError("distegnn_b200 has no CPU path: tensors must be on a CUDA device")
        return _lib.stream_ptr(t.device)

    # ---- graph preprocessing -------------------------------------------------------------------
    def build_csr(self, edge_index: Tensor, n_nodes: int, validate: bool = True
                  ) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """int64 COO -> int32 CSR by destination, rows in id order.  `validate`: read back the out-of-range counter (one
        host sync per build; builds are cached per edge_index) and raise ValueError like the reference's index assert
        would; validate="defer" hands the device counter back as a fifth value instead (the caller reads it together with
        the data_batch counter after the embed kernel: one pipeline drain for both checks; ids are clamped meanwhile)."""
        return self._build_csr(edge_index, n_nodes, validate, None, None, 1)

    def build_csr_cells(self, edge_index: Tensor, n_nodes: int, pos: Tensor, batch: Optional[Tensor], n_graphs: int,
                        validate: bool = True):
        """`build_csr` with the rows in (graph, cell of `pos`, id) order (DESIGN §3): the same rowptr, the edges of every
        row contiguous, the rows of nearby destinations next to each other.  `pos` float32 [N,3] contiguous, `batch`
        int64 sorted or None for one graph."""
        return self._build_csr(edge_index, n_nodes, validate, pos, batch, n_graphs)

    def _build_csr(self, edge_index, n_nodes, validate, pos, batch, n_graphs):
        E = int(edge_index.shape[1])
        dev = edge_index.device
        stream = self._s(edge_index)
        rowptr = torch.empty(n_nodes + 1, dtype=torch.int32, device=dev)
        row = torch.empty(E, dtype=torch.int32, device=dev)
        col = torch.empty(E, dtype=torch.int32, device=dev)
        perm = torch.empty(E, dtype=torch.int32, device=dev)
        nbytes = C.c_int64(0)
        check(self.lib.distegnn_csr_workspace_bytes(n_nodes, E, C.byref(nbytes)), "csr_workspace_bytes")
        ws = torch.empty(max(int(nbytes.value), 1), dtype=torch.uint8, device=dev)
        bad = torch.empty(1, dtype=torch.int32, device=dev) if validate else None
        if pos is None:
            check(self.lib.distegnn_build_csr(ptr(edge_index), n_nodes, E, ptr(rowptr), ptr(row), ptr(col),
                                              ptr(perm), ptr(ws), ws.numel(), ptr(bad), stream), "build_csr")
        else:
            check(self.lib.distegnn_build_csr_cells(ptr(edge_index), n_nodes, E, ptr(pos), ptr(batch), n_graphs,
                                                    ptr(rowptr), ptr(row), ptr(col), ptr(perm), ptr(ws), ws.numel(),
                                                    ptr(bad), stream), "build_csr_cells")
        self.launches += (6 + (7 if pos is not None else 0) if E else 1) + (1 if validate else 0)
        if validate == "defer":
            return rowptr, row, col, perm, (bad if E else None)
        if validate and E and int(bad.item()) != 0:
            raise ValueError(f"edge_index has {int(bad.item())} edge(s) with a node id outside [0, {n_nodes})")
        return rowptr, row, col, perm

    def gather_rows(self, src: Tensor, perm: Tensor, inverse: bool = False) -> Tensor:
        """dst[i] = src[perm[i]]; with `inverse` dst[perm[i]] = src[i] (CSR order back to the caller's edge order)."""
        dst = torch.empty_like(src)
        if src.numel():
            fn = self.lib.distegnn_scatter_rows if inverse else self.lib.distegnn_gather_rows
            check(fn(ptr(src), ptr(perm), src.shape[0], src.shape[1], ptr(dst), self._s(src)),
                  "scatter_rows" if inverse else "gather_rows")
            self.launches += 1
        return dst

    # ---- layer stages --------------------------------------------------------------------------
    def embed(self, dims, node_feat, node_loc, data_batch, emb_wt, emb_b, layer0, h, x4, batch32, P, Q,
              Hn, vsum, n_invalid=None, det_ws=None) -> None:
        """`n_invalid`: zeroed int32 [1] device counter of data_batch entries that are unsorted / outside [0,B).  `det_ws`
        (deterministic mode): the statistics in vsum are then recomputed from x4 in a fixed order."""
        N, B, F, A, Cn, Na = dims
        check(self.lib.distegnn_embed_fwd(N, B, F, A, Cn, Na, ptr(node_feat), ptr(node_loc),
                                          ptr(data_batch), ptr(emb_wt), ptr(emb_b), ptr(layer0), ptr(h),
                                          ptr(x4), ptr(batch32), ptr(P), ptr(Q), ptr(Hn), ptr(vsum),
                                          ptr(n_invalid), self._s(h)), "embed_fwd")
        self.launches += 1 if N else 0
        if det_ws is not None:
            self._vsum_combine(N, B, Cn, _lib.FLAG_INIT, batch32, x4, vsum, det_ws)

    def edge_layer(self, dims, flags, row, col, ea, x4, P, Q, lp, agg_m, agg_x, n_edges_dev=None, det_ws=None) -> None:
        """`n_edges_dev`: int32 [1] on the device with the true edge count when E is only a capacity (CSRGraph built on the
        device without a host round trip).  `det_ws` (uint8, deterministic_workspace_bytes): the deterministic kernel and
        its combine pass instead."""
        N, E, A, Cn, Na = dims
        if det_ws is None:
            check(self.lib.distegnn_edge_layer_fwd(N, E, A, Cn, Na, flags, ptr(row), ptr(col), ptr(ea),
                                                   ptr(x4), ptr(P), ptr(Q), ptr(lp), ptr(agg_m), ptr(agg_x),
                                                   ptr(n_edges_dev), self._s(x4)), "edge_layer_fwd")
            self.launches += 1 if E else 0
            return
        check(self.lib.distegnn_edge_layer_fwd_det(N, E, A, Cn, Na, flags, ptr(row), ptr(col), ptr(ea), ptr(x4), ptr(P),
                                                   ptr(Q), ptr(lp), ptr(agg_m), ptr(agg_x), ptr(n_edges_dev),
                                                   ptr(det_ws), det_ws.numel(), self._s(x4)), "edge_layer_fwd_det")
        check(self.lib.distegnn_edge_combine_det(N, E, Cn, ptr(row), ptr(n_edges_dev), ptr(agg_m), ptr(agg_x),
                                                 ptr(det_ws), det_ws.numel(), self._s(x4)), "edge_combine_det")
        self.launches += 2 if E else 0

    def _vsum_combine(self, N, B, Cn, flags, batch32, x4, vsum, det_ws) -> None:
        """Deterministic mode: vsum[:, 0:4] = Σ(x, 1) of x4 per graph in a fixed order; unless FLAG_INIT also the slots of
        the deterministic real<->virtual kernel, in chunk order."""
        check(self.lib.distegnn_vsum_combine_det(N, B, Cn, flags, ptr(batch32), ptr(x4), ptr(vsum), ptr(det_ws),
                                                 det_ws.numel(), self._s(vsum)), "vsum_combine_det")
        self.launches += 1

    def edge_layer_bwd(self, dims, flags, row, col, ea, x4, P, Q, lp, g_agg_m, g_agg_x, g_P, g_Q, g_x4, g_lp,
                       n_edges_dev=None, g_ea=None) -> None:
        """Backward of edge_layer: accumulates into g_P, g_Q, g_x4 and the parameter-gradient block g_lp; with `g_ea`
        ([E,A], CSR order) also into the gradient w.r.t. the edge attributes."""
        N, E, A, Cn, Na = dims
        args = (N, E, A, Cn, Na, flags, ptr(row), ptr(col), ptr(ea), ptr(x4), ptr(P), ptr(Q), ptr(lp), ptr(g_agg_m),
                ptr(g_agg_x), ptr(g_P), ptr(g_Q), ptr(g_x4), ptr(g_lp), ptr(n_edges_dev))
        if g_ea is None:
            check(self.lib.distegnn_edge_layer_bwd(*args, self._s(x4)), "edge_layer_bwd")
        else:
            check(self.lib.distegnn_edge_layer_bwd_inputs(*args, ptr(g_ea), self._s(x4)), "edge_layer_bwd_inputs")
        self.launches += 1 if E else 0

    def virtual_bwd_prepare(self, A, Cn, Na, lp) -> "torch.Tensor":
        """fp16 hi/lo operand images of the virtual stage's weights and their transposes (96 KB) for virtual_layer_bwd."""
        import torch
        img = torch.empty(6 * 2 * 64 * 64, dtype=torch.float16, device=lp.device)
        check(self.lib.distegnn_virtual_bwd_prepare(A, Cn, Na, ptr(lp), ptr(img), self._s(lp)), "virtual_bwd_prepare")
        self.launches += 1
        return img

    def virtual_layer_bwd(self, dims, flags, batch32, x4, Hn, Xv, G, lp, wimg, g_agg_v, g_trans_v, g_vsum, g_Hn, g_xv,
                          g_G, g_Xv, g_lp) -> None:
        """Backward of virtual_layer (tensor cores): writes g_Hn, g_xv; accumulates into g_G, g_Xv and the parameter gradients.
        `wimg` comes from virtual_bwd_prepare(lp)."""
        N, B, A, Cn, Na = dims
        check(self.lib.distegnn_virtual_layer_bwd(N, B, A, Cn, Na, flags, ptr(batch32), ptr(x4), ptr(Hn), ptr(Xv),
                                                  ptr(G), ptr(lp), ptr(wimg), ptr(g_agg_v), ptr(g_trans_v), ptr(g_vsum),
                                                  ptr(g_Hn), ptr(g_xv), ptr(g_G), ptr(g_Xv), ptr(g_lp), self._s(x4)),
              "virtual_layer_bwd")
        self.launches += 1 if N else 0

    def virtual_layer(self, dims, flags, batch32, x4, Hn, Xv, G, lp, agg_v, trans_v, vsum, det_ws=None) -> None:
        """`det_ws`: the deterministic kernel (vsum is complete only after vsum_combine)."""
        N, B, A, Cn, Na = dims
        args = (N, B, A, Cn, Na, flags, ptr(batch32), ptr(x4), ptr(Hn), ptr(Xv), ptr(G), ptr(lp), ptr(agg_v), ptr(trans_v),
                ptr(vsum))
        if det_ws is None:
            check(self.lib.distegnn_virtual_layer_fwd(*args, self._s(x4)), "virtual_layer_fwd")
        else:
            check(self.lib.distegnn_virtual_layer_fwd_det(*args, ptr(det_ws), det_ws.numel(), self._s(x4)),
                  "virtual_layer_fwd_det")
        self.launches += 1 if N else 0

    def node_layer(self, dims, flags, rowptr, batch32, h, x4, vel, attr, agg_m, agg_x, agg_v, trans_v,
                   lp, lp_next, h_out, x4_out, P, Q, Hn, loc_out, vsum, det_ws=None) -> None:
        """`det_ws` (deterministic mode): vsum is completed by the combine pass (Σ(x, 1) from x4_out in a fixed order, and
        the slots of the deterministic real<->virtual kernel)."""
        N, B, A, Cn, Na = dims
        check(self.lib.distegnn_node_layer_fwd(N, B, A, Cn, Na, flags, ptr(rowptr), ptr(batch32), ptr(h),
                                               ptr(x4), ptr(vel), ptr(attr), ptr(agg_m), ptr(agg_x),
                                               ptr(agg_v), ptr(trans_v), ptr(lp), ptr(lp_next),
                                               ptr(h_out), ptr(x4_out), ptr(P), ptr(Q), ptr(Hn),
                                               ptr(loc_out), ptr(vsum), self._s(x4)), "node_layer_fwd")
        self.launches += 1 if N else 0
        if det_ws is not None:
            self._vsum_combine(N, B, Cn, flags & _lib.FLAG_LAST, batch32, x4_out, vsum, det_ws)

    def node_layer_bwd(self, dims, flags, rowptr, batch32, h, vel, attr, agg_m, agg_v, lp, lp_next, g_x_out, g_vsum,
                       g_h_out, g_P, g_Q, g_Hn, g_h, g_x, g_agg_x, g_trans_v, g_agg_m, g_agg_v, g_lp, g_lp_next,
                       g_vel=None, g_attr=None) -> None:
        """Backward of node_layer (csrc/node_layer_bwd.cu): writes g_h, g_x [N,3], g_agg_x, g_trans_v [N,4], g_agg_m, g_agg_v;
        accumulates parameter gradients into g_lp (this layer) and g_lp_next (the projections of the next layer), and, when
        given, the input gradients g_vel [N,3] and g_attr [N,Na]."""
        N, B, A, Cn, Na = dims
        args = (N, A, Cn, Na, flags, ptr(rowptr), ptr(h), ptr(vel), ptr(attr), ptr(agg_m), ptr(agg_v), ptr(lp),
                ptr(lp_next), ptr(g_x_out), ptr(g_vsum), ptr(batch32), ptr(g_h_out), ptr(g_P), ptr(g_Q), ptr(g_Hn),
                ptr(g_h), ptr(g_x), ptr(g_agg_x), ptr(g_trans_v), ptr(g_agg_m), ptr(g_agg_v), ptr(g_lp), ptr(g_lp_next))
        if g_vel is None and g_attr is None:
            check(self.lib.distegnn_node_layer_bwd(*args, self._s(h)), "node_layer_bwd")
        else:
            check(self.lib.distegnn_node_layer_bwd_inputs(*args, ptr(g_vel), ptr(g_attr), self._s(h)),
                  "node_layer_bwd_inputs")
        self.launches += 1 if N else 0

    def embed_bwd(self, dims, node_feat, h0, lp0, g_h, g_P, g_Q, g_Hn, g_emb_wt, g_emb_b, g_lp0, g_feat=None, g_loc=None,
                  emb_wt=None, batch32=None, g_x0=None, g_vsum0=None) -> None:
        """Backward of embed: accumulates g_emb_wt [F,64], g_emb_b [64] and layer 0's projection gradients into g_lp0.  With
        `g_feat` writes the gradient w.r.t. node_feat (needs `emb_wt`); with `g_loc` the gradient w.r.t. node_loc,
        g_x0 + g_vsum0[batch, 0:3] (g_x0: w.r.t. layer 0's coordinates; g_vsum0: w.r.t. the initial statistics)."""
        N, B, F, A, Cn, Na = dims
        args = (N, F, A, Cn, Na, ptr(node_feat), ptr(h0), ptr(lp0), ptr(g_h), ptr(g_P), ptr(g_Q), ptr(g_Hn), ptr(g_emb_wt),
                ptr(g_emb_b), ptr(g_lp0))
        if g_feat is None and g_loc is None:
            check(self.lib.distegnn_embed_bwd(*args, self._s(h0)), "embed_bwd")
        else:
            check(self.lib.distegnn_embed_bwd_inputs(*args, ptr(emb_wt), ptr(batch32), ptr(g_x0), ptr(g_vsum0),
                                                     ptr(g_feat), ptr(g_loc), self._s(h0)), "embed_bwd_inputs")
        self.launches += 1 if N else 0

    def virtual_update(self, dims, flags, vsum, Xv, Hv, lp, lp_next, G, init_loc_mean=None, init_hv0=None,
                       comm: "Optional[Comm]" = None) -> None:
        """Virtual-node update; with `comm` the same kernel first all-reduces vsum over the partitions (NVLink peer
        memory) — the fused form of weighted_average_reduce + update."""
        B, A, Cn, Na = dims
        check(self.lib.distegnn_virtual_update_fwd(B, A, Cn, Na, flags, ptr(vsum), ptr(Xv), ptr(Hv),
                                                   ptr(lp), ptr(lp_next), ptr(G), ptr(init_loc_mean), ptr(init_hv0),
                                                   comm.handle if comm is not None else None, self._s(vsum)),
              "virtual_update_fwd")
        self.launches += 1 if B else 0

    def virtual_update_bwd(self, dims, flags, vsum, Xv, Hv, lp, lp_next, g_Xn, g_Hn, g_G, g_vsum, g_Xv, g_Hv, g_lp,
                           g_lp_next) -> None:
        """Backward of virtual_update (csrc/virtual_update.cu): writes g_vsum, g_Xv, g_Hv; accumulates into g_lp / g_lp_next."""
        B, A, Cn, Na = dims
        check(self.lib.distegnn_virtual_update_bwd(B, A, Cn, Na, flags, ptr(vsum), ptr(Xv), ptr(Hv), ptr(lp), ptr(lp_next),
                                                   ptr(g_Xn), ptr(g_Hn), ptr(g_G), ptr(g_vsum), ptr(g_Xv), ptr(g_Hv),
                                                   ptr(g_lp), ptr(g_lp_next), self._s(vsum)), "virtual_update_bwd")
        self.launches += 1 if B else 0

    # ---- rollout (csrc/rollout.cu) -------------------------------------------------------------------------------------
    def graph_buffers(self, n_nodes: int, capacity: int, edge_attr_nf: int, device):
        from .partition import RadiusGraphBuffers
        return RadiusGraphBuffers(n_nodes, capacity, edge_attr_nf, device)

    def radius_graph_into(self, buf, pos: Tensor, r: float, batch: Optional[Tensor], n_graphs: int, loop: bool) -> None:
        """Capacity-mode radius graph of `pos` into the preallocated `partition.RadiusGraphBuffers` (no host sync)."""
        from .partition import radius_graph_csr
        radius_graph_csr(pos, r, batch, loop=loop, edge_attr_nf=buf.edge_attr_nf, n_graphs=n_graphs, out=buf)
        self.launches += 7 if pos.shape[0] else 0            # ours; the cub scans and the radix sort come on top

    def cutoff_into(self, buf, graph, pos: Tensor, rate: float, batch: Optional[Tensor], n_graphs: int) -> None:
        """The kept edges of `graph` (the shortest int(E_b·(1 − rate)) of every graph) into the preallocated
        `partition.RadiusGraphBuffers` `buf` (csrc/cutoff_csr.cu; no host sync)."""
        from .partition import cutoff_edges_csr
        cutoff_edges_csr(graph, pos, rate, batch, n_graphs, buf.edge_attr_nf, out=buf)
        self.launches += (14 if graph.num_edges else 3) if pos.shape[0] else 0   # ours; two cub scans on top

    def edge_lengths(self, row: Tensor, col: Tensor, pos: Tensor, n_edges_dev: Optional[Tensor], ea: Tensor) -> None:
        """edge_attr[e, :] = ‖pos[row[e]] − pos[col[e]]‖ in CSR order, in place."""
        E, A = int(ea.shape[0]), int(ea.shape[1])
        check(self.lib.distegnn_edge_lengths_csr(E, A, ptr(row), ptr(col), ptr(pos), ptr(n_edges_dev), ptr(ea),
                                                 self._s(pos)), "edge_lengths_csr")
        self.launches += 1 if E and A else 0

    def rollout_advance(self, speed_col: int, tau: float, pred: Tensor, loc: Tensor, vel: Tensor, feat: Optional[Tensor],
                        traj: Optional[Tensor], edge_count: Tensor, overflow: Optional[Tensor], n_edges: Tensor,
                        counter: Tensor) -> None:
        """One step's state update (see distegnn_rollout_advance); `feat` None = no speed feature."""
        N, F = int(loc.shape[0]), (int(feat.shape[1]) if feat is not None else 0)
        check(self.lib.distegnn_rollout_advance(N, F, speed_col if feat is not None else -1, float(tau), int(n_edges.numel()),
                                                ptr(pred), ptr(loc), ptr(vel), ptr(feat), ptr(traj), ptr(edge_count),
                                                ptr(overflow), ptr(n_edges), ptr(counter), self._s(loc)), "rollout_advance")
        self.launches += 1

    def edge_lengths_bwd(self, row: Tensor, col: Tensor, pos: Tensor, n_edges_dev: Optional[Tensor], g_ea: Tensor,
                         g_pos: Tensor) -> None:
        """g_pos [N,3] += the gradient of edge_attr[e, :] = ‖pos[row[e]] − pos[col[e]]‖ given g_ea [E,A] (CSR order)."""
        E, A = int(g_ea.shape[0]), int(g_ea.shape[1])
        check(self.lib.distegnn_edge_lengths_bwd(E, A, ptr(row), ptr(col), ptr(pos), ptr(n_edges_dev), ptr(g_ea),
                                                 ptr(g_pos), self._s(pos)), "edge_lengths_bwd")
        self.launches += 1 if E and A else 0

    def rollout_advance_bwd(self, speed_col: Optional[int], tau: float, x_next: Tensor, x: Tensor,
                            g_traj: Optional[Tensor], g_x_next: Optional[Tensor], g_v_next: Optional[Tensor],
                            g_feat_next: Optional[Tensor], g_pred: Tensor, g_x: Tensor) -> None:
        """Backward of one rollout_advance: writes g_pred (upstream of the step's prediction) and g_x (the advance's part
        of the gradient of x_t); reads and zeroes g_feat_next[:, speed_col]."""
        N = int(x.shape[0])
        F = int(g_feat_next.shape[1]) if g_feat_next is not None else 0
        check(self.lib.distegnn_rollout_advance_bwd(N, F, speed_col if g_feat_next is not None else -1, float(tau),
                                                    ptr(x_next), ptr(x), ptr(g_traj), ptr(g_x_next), ptr(g_v_next),
                                                    ptr(g_feat_next), ptr(g_pred), ptr(g_x), self._s(x)),
              "rollout_advance_bwd")
        self.launches += 1 if N else 0

    def rollout_centroid(self, pos: Tensor, batch: Optional[Tensor], sums: Tensor, deterministic: bool = False) -> None:
        """sums float64 [B,4] += per-graph (Σx, Σy, Σz, count); `deterministic`: in a fixed order."""
        fn = self.lib.distegnn_rollout_centroid_det if deterministic else self.lib.distegnn_rollout_centroid
        check(fn(int(pos.shape[0]), int(sums.shape[0]), ptr(pos), ptr(batch), ptr(sums), self._s(pos)), "rollout_centroid")
        self.launches += 1 if pos.shape[0] else 0

    def rollout_sq_err(self, pred: Tensor, targets: Tensor, batch: Optional[Tensor], counter: Tensor, sq_err: Tensor,
                       ws: Tensor) -> None:
        """sq_err float64 [steps,B] row counter[0] = per-graph Σ‖pred − targets[counter[0]]‖² (see
        distegnn_rollout_sq_err; `ws` from rollout_sq_err_workspace, zeroed)."""
        N = int(pred.shape[0])
        check(self.lib.distegnn_rollout_sq_err(N, int(sq_err.shape[1]), int(sq_err.shape[0]), ptr(pred), ptr(targets),
                                               ptr(batch), ptr(counter), ptr(sq_err), ptr(ws), ws.numel(),
                                               self._s(pred)), "rollout_sq_err")
        self.launches += 1 if N else 0

    def rollout_sq_err_workspace(self, n_nodes: int, device) -> Tensor:
        nbytes = C.c_int64(0)
        check(self.lib.distegnn_rollout_sq_err_workspace_bytes(n_nodes, C.byref(nbytes)), "rollout_sq_err_workspace_bytes")
        return torch.zeros(int(nbytes.value), dtype=torch.uint8, device=device)

    def rollout_chamfer(self, pred: Tensor, targets: Tensor, batch: Optional[Tensor], counter: Tensor, chamfer: Tensor,
                        ws: Tensor) -> None:
        """chamfer float64 [steps,B,2] row counter[0] = per-graph Chamfer sums of pred against targets[counter[0]], both
        directions (see distegnn_rollout_chamfer; `ws` from rollout_chamfer_workspace)."""
        N = int(pred.shape[0])
        check(self.lib.distegnn_rollout_chamfer(N, int(chamfer.shape[1]), int(chamfer.shape[0]), ptr(pred),
                                                ptr(targets), ptr(batch), ptr(counter), ptr(chamfer), ptr(ws),
                                                ws.numel(), self._s(pred)), "rollout_chamfer")
        self.launches += 7 if N else 0                         # ours; the cub scan comes on top

    def rollout_chamfer_workspace(self, n_nodes: int, n_graphs: int, device) -> Tensor:
        nbytes = C.c_int64(0)
        check(self.lib.distegnn_rollout_chamfer_workspace_bytes(n_nodes, n_graphs, C.byref(nbytes)),
              "rollout_chamfer_workspace_bytes")
        return torch.empty(int(nbytes.value), dtype=torch.uint8, device=device)

    def chamfer_distance(self, pred: Tensor, target: Tensor, batch: Optional[Tensor], out: Tensor, nearest: Tensor,
                         ws: Tensor) -> None:
        """out float64 [B,2] = per-graph Chamfer sums of pred against target, nearest int32 [2N] the minimiser of every
        minimum (see distegnn_chamfer_distance; `ws` from rollout_chamfer_workspace)."""
        N = int(pred.shape[0])
        check(self.lib.distegnn_chamfer_distance(N, int(out.shape[0]), ptr(pred), ptr(target), ptr(batch), ptr(out),
                                                 ptr(nearest), ptr(ws), ws.numel(), self._s(pred)), "chamfer_distance")
        self.launches += 7 if N else 0                         # ours; the cub scan comes on top

    def chamfer_distance_bwd(self, pred: Tensor, target: Tensor, batch: Optional[Tensor], nearest: Tensor, g: Tensor,
                             g_pred: Optional[Tensor], g_target: Optional[Tensor], ws: Tensor) -> None:
        """g_pred / g_target [N,3] (either may be None: not written) = the gradient of chamfer_distance's sums given the
        upstream g float64 [B,2] (see distegnn_chamfer_distance_bwd; `ws` from chamfer_distance_bwd_workspace)."""
        N = int(pred.shape[0])
        check(self.lib.distegnn_chamfer_distance_bwd(N, int(g.shape[0]), ptr(pred), ptr(target), ptr(batch),
                                                     ptr(nearest), ptr(g), ptr(g_pred), ptr(g_target), ptr(ws),
                                                     ws.numel(), self._s(pred)), "chamfer_distance_bwd")
        self.launches += 2 if N and (g_pred is not None or g_target is not None) else 0   # ours; the cub sort on top

    def chamfer_distance_bwd_workspace(self, n_nodes: int, device) -> Tensor:
        nbytes = C.c_int64(0)
        check(self.lib.distegnn_chamfer_distance_bwd_workspace_bytes(n_nodes, C.byref(nbytes)),
              "chamfer_distance_bwd_workspace_bytes")
        return torch.empty(int(nbytes.value), dtype=torch.uint8, device=device)

    def allreduce_packed(self, comm: "Comm", buf: Tensor) -> None:
        """In-place SUM of `buf` over the partitions through the communicator's peer-mapped segments."""
        check(self.lib.distegnn_allreduce_packed(comm.handle, ptr(buf), buf.numel(), self._s(buf)), "allreduce_packed")
        self.launches += 1 if buf.numel() else 0


class Comm:
    """Communicator of the virtual-node sync (C ABI: distegnn_comm_*).  One per (process group, capacity).  The IPC
    handles are all-gathered with torch.distributed (plumbing); the exchange itself is the library's own kernel."""

    def __init__(self, lib, device: torch.device, group, max_slots: int, slot_floats: int):
        import torch.distributed as dist
        self.lib, self.group, self.handle = lib, group, None
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.max_slots, self.slot_floats = int(max_slots), int(slot_floats)
        nb = lib.distegnn_comm_handle_bytes()
        mine = (C.c_ubyte * nb)()
        h = C.c_void_p()
        with torch.cuda.device(device):
            check(lib.distegnn_comm_init(self.rank, self.world, self.max_slots, self.slot_floats, C.byref(h), mine),
                  "comm_init")
            self.handle = h
            gathered = [None] * self.world
            dist.all_gather_object(gathered, bytes(mine), group=group)
            allh = (C.c_ubyte * (nb * self.world)).from_buffer_copy(b"".join(gathered))
            rc = lib.distegnn_comm_connect(self.handle, allh)
            # every rank must agree on the outcome: a half-connected group would dead-lock in the first exchange
            oks = [None] * self.world
            dist.all_gather_object(oks, rc == 0, group=group)
            if not all(oks):
                msg = lib.distegnn_last_error().decode("utf-8", "replace") if rc != 0 else "a peer failed to connect"
                self.destroy()
                raise _lib.DistEGNNError(f"comm_connect failed: {msg}")

    def status(self) -> int:
        v = C.c_int(0)
        check(self.lib.distegnn_comm_status(self.handle, C.byref(v)), "comm_status")
        return int(v.value)

    def destroy(self) -> None:
        """Collective teardown: unmap the peers, wait until every rank has done so, then free the own segment."""
        if self.handle is not None:
            import torch.distributed as dist
            self.lib.distegnn_comm_disconnect(self.handle)
            try:
                dist.barrier(group=self.group)
            except Exception:        # noqa: BLE001 — process group already gone: nothing left to order against
                pass
            self.lib.distegnn_comm_destroy(self.handle)
            self.handle = None


_cuda_backend: Optional[CudaBackend] = None


def cuda_backend() -> CudaBackend:
    global _cuda_backend
    if _cuda_backend is None:
        _cuda_backend = CudaBackend()
    return _cuda_backend
