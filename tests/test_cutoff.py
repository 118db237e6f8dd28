"""Edge cutoff (FastEGNN's cutoff_edges mode): keep the shortest int(E_b·(1 − rate)) edges of every graph (DESIGN §16).

CPU: the C-ABI argument checks, Python validation, the oracle against the reference's own `cutoff_edge` (fixtures from
oracle/make_golden_cutoff.py), and rollouts with a torch stand-in for the kernels: overflow regrowth from the candidate
count, kept counts in n_edges, differentiable_rollout against float64 autograd of the oracle pipeline.
GPU: the kernel against the fixtures (tie-robust) and the oracle (exact on lattices), the count rule, edge shapes,
rate 0 leaving the default path alone, rollouts against the float64 oracle, no host sync, graphed == eager, SE(3)
equivariance, training through a cut rollout, and the entry point."""
import glob
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distegnn_b200 import FastEGNN, _lib, cutoff_edges_csr, differentiable_rollout, radius_graph_csr, rollout, synth
from distegnn_b200.backend import CudaBackend
from distegnn_b200.shards import CSRGraph
from oracle import cutoff_oracle as co
from oracle import fastegnn_oracle as orc
from tests.test_rollout import FLUID, MARGIN, RUN_TO_RUN
from tests.test_rollout_grad import (RolloutGradStandIn, _cots, _compare, _leaves, _oracle_grads, _radius_edges, _rel)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "cutoff_*.npz")))


def _golden(path):
    z = np.load(path)
    return {k: z[k] for k in z.files}


def _per_graph(ei, batch, B):
    g = batch[ei[0]]
    return [ei[:, g == b] for b in range(B)]


# ---- torch stand-in of the cutoff kernel (CPU tests only) ---------------------------------------------------------------
class CutoffStandIn(RolloutGradStandIn):
    """RolloutGradStandIn plus the cutoff: the oracle's selection on the fp32 lengths, into the same buffer fields."""

    def __init__(self, inflate=None):
        super().__init__(inflate)
        self.cuts = 0

    def cutoff_into(self, buf, graph, pos, rate, batch, n_graphs):
        cap = graph.num_edges
        nc = int(graph.n_edges_dev[0]) if graph.n_edges_dev is not None else int(graph.rowptr[-1])
        valid = min(nc, cap)
        rowptr = graph.rowptr.clamp(max=valid).long()
        row, col = graph.rows()[:valid].long(), graph.col[:valid].long()
        length = (pos[row] - pos[col]).norm(dim=1)
        rp, r_out, c_out, l_out, _ = co.cutoff_csr(rowptr.numpy(), row.numpy(), col.numpy(), pos.numpy(), rate,
                                                   None if batch is None else batch.numpy(), n_graphs,
                                                   lengths=length.numpy())
        k = r_out.shape[0]
        buf.rowptr.copy_(torch.from_numpy(rp).to(torch.int32))
        buf.row[:k], buf.col[:k] = torch.from_numpy(r_out).to(torch.int32), torch.from_numpy(c_out).to(torch.int32)
        if buf.edge_attr is not None:
            buf.edge_attr[:k] = torch.from_numpy(l_out).float()[:, None]
        overflow = graph.info is not None and int(graph.info[1]) != 0
        buf.info[0], buf.info[1], buf.info[2] = k, int(nc > cap or overflow), nc
        self.cuts += 1


def _cpu_case(n=160, seed=0, layers=2):
    w = synth.WORKLOADS["fluid113k"]
    inp = synth.make_partitions(w, n_nodes=n, seed=seed)[0]
    sd = orc.init_state_dict(3, 2, 2, 64, 5, layers, seed=1, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, **dict(FLUID, n_layers=layers))
    m.load_state_dict(sd)
    node = {k: v for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
    return m, node, w.radius, sd


def _kept_graphs(states, r, batch, rate, B):
    """The oracle's kept edges of each state's radius candidates (destination-major order, fp32 lengths)."""
    out = []
    for x in states:
        ei = _radius_edges(x, r, batch)
        length = (x.float()[ei[0]] - x.float()[ei[1]]).norm(dim=1).numpy()
        out.append(torch.from_numpy(co.cutoff_edge_index(ei.numpy(), x.numpy(), rate, batch.numpy(), B, length)))
    return out


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_cabi_argument_checks():
    import ctypes as C
    lib = _lib.load()
    p = 256                                                    # any non-null pointer: never dereferenced
    cut = lib.distegnn_cutoff_csr

    def call(rate=0.5, pos=p, rowptr_out=p, row_in=p, ws=p, ws_bytes=1 << 40, n=10, B=1, batch=None, A=2):
        return cut(n, B, pos, batch, rate, A, p, row_in, p, None, 100, None, rowptr_out, p, p, p, p, ws, ws_bytes, None)

    for rate in (-0.1, 1.5, float("nan"), float("inf")):
        assert call(rate=rate) == -1
        assert "cutoff_rate" in lib.distegnn_last_error().decode()
    assert call(pos=None) == -1 and "null pointer" in lib.distegnn_last_error().decode()
    assert call(rowptr_out=None) == -1
    assert call(row_in=None) == -1
    assert call(ws=None) == -1
    assert call(B=2) == -1 and "data_batch" in lib.distegnn_last_error().decode()
    assert call(n=0) == -1
    assert call(A=_lib.MAX_EDGE_ATTR + 1) == -1
    assert call(ws_bytes=16) == -3 and "workspace" in lib.distegnn_last_error().decode()
    nb = C.c_int64(0)
    assert lib.distegnn_cutoff_csr_workspace_bytes(10, 0, 100, C.byref(nb)) == -1
    assert lib.distegnn_cutoff_csr_workspace_bytes(10, 1, -1, C.byref(nb)) == -1
    assert lib.distegnn_abi_version() == 3


def test_python_validation():
    pos = torch.zeros(4, 3)
    g = CSRGraph(torch.zeros(5, dtype=torch.int32), torch.zeros(0, dtype=torch.int32))
    for bad in (-0.1, 1.01, float("nan"), "0.5", True, None):
        with pytest.raises(ValueError):
            cutoff_edges_csr(g, pos, bad)
        with pytest.raises(ValueError):
            radius_graph_csr(pos, 0.1, cutoff_rate=bad)
    with pytest.raises(_lib.DistEGNNError):                    # CPU tensors: no CPU path
        cutoff_edges_csr(g, pos, 0.5)
    with pytest.raises(_lib.DistEGNNError):
        radius_graph_csr(pos, 0.1, cutoff_rate=0.5)
    m, node, r, _ = _cpu_case(n=40)
    m._backend = CutoffStandIn()
    for fn in (rollout, differentiable_rollout):
        with pytest.raises(ValueError):
            fn(m, **node, steps=2, radius=r, cutoff_rate=1.5)
        with pytest.raises(ValueError):
            fn(m, **node, steps=2, radius=r, cutoff_rate="half")
    m2 = FastEGNN(hidden_nf=64, world_size=2, **dict(FLUID, n_layers=2))
    m2._backend = CutoffStandIn()
    for fn in (rollout, differentiable_rollout):               # the cutoff mode is single-device
        with pytest.raises(ValueError, match="single-device"):
            fn(m2, **node, steps=2, radius=r, cutoff_rate=0.5)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[7:-4] for p in GOLDEN])
def test_oracle_against_the_reference_fixtures(path):
    """The reference's tie order is torch.sort's; the oracle's is candidate order.  So: per-graph counts, the length
    multisets and the edges strictly below each graph's threshold agree exactly (bitwise on the lattices, where fp32
    lengths are exact); the whole kept set agrees wherever the only ties are mirror pairs split the same way."""
    z = _golden(path)
    pos, batch, cand, kept, rate = z["pos"], z["batch"], z["candidates"], z["kept"], float(z["rate"])
    B = int(batch.max()) + 1
    l32 = lambda ei: (torch.from_numpy(pos)[ei[0]] - torch.from_numpy(pos)[ei[1]]).norm(dim=1).numpy()
    mine = co.cutoff_edge_index(cand, pos, rate, batch, B, l32(cand))
    for b, (ref_b, mine_b, cand_b) in enumerate(zip(_per_graph(kept, batch, B), _per_graph(mine, batch, B),
                                                    _per_graph(cand, batch, B))):
        assert ref_b.shape[1] == mine_b.shape[1] == co.k_of(cand_b.shape[1], rate)
        lr, lm = np.sort(l32(ref_b)), np.sort(l32(mine_b))
        assert np.array_equal(lr.view(np.uint32), lm.view(np.uint32)), f"graph {b}: length multisets differ"
        thr = lr[-1]
        below = lambda ei: set(map(tuple, ei[:, l32(ei) < thr].T.tolist()))
        assert below(ref_b) == below(mine_b)
    if "lattice" not in path:
        assert set(map(tuple, kept.T.tolist())) == set(map(tuple, mine.T.tolist()))


def test_rollout_overflow_regrows_from_the_candidate_count():
    m, node, r, _ = _cpu_case(n=160, layers=4)
    m.load_state_dict(orc.init_state_dict(3, 2, 2, 64, 5, 4, seed=1, coord_gain=0.05))
    m._backend = be0 = CutoffStandIn()
    ref = rollout(m, **node, steps=6, radius=r, speed_col=0, check_every=3, return_trajectory=True, cutoff_rate=0.5)
    cap = ref.capacity
    states = [node["node_loc"]] + list(ref.trajectory[:-1])
    cands = [_radius_edges(x, r, node["data_batch"]).shape[1] for x in states]
    assert cap == math.ceil(1.25 * cands[0]) and be0.cuts == 6
    assert ref.n_edges.tolist() == [co.k_of(c, 0.5) for c in cands]           # the kept counts
    assert int(ref.status[6]) == max(cands)
    forced = 4 * cap
    m._backend = be = CutoffStandIn(inflate={3: forced})
    res = rollout(m, **node, steps=6, radius=r, speed_col=0, check_every=3, capacity=cap, return_trajectory=True,
                  cutoff_rate=0.5)
    grown = math.ceil(1.25 * forced)                                            # from the candidates, not the kept
    assert res.regrowths == [grown] and res.capacity == grown
    assert be.builds == [(s, cap) for s in range(6)] + [(s, grown) for s in range(3, 6)]
    for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "virtual_loc", "trajectory", "n_edges"):
        assert torch.equal(getattr(res, k), getattr(ref, k)), k
    res.check()
    # rate 0 is the default path: no cutoff call at all
    m._backend = be = CutoffStandIn()
    rollout(m, **node, steps=2, radius=r, cutoff_rate=0.0)
    assert be.cuts == 0


def test_differentiable_rollout_with_cutoff_against_oracle_autograd():
    """3 steps, radius candidates, cutoff 0.5: every parameter and all five inputs against float64 autograd of the oracle
    pipeline on the kept graphs."""
    m, node, r, sd = _cpu_case(n=160, seed=2)
    m._backend = CutoffStandIn()
    leaf = _leaves(node)
    steps, tau, C = 3, 0.5, FLUID["virtual_channels"]
    cot, cotX = _cots(steps, 160, 1, C)
    res = differentiable_rollout(m, **leaf, steps=steps, radius=r, speed_col=0, tau=tau, cutoff_rate=0.5)
    ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
    res.check()
    states = [node["node_loc"]] + list(res.trajectory.detach()[:-1])
    graphs = _kept_graphs(states, r, node["data_batch"], 0.5, 1)
    assert [g.shape[1] for g in graphs] == res.n_edges.tolist()
    ref_in, ref_p, traj64 = _oracle_grads(sd, node, steps, 2, tau, 0, False, graphs, cot, cotX)
    assert _rel(res.trajectory, traj64) <= 1e-4
    _compare(m, leaf, ref_in, ref_p, 5e-4, "cutoff, radius mode")


def test_fixed_graph_cutoff_reselects_every_step():
    from tests.test_rollout_grad import _nbody_case
    m, node, ei, sd, kw = _nbody_case()
    m._backend = CutoffStandIn()
    g, _ = CSRGraph.from_edge_index(ei, node["node_loc"].shape[0])
    leaf = _leaves(node)
    cot, cotX = _cots(3, node["node_loc"].shape[0], 2, kw["virtual_channels"], seed=9)
    res = differentiable_rollout(m, **leaf, steps=3, graph=g, speed_col=1, cutoff_rate=0.3)
    ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
    res.check()
    eic = g.edge_index()
    states = [node["node_loc"]] + list(res.trajectory.detach()[:-1])
    graphs = []
    for x in states:
        length = (x.float()[eic[0]] - x.float()[eic[1]]).norm(dim=1).numpy()
        graphs.append(torch.from_numpy(co.cutoff_edge_index(eic.numpy(), x.numpy(), 0.3, node["data_batch"].numpy(), 2,
                                                            length)))
    assert res.n_edges.tolist() == [2 * co.k_of(132, 0.3)] * 3
    ref_in, ref_p, _ = _oracle_grads(sd, node, 3, 2, 1.0, 1, True, graphs, cot, cotX)
    _compare(m, leaf, ref_in, ref_p, 5e-4, "cutoff, fixed graph")


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def _valid(g, n=None):
    """The first n (default: n_edges_dev or all) edges of g as host arrays, after the CSR checks."""
    n = int(g.n_edges_dev) if n is None and g.n_edges_dev is not None else (g.num_edges if n is None else n)
    rp = g.rowptr.cpu().numpy().astype(np.int64)
    row, col = g.row[:n].cpu().numpy(), g.col[:n].cpu().numpy()
    assert rp[0] == 0 and rp[-1] == n and (np.diff(rp) >= 0).all()
    assert np.array_equal(row, np.repeat(np.arange(rp.shape[0] - 1), np.diff(rp)))
    return rp, row, col


def _check_against_oracle(cand, out, ea, pos, rate, batch=None, B=1, exact_lengths=False):
    """The device output against the oracle run on the device's own candidates with the kernel's fp32 lengths."""
    crp, crow, ccol = _valid(cand)
    rp, row, col = _valid(out)
    p = pos.cpu().numpy()
    ea32 = torch.empty(crow.shape[0], 1, dtype=torch.float32, device=pos.device)  # the kernel's own fp32 lengths
    CudaBackend().edge_lengths(torch.from_numpy(crow).to(pos.device), torch.from_numpy(ccol).to(pos.device), pos, None,
                               ea32)
    l32 = ea32[:, 0].cpu().numpy()
    lengths = co.lengths64(p, crow, ccol) if exact_lengths else l32
    orp, orow, ocol, _, mask = co.cutoff_csr(crp, crow, ccol, p, rate, None if batch is None else batch.cpu().numpy(), B,
                                             lengths=lengths)
    assert np.array_equal(rp, orp) and np.array_equal(row, orow) and np.array_equal(col, ocol)
    if ea is not None:
        e = ea[:row.shape[0]].cpu().numpy()
        assert (e == e[:, :1]).all()
        # the kernel's length of every kept edge is the fp32 length of the candidate it came from
        assert np.allclose(e[:, 0], l32[mask], rtol=2e-7, atol=0)
    return mask


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[7:-4] for p in GOLDEN])
def test_device_against_the_reference_fixtures(path):
    z = _golden(path)
    d = dev()
    pos, batch = torch.from_numpy(z["pos"]).to(d), torch.from_numpy(z["batch"]).to(d)
    cand_ref, kept, rate, radius = z["candidates"], z["kept"], float(z["rate"]), float(z["radius"])
    B = int(z["batch"].max()) + 1
    if radius > 0:
        g, _ = radius_graph_csr(pos, radius, batch, n_graphs=B, edge_attr_nf=0)
        gi = g.edge_index().cpu().numpy()
        assert set(map(tuple, gi.T.tolist())) == set(map(tuple, cand_ref.T.tolist())), "candidate sets differ"
        out, ea = radius_graph_csr(pos, radius, batch, n_graphs=B, cutoff_rate=rate)
        out2, ea2 = cutoff_edges_csr(g, pos, rate, batch, B)
        assert torch.equal(out.col, out2.col) and torch.equal(out.rowptr, out2.rowptr) and torch.equal(ea, ea2)
    else:
        g, _ = CSRGraph.from_edge_index(torch.from_numpy(cand_ref).to(d), pos.shape[0])
        out, ea = cutoff_edges_csr(g, pos, rate, batch, B)
    lattice = "lattice" in path
    _check_against_oracle(g, out, ea, pos, rate, batch, B, exact_lengths=lattice)
    got = out.edge_index().cpu().numpy()
    l32 = lambda ei: (torch.from_numpy(z["pos"])[ei[0]] - torch.from_numpy(z["pos"])[ei[1]]).norm(dim=1).numpy()
    for b, (ref_b, got_b) in enumerate(zip(_per_graph(kept, z["batch"], B), _per_graph(got, z["batch"], B))):
        assert ref_b.shape[1] == got_b.shape[1], f"graph {b}: kept count"
        lr, lg = np.sort(l32(ref_b)), np.sort(l32(got_b))
        if lattice:
            assert np.array_equal(lr.view(np.uint32), lg.view(np.uint32))
        else:
            assert np.allclose(lr, lg, rtol=1e-6, atol=0)
        thr = lr[-1] * (1 - 1e-6 * (not lattice))
        below = lambda ei: set(map(tuple, ei[:, l32(ei) < thr].T.tolist()))
        assert below(ref_b) == below(got_b), f"graph {b}: edges below the threshold differ"


@pytest.mark.gpu
def test_count_rule_over_2000_graphs():
    """Graph b has two nodes and b parallel edges (equal lengths): k_b must be Python's int(b * (1 - r))."""
    d = dev()
    Bn = 2000
    E_b = torch.arange(Bn)
    deg = torch.zeros(2 * Bn, dtype=torch.int64)
    deg[0::2] = E_b
    rowptr = torch.zeros(2 * Bn + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).to(torch.int32)
    col = torch.repeat_interleave(torch.arange(1, 2 * Bn, 2), E_b).to(torch.int32)
    g = CSRGraph(rowptr.to(d), col.to(d))
    pos = torch.randn(2 * Bn, 3, device=d)
    batch = torch.arange(Bn, device=d).repeat_interleave(2)
    for r in (0.1, 0.3, 0.7, 0.9, 1 / 3, 1.0):
        out, _ = cutoff_edges_csr(g, pos, r, batch, Bn)
        k = (out.rowptr[2::2] - out.rowptr[0:-1:2]).cpu().tolist()
        assert k == [int(e * (1 - r)) for e in range(Bn)], r


def _nbody_batch(B=3, n=100, seed=0):
    gen = torch.Generator().manual_seed(seed)
    pos = torch.randn(B * n, 3, generator=gen)
    i, j = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    keep = i != j
    ei = torch.cat([torch.stack([i[keep], j[keep]]) + n * b for b in range(B)], 1)
    return pos, torch.arange(B).repeat_interleave(n), ei


@pytest.mark.gpu
def test_shapes_against_the_oracle():
    d = dev()
    # k_b = 0 (rate 1) on a radius graph; k_b = E_b through the direct call at rate 0
    x = torch.rand(3000, 3, device=d)
    g, _ = radius_graph_csr(x, 0.08, edge_attr_nf=0)
    for rate in (1.0, 0.0, 0.5, 0.25):
        out, ea = cutoff_edges_csr(g, x, rate)
        _check_against_oracle(g, out, ea, x, rate)
    # graphs with no nodes (batch ids skipped) and with no edges, mixed with ordinary ones
    pos, batch, ei = _nbody_batch(B=3, n=30)
    iso = torch.randn(5, 3)                                     # graph 4: five nodes without edges
    pos = torch.cat([pos, iso])
    batch = torch.cat([torch.tensor([0] * 30 + [2] * 30 + [3] * 30), torch.full((5,), 4)])   # graph 1 and 5 empty
    g, _ = CSRGraph.from_edge_index(ei.to(d), pos.shape[0])
    pos, batch = pos.to(d), batch.to(d)
    for rate in (0.5, 0.3):
        out, ea = cutoff_edges_csr(g, pos, rate, batch, 6)
        _check_against_oracle(g, out, ea, pos, rate, batch, 6)
    # a 6,000-edge hub, and a graph whose lengths are all equal (parallel edges)
    hub_pos = torch.randn(6001, 3, device=d)
    hub = CSRGraph(torch.tensor([0] + [6000] * 6001, dtype=torch.int32, device=d),
                   torch.arange(1, 6001, dtype=torch.int32, device=d))
    out, ea = cutoff_edges_csr(hub, hub_pos, 0.5)
    _check_against_oracle(hub, out, ea, hub_pos, 0.5)
    same = CSRGraph(torch.tensor([0, 999, 999], dtype=torch.int32, device=d), torch.ones(999, dtype=torch.int32, device=d))
    p2 = torch.randn(2, 3, device=d)
    out, ea = cutoff_edges_csr(same, p2, 0.5)
    _check_against_oracle(same, out, ea, p2, 0.5)
    assert int(out.rowptr[-1]) == 499
    # two runs are bitwise equal
    a = cutoff_edges_csr(hub, hub_pos, 0.37)
    b = cutoff_edges_csr(hub, hub_pos, 0.37)
    assert torch.equal(a[0].rowptr, b[0].rowptr) and torch.equal(a[0].col, b[0].col) and torch.equal(a[1], b[1])


@pytest.mark.gpu
def test_capacity_tail_is_never_read_and_overflow_flags():
    d = dev()
    x = torch.rand(2000, 3, device=d)
    g, _ = radius_graph_csr(x, 0.1, edge_attr_nf=0)
    E = g.num_edges
    # the tail of a capacity-sized candidate graph points at an extra node at NaN: reading it would show up as NaN
    xn = torch.cat([x, torch.full((1, 3), float("nan"), device=d)])
    tail = torch.full((1000,), 2000, dtype=torch.int32, device=d)
    rowptr = torch.cat([g.rowptr, g.rowptr[-1:]])
    big = CSRGraph(rowptr, torch.cat([g.col, tail]), torch.cat([g.rows(), tail]))
    big.n_edges_dev = torch.tensor([E], dtype=torch.int32, device=d)
    out, ea = cutoff_edges_csr(big, xn, 0.5, capacity=E + 1000)
    n = int(out.n_edges_dev)
    ref, ref_ea = cutoff_edges_csr(g, x, 0.5)
    assert n == ref.num_edges and torch.equal(out.col[:n], ref.col) and torch.equal(ea[:n], ref_ea)
    assert not torch.isnan(ea[:n]).any() and torch.equal(out.rowptr[:-1], ref.rowptr)
    # an overflowed candidate build: flagged, the true count reported, nothing past the capacity read
    cg, _ = radius_graph_csr(x, 0.1, edge_attr_nf=0, capacity=E // 2)
    out, _ = cutoff_edges_csr(cg, x, 0.5, capacity=E // 2)
    info = out.info.tolist()
    assert info[1] == 1 and info[2] == E and info[0] <= E // 2
    with pytest.raises(ValueError, match="overflowed"):
        cutoff_edges_csr(cg, x, 0.5)


@pytest.mark.gpu
def test_rate_zero_is_the_default_path():
    d = dev()
    x = torch.rand(5000, 3, device=d)
    a = radius_graph_csr(x, 0.06)
    b = radius_graph_csr(x, 0.06, cutoff_rate=0.0)
    assert torch.equal(a[0].rowptr, b[0].rowptr) and torch.equal(a[0].col, b[0].col) and torch.equal(a[1], b[1])
    m, node, w, ref = _clear(steps=3, rate=0.0)
    be = m._get_backend(d)
    n0 = be.launches
    r0 = rollout(m, **node, steps=3, radius=w.radius, speed_col=0, capacity=ref.capacity, return_trajectory=True)
    n1 = be.launches
    r1 = rollout(m, **node, steps=3, radius=w.radius, speed_col=0, capacity=ref.capacity, return_trajectory=True,
                 cutoff_rate=0.0)
    assert be.launches - n1 == n1 - n0
    assert torch.equal(r0.n_edges, r1.n_edges)
    for t in range(3):
        assert float((r0.trajectory[t] - r1.trajectory[t]).abs().max()) <= RUN_TO_RUN * (t + 1)


# ---- rollouts against the float64 oracle ------------------------------------------------------------------------------
THR_MARGIN = 1e-5          # relative gap between the threshold length and any other pair's length across it


def _clear_of_threshold(x, rate, batch, B, r=None, ei=None):
    """No pair (other than the threshold edge's own mirror) within THR_MARGIN of a graph's threshold length; for
    radius candidates also no pair within MARGIN of r."""
    xd = x.double()
    if r is not None:
        dist = torch.cdist(xd, xd)
        if bool(((dist - r).abs() < MARGIN * r).any()):
            return False
        ei = _radius_edges(x.cpu(), r, batch.cpu()).to(x.device)
    length = (xd[ei[0]] - xd[ei[1]]).norm(dim=1)
    gb = batch[ei[0]]
    for b in range(B):
        lb = length[gb == b]
        k = co.k_of(int(lb.numel()), rate)
        if k == 0 or k == lb.numel():
            continue
        s, _ = torch.sort(lb)
        thr = s[k - 1]
        near = ((lb - thr).abs() <= THR_MARGIN * thr).sum()
        if int(near) > 2:                                      # the threshold pair itself and its mirror
            return False
    return True


def _gpu_model(kw, sd, normalize=False):
    m = FastEGNN(hidden_nf=64, world_size=1, normalize=normalize, **kw)
    m.load_state_dict(sd)
    return m.to(dev()).eval()


def _clear(steps, rate=0.5, r=0.05, sizes=None, n=300, layers=4):
    """The first seed of a fluid case whose rollout states are clear of r and of every threshold tie."""
    kw = dict(FLUID, n_layers=layers)
    sd = orc.init_state_dict(3, 2, 2, 64, 5, layers, seed=1, coord_gain=0.05)
    m = _gpu_model(kw, sd)
    for seed in range(60):
        inp = synth.make_partitions(synth.WORKLOADS["fluid113k"], n_nodes=n, seed=seed)[0]
        node = {k: (v.to(dev()) if v is not None else None) for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
        B = 1
        if sizes is not None:
            B = len(sizes)
            node["data_batch"] = torch.arange(B, device=dev()).repeat_interleave(torch.tensor(sizes, device=dev()))
            node["loc_mean"] = torch.stack([node["node_loc"][node["data_batch"] == b].mean(0) for b in range(B)])
        ref = rollout(m, **node, steps=steps, radius=r, speed_col=0, return_trajectory=True, cutoff_rate=rate)
        states = [node["node_loc"]] + list(ref.trajectory[:-1])
        if all(_clear_of_threshold(x, rate, node["data_batch"], B, r=r) for x in states):
            return m, node, SimpleNamespace(radius=r, sd=sd, B=B), ref
    pytest.fail("no seed clear of r and of the thresholds")


def _oracle_graph_kdtree(x, r, batch, rate, B):
    from scipy.spatial import cKDTree
    p = x.double().cpu().numpy()
    bt = batch.cpu().numpy()
    pairs = cKDTree(p).query_pairs(r, output_type="ndarray")
    pairs = pairs[bt[pairs[:, 0]] == bt[pairs[:, 1]]]
    ei = np.concatenate([pairs.T, pairs.T[::-1]], 1)
    ei = ei[:, np.lexsort((ei[1], ei[0]))]                    # destination-major, as a CSR
    return torch.from_numpy(co.cutoff_edge_index(ei, p, rate, bt, B)).to(x.device)


def _oracle_step(sd, normalize, feat, x, v, lm, ei, batch, attr, A):
    dd = lambda t: None if t is None else t.double()
    ea = (x.double()[ei[0]] - x.double()[ei[1]]).norm(dim=1, keepdim=True).expand(-1, A).contiguous()
    return orc.forward({k: v_.to(x.device).double() for k, v_ in sd.items()}, dd(feat), dd(x), dd(v), dd(lm), ei, batch,
                       ea, dd(attr), normalize=normalize)


def _gate(out, ref, pos, what):
    e_abs = float((out.double() - ref).abs().max())
    den = float((ref - pos.double()).abs().max())
    assert e_abs <= 1e-5 * max(1.0, float(ref.abs().max())), f"{what}: abs {e_abs:.3e}"
    assert e_abs / max(den, 1e-30) <= 1e-4, f"{what}: rel-disp {e_abs / den:.3e}"


def _walk(res, node, sd, normalize, graph_of, steps, B, speed_col=0):
    x, v, feat, lm, batch = (node[k] for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "data_batch"))
    for t in range(steps):
        ei = graph_of(x)
        assert int(res.n_edges[t]) == ei.shape[1], f"step {t}: kept count"
        ref, _ = _oracle_step(sd, normalize, feat, x, v, lm, ei, batch, node.get("node_attr"), 2)
        _gate(res.trajectory[t], ref, x, f"step {t}")
        xd = res.trajectory[t].double()
        v = xd - x.double()
        feat = feat.double().clone()
        feat[:, speed_col] = v.norm(dim=1)
        lm = torch.stack([xd[batch == b].mean(0) for b in range(B)])
        x = res.trajectory[t]


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", [None, [170, 60, 100]], ids=["B1", "B3_unequal"])
def test_rollout_with_cutoff_every_step_against_the_oracle(sizes):
    m, node, w, res = _clear(steps=4, sizes=sizes, n=300 if sizes is None else 330)
    graph_of = lambda x: _oracle_graph_kdtree(x, w.radius, node["data_batch"], 0.5, w.B)
    _walk(res, node, w.sd, False, graph_of, 4, w.B)
    g, ea = res.graph, res.edge_attr                           # the last step's kept graph, from the same buffers
    n = int(g.n_edges_dev)
    assert n == int(res.n_edges[-1]) and (ea[:n, 0] == ea[:n, 1]).all()


@pytest.mark.gpu
def test_rollout_with_cutoff_fixed_nbody_graph():
    kw = dict(node_feat_nf=2, node_attr_nf=0, edge_attr_nf=2, virtual_channels=3, n_layers=4)
    sd = orc.init_state_dict(2, 0, 2, 64, 3, 4, seed=1, coord_gain=0.05)
    m = _gpu_model(kw, sd, normalize=True)
    w = synth.WORKLOADS["nbody100"]
    for seed in range(40):
        parts = [synth.make_partitions(w, n_nodes=100, seed=seed * 8 + s)[0] for s in range(4)]
        cat = lambda k: torch.cat([p[k] for p in parts]).to(dev())
        node = dict(node_feat=cat("node_feat"), node_loc=cat("node_loc"), node_vel=cat("node_vel"),
                    loc_mean=torch.stack([p["node_loc"].mean(0) for p in parts]).to(dev()),
                    data_batch=torch.arange(4, device=dev()).repeat_interleave(100))
        ei = torch.cat([p["edge_index"] + 100 * b for b, p in enumerate(parts)], 1).to(dev())
        g, _ = CSRGraph.from_edge_index(ei, 400)
        res = rollout(m, **node, steps=4, graph=g, speed_col=1, return_trajectory=True, cutoff_rate=0.5)
        eic = g.edge_index()
        states = [node["node_loc"]] + list(res.trajectory[:-1])
        if all(_clear_of_threshold(x, 0.5, node["data_batch"], 4, ei=eic) for x in states):
            break
    else:
        pytest.fail("no seed clear of the thresholds")
    bt = node["data_batch"].cpu().numpy()
    graph_of = lambda x: torch.from_numpy(co.cutoff_edge_index(eic.cpu().numpy(), x.double().cpu().numpy(), 0.5, bt,
                                                               4)).to(dev())
    _walk(res, node, sd, True, graph_of, 4, 4, speed_col=1)
    assert res.n_edges.tolist() == [4 * co.k_of(9900, 0.5)] * 4


def _same_run(ref, other, what):
    assert torch.equal(other.n_edges, ref.n_edges), what
    for t in range(ref.trajectory.shape[0]):
        err = float((other.trajectory[t] - ref.trajectory[t]).abs().max())
        assert err <= RUN_TO_RUN * (t + 1), f"{what}, step {t}: {err:.3e}"


@pytest.mark.gpu
def test_no_host_sync_and_graphed_equals_eager():
    m, node, w, eager = _clear(steps=5)
    cap = eager.capacity
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = rollout(m, **node, steps=5, radius=w.radius, speed_col=0, capacity=cap, check_every=0,
                      return_trajectory=True, cutoff_rate=0.5)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    res.check()
    _same_run(eager, res, "no-sync rollout")
    m.cuda_graph = True
    be = m._get_backend(dev())
    n0 = be.launches
    graphed = rollout(m, **node, steps=5, radius=w.radius, speed_col=0, capacity=cap, return_trajectory=True,
                      cutoff_rate=0.5)
    per_step = (be.launches - n0) / 5
    m.cuda_graph = False
    n1 = be.launches
    rollout(m, **node, steps=5, radius=w.radius, speed_col=0, capacity=cap, cutoff_rate=0.5)
    assert graphed.replays == 4 and per_step == (be.launches - n1) / 5
    _same_run(eager, graphed, "graphed rollout")


@pytest.mark.gpu
def test_rollout_with_cutoff_is_se3_equivariant():
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(0), dtype=torch.float64))
    Rm = q.float().to(dev())
    s = torch.tensor([[0.3, -0.2, 0.5]], device=dev())
    m, node, w, a = _clear(steps=3)
    rot = dict(node, node_loc=node["node_loc"] @ Rm.T + s, node_vel=node["node_vel"] @ Rm.T,
               loc_mean=node["loc_mean"] @ Rm.T + s)
    b = rollout(m, **rot, steps=3, radius=w.radius, speed_col=0, return_trajectory=True, cutoff_rate=0.5)
    states = [rot["node_loc"]] + list(b.trajectory[:-1])
    assert all(_clear_of_threshold(x, 0.5, node["data_batch"], 1, r=w.radius) for x in states)
    assert torch.equal(a.n_edges, b.n_edges)
    assert float((b.trajectory - (a.trajectory @ Rm.T + s)).abs().max()) <= 1e-4


@pytest.mark.gpu
def test_differentiable_rollout_with_cutoff_against_oracle_autograd_gpu():
    m, node, w, _ = _clear(steps=4, layers=2)
    leaf = _leaves(node)
    cot, cotX = _cots(4, node["node_loc"].shape[0], 1, FLUID["virtual_channels"], device=dev())
    res = differentiable_rollout(m, **leaf, steps=4, radius=w.radius, speed_col=0, cutoff_rate=0.5)
    ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
    res.check()
    assert int(res.status[5]) == 0                             # every rebuilt kept graph matched the forward's
    states = [node["node_loc"]] + list(res.trajectory.detach()[:-1])
    graphs = [_oracle_graph_kdtree(x, w.radius, node["data_batch"], 0.5, 1) for x in states]
    assert [g.shape[1] for g in graphs] == res.n_edges.tolist()
    sd = {k: v.to(dev()) for k, v in w.sd.items()}
    ref_in, ref_p, _ = _oracle_grads(sd, node, 4, 2, 1.0, 0, False, graphs, cot, cotX)
    _compare(m, leaf, ref_in, ref_p, 5e-4, "cutoff, GPU, K=4")


@pytest.mark.gpu
def test_main_with_the_fastegnn_config():
    cfg = os.path.join(ROOT, "config", "nbody_fastegnn.yaml")
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--config_path", cfg, "--cutoff_rate", "0.5", "--eval_steps",
           "2", "--train_steps", "2", "--rollout_steps", "3", "--batch_size", "4"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0
    E = 4 * 100 * 99
    assert f"kept {int(E * 0.5)} of {E} candidate edges" in p.stdout
    assert "rollout 3 steps" in p.stdout and "train step 1" in p.stdout and "NOT used" not in p.stdout
