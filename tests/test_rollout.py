"""rollout(): multi-step inference that rebuilds the graph and advances the state on the device (DESIGN §14).

CPU: argument validation, the overflow / rollback policy and the exchange count under gloo with a torch stand-in for the
kernels, the new C-ABI symbols.  GPU: every step against the float64 oracle on the state the rollout produced, against
the hand-written loop of public calls, no host sync, graphed == eager, overflow recovery, fixed graphs, batches, SE(3)
equivariance, the caller's tensors left alone."""
import math
import os
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from distegnn_b200 import FastEGNN, _lib, rollout, synth
from distegnn_b200.shards import CSRGraph
from oracle import fastegnn_oracle as orc
from tests.shadow_backend import ShadowBackend

FLUID = dict(node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2, virtual_channels=5, n_layers=4)


# ---- torch stand-in for the rollout's device work (CPU tests only) ------------------------------------------------------
class RolloutStandIn(ShadowBackend):
    """ShadowBackend plus brute-force radius graph into capacity buffers, the advance step, edge lengths and the centroid.
    `inflate = {step: count}` reports `count` edges for that step's first build (a transient overflow)."""

    def __init__(self, inflate=None):
        super().__init__()
        self.inflate = dict(inflate or {})
        self.builds = []                       # (step, capacity) of every graph build
        self.counter = None

    def graph_buffers(self, n, cap, A, device):
        z = lambda *s, dt=torch.int32: torch.zeros(*s, dtype=dt, device=device)
        info = z(4)
        b = SimpleNamespace(n_nodes=n, capacity=cap, edge_attr_nf=A, rowptr=z(n + 1), row=z(cap), col=z(cap), info=info,
                            edge_attr=z(cap, A, dt=torch.float32) if A else None)
        b.graph = CSRGraph(b.rowptr, b.col, b.row)
        b.graph.n_edges_dev, b.graph.info = info[0:1], info
        return b

    def radius_graph_into(self, buf, pos, r, batch, n_graphs, loop):
        step = int(self.counter[0]) if self.counter is not None else 0
        n = pos.shape[0]
        b = batch if batch is not None else torch.zeros(n, dtype=torch.int64)
        ok = (torch.cdist(pos.double(), pos.double()) < r) & (b[:, None] == b[None, :])
        if not loop:
            ok &= ~torch.eye(n, dtype=torch.bool)
        i, j = ok.nonzero(as_tuple=True)                      # row-major: grouped by destination i
        true = int(i.numel())
        count = max(true, self.inflate.pop(step)) if step in self.inflate else true
        k = min(true, buf.capacity)
        buf.row.zero_(); buf.col.zero_()
        buf.row[:k], buf.col[:k] = i[:k].to(torch.int32), j[:k].to(torch.int32)
        buf.rowptr[1:] = torch.cumsum(torch.bincount(i, minlength=n), 0).to(torch.int32)
        if buf.edge_attr is not None:
            buf.edge_attr[:k] = (pos[i[:k]] - pos[j[:k]]).norm(dim=1, keepdim=True)
        buf.info[0], buf.info[1] = count, int(count > buf.capacity)
        self.builds.append((step, buf.capacity))

    def edge_layer(self, dims, flags, row, col, ea, x4, P, Q, lp, agg_m, agg_x, n_edges_dev=None):
        N, E, A, C, Na = dims
        if n_edges_dev is not None:
            E = min(int(n_edges_dev[0]), E)
            row, col, ea = row[:E], col[:E], (ea[:E] if ea is not None else None)
        super().edge_layer((N, E, A, C, Na), flags, row, col, ea, x4, P, Q, lp, agg_m, agg_x)

    def virtual_update(self, dims, flags, vsum, Xv, Hv, lp, lp_next, G, init_loc_mean=None, init_hv0=None, comm=None):
        if flags & _lib.FLAG_INIT_CENTROID:
            assert init_loc_mean is None
            init_loc_mean = vsum[:, :3] / vsum[:, 3:4].clamp(min=1)
            flags &= ~_lib.FLAG_INIT_CENTROID
        super().virtual_update(dims, flags, vsum, Xv, Hv, lp, lp_next, G, init_loc_mean, init_hv0, comm)

    def edge_lengths(self, row, col, pos, n_edges_dev, ea):
        ea[:] = (pos[row.long()] - pos[col.long()]).norm(dim=1, keepdim=True)

    def rollout_advance(self, speed_col, tau, pred, loc, vel, feat, traj, edge_count, overflow, n_edges, counter):
        self.counter = counter
        step = int(counter[0])
        vel.copy_((pred - loc) / tau)
        if feat is not None:
            feat[:, speed_col] = vel.norm(dim=1)
        loc.copy_(pred)
        if traj is not None:
            traj[step] = pred
        n_edges[step] = edge_count[0]
        if overflow is not None and int(overflow[0]) and int(counter[1]) == 0:
            counter[1], counter[2] = 1, step
        counter[3] = max(int(counter[3]), int(edge_count[0]))
        counter[0] += 1

    def rollout_centroid(self, pos, batch, sums):
        b = batch if batch is not None else torch.zeros(pos.shape[0], dtype=torch.int64)
        sums[:, :3].index_add_(0, b, pos.double())
        sums[:, 3].index_add_(0, b, torch.ones(pos.shape[0], dtype=torch.float64))


def _cpu_case(n=160, seed=0, world=1, rank=0):
    w = synth.WORKLOADS["fluid113k"]
    inp = synth.make_partitions(w, world_size=world, n_nodes=n, seed=seed)[rank]
    sd = orc.init_state_dict(3, 2, 2, 64, 5, 4, seed=1, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=world, **FLUID)
    m.load_state_dict(sd)
    node = {k: v for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
    return m, node, w.radius, sd


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_rollout_symbols_in_library():
    lib = _lib.load()
    for name in ("distegnn_rollout_advance", "distegnn_edge_lengths_csr", "distegnn_rollout_centroid"):
        assert hasattr(lib, name)
    assert lib.distegnn_abi_version() == 3 and _lib.FLAG_INIT_CENTROID == 32


def test_rollout_argument_validation():
    m, node, r, _ = _cpu_case(n=40)
    ok = dict(steps=2, radius=r)
    m._backend = RolloutStandIn()
    bad = [dict(steps=0, radius=r), dict(steps=2.0, radius=r), dict(steps=2, radius=r, tau=0.0), dict(steps=2),
           dict(steps=2, radius=r, graph=CSRGraph(torch.zeros(41, dtype=torch.int32), torch.zeros(0, dtype=torch.int32))),
           dict(steps=2, radius=-1.0), dict(steps=2, radius=r, speed_col=3), dict(steps=2, radius=r, speed_col=-1),
           dict(steps=2, radius=r, capacity=0), dict(steps=2, radius=r, check_every=-1), dict(steps=2, graph="edges"),
           dict(steps=True, radius=r), dict(steps=2, radius=r, speed_col=False), dict(steps=2, radius=r, check_every=True),
           dict(steps=2, radius=r, capacity=True)]
    for kw in bad:
        with pytest.raises(ValueError):
            rollout(m, **node, **kw)
    with pytest.raises(ValueError):
        rollout(m, **dict(node, node_vel=node["node_vel"][:-1]), **ok)
    with pytest.raises(ValueError):
        rollout(m, **dict(node, data_batch=node["data_batch"].int()), **ok)
    with pytest.raises(TypeError):
        rollout(torch.nn.Linear(2, 2), **node, **ok)
    m._backend = None                                          # the product backend: CPU tensors are refused
    with pytest.raises(_lib.DistEGNNError):
        rollout(m, **node, **ok)


def test_init_centroid_flag_is_inference_only():
    """The backward of the virtual update rejects FLAG_INIT_CENTROID (no gradient through x̄), and the forward accepts it
    only with FLAG_INIT and without init_loc_mean.  The argument checks return before anything is touched."""
    lib = _lib.load()
    p = 256                                                    # any non-null pointer: never dereferenced
    flags = _lib.FLAG_INIT | _lib.FLAG_INIT_CENTROID
    assert lib.distegnn_virtual_update_bwd(1, 2, 5, 2, flags, *([p] * 13), None) == -1
    assert "FLAG_INIT_CENTROID" in lib.distegnn_last_error().decode()
    assert lib.distegnn_virtual_update_fwd(1, 2, 5, 2, _lib.FLAG_INIT_CENTROID, p, p, p, p, p, p, None, None, None,
                                           None) == -1
    assert lib.distegnn_virtual_update_fwd(1, 2, 5, 2, flags, p, p, p, p, p, p, p, None, None, None) == -1
    assert "FLAG_INIT_CENTROID" in lib.distegnn_last_error().decode()


def test_overflow_reruns_exactly_the_chunk_with_a_larger_capacity():
    m, node, r, _ = _cpu_case()
    m._backend = be0 = RolloutStandIn()
    ref = rollout(m, **node, steps=10, radius=r, speed_col=0, check_every=5, return_trajectory=True)
    cap = ref.capacity                                         # 1.25 x step 0's count
    assert be0.builds[0] == (0, 0) and cap == math.ceil(1.25 * int(ref.n_edges[0]))
    assert [s for s, _ in be0.builds[1:]] == list(range(10)) and ref.regrowths == []
    forced = 4 * cap
    m._backend = be = RolloutStandIn(inflate={3: forced})
    res = rollout(m, **node, steps=10, radius=r, speed_col=0, check_every=5, capacity=cap, return_trajectory=True)
    grown = math.ceil(1.25 * forced)
    assert be.builds == [(s, cap) for s in range(5)] + [(s, grown) for s in range(10)]
    assert res.regrowths == [grown] and res.capacity == grown
    for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "virtual_loc", "trajectory", "n_edges"):
        assert torch.equal(getattr(res, k), getattr(ref, k)), k
    # the caller's tensors are untouched and the state follows the table of DESIGN §14
    assert torch.equal(res.node_loc, res.trajectory[-1])
    assert torch.allclose(res.node_vel, res.trajectory[-1] - res.trajectory[-2])
    assert torch.allclose(res.node_feat[:, 0], res.node_vel.norm(dim=1)) and torch.equal(res.node_feat[:, 1:],
                                                                                          node["node_feat"][:, 1:])
    assert torch.allclose(res.loc_mean, res.node_loc.mean(0, keepdim=True))


def test_overflow_after_the_regrowth_limit_raises_with_the_counts():
    m, node, r, _ = _cpu_case(n=60)

    class NeverEnough(RolloutStandIn):
        def radius_graph_into(self, buf, *a):
            super().radius_graph_into(buf, *a)
            buf.info[0], buf.info[1] = 2 * buf.capacity + 1, 1

    m._backend = be = NeverEnough()
    with pytest.raises(RuntimeError, match="still overflow"):
        rollout(m, **node, steps=3, radius=r, capacity=100, check_every=3)
    caps = sorted({c for _, c in be.builds})
    assert len(caps) == 5 and caps[0] == 100                  # the first capacity and four regrowths


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_rank(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        m, node, r, _ = _cpu_case(n=240, world=2, rank=rank)
        m._backend = RolloutStandIn()
        ref = rollout(m, **node, steps=4, radius=r, speed_col=0, check_every=4)
        cap = ref.capacity
        m._backend = be = RolloutStandIn(inflate={1: 3 * cap} if rank == 0 else None)
        calls = []
        orig = dist.all_reduce

        def counting(t, *a, **k):
            calls.append((tuple(t.shape), t.dtype))
            return orig(t, *a, **k)

        dist.all_reduce = counting
        res = rollout(m, **node, steps=4, radius=r, speed_col=0, check_every=4, capacity=cap)
        dist.all_reduce = orig
        same = all(torch.equal(getattr(res, k), getattr(ref, k)) for k in ("node_loc", "node_vel", "loc_mean",
                                                                          "virtual_loc"))
        q.put((rank, calls, be.builds, res.regrowths, cap, res.loc_mean.numpy(), res.virtual_loc.numpy(), same))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_ranks_roll_back_together_and_exchange_L_plus_1_per_step():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_rank, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in procs], key=lambda t: t[0])
    [p.join(timeout=60) for p in procs]
    L, C = FLUID["n_layers"], FLUID["virtual_channels"]
    K = 4 + 3 * C + 64 * C
    for rank, calls, builds, grown, cap, lm, X, same in res:
        assert same, f"rank {rank}: the rerun differs from the run without overflow"
        assert [s for s, _ in builds] == list(range(4)) * 2   # both ranks rerun the chunk
        assert grown == ([math.ceil(1.25 * 3 * cap)] if rank == 0 else [])
        stats = [c for c in calls if c == ((1, K), torch.float32)]
        assert len(stats) == (L + 1) * 8                      # L+1 per executed step (4 steps, twice)
        assert calls.count(((1, 4), torch.float64)) == 1      # the final loc_mean (fp64 sums)
        assert calls.count(((1,), torch.int32)) == 2          # the per-chunk overflow OR (overflow, then clean)
        assert len(calls) == len(stats) + 3
    assert (res[0][5] == res[1][5]).all() and (res[0][6] == res[1][6]).all()


# ---- GPU ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_gpu_rollout_under_torchrun():
    """2 ranks (2 GPUs) under torchrun, random partitions, 3 steps, graphed, rank 0 with too small a capacity (it alone
    regrows; both roll back and recapture): every step against oracle.forward_partitions on the gathered state, loc_mean
    and virtual_loc bit-identical on both ranks (scripts/rollout_dist_check.py).  Skipped with a single GPU."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29547", os.path.join(root, "scripts", "rollout_dist_check.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    print(p.stdout[-3000:], p.stderr[-1500:])
    assert p.returncode == 0 and "ROLLOUT_DIST PASS" in p.stdout


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def _gpu_case(w_name="fluid113k", n=20_000, seed=3, kw=FLUID, coord_gain=0.05):
    w = synth.WORKLOADS[w_name]
    inp = synth.make_partitions(w, n_nodes=n, seed=seed)[0]
    F, Na, A, C, L = kw["node_feat_nf"], kw["node_attr_nf"], kw["edge_attr_nf"], kw["virtual_channels"], kw["n_layers"]
    sd = orc.init_state_dict(F, Na, A, 64, C, L, seed=1, coord_gain=coord_gain)
    m = FastEGNN(hidden_nf=64, world_size=1, normalize=w.normalize, **kw)
    m.load_state_dict(sd)
    m = m.to(dev()).eval()
    node = {k: (v.to(dev()) if v is not None else None) for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
    return m, node, w, sd


def _oracle_step(sd, normalize, feat, x, v, lm, g, batch, attr, A):
    """float64 oracle on the GPU for one step on graph `g` (CSR, first n valid edges)."""
    d = lambda t: None if t is None else t.double()
    ei = g.edge_index()
    ea = (x[ei[0]] - x[ei[1]]).norm(dim=1, keepdim=True).expand(-1, A).contiguous()
    return orc.forward({k: v_.to(x.device).double() for k, v_ in sd.items()}, d(feat), d(x), d(v), d(lm), ei, batch,
                       d(ea), d(attr), normalize=normalize)


def _exact_graph(x, r, batch=None, B=1, loop=False):
    from distegnn_b200.partition import radius_graph_csr
    return radius_graph_csr(x.float().contiguous(), r, batch if B > 1 else None, loop=loop, n_graphs=B)[0]


def _check_vs_kdtree(g, x, r):
    from scipy.spatial import cKDTree
    pos = x.double().cpu().numpy()
    want, near = set(), set()
    for i, j in cKDTree(pos).query_pairs(r * (1 + 1e-6), output_type="ndarray"):
        dd = float(np.linalg.norm(pos[i] - pos[j]))
        (near if abs(dd - r) <= 2e-7 * max(r, 1.0) else want).update({(int(i), int(j)), (int(j), int(i))})
    ei = g.edge_index().cpu().numpy()
    got = set(zip(ei[0].tolist(), ei[1].tolist()))
    assert len(got) == ei.shape[1] and want - near <= got <= want | near


def _gate(out, ref, pos, what):
    e_abs = float((out.double() - ref).abs().max())
    den = float((ref - pos.double()).abs().max())
    assert e_abs <= 1e-5 * max(1.0, float(ref.abs().max())), f"{what}: abs {e_abs:.3e}"
    assert e_abs / max(den, 1e-30) <= 1e-4, f"{what}: rel-disp {e_abs / den:.3e}"


def _own_graph(res):
    """The valid part of a rollout's own (capacity-sized) graph and edge_attr."""
    g, n = res.graph, int(res.graph.n_edges_dev)
    return CSRGraph(g.rowptr, g.col[:n], g.row[:n]), res.edge_attr[:n]


@pytest.mark.gpu
def test_rollout_every_step_against_the_oracle_and_the_table():
    """Every step of a 5-step rollout against the float64 oracle run on the state the rollout produced.  The graph of step
    t is the rollout's own: a one-step rollout from x_t (same kernel, same positions, same buffers' contents as step t of
    the long one) hands it back, and it is compared with cKDTree's and with n_edges[t]."""
    m, node, w, sd = _gpu_case()
    before = {k: v.clone() for k, v in node.items() if v is not None}
    res = rollout(m, **node, steps=5, radius=w.radius, speed_col=0, tau=0.5, return_trajectory=True)
    for k, v in before.items():
        assert torch.equal(node[k], v), f"caller's {k} was modified"
    traj = res.trajectory
    x, v, feat, lm = node["node_loc"], node["node_vel"], node["node_feat"], node["loc_mean"]
    n_edges = res.n_edges.tolist()
    for t in range(5):
        one = rollout(m, feat, x, v, lm, node["data_batch"], node["node_attr"], steps=1, radius=w.radius,
                      capacity=res.capacity)
        g, ea = _own_graph(one)
        _check_vs_kdtree(g, x, w.radius)
        assert n_edges[t] == g.num_edges
        ei = g.edge_index()
        assert float((ea[:, 0] - (x[ei[0]] - x[ei[1]]).norm(dim=1)).abs().max()) <= 1e-6 and torch.equal(ea[:, 0], ea[:, 1])
        ref, refX = _oracle_step(sd, w.normalize, feat, x, v, lm, g, node["data_batch"], node["node_attr"], 2)
        _gate(traj[t], ref, x, f"step {t}")
        xd = traj[t].double()
        v = (xd - x.double()) / 0.5                            # float64 restatement of the table
        feat = feat.double().clone()
        feat[:, 0] = v.norm(dim=1)
        lm = xd.mean(0, keepdim=True)
        x = traj[t]
    assert float((res.virtual_loc.double() - refX).abs().max()) <= 1e-5 * max(1.0, float(refX.abs().max()))
    assert float((res.node_vel.double() - v).abs().max()) <= 1e-5 * max(1.0, float(v.abs().max()))
    assert float((res.node_feat.double() - feat).abs().max()) <= 1e-5 * max(1.0, float(feat.abs().max()))
    assert float((res.loc_mean.double() - lm).abs().max()) <= 1e-6
    assert torch.equal(res.node_loc, traj[-1])


# ---- comparisons of independent runs ------------------------------------------------------------------------------------
# Two runs of the same rollout differ by the run-to-run rounding of the forward's fp32 atomics: at most 2e-6 per forward
# (DESIGN §7).  A pair whose distance is within that of r can enter one run's graph and not the other's, which moves its
# nodes by far more than 2e-6.  So these tests use a case whose states (every position a graph is built from) have no pair
# within MARGIN of r, in every run compared — asserted, not assumed — and then require identical edge counts.  With the
# same graphs every step adds at most the one-forward bound, and a step's map is close to the identity (displacements are
# ~1e-3 of the positions), so after step t the runs differ by at most 2e-6 * (t + 1).
MARGIN = 1e-4                      # relative to r
RUN_TO_RUN = 2e-6


def _states(x0, traj):
    return [x0] + list(traj[:-1])


def _clear_of_r(states, r):
    for x in states:
        d = torch.cdist(x.double(), x.double())
        if bool(((d - r).abs() < MARGIN * r).any()):
            return False
    return True


def _clear_case(steps, r=0.05):
    """The first seed of a 300-node fluid case whose rollout with radius `r` stays clear of r.  A 20k-node case has ~150k
    pairs within r, so some pair lands next to r at almost every step; here ~0.2 per state are expected."""
    for seed in range(60):
        m, node, _, _ = _gpu_case(n=300, seed=seed)
        ref = rollout(m, **node, steps=steps, radius=r, speed_col=0, return_trajectory=True)
        if _clear_of_r(_states(node["node_loc"], ref.trajectory), r):
            return m, node, SimpleNamespace(radius=r), ref
    pytest.fail("no seed without pairs near r")


def _same_run(ref, other, x0, r, what):
    assert _clear_of_r(_states(x0, other.trajectory), r), f"{what}: a pair came within {MARGIN} r of r"
    assert torch.equal(other.n_edges, ref.n_edges), what
    for t in range(ref.trajectory.shape[0]):
        err = float((other.trajectory[t] - ref.trajectory[t]).abs().max())
        assert err <= RUN_TO_RUN * (t + 1), f"{what}, step {t}: {err:.3e}"


@pytest.mark.gpu
def test_rollout_matches_the_hand_written_loop():
    from distegnn_b200 import radius_graph_csr
    m, node, w, res = _clear_case(steps=5)
    x, v, feat, lm = node["node_loc"].clone(), node["node_vel"].clone(), node["node_feat"].clone(), node["loc_mean"]
    traj, n_edges = [], []
    with torch.no_grad():
        for t in range(5):
            g, ea = radius_graph_csr(x, w.radius)
            out, X = m(feat, x, v, lm, g, node["data_batch"], ea, node["node_attr"])
            v = out - x
            feat[:, 0] = v.norm(dim=1)
            lm = out.mean(0, keepdim=True)
            x = out
            traj.append(out)
            n_edges.append(g.num_edges)
    hand = SimpleNamespace(trajectory=torch.stack(traj), n_edges=torch.tensor(n_edges, dtype=torch.int32, device=dev()))
    _same_run(res, hand, node["node_loc"], w.radius, "hand-written loop")
    assert float((res.loc_mean - lm).abs().max()) <= RUN_TO_RUN * 5


@pytest.mark.gpu
def test_rollout_enqueues_without_host_sync_and_graphed_equals_eager():
    m, node, w, eager = _clear_case(steps=6)                  # its first rollout also validated data_batch
    cap = eager.capacity
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = rollout(m, **node, steps=6, radius=w.radius, speed_col=0, capacity=cap, check_every=0,
                      return_trajectory=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    res.check()
    _same_run(eager, res, node["node_loc"], w.radius, "no-sync rollout")
    m.cuda_graph = True
    be = m._get_backend(dev())
    n0 = be.launches
    graphed = rollout(m, **node, steps=6, radius=w.radius, speed_col=0, capacity=cap, return_trajectory=True)
    per_step = (be.launches - n0) / 6
    m.cuda_graph = False
    n1 = be.launches
    rollout(m, **node, steps=6, radius=w.radius, speed_col=0, capacity=cap)
    assert graphed.replays == 5 and per_step == (be.launches - n1) / 6   # step 0 eager, one replay per later step
    _same_run(eager, graphed, node["node_loc"], w.radius, "graphed rollout")


@pytest.mark.gpu
def test_rollout_overflow_regrows_and_gives_the_same_trajectory():
    m, node, w, ref = _clear_case(steps=4)
    e0 = int(ref.n_edges[0])
    small = rollout(m, **node, steps=4, radius=w.radius, speed_col=0, capacity=e0 // 2, check_every=2,
                    return_trajectory=True)
    assert small.regrowths and small.capacity > e0 // 2
    _same_run(ref, small, node["node_loc"], w.radius, "regrown rollout")
    with pytest.raises(RuntimeError, match="capacity"):
        rollout(m, **node, steps=2, radius=w.radius, capacity=e0 // 2, check_every=0).check()


@pytest.mark.gpu
def test_rollout_fixed_fully_connected_graph_nbody():
    kw = dict(node_feat_nf=2, node_attr_nf=0, edge_attr_nf=2, virtual_channels=3, n_layers=4)
    w = synth.WORKLOADS["nbody100"]
    parts = [synth.make_partitions(w, n_nodes=100, seed=s)[0] for s in range(8)]
    B = len(parts)
    cat = lambda k: torch.cat([p[k] for p in parts])
    node = dict(node_feat=cat("node_feat"), node_loc=cat("node_loc"), node_vel=cat("node_vel"),
                loc_mean=torch.cat([p["node_loc"].mean(0, keepdim=True) for p in parts]),
                data_batch=torch.arange(B).repeat_interleave(100))
    ei = torch.cat([p["edge_index"] + 100 * b for b, p in enumerate(parts)], 1)
    g, _ = CSRGraph.from_edge_index(ei, 100 * B)
    sd = orc.init_state_dict(2, 0, 2, 64, 3, 4, seed=1, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, normalize=True, **kw)
    m.load_state_dict(sd)
    m = m.to(dev()).eval()
    node = {k: v.to(dev()) for k, v in node.items()}
    g = CSRGraph(g.rowptr.to(dev()), g.col.to(dev()), g.row.to(dev()))
    res = rollout(m, **node, steps=4, graph=g, speed_col=1, return_trajectory=True)
    x, v, feat, lm = node["node_loc"], node["node_vel"], node["node_feat"], node["loc_mean"]
    for t in range(4):
        ref, _ = _oracle_step(sd, True, feat, x, v, lm, g, node["data_batch"], None, 2)
        _gate(res.trajectory[t], ref, x, f"step {t}")
        xd = res.trajectory[t].double()
        v = xd - x.double()
        feat = feat.double().clone()
        feat[:, 1] = v.norm(dim=1)
        lm = torch.stack([xd[node["data_batch"] == b].mean(0) for b in range(B)])
        x = res.trajectory[t]
    assert res.n_edges.tolist() == [g.num_edges] * 4
    assert float((res.loc_mean.double() - lm).abs().max()) <= 1e-6


@pytest.mark.gpu
def test_rollout_batched_graphs_of_unequal_sizes():
    from scipy.spatial import cKDTree  # noqa: F401  (the kd-tree check runs per graph below)
    m, node0, w, sd = _gpu_case(n=3000, seed=5)
    sizes = [1700, 300, 1000]
    batch = torch.arange(3, device=dev()).repeat_interleave(torch.tensor(sizes, device=dev()))
    node = dict(node0, data_batch=batch,
                loc_mean=torch.stack([node0["node_loc"][batch == b].mean(0) for b in range(3)]))
    res = rollout(m, **node, steps=3, radius=w.radius, speed_col=0, return_trajectory=True)
    x, v, feat, lm = node["node_loc"], node["node_vel"], node["node_feat"], node["loc_mean"]
    for t in range(3):
        g = _exact_graph(x, w.radius, batch, 3)
        ref, refX = _oracle_step(sd, w.normalize, feat, x, v, lm, g, batch, node["node_attr"], 2)
        _gate(res.trajectory[t], ref, x, f"step {t}")
        xd = res.trajectory[t].double()
        v = xd - x.double()
        feat = feat.double().clone()
        feat[:, 0] = v.norm(dim=1)
        lm = torch.stack([xd[batch == b].mean(0) for b in range(3)])
        x = res.trajectory[t]
    assert float((res.loc_mean.double() - lm).abs().max()) <= 1e-6
    assert float((res.virtual_loc.double() - refX).abs().max()) <= 1e-5 * max(1.0, float(refX.abs().max()))


@pytest.mark.gpu
def test_rollout_is_se3_equivariant():
    """A rotation + translation of (x0, v0) commutes with a 3-step rollout.  The radius graph is only equivariant away from
    pairs at distance ~r (their membership can flip under rounding), so the case is the first seed whose trajectories
    have none within 1e-4 r of r — asserted for both."""
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(0), dtype=torch.float64))
    Rm = q.float().to(dev())
    s = torch.tensor([[0.3, -0.2, 0.5]], device=dev())

    for seed in range(40):
        m, node, w, _ = _gpu_case(n=300, seed=seed)
        a = rollout(m, **node, steps=3, radius=w.radius, speed_col=0, return_trajectory=True)
        if _clear_of_r(_states(node["node_loc"], a.trajectory), w.radius):
            break
    else:
        pytest.fail("no seed without near-r pairs")
    rot = dict(node, node_loc=node["node_loc"] @ Rm.T + s, node_vel=node["node_vel"] @ Rm.T,
               loc_mean=node["loc_mean"] @ Rm.T + s)
    b = rollout(m, **rot, steps=3, radius=w.radius, speed_col=0, return_trajectory=True)
    assert _clear_of_r(_states(rot["node_loc"], b.trajectory), w.radius)
    want = a.trajectory @ Rm.T + s
    assert float((b.trajectory - want).abs().max()) <= 1e-4
    assert torch.equal(a.n_edges, b.n_edges)
