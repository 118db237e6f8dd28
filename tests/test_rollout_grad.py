"""differentiable_rollout(): back-propagation through multi-step rollouts, each step recomputed in the backward (DESIGN §15).

CPU: argument validation, the new C-ABI symbols and their argument checks, the host orchestration with the kernels
replaced by torch stand-ins against float64 autograd of the oracle through the same steps (fixed graph and radius mode),
and two ranks under gloo (state gradients per rank, summed parameter gradients, exchanges per backward step).
GPU: the two new kernels against float64 autograd, the whole feature against the oracle and against the hand-written
loop, rebuilt graphs equal to the forward's, no host sync, and memory that grows with K by O(K·N) only."""
import os
import socket
from types import SimpleNamespace

import pytest
import torch
import torch.multiprocessing as mp

from distegnn_b200 import FastEGNN, _lib, differentiable_rollout, rollout, synth
from distegnn_b200.shards import CSRGraph
from oracle import fastegnn_oracle as orc
from tests.test_input_grads import InputGradShadowBackend
from tests.test_rollout import FLUID, RolloutStandIn, _same_run

STATE = ["node_feat", "node_loc", "node_vel", "loc_mean", "node_attr"]


# ---- torch stand-ins of the two new kernels (CPU tests only) ---------------------------------------------------------
class RolloutGradStandIn(RolloutStandIn, InputGradShadowBackend):
    """RolloutStandIn + InputGradShadowBackend, plus the edge-length backward and the advance backward in torch, and the
    input-gradient edge backward limited to the valid edges of a capacity-sized graph."""

    def edge_layer_bwd(self, dims, flags, row, col, ea, x4, P, Q, lp, g_agg_m, g_agg_x, g_P, g_Q, g_x4, g_lp,
                       n_edges_dev=None, g_ea=None):
        N, E, A, C, Na = dims
        if n_edges_dev is not None:
            E = min(int(n_edges_dev[0]), E)
            row, col, ea = row[:E], col[:E], (ea[:E] if ea is not None else None)
            g_ea = g_ea[:E] if g_ea is not None else None
        InputGradShadowBackend.edge_layer_bwd(self, (N, E, A, C, Na), flags, row, col, ea, x4, P, Q, lp, g_agg_m, g_agg_x,
                                              g_P, g_Q, g_x4, g_lp, None, g_ea)

    def edge_lengths_bwd(self, row, col, pos, n_edges_dev, g_ea, g_pos):
        E = g_ea.shape[0] if n_edges_dev is None else min(int(n_edges_dev[0]), g_ea.shape[0])
        r, c = row[:E].long(), col[:E].long()
        d = pos[r] - pos[c]
        n = d.norm(dim=1, keepdim=True)
        contrib = torch.where(n > 0, g_ea[:E].sum(1, keepdim=True) * d / n.clamp(min=1e-30), torch.zeros_like(d))
        g_pos.index_add_(0, r, contrib)
        g_pos.index_add_(0, c, -contrib)

    def rollout_advance_bwd(self, speed_col, tau, x_next, x, g_traj, g_x_next, g_v_next, g_feat_next, g_pred, g_x):
        v = (x_next - x) * (1.0 / tau)
        gv = torch.zeros_like(v) if g_v_next is None else g_v_next.clone()
        if g_feat_next is not None:
            s = v.norm(dim=1, keepdim=True)
            gv += torch.where(s > 0, g_feat_next[:, speed_col:speed_col + 1] * v / s.clamp(min=1e-30), torch.zeros_like(v))
            g_feat_next[:, speed_col] = 0
        a = gv / tau
        g_pred.copy_(a + (0 if g_traj is None else g_traj) + (0 if g_x_next is None else g_x_next))
        g_x.copy_(-a)


def _radius_edges(x, r, batch):
    """The stand-in's radius graph of x (row-major pairs, grouped by destination): the same edges the rollout used."""
    ok = (torch.cdist(x.double(), x.double()) < r) & (batch[:, None] == batch[None, :])
    ok &= ~torch.eye(x.shape[0], dtype=torch.bool, device=x.device)
    i, j = ok.nonzero(as_tuple=True)
    return torch.stack([i, j])


def _group_mean(x, batch, B):
    return torch.stack([x[batch == b].mean(0) for b in range(B)])


def oracle_rollout(sd64, node, steps, A, tau, speed_col, normalize, graphs):
    """float64 autograd through `steps` steps of the table of DESIGN §14, the oracle as the model.  graphs[t] is step t's
    edge_index (the rollout's own: topology is piecewise constant); edge_attr = the lengths, differentiable."""
    x, v, feat, lm, attr, batch = (node[k] for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "node_attr",
                                                     "data_batch"))
    B = lm.shape[0]
    traj, Xs = [], []
    for t in range(steps):
        ei = graphs[t]
        ea = (x[ei[0]] - x[ei[1]]).norm(dim=1, keepdim=True).expand(-1, A)
        out, X = orc.forward(sd64, feat, x, v, lm, ei, batch, ea, attr, normalize=normalize)
        v = (out - x) / tau
        if speed_col is not None:
            feat = torch.cat([feat[:, :speed_col], v.norm(dim=1, keepdim=True), feat[:, speed_col + 1:]], 1)
        lm = _group_mean(out, batch, B)
        x = out
        traj.append(out)
        Xs.append(X)
    return torch.stack(traj), torch.stack(Xs)


def _rel(a, b, floor=1e-30):
    """max |a − b| / max |b|.  `floor`: lower bound of the denominator (see _param_errs)."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / max(float(b.abs().max()), floor))


FLOOR = 1e-3     # of the largest parameter gradient


def _param_errs(got, ref):
    """Relative error of each parameter gradient, the denominator floored at FLOOR × the largest reference parameter
    gradient.  A few gradients (the φ_X bias of a layer) cancel to ~1e-6 of the others; fp32 accumulation noise is set by
    the size of the summed terms, not of their sum, so their plain relative error only measures that noise (2.5e-4 to
    4.9e-4 over five H100 runs of the same case)."""
    big = max(float(r.abs().max()) for r in ref.values() if r is not None)
    return {k: _rel(got[k], r, FLOOR * big) for k, r in ref.items() if r is not None and float(r.abs().max()) > 0}


def _leaves(node, dtype=None):
    return {k: (v.to(dtype or v.dtype).clone().requires_grad_(True) if (v is not None and v.is_floating_point()) else v)
            for k, v in node.items()}


def _cots(steps, N, B, C, seed=7, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(steps, N, 3, generator=g).to(device), torch.randn(steps, B, 3, C, generator=g).to(device)


def _compare(m, leaf, ref_in, ref_p, tol, what):
    errs = {}
    for k in STATE:
        if leaf.get(k) is None:
            continue
        assert leaf[k].grad is not None and leaf[k].grad.dtype == leaf[k].dtype, k
        errs[k] = _rel(leaf[k].grad, ref_in[k])
    errs.update(_param_errs({k: p.grad for k, p in m.named_parameters()}, ref_p))
    worst = max(errs, key=errs.get)
    print(f"{what}: " + ", ".join(f"{k} {errs[k]:.1e}" for k in STATE if k in errs) + f"; worst {worst} {errs[worst]:.1e}")
    assert errs[worst] <= tol, (worst, errs[worst])
    return errs


def _oracle_grads(sd, node, steps, A, tau, speed_col, normalize, graphs, cot, cotX):
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    leaf64 = _leaves(node, torch.float64)
    traj, Xs = oracle_rollout(sd64, leaf64, steps, A, tau, speed_col, normalize, graphs)
    loss = (traj * cot.double()).sum() + (Xs * cotX.double()).sum()
    keys = list(sd64)
    ins = [k for k in STATE if leaf64.get(k) is not None]
    gr = torch.autograd.grad(loss, [leaf64[k] for k in ins] + [sd64[k] for k in keys], allow_unused=True)
    return dict(zip(ins, gr[:len(ins)])), dict(zip(keys, gr[len(ins):])), traj


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def _cpu_case(n=160, seed=0, world=1, rank=0):
    w = synth.WORKLOADS["fluid113k"]
    inp = synth.make_partitions(w, world_size=world, n_nodes=n, seed=seed)[rank]
    sd = orc.init_state_dict(3, 2, 2, 64, 5, 2, seed=1, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=world, **dict(FLUID, n_layers=2))
    m.load_state_dict(sd)
    node = {k: v for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
    return m, node, w.radius, sd


def test_new_symbols_and_their_argument_checks():
    lib = _lib.load()
    assert lib.distegnn_abi_version() == 3
    p = 256                                                    # any non-null pointer: never dereferenced
    bwd = lib.distegnn_edge_lengths_bwd
    assert bwd(-1, 2, p, p, p, None, p, p, None) == -1         # bad size
    assert bwd(10, _lib.MAX_EDGE_ATTR + 1, p, p, p, None, p, p, None) == -1
    assert bwd(10, 2, p, None, p, None, p, p, None) == -1      # null pointers
    assert bwd(10, 2, p, p, p, None, p, None, None) == -1
    assert "null pointer" in lib.distegnn_last_error().decode()
    assert bwd(0, 2, None, None, None, None, None, None, None) == 0      # nothing to do
    adv = lib.distegnn_rollout_advance_bwd
    assert adv(-1, 3, 0, 1.0, p, p, p, p, p, p, p, p, None) == -1
    assert adv(10, 3, 0, 0.0, p, p, p, p, p, p, p, p, None) == -1      # tau <= 0
    assert "tau" in lib.distegnn_last_error().decode()
    assert adv(10, 3, 0, -1.0, p, p, p, p, p, p, p, p, None) == -1
    assert adv(10, 3, 3, 1.0, p, p, p, p, p, p, p, p, None) == -1      # speed_col outside [0, F)
    assert adv(10, 3, 0, 1.0, None, p, p, p, p, p, p, p, None) == -1   # null pointers
    assert adv(10, 3, 0, 1.0, p, p, p, p, p, p, p, None, None) == -1
    assert adv(0, 3, 0, 1.0, None, None, None, None, None, None, None, None, None) == 0


def test_differentiable_rollout_argument_validation_and_input_grads_flag():
    m, node, r, _ = _cpu_case(n=40)
    m._backend = RolloutGradStandIn()
    bad = [dict(steps=0, radius=r), dict(steps=2.0, radius=r), dict(steps=2, radius=r, tau=0.0), dict(steps=2),
           dict(steps=2, radius=-1.0), dict(steps=2, radius=r, speed_col=3), dict(steps=2, radius=r, capacity=0),
           dict(steps=2, radius=r, check_every=-1), dict(steps=2, graph="edges"), dict(steps=True, radius=r)]
    for kw in bad:
        for fn in (rollout, differentiable_rollout):           # the same errors as rollout()
            with pytest.raises(ValueError):
                fn(m, **node, **kw)
    with pytest.raises(ValueError):
        differentiable_rollout(m, **dict(node, node_vel=node["node_vel"][:-1]), steps=2, radius=r)
    with pytest.raises(TypeError):
        differentiable_rollout(torch.nn.Linear(2, 2), **node, steps=2, radius=r)
    for flag in (False, True):                                 # model.input_grads is neither needed nor changed
        m.input_grads = flag
        leaf = _leaves(node)
        res = differentiable_rollout(m, **leaf, steps=2, radius=r, speed_col=0)
        (res.trajectory.sum() + res.virtual_locs.sum()).backward()
        assert m.input_grads is flag
        assert all(leaf[k].grad is not None for k in STATE)
        assert res.trajectory.shape == (2, 40, 3) and res.virtual_locs.shape == (2, 1, 3, 5)
        for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "virtual_loc", "n_edges"):
            assert not getattr(res, k).requires_grad, k
        res.check()
    m._backend = None                                          # the product backend: CPU tensors are refused
    with pytest.raises(_lib.DistEGNNError):
        differentiable_rollout(m, **node, steps=2, radius=r)


def test_rollout_result_is_unchanged_by_the_new_field():
    m, node, r, _ = _cpu_case(n=60)
    m._backend = RolloutStandIn()
    res = rollout(m, **node, steps=2, radius=r, speed_col=0, return_trajectory=True)
    assert res.virtual_locs is None
    m._backend = RolloutGradStandIn()
    dres = differentiable_rollout(m, **node, steps=2, radius=r, speed_col=0)
    for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "virtual_loc", "trajectory", "n_edges"):
        assert torch.allclose(getattr(dres, k).detach(), getattr(res, k), rtol=0, atol=1e-6), k
    assert torch.allclose(dres.virtual_locs[-1].detach(), res.virtual_loc, rtol=0, atol=1e-6)


def test_radius_mode_gradients_against_oracle_autograd():
    """3 steps, radius graph rebuilt every step, speed column, tau != 1: every parameter and all five inputs."""
    m, node, r, sd = _cpu_case(n=160, seed=2)
    m._backend = RolloutGradStandIn()
    leaf = _leaves(node)
    steps, tau, C = 3, 0.5, FLUID["virtual_channels"]
    cot, cotX = _cots(steps, 160, 1, C)
    res = differentiable_rollout(m, **leaf, steps=steps, radius=r, speed_col=0, tau=tau)
    ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
    res.check()
    states = [node["node_loc"]] + list(res.trajectory.detach()[:-1])
    graphs = [_radius_edges(x, r, node["data_batch"]) for x in states]
    assert [g.shape[1] for g in graphs] == res.n_edges.tolist()
    ref_in, ref_p, traj64 = _oracle_grads(sd, node, steps, 2, tau, 0, False, graphs, cot, cotX)
    assert _rel(res.trajectory, traj64) <= 1e-4
    _compare(m, leaf, ref_in, ref_p, 5e-4, "radius mode")


def _nbody_case(B=2, n=12, seed=0):
    kw = dict(node_feat_nf=2, node_attr_nf=1, edge_attr_nf=2, virtual_channels=3, n_layers=2)
    g = torch.Generator().manual_seed(seed)
    N = B * n
    node = dict(node_feat=torch.randn(N, 2, generator=g), node_loc=torch.randn(N, 3, generator=g),
                node_vel=0.1 * torch.randn(N, 3, generator=g), data_batch=torch.arange(B).repeat_interleave(n),
                node_attr=torch.randn(N, 1, generator=g))
    node["loc_mean"] = _group_mean(node["node_loc"], node["data_batch"], B)
    i, j = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    keep = i != j
    ei = torch.cat([torch.stack([i[keep], j[keep]]) + n * b for b in range(B)], 1)
    sd = orc.init_state_dict(2, 1, 2, 64, 3, 2, seed=3, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, normalize=True, **kw)
    m.load_state_dict(sd)
    return m, node, ei, sd, kw


def test_fixed_graph_gradients_against_oracle_autograd():
    """3 steps on a kept fully connected graph (two graphs of a batch: per-graph centroids), normalize=True."""
    m, node, ei, sd, kw = _nbody_case()
    m._backend = RolloutGradStandIn()
    g, _ = CSRGraph.from_edge_index(ei, node["node_loc"].shape[0])
    leaf = _leaves(node)
    steps, C = 3, kw["virtual_channels"]
    cot, cotX = _cots(steps, node["node_loc"].shape[0], 2, C, seed=9)
    res = differentiable_rollout(m, **leaf, steps=steps, graph=g, speed_col=1)
    ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
    eic = g.edge_index()
    ref_in, ref_p, _ = _oracle_grads(sd, node, steps, 2, 1.0, 1, True, [eic] * steps, cot, cotX)
    _compare(m, leaf, ref_in, ref_p, 5e-4, "fixed graph")


# ---- two ranks under gloo ---------------------------------------------------------------------------------------------
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
        m._backend = RolloutGradStandIn()
        leaf = _leaves(node)
        N = node["node_loc"].shape[0]
        cot, cotX = _cots(2, N, 1, FLUID["virtual_channels"], seed=11 + rank)
        calls = []
        orig = dist.all_reduce

        def counting(t, *a, **k):
            calls.append((tuple(t.shape), t.dtype))
            return orig(t, *a, **k)

        dist.all_reduce = counting
        res = differentiable_rollout(m, **leaf, steps=2, radius=r, speed_col=0, tau=0.5)
        n_fwd = len(calls)
        ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
        dist.all_reduce = orig
        bwd = calls[n_fwd:]
        q.put((rank, {k: leaf[k].grad.numpy() for k in STATE}, {k: p.grad.numpy() for k, p in m.named_parameters()},
               res.trajectory.detach().numpy(), bwd))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_ranks_gradients_against_the_partitioned_oracle():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_rank, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=600) for _ in procs], key=lambda t: t[0])
    [p.join(timeout=60) for p in procs]
    _, node0, r, sd = _cpu_case(n=240, world=2, rank=0)
    parts = [node0, _cpu_case(n=240, world=2, rank=1)[1]]
    L, C, tau = 2, FLUID["virtual_channels"], 0.5
    K = 4 + 3 * C + 64 * C
    # the oracle over both partitions: float64 autograd through 2 steps, each rank's graphs rebuilt from its trajectory
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    leaves64 = [_leaves(p, torch.float64) for p in parts]
    xs = [lf["node_loc"] for lf in leaves64]
    vs = [lf["node_vel"] for lf in leaves64]
    fs = [lf["node_feat"] for lf in leaves64]
    lm = leaves64[0]["loc_mean"]
    loss = 0
    for t in range(2):
        pin = []
        for k, lf in enumerate(leaves64):
            state = torch.from_numpy(res[k][3][t - 1]) if t else parts[k]["node_loc"]
            ei = _radius_edges(state, r, lf["data_batch"])
            pin.append(dict(node_feat=fs[k], node_loc=xs[k], node_vel=vs[k], edge_index=ei, data_batch=lf["data_batch"],
                            edge_attr=(xs[k][ei[0]] - xs[k][ei[1]]).norm(dim=1, keepdim=True).expand(-1, 2),
                            node_attr=lf["node_attr"]))
        outs, X = orc.forward_partitions(sd64, pin, lm if t == 0 else lm_t)
        for k in range(2):
            cot, cotX = _cots(2, parts[k]["node_loc"].shape[0], 1, C, seed=11 + k)
            loss = loss + (outs[k] * cot[t].double()).sum() + (X * cotX[t].double()).sum()
            vs[k] = (outs[k] - xs[k]) / tau
            fs[k] = torch.cat([vs[k].norm(dim=1, keepdim=True), fs[k][:, 1:]], 1)
        lm_t = torch.cat(outs).mean(0, keepdim=True)
        xs = outs
    loss.backward()
    # loc_mean is replicated: each rank's copy gets what its own chain carries, and the copies sum to the oracle's
    e = _rel(torch.from_numpy(res[0][1]["loc_mean"] + res[1][1]["loc_mean"]), leaves64[0]["loc_mean"].grad)
    assert e <= 5e-4, ("loc_mean", e)
    for k, (rank, g_in, g_p, traj, bwd) in enumerate(res):
        for name in ("node_feat", "node_loc", "node_vel", "node_attr"):
            e = _rel(torch.from_numpy(g_in[name]), leaves64[k][name].grad)
            assert e <= 5e-4, (rank, name, e)
        # per backward step: the recompute's L+1 exchanges, then L for the statistics' gradient and 1 for g_vsum0
        stats = [c for c in bwd if c == ((1, K), torch.float32)]
        assert len(stats) == 2 * (2 * (L + 1)) and len(bwd) == len(stats), bwd
    for name, p in sd64.items():
        if p.grad is None or float(p.grad.abs().max()) == 0:
            continue
        tot = torch.from_numpy(res[0][2][name]) + torch.from_numpy(res[1][2][name])
        assert _rel(tot, p.grad) <= 5e-4, name


# ======================================================================================================================
# GPU
# ======================================================================================================================
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def _row_gate(got, ref, what, tol=2e-5):
    """Per row: |got − ref| <= tol · that row's largest |ref|; rows whose reference is exactly zero must be exactly zero."""
    got, ref = got.double(), ref.double()
    scale = ref.abs().amax(1, keepdim=True)
    zero = scale[:, 0] == 0
    assert float(got[zero].abs().max()) == 0.0 if bool(zero.any()) else True, f"{what}: nonzero structurally-zero row"
    bad = (got - ref).abs() > tol * scale
    assert not bool(bad[~zero].any()), f"{what}: {int(bad.any(1).sum())} rows off, worst " \
        f"{float(((got - ref).abs() / scale.clamp(min=1e-300))[~zero].max()):.2e}"


def _edge_case(N, E, A, hub=0, loops=0, coincident=0, seed=0):
    g = torch.Generator().manual_seed(seed)
    pos = torch.rand(N, 3, generator=g)
    row = torch.randint(0, N, (E,), generator=g)
    col = torch.randint(0, N, (E,), generator=g)
    if hub:
        row[:hub] = 5
    if loops:
        col[hub:hub + loops] = row[hub:hub + loops]
    if coincident:                                             # distinct nodes at the same place
        a, b = row[hub + loops:hub + loops + coincident], col[hub + loops:hub + loops + coincident]
        keep = a != b
        pos[b[keep]] = pos[a[keep]]
    row, order = torch.sort(row, stable=True)
    col = col[order]
    return pos, row, col


@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 2, 8])
@pytest.mark.parametrize("case", ["ragged", "empty", "capacity", "hub", "loops"])
def test_edge_lengths_bwd_against_float64_autograd(A, case):
    from distegnn_b200.backend import cuda_backend
    be = cuda_backend()
    N, E, nE = 3000, {"ragged": 20_011, "empty": 0, "capacity": 20_000, "hub": 12_000, "loops": 9_001}[case], None
    pos, row, col = _edge_case(N, E, A, hub=6000 if case == "hub" else 0, loops=500 if case == "loops" else 0,
                               coincident=300 if case == "loops" else 0, seed=A)
    g = torch.Generator().manual_seed(100 + A)
    g_ea = torch.randn(E, A, generator=g)
    if case == "capacity":                                     # only the first 13,337 edges are valid
        nE = 13_337
        g_ea[nE:] = float("nan")
    valid = E if nE is None else nE
    # float64 autograd of (x[row] − x[col]).norm() repeated A times (torch's norm backward: 0 at zero length)
    x64 = pos.double().requires_grad_(True)
    r, c = row[:valid], col[:valid]
    d = (x64[r] - x64[c]).norm(dim=1, keepdim=True).expand(-1, A)
    (ref,) = torch.autograd.grad((d * g_ea[:valid].double()).sum(), x64) if valid else (torch.zeros(N, 3,
                                                                                                    dtype=torch.float64),)
    dv = lambda t: t.to(dev()).contiguous()
    gp = torch.zeros(N, 3, device=dev())
    n_dev = torch.tensor([nE], dtype=torch.int32, device=dev()) if nE is not None else None
    be.edge_lengths_bwd(dv(row.int()), dv(col.int()), dv(pos), n_dev, dv(g_ea), gp)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(gp).all())
    _row_gate(gp.cpu(), ref, f"A={A} {case}")
    if case == "loops":                                        # nodes touched only by zero-length edges get exactly 0
        zero_len = (pos[row] - pos[col]).norm(dim=1) == 0
        only = torch.zeros(N, dtype=torch.bool)
        only[row[zero_len]] = True
        only[col[zero_len]] = True
        touched = torch.zeros(N, dtype=torch.bool)
        touched[row[~zero_len]] = True
        touched[col[~zero_len]] = True
        iso = only & ~touched
        assert bool(iso.any()) and float(gp.cpu()[iso].abs().max()) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("tau", [1.0, 0.5, 3.0])
@pytest.mark.parametrize("speed_col", [None, 1])
def test_rollout_advance_bwd_against_float64_autograd(tau, speed_col):
    from distegnn_b200.backend import cuda_backend
    be = cuda_backend()
    N, F = 5000, 3
    g = torch.Generator().manual_seed(int(tau * 10) + (speed_col or 0))
    x = torch.rand(N, 3, generator=g)
    x_next = x + 0.01 * torch.randn(N, 3, generator=g)
    x_next[:300] = x[:300]                                     # v = 0 rows
    g_traj, g_xn, g_vn = (torch.randn(N, 3, generator=g) for _ in range(3))
    g_fn = torch.randn(N, F, generator=g)
    # float64 autograd of the advance table: v = (x' − x)/tau, speed = ‖v‖ (norm backward 0 at v = 0)
    xn64, x64 = x_next.double().requires_grad_(True), x.double().requires_grad_(True)
    v = (xn64 - x64) / tau
    loss = (xn64 * (g_traj + g_xn).double()).sum() + (v * g_vn.double()).sum()
    if speed_col is not None:
        loss = loss + (v.norm(dim=1) * g_fn[:, speed_col].double()).sum()
    ref_pred, ref_x = torch.autograd.grad(loss, (xn64, x64))
    dv = lambda t: t.to(dev()).contiguous()
    g_pred, g_x = torch.empty(N, 3, device=dev()), torch.empty(N, 3, device=dev())
    gf = dv(g_fn) if speed_col is not None else None
    be.rollout_advance_bwd(speed_col, tau, dv(x_next), dv(x), dv(g_traj), dv(g_xn), dv(g_vn), gf, g_pred, g_x)
    torch.cuda.synchronize()
    # g_x here is the advance's own part, −g_v/tau: the g_x' pass-through belongs to g_pred only
    _row_gate(g_pred.cpu(), ref_pred, "g_pred")
    _row_gate(g_x.cpu(), ref_x, "g_x")
    if speed_col is not None:
        want = g_fn.clone()
        want[:, speed_col] = 0
        assert torch.equal(gf.cpu(), want)                     # the speed column is consumed, the others untouched


def _gpu_model(kw, sd, normalize=False):
    m = FastEGNN(hidden_nf=64, world_size=1, normalize=normalize, **kw)
    m.load_state_dict(sd)
    return m.to(dev()).train()


def _clear_fluid(steps, B=1, sizes=None, r=0.05, kw=None, sd_seed=1):
    """The first seed of a ~300-node fluid case whose rollout states have no pair within 1e-4·r of r (the oracle's graphs
    then equal the rollout's)."""
    from tests.test_rollout import _clear_of_r, _states  # noqa: F401
    kw = kw or dict(FLUID, n_layers=2)
    sd = orc.init_state_dict(kw["node_feat_nf"], kw["node_attr_nf"], kw["edge_attr_nf"], 64, kw["virtual_channels"],
                             kw["n_layers"], seed=sd_seed, coord_gain=0.05)
    n = sum(sizes) if sizes else 300
    for seed in range(60):
        inp = synth.make_partitions(synth.WORKLOADS["fluid113k"], n_nodes=n, seed=seed)[0]
        node = {k: v.to(dev()) for k, v in inp.items() if k not in ("edge_index", "edge_attr") and v is not None}
        if sizes:
            batch = torch.arange(B, device=dev()).repeat_interleave(torch.tensor(sizes, device=dev()))
            node.update(data_batch=batch, loc_mean=_group_mean(node["node_loc"], batch, B))
        m = _gpu_model(kw, sd)
        with torch.no_grad():
            ref = rollout(m, **node, steps=steps, radius=r, speed_col=0, tau=0.5, return_trajectory=True)
        if _clear_of_r(_states(node["node_loc"], ref.trajectory), r):
            return m, node, sd, ref, r
    pytest.fail("no seed without pairs near r")


def _radius_graphs(states, r, batch, B):
    from distegnn_b200.partition import radius_graph_csr
    out = []
    for x in states:
        g = radius_graph_csr(x.float().contiguous(), r, batch if B > 1 else None, n_graphs=B)[0]
        out.append(g.edge_index())
    return out


def _run_against_oracle(m, node, sd, steps, graphs_of, normalize, A, what, **kw):
    B, C = node["loc_mean"].shape[0], m.virtual_channels
    N = node["node_loc"].shape[0]
    cot, cotX = _cots(steps, N, B, C, seed=21, device=dev())
    leaf = _leaves(node)
    res = differentiable_rollout(m, **leaf, steps=steps, **kw)
    ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
    res.check()
    states = [node["node_loc"]] + list(res.trajectory.detach()[:-1])
    graphs = graphs_of(states)
    ref_in, ref_p, _ = _oracle_grads({k: v.to(dev()) for k, v in sd.items()}, node, steps, A, kw.get("tau", 1.0),
                                     kw.get("speed_col"), normalize, graphs, cot, cotX)
    return _compare(m, leaf, ref_in, ref_p, 5e-4, what), res


@pytest.mark.gpu
def test_gradients_against_oracle_radius_mode():
    m, node, sd, ref, r = _clear_fluid(4)
    _, res = _run_against_oracle(m, node, sd, 4, lambda s: _radius_graphs(s, r, node["data_batch"], 1), False, 2,
                                 "radius B=1", radius=r, speed_col=0, tau=0.5)
    # the forward is rollout()'s step: the same graphs, and positions within the forward's run-to-run rounding (its fp32
    # atomics make two runs of rollout() itself differ by that much, so bit equality between runs is not defined)
    _same_run(ref, SimpleNamespace(trajectory=res.trajectory.detach(), n_edges=res.n_edges), node["node_loc"], r,
              "differentiable_rollout vs rollout")


@pytest.mark.gpu
def test_gradients_against_oracle_unequal_batch():
    m, node, sd, ref, r = _clear_fluid(4, B=3, sizes=[170, 60, 110])
    _run_against_oracle(m, node, sd, 4, lambda s: _radius_graphs(s, r, node["data_batch"], 3), False, 2, "radius B=3",
                        radius=r, speed_col=0, tau=0.5)


@pytest.mark.gpu
def test_gradients_against_oracle_fixed_nbody_normalized():
    m, node, ei, sd, kw = _nbody_case(B=4, n=25, seed=1)
    m = m.to(dev()).train()
    node = {k: v.to(dev()) for k, v in node.items()}
    g, _ = CSRGraph.from_edge_index(ei.to(dev()), node["node_loc"].shape[0])
    eic = g.edge_index()
    _run_against_oracle(m, node, sd, 4, lambda s: [eic] * 4, True, 2, "fixed N-body", graph=g, speed_col=1)


@pytest.mark.gpu
def test_gradients_match_the_hand_written_loop():
    """K = 3: the loop of public calls with model.input_grads, radius_graph_csr per step, edge_attr recomputed in torch
    from the CSR, the advance in torch."""
    from distegnn_b200 import radius_graph_csr
    m, node, sd, ref, r = _clear_fluid(3)
    B, C, N = 1, m.virtual_channels, node["node_loc"].shape[0]
    cot, cotX = _cots(3, N, B, C, seed=5, device=dev())
    leaf = _leaves(node)
    res = differentiable_rollout(m, **leaf, steps=3, radius=r, speed_col=0, tau=0.5)
    ((res.trajectory * cot).sum() + (res.virtual_locs * cotX).sum()).backward()
    res.check()
    mine = {k: leaf[k].grad.clone() for k in STATE}
    mine_p = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    m.input_grads = True
    hand = _leaves(node)
    x, v, feat, lm = hand["node_loc"], hand["node_vel"], hand["node_feat"], hand["loc_mean"]
    loss = 0
    for t in range(3):
        g, _ = radius_graph_csr(x.detach(), r)
        ei = g.edge_index()
        ea = (x[ei[0]] - x[ei[1]]).norm(dim=1, keepdim=True).expand(-1, 2).contiguous()
        out, X = m(feat, x, v, lm, g, hand["data_batch"], ea, hand["node_attr"])
        loss = loss + (out * cot[t]).sum() + (X * cotX[t]).sum()
        v = (out - x) / 0.5
        feat = torch.cat([v.norm(dim=1, keepdim=True), feat[:, 1:]], 1)
        lm = out.mean(0, keepdim=True)
        x = out
    loss.backward()
    m.input_grads = False
    errs = {k: _rel(mine[k], hand[k].grad) for k in STATE}
    errs.update(_param_errs(mine_p, {k: p.grad for k, p in m.named_parameters()}))
    worst = max(errs, key=errs.get)
    print("vs hand-written loop:", {k: f"{errs[k]:.1e}" for k in STATE}, "worst", worst, f"{errs[worst]:.1e}")
    assert errs[worst] <= 1e-4


@pytest.mark.gpu
def test_no_host_sync_in_forward_and_backward():
    m, node, sd, ref, r = _clear_fluid(3)
    leaf = _leaves(node)
    differentiable_rollout(m, **_leaves(node), steps=3, radius=r, speed_col=0, tau=0.5)   # validates data_batch once
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = differentiable_rollout(m, **leaf, steps=3, radius=r, speed_col=0, tau=0.5, capacity=ref.capacity,
                                     check_every=0)
        (res.trajectory.square().sum() + res.virtual_locs.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    res.check()
    assert all(leaf[k].grad is not None for k in STATE)


@pytest.mark.gpu
def test_memory_grows_by_O_K_N_only():
    """~50k nodes: max_memory_allocated over forward + backward for K = 2 and K = 8 differ by less than a quarter of one
    training step's peak (measured here); the hand-written loop's growth is printed for contrast."""
    from distegnn_b200 import radius_graph_csr
    w = synth.WORKLOADS["fluid113k"]
    inp = synth.make_partitions(w, n_nodes=50_000, seed=0)[0]
    node = {k: v.to(dev()) for k, v in inp.items() if v is not None}
    ei, ea = node.pop("edge_index"), node.pop("edge_attr")
    kw = dict(FLUID)
    sd = orc.init_state_dict(3, 2, 2, 64, 5, 4, seed=1, coord_gain=0.05)
    m = _gpu_model(kw, sd)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    def one_step():
        g, e = radius_graph_csr(node["node_loc"], w.radius)
        out, X = m(node["node_feat"], node["node_loc"], node["node_vel"], node["loc_mean"], g, node["data_batch"], e,
                   node["node_attr"])
        (out.sum() + X.sum()).backward()

    def diff(K):
        def run():
            leaf = _leaves(node)
            res = differentiable_rollout(m, **leaf, steps=K, radius=w.radius, speed_col=0)
            (res.trajectory.sum() + res.virtual_locs.sum()).backward()
        return run

    def hand(K):
        def run():
            m.input_grads = True
            leaf = _leaves(node)
            x, v, f, lm = leaf["node_loc"], leaf["node_vel"], leaf["node_feat"], leaf["loc_mean"]
            loss = 0
            for _ in range(K):
                g, _ = radius_graph_csr(x.detach(), w.radius)
                e = g.edge_index()
                a = (x[e[0]] - x[e[1]]).norm(dim=1, keepdim=True).expand(-1, 2).contiguous()
                out, X = m(f, x, v, lm, g, leaf["data_batch"], a, leaf["node_attr"])
                loss = loss + out.sum() + X.sum()
                v = out - x
                f = torch.cat([v.norm(dim=1, keepdim=True), f[:, 1:]], 1)
                lm = out.mean(0, keepdim=True)
                x = out
            loss.backward()
            m.input_grads = False
        return run

    step = peak(one_step)
    peak(diff(2))                                              # first call: the model's persistent workspace
    p2, p8 = peak(diff(2)), peak(diff(8))
    h2, h8 = peak(hand(2)), peak(hand(8))
    mb = lambda b: f"{b / 2**20:.1f} MB"
    print(f"one training step {mb(step)}; differentiable_rollout K=2 {mb(p2)}, K=8 {mb(p8)} (+{mb(p8 - p2)}); "
          f"hand-written loop K=2 {mb(h2)}, K=8 {mb(h8)} (+{mb(h8 - h2)})")
    assert p8 - p2 < step / 4
