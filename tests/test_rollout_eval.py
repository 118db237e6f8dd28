"""Rollouts against recorded trajectories (DESIGN §19): FrameLoader(horizon=K)'s multi-step targets and the per-step,
per-graph squared error that rollout(targets=...) computes inside each step.

CPU: horizon validation, the staged frames per recipe against a float64 restatement (oracle/targets_oracle.py), the
argument checks of rollout(targets=), and two gloo ranks with a torch stand-in for the kernels.  GPU: the targets
gather against the oracle, the error kernel against float64, what targets change and what they do not, bitwise
reproducibility, no host synchronisation, the training loss, a differentiable rollout's loss, and main.py."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from distegnn_b200 import FastEGNN, _lib, rollout
from distegnn_b200.frames import FrameLoader, check_samples, load_nbody, load_scenes, sample_list
from oracle import targets_oracle as to
from tests.test_rollout import FLUID, RolloutStandIn, _cpu_case, _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- trajectories (seeded random walks in the loader's input layout) ------------------------------------------------
def _walk(rng, T, n, step=0.01):
    steps = rng.normal(0.0, step, (T, n, 3))
    steps[0] = rng.random((n, 3))
    return np.cumsum(steps, 0).astype(np.float32)


def _water(d, sizes, T=10, seed=0, step=0.01):
    rng = np.random.default_rng(seed)
    paths = []
    for k, n in enumerate(sizes):
        p = str(d / f"water_{k}.npz")
        np.savez(p, position=_walk(rng, T, n, step), particle_type=rng.integers(1, 9, n))
        paths.append(p)
    return paths


def _fluid(d, sizes, T=10, seed=1, step=0.01):
    rng = np.random.default_rng(seed)
    paths = []
    for k, n in enumerate(sizes):
        p = str(d / f"fluid_{k}.npz")
        np.savez(p, position=_walk(rng, T, n, step), velocity=rng.normal(0, 1, (T, n, 3)).astype(np.float32),
                 viscosity=rng.random(n).astype(np.float32), mass=rng.random(n).astype(np.float32))
        paths.append(p)
    return paths


def _nbody(d, part="train", S=4, T=10, n=5, seed=2, step=0.1):
    rng = np.random.default_rng(seed)
    d.mkdir(exist_ok=True)
    np.save(d / f"loc_{part}_charged100_0_0_1.npy", np.stack([_walk(rng, T, n, step) for _ in range(S)]))
    np.save(d / f"vel_{part}_charged100_0_0_1.npy", rng.normal(0, 1, (S, T, n, 3)).astype(np.float32))
    np.save(d / f"charges_{part}_charged100_0_0_1.npy", rng.choice([-1.0, 1.0], (S, n, 1)).astype(np.float32))
    return str(d)


def _traj(tmp_path, recipe, sizes=(40, 30, 50, 35)):
    if recipe == "nbody":
        return load_nbody(_nbody(tmp_path / "nbody"))
    paths = _water(tmp_path, sizes) if recipe == "water3d" else _fluid(tmp_path, sizes)
    return load_scenes(paths, recipe)


def _position(traj, s):
    return torch.from_numpy(np.array(traj.scenes[s].position))


# ---- CPU: horizon validation and staging -----------------------------------------------------------------------------
def test_horizon_validation(tmp_path):
    traj = _traj(tmp_path, "water3d")                         # 10 frames per scene
    check_samples(traj, [(0, 3)], delta_t=2, horizon=3)       # frames 5, 7, 9
    with pytest.raises(ValueError, match=r"sample \(0, 4\).*horizon=3 needs frame 10"):
        check_samples(traj, [(0, 3), (0, 4)], delta_t=2, horizon=3)
    with pytest.raises(ValueError, match=r"sample \(1, 4\)"):
        FrameLoader(traj, [(0, 0), (1, 4)], delta_t=2, horizon=3)
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match="horizon"):
            check_samples(traj, [(0, 0)], delta_t=1, horizon=bad)
        with pytest.raises(ValueError, match="horizon"):
            FrameLoader(traj, [(0, 0)], delta_t=1, horizon=bad)
    # sample_list follows the horizon through check_samples: a frame draw that cannot hold it raises
    sample_list(traj, seed=0, max_samples=4, delta_t=1, frames_per_scene=1, max_frame=5)
    FrameLoader(traj, sample_list(traj, seed=0, max_samples=4, delta_t=1, frames_per_scene=1, max_frame=5),
                horizon=4)


def test_nbody_horizon_limit_of_the_reference_files(tmp_path):
    """The reference's N-body files hold 50 frames, frame_0 = 30 and Δ = 10: a horizon of 1 only."""
    traj = load_nbody(_nbody(tmp_path / "nb", S=2, T=50, n=3))
    samples = sample_list(traj, frame_0=30, delta_t=10)
    FrameLoader(traj, samples, delta_t=10, horizon=1)
    with pytest.raises(ValueError, match=r"frame 50.*only 1 step\(s\) of 10 frames fit after frame 30 \(at most "
                                         r"horizon 1\)"):
        FrameLoader(traj, samples, delta_t=10, horizon=2)


@pytest.mark.parametrize("recipe", ["nbody", "water3d", "largefluid"])
@pytest.mark.parametrize("K", [1, 3])
def test_staged_frames_per_recipe_are_the_float64_targets(tmp_path, recipe, K):
    """2 + K frames per sample cross PCIe: pos[f], the velocity frame, then pos[f + tΔ], t = 1..K (the oracle's)."""
    traj = _traj(tmp_path, recipe)
    dt = 2
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=dt, frames_per_scene=2, max_frame=9 - 1 - K * dt,
                          frame_0=1)
    ld = FrameLoader(traj, samples, delta_t=dt, batch_size=2, horizon=K)
    host = ld._host_batch([0, 1])
    fr = host["frames"]
    assert fr.shape == (2 + K, host["n_frame"], 3) and fr.dtype == torch.float32
    off = 0
    for i in (0, 1):
        s, f = samples[i]
        pos = _position(traj, s)
        n = pos.shape[1]
        want = to.targets(recipe, pos, f, dt, K)
        assert torch.equal(fr[2:, off:off + n].double(), want)
        assert torch.equal(fr[0, off:off + n], pos[f])
        off += n
    # K = 1 stages exactly the three frames of a loader without a horizon
    if K == 1:
        assert torch.equal(fr, FrameLoader(traj, samples, delta_t=dt, batch_size=2)._host_batch([0, 1])["frames"])


def test_abi_symbols_are_exported():
    lib = _lib.load()
    assert lib.distegnn_abi_version() == 3
    for name in ("distegnn_frames_targets", "distegnn_rollout_sq_err", "distegnn_rollout_sq_err_workspace_bytes"):
        assert hasattr(lib, name)
    p = 256                                                    # never dereferenced: the checks return first
    assert lib.distegnn_frames_targets(1, 4, 4, 0, p, p, p, None, p, None) == -1
    assert lib.distegnn_rollout_sq_err(4, 2, 1, p, p, None, p, p, p, 1 << 20, None) == -1
    assert b"data_batch" in lib.distegnn_last_error()
    assert lib.distegnn_rollout_sq_err(5000, 1, 1, p, p, None, p, p, p, 8, None) != 0   # workspace too small


# ---- CPU: rollout(targets=) ------------------------------------------------------------------------------------------
class ErrStandIn(RolloutStandIn):
    """RolloutStandIn plus the per-step error in torch (row counter[0], plain stores)."""

    def rollout_sq_err_workspace(self, n, device):
        return torch.zeros(16, dtype=torch.uint8, device=device)

    def rollout_sq_err(self, pred, targets, batch, counter, sq_err, ws):
        t = int(counter[0])
        if 0 <= t < sq_err.shape[0]:
            sq_err[t] = to.sq_err(pred, targets[t], batch, sq_err.shape[1])
        self.launches += 1


def test_rollout_targets_argument_checks():
    m, node, r, _ = _cpu_case(n=40)
    m._backend = be = ErrStandIn()
    N = node["node_loc"].shape[0]
    good = torch.zeros(3, N, 3)
    for bad in (good.double(), good[:2], good[:, :-1], good[..., :2], good.numpy(), torch.zeros(3, N, 3, device="meta")):
        with pytest.raises(ValueError, match="targets"):
            rollout(m, **node, steps=3, radius=r, targets=bad)
    assert be.launches == 0 and be.builds == []               # rejected before anything was enqueued
    res = rollout(m, **node, steps=3, radius=r, speed_col=0, targets=good, return_trajectory=True)
    assert res.sq_err.shape == (3, 1) and res.sq_err.dtype == torch.float64
    assert res.graph_nodes.tolist() == [N] and res.graph_nodes.dtype == torch.int64
    want = torch.stack([to.sq_err(res.trajectory[t], good[t], None, 1) for t in range(3)])
    assert torch.equal(res.sq_err, want)
    assert torch.allclose(res.mse, want[:, 0] / (3 * N), rtol=1e-15, atol=0)
    plain = rollout(m, **node, steps=3, radius=r, speed_col=0)
    assert plain.sq_err is None and plain.graph_nodes is None and plain.mse is None


def _gloo_rank(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        m, node, r, _ = _cpu_case(n=240, world=2, rank=rank)
        N = node["node_loc"].shape[0]
        tg = node["node_loc"] + torch.randn(4, N, 3, generator=torch.Generator().manual_seed(rank)) * 0.01
        m._backend = ErrStandIn()
        ref = rollout(m, **node, steps=4, radius=r, speed_col=0, check_every=4)
        m._backend = ErrStandIn()
        calls = []
        orig = dist.all_reduce

        def counting(t, *a, **k):
            calls.append((tuple(t.shape), t.dtype))
            return orig(t, *a, **k)

        dist.all_reduce = counting
        res = rollout(m, **node, steps=4, radius=r, speed_col=0, check_every=4, capacity=ref.capacity, targets=tg,
                      return_trajectory=True)
        dist.all_reduce = orig
        own = torch.stack([to.sq_err(res.trajectory[t], tg[t], None, 1) for t in range(4)])
        same = torch.equal(res.node_loc, ref.node_loc) and torch.equal(res.loc_mean, ref.loc_mean)
        q.put((rank, calls, own, res.sq_err, res.graph_nodes, res.mse, N, same))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_ranks_sum_sq_err_in_the_final_reduction():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_rank, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in procs], key=lambda t: t[0])
    [p.join(timeout=60) for p in procs]
    L, C = FLUID["n_layers"], FLUID["virtual_channels"]
    K = 4 + 3 * C + 64 * C
    total = res[0][2] + res[1][2]
    n_all = res[0][6] + res[1][6]
    for rank, calls, own, sq, nodes, mse, N, same in res:
        assert same, f"rank {rank}: targets changed the rollout"
        assert torch.equal(sq, total), f"rank {rank}: sq_err is not the sum over the ranks"
        assert nodes.tolist() == [n_all]
        assert torch.allclose(mse, total[:, 0] / (3 * n_all), rtol=1e-15, atol=0)
        stats = [c for c in calls if c == ((1, K), torch.float32)]
        assert len(stats) == (L + 1) * 4                      # L+1 exchanges per step, as without targets
        assert calls.count(((1 * 4 + 4 * 1,), torch.float64)) == 1   # ONE end-of-rollout reduction: centroid + sq_err
        assert calls.count(((1,), torch.int32)) == 1          # the overflow OR of the one chunk
        assert len(calls) == len(stats) + 2


# ---- GPU ------------------------------------------------------------------------------------------------------------
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


TARGET_CASES = [("nbody", 1, "random"), ("water3d", 1, "random"), ("water3d", 2, "random"), ("water3d", 2, "kmeans"),
                ("largefluid", 1, "random"), ("largefluid", 3, "random"), ("largefluid", 2, "kmeans")]


@pytest.mark.gpu
@pytest.mark.parametrize("recipe,P,split", TARGET_CASES)
def test_targets_gather_equals_the_oracle(tmp_path, recipe, P, split):
    traj = _traj(tmp_path, recipe)
    dt, K = (2, 3) if recipe != "nbody" else (2, 4)
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=dt, frames_per_scene=2, max_frame=9 - K * dt,
                          frame_0=1)
    for rank in range(P):
        kw = dict(delta_t=dt, radius=0.25, batch_size=2, shuffle=True, seed=5, device=dev(), world_size=P, rank=rank,
                  split_mode=split)
        ld = FrameLoader(traj, samples, horizon=K, **kw)
        one = FrameLoader(traj, samples, horizon=1, **kw)
        base = FrameLoader(traj, samples, **kw)
        order = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=5).batches()
        for (k3, e3), (k1, e1), (k0, e0), idx in zip(ld, one, base, order):
            tg = e3["targets"]
            assert tg.shape == (K, k3["node_loc"].shape[0], 3) and tg.dtype == torch.float32
            assert torch.equal(tg[0], e3["target"]) and torch.equal(e3["target"], e0["target"])
            for b, i in enumerate(idx):
                s, f = ld.samples[i]
                index, _ = ld.partition(i)
                want = to.targets(recipe, _position(traj, s), f, dt, K, None if index is None else index.long())
                lo, hi = e3["ptr"][b], e3["ptr"][b + 1]
                assert torch.equal(tg[:, lo:hi].cpu().double(), want), f"rank {rank}, sample {i}"
            # horizon 1 gives today's tensors
            for k in k0:
                if k != "edge_index" and k0[k] is not None:
                    assert torch.equal(k1[k], k0[k]) and torch.equal(k3[k], k0[k]), k
            assert torch.equal(k1["edge_index"].col, k0["edge_index"].col)
            assert torch.equal(e1["targets"][0], e0["target"]) and e1["targets"].shape[0] == 1


def _sq_err_kernel(pred, tg, batch, B, t, steps):
    be = _backend()
    N = pred.shape[0]
    full = torch.zeros(steps, N, 3, device=dev())
    full[t] = tg
    counter = torch.zeros(8, dtype=torch.int32, device=dev())
    counter[0] = t
    out = torch.full((steps, B), -7.0, dtype=torch.float64, device=dev())
    be.rollout_sq_err(pred, full, batch, counter, out, be.rollout_sq_err_workspace(N, dev()))
    return out


def _backend():
    from distegnn_b200.backend import CudaBackend
    return CudaBackend()


def _case(sizes, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    N = sum(sizes)
    pred = torch.rand(N, 3, generator=g) * scale
    tg = pred + torch.randn(N, 3, generator=g) * 1e-2
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    return pred, tg, batch


def _check_rel(got, want, what):
    rel = ((got - want).abs() / want.abs().clamp(min=1e-300)).max()
    assert float(rel) <= 1e-12, f"{what}: rel {float(rel):.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", [[0, 1, 31, 33, 255, 257], [2047, 1, 2049, 0, 4097, 6000], [2_000_000],
                                   [100] * 250])
def test_error_kernel_against_float64(sizes):
    """Per-graph sums within 1e-12 of float64, empty graph ids (and a leading one) included; only row t is written."""
    pred, tg, batch = _case(sizes)
    B, steps, t = len(sizes), 3, 1
    out = _sq_err_kernel(pred.to(dev()), tg.to(dev()), batch.to(dev()) if B > 1 else None, B, t, steps).cpu()
    want = to.sq_err(pred, tg, batch, B)
    assert (out[[0, 2]] == -7.0).all(), "rows other than the counter's step were written"
    nz = torch.tensor(sizes) > 0
    assert (out[t][~nz] == 0).all()
    _check_rel(out[t][nz], want[nz], f"sizes {sizes[:6]}")
    if B > 1:                                                  # one graph's NaN / inf stays in that graph
        for bad in (float("nan"), float("inf")):
            p2 = pred.clone()
            k = int(np.argmax(sizes))
            p2[sum(sizes[:k]) + sizes[k] // 2, 1] = bad
            o2 = _sq_err_kernel(p2.to(dev()), tg.to(dev()), batch.to(dev()), B, t, steps).cpu()
            assert not math.isfinite(float(o2[t, k]))
            others = torch.arange(B) != k
            assert torch.equal(o2[t][others], out[t][others])


@pytest.mark.gpu
def test_error_kernel_outside_the_steps_writes_nothing():
    pred, tg, batch = _case([500, 7000])
    be = _backend()
    ws = be.rollout_sq_err_workspace(7500, dev())
    for t in (-1, 3, 2):
        counter = torch.zeros(8, dtype=torch.int32, device=dev())
        counter[0] = t
        o = torch.full((3, 2), -7.0, dtype=torch.float64, device=dev())
        be.rollout_sq_err(pred.to(dev()), tg.to(dev()).expand(3, -1, -1).contiguous(), batch.to(dev()), counter, o, ws)
        if t == 2:                                             # the same workspace serves the next call
            _check_rel(o[2].cpu(), to.sq_err(pred, tg, batch, 2), "after skipped calls")
            assert (o[:2] == -7.0).all()
        else:
            assert (o == -7.0).all(), f"step {t} is outside [0, steps): nothing may be written"


# ---- GPU: rollouts with targets -------------------------------------------------------------------------------------
def _fluid_batch(tmp_path, K, sizes=(400, 300), step=0.02, radius=0.12, rate=0.0, capacity=None):
    paths = _fluid(tmp_path, list(sizes), T=2 + K, step=step)
    traj = load_scenes(paths, "largefluid")
    samples = [(s, 0) for s in range(len(sizes))]
    ld = FrameLoader(traj, samples, delta_t=1, radius=radius, batch_size=len(sizes), device=dev(), horizon=K,
                     cutoff_rate=rate, capacity=capacity)
    (kw, ex), = list(ld)
    return ld, kw, ex


def _model(F=3, Na=2, deterministic=False):
    from oracle import fastegnn_oracle as orc
    sd = orc.init_state_dict(F, Na, 2, 64, 5, 4, seed=1, coord_gain=0.05)
    m = FastEGNN(node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=2, hidden_nf=64, virtual_channels=5, world_size=1,
                 n_layers=4)
    m.load_state_dict(sd)
    m = m.to(dev()).eval()
    m.deterministic = deterministic
    return m


def _node(kw):
    return dict(node_feat=kw["node_feat"], node_loc=kw["node_loc"], node_vel=kw["node_vel"], loc_mean=kw["loc_mean"],
                data_batch=kw["data_batch"], node_attr=kw["node_attr"])


def _float64_sq_err(traj, targets, batch, B):
    return torch.stack([to.sq_err(traj[t], targets[t], batch, B) for t in range(traj.shape[0])])


@pytest.mark.gpu
def test_targets_change_nothing_else_and_add_one_launch_per_step(tmp_path):
    K = 5
    ld, kw, ex = _fluid_batch(tmp_path, K)
    m = _model(deterministic=True)
    be = m._get_backend(dev())
    common = dict(steps=K, radius=ld.radius, speed_col=2, tau=1.0, return_trajectory=True)
    plain = rollout(m, **_node(kw), **common)                  # warm-up: sizes the capacity, validates data_batch
    cap = plain.capacity
    n0 = be.launches
    plain = rollout(m, **_node(kw), capacity=cap, **common)
    n1 = be.launches
    res = rollout(m, **_node(kw), capacity=cap, targets=ex["targets"], **common)
    n2 = be.launches
    assert (n2 - n1) - (n1 - n0) == K                          # one launch per step, none without targets
    for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "virtual_loc", "trajectory", "n_edges"):
        assert torch.equal(getattr(res, k), getattr(plain, k)), k
    want = _float64_sq_err(res.trajectory, ex["targets"], kw["data_batch"], 2)
    _check_rel(res.sq_err.cpu(), want, "rollout sq_err")
    assert res.graph_nodes.tolist() == ex["node_counts"]
    assert torch.allclose(res.mse.cpu(), want.sum(1) / (3 * sum(ex["node_counts"])), rtol=1e-12, atol=0)


@pytest.mark.gpu
def test_sq_err_is_bitwise_reproducible(tmp_path):
    """Deterministic mode: eager == graphed, two capacities, and a forced overflow rerun == an ample capacity."""
    K = 6
    ld, kw, ex = _fluid_batch(tmp_path, K)
    m = _model(deterministic=True)
    common = dict(steps=K, radius=ld.radius, speed_col=2, targets=ex["targets"])
    ref = rollout(m, **_node(kw), **common)
    cap = ref.capacity
    e0 = int(ref.n_edges.max())
    runs = {"eager, 2x capacity": rollout(m, **_node(kw), capacity=2 * cap, **common),
            "eager, 4x capacity": rollout(m, **_node(kw), capacity=4 * cap, **common)}
    m.cuda_graph = True
    runs["graphed"] = rollout(m, **_node(kw), capacity=2 * cap, **common)
    m.cuda_graph = False
    small = rollout(m, **_node(kw), capacity=max(1, e0 // 2), check_every=2, **common)
    assert small.regrowths
    runs["overflow rerun"] = small
    assert runs["graphed"].replays == K - 1
    for what, r in runs.items():
        assert torch.equal(r.sq_err, ref.sq_err), what
        assert torch.equal(r.mse, ref.mse), what


@pytest.mark.gpu
def test_rollout_with_targets_never_synchronises(tmp_path):
    K = 4
    ld, kw, ex = _fluid_batch(tmp_path, K)
    m = _model()
    warm = rollout(m, **_node(kw), steps=K, radius=ld.radius, speed_col=2, targets=ex["targets"])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = rollout(m, **_node(kw), steps=K, radius=ld.radius, speed_col=2, capacity=2 * warm.capacity,
                      check_every=0, targets=ex["targets"], return_trajectory=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    res.check()
    _check_rel(res.sq_err.cpu(), _float64_sq_err(res.trajectory, ex["targets"], kw["data_batch"], 2), "no-sync")


@pytest.mark.gpu
def test_first_step_mse_is_the_training_loss(tmp_path):
    from distegnn_b200 import train_loss
    ld, kw, ex = _fluid_batch(tmp_path, 1, step=0.5)
    m = _model()
    res = rollout(m, **_node(kw), steps=1, radius=ld.radius, speed_col=2, targets=ex["targets"])
    with torch.no_grad():
        pred, X = m(**kw)
        _, info = train_loss(pred, ex["target"], X, kw["data_batch"], world_size=1, mmd_samples=8,
                             loc_mean=kw["loc_mean"], node_counts=ex["node_counts"])
    logged = float(info["logged"])
    assert abs(float(res.mse[0]) - logged) <= 1e-5 * abs(logged)


@pytest.mark.gpu
def test_differentiable_rollout_loss_against_targets(tmp_path):
    """The INTEGRATION §1 loss on a differentiable rollout equals Σ sq_err / (3·N·K) of a rollout on the same batch; its
    gradient reaches the parameters."""
    from distegnn_b200 import differentiable_rollout
    K = 3
    ld, kw, ex = _fluid_batch(tmp_path, K, step=0.5)
    m = _model().train()
    res = differentiable_rollout(m, **_node(kw), steps=K, radius=ld.radius, speed_col=2)
    loss = ((res.trajectory - ex["targets"]) ** 2).mean()
    loss.backward()
    assert any(p.grad is not None and float(p.grad.abs().max()) > 0 for p in m.parameters())
    m.eval()
    ev = rollout(m, **_node(kw), steps=K, radius=ld.radius, speed_col=2, targets=ex["targets"])
    N = kw["node_loc"].shape[0]
    want = float(ev.sq_err.sum()) / (3 * N * K)
    assert abs(float(loss) - want) <= 1e-5 * want


@pytest.mark.gpu
def test_main_rollout_evaluation_on_raw_frames(tmp_path):
    import subprocess
    import yaml

    def run(cfg, K, *extra):
        p = tmp_path / "cfg.yaml"
        with open(p, "w") as f:
            yaml.safe_dump(cfg, f)
        return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--config_path", str(p), "--trajectory",
                               str(data), "--train_steps", "1", "--rollout_steps", str(K), *extra],
                              capture_output=True, text=True, timeout=600, cwd=ROOT)

    # Water-3D: tau defaults to delta_t
    data = tmp_path / "water"
    for part, sizes, seed in (("train", [60, 50], 1), ("valid", [40, 45], 3)):
        (data / part).mkdir(parents=True)
        _water(data / part, sizes, T=10, seed=seed)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"].update(node_feat_nf=2, node_attr_nf=1)
    cfg["data"].update(dataset_name="Water3D", inner_radius=0.3, max_samples=4, split_mode="random", delta_t=2)
    r = run(cfg, 3)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "rollout evaluation over 4 batches (valid), 3 steps, tau=2" in r.stdout, r.stdout
    for t in (1, 2, 3):
        assert f"rollout step {t}: MSE" in r.stdout
    # N-body: fully connected with the cutoff, --rollout_tau required; a horizon past the files exits with a message
    data = tmp_path / "nbody"
    _nbody(data, "train", S=4, T=10)
    _nbody(data, "valid", S=2, T=10, seed=5)
    with open(os.path.join(ROOT, "config", "nbody_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(batch_size=2, frame_0=1, frame_T=3, cutoff_rate=0.5)
    r = run(cfg, 3)
    assert r.returncode != 0 and "--rollout_tau" in r.stdout, r.stdout + r.stderr[-2000:]
    r = run(cfg, 3, "--rollout_tau", "0.5")
    assert r.returncode == 0, r.stderr[-3000:]
    assert "rollout evaluation over 1 batches (valid), 3 steps" in r.stdout and "rollout step 3: MSE" in r.stdout
    r = run(cfg, 5, "--rollout_tau", "0.5")
    assert r.returncode != 0 and "horizon=5 needs frame 11" in r.stdout, r.stdout + r.stderr[-2000:]
