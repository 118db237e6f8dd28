"""FrameLoader (distegnn_b200/frames.py): training batches assembled on the device from raw trajectories, against the
reference's per-sample lines restated in oracle/frames_oracle.py.  Trajectories are seeded random walks written to
tmp_path in the loader's input layout."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from distegnn_b200 import _lib
from distegnn_b200.frames import (FrameLoader, check_samples, complete_graph_edges, load_nbody, load_scenes,
                                  sample_list)
from distegnn_b200.loader import ShardLoader
from distegnn_b200.partition import node_chunks
from distegnn_b200.shards import CSRGraph
from oracle import frames_oracle as fo


# ---- trajectories -------------------------------------------------------------------------------------------------
def _walk(rng, T, n, step=0.01):
    steps = rng.normal(0.0, step, (T, n, 3))
    steps[0] = rng.random((n, 3))
    return np.cumsum(steps, 0).astype(np.float32)


def _water(tmp_path, sizes, T=8, seed=0, step=0.01):
    rng = np.random.default_rng(seed)
    paths = []
    for k, n in enumerate(sizes):
        p = str(tmp_path / f"water_{k}.npz")
        np.savez(p, position=_walk(rng, T, n, step), particle_type=rng.integers(1, 9, n))
        paths.append(p)
    return paths


def _fluid(tmp_path, sizes, T=8, seed=1, step=0.01):
    rng = np.random.default_rng(seed)
    paths = []
    for k, n in enumerate(sizes):
        p = str(tmp_path / f"fluid_{k}.npz")
        np.savez(p, position=_walk(rng, T, n, step), velocity=rng.normal(0, 1, (T, n, 3)).astype(np.float32),
                 viscosity=rng.random(n).astype(np.float32), mass=rng.random(n).astype(np.float32))
        paths.append(p)
    return paths


def _nbody(tmp_path, S=4, T=6, n=5, seed=2):
    rng = np.random.default_rng(seed)
    d = tmp_path / "nbody"
    d.mkdir(exist_ok=True)
    np.save(d / "loc_train_charged100_0_0_1.npy", np.stack([_walk(rng, T, n, 0.1) for _ in range(S)]))
    np.save(d / "vel_train_charged100_0_0_1.npy", rng.normal(0, 1, (S, T, n, 3)).astype(np.float32))
    np.save(d / "charges_train_charged100_0_0_1.npy", rng.choice([-1.0, 1.0], (S, n, 1)).astype(np.float32))
    return str(d)


def _traj(tmp_path, recipe, sizes=(40, 30, 50, 35)):
    if recipe == "nbody":
        return load_nbody(_nbody(tmp_path))
    paths = _water(tmp_path, sizes) if recipe == "water3d" else _fluid(tmp_path, sizes)
    return load_scenes(paths, recipe)


def _scene_tensors(traj, s):
    sc = traj.scenes[s]
    vel = None if sc.velocity is None else torch.from_numpy(np.array(sc.velocity))
    static = {k: torch.from_numpy(sc.static[:, c].copy()) for c, k in enumerate(traj.recipe.static_keys)}
    return torch.from_numpy(np.array(sc.position)), vel, static


# ---- host side (no GPU) -------------------------------------------------------------------------------------------
def test_sample_list_is_seeded_capped_per_scene_and_in_bounds(tmp_path):
    traj = _traj(tmp_path, "water3d")
    a = sample_list(traj, seed=3, max_samples=10, delta_t=2, frames_per_scene=3, max_frame=5)
    assert a == sample_list(traj, seed=3, max_samples=10, delta_t=2, frames_per_scene=3, max_frame=5)
    assert a != sample_list(traj, seed=4, max_samples=10, delta_t=2, frames_per_scene=3, max_frame=5)
    assert [s for s, _ in a] == [0, 0, 0, 1, 1, 1, 2, 2, 2, 3]        # 3 per scene, capped at max_samples
    assert all(0 <= f <= 5 for _, f in a)
    # the reference's defaults: randint(0, 250) 15 times per scene; these 8-frame scenes cannot hold them
    with pytest.raises(ValueError, match="outside scene"):
        sample_list(traj, seed=0, max_samples=4)
    with pytest.raises(ValueError, match="outside scene"):                # f + 1 (the Water-3D velocity) past the end
        check_samples(traj, [(0, 7)], delta_t=0)
    check_samples(traj, [(0, 6)], delta_t=1)
    with pytest.raises(ValueError, match="no scene"):
        check_samples(traj, [(9, 0)], delta_t=1)
    nb = _traj(tmp_path, "nbody")
    assert sample_list(nb, max_samples=3, frame_0=1, delta_t=4) == [(0, 1), (1, 1), (2, 1)]
    with pytest.raises(ValueError, match="outside scene"):
        sample_list(nb, frame_0=1, delta_t=5)


def test_sampler_order_is_shardloaders(tmp_path):
    from torch.utils.data import RandomSampler
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=0, max_samples=7, delta_t=1, frames_per_scene=2, max_frame=5)
    gen = torch.Generator()
    gen.manual_seed(43)
    want = list(RandomSampler(range(7), replacement=False, generator=gen))
    fl = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=43)
    sl = ShardLoader([str(i) for i in range(7)], batch_size=2, shuffle=True, seed=43)
    assert len(fl) == len(sl) == 3
    assert fl.batches() == [want[0:2], want[2:4], want[4:6]]
    from distegnn_b200.loader import sampler_batches
    assert sampler_batches(7, 2, True, torch.Generator().manual_seed(43), True) == [want[0:2], want[2:4], want[4:6]]
    assert FrameLoader(traj, samples, batch_size=3, drop_last=False).batches() == [[0, 1, 2], [3, 4, 5], [6]]


def test_malformed_inputs_are_rejected(tmp_path):
    rng = np.random.default_rng(0)
    pos = _walk(rng, 4, 6)
    cases = [(dict(particle_type=np.ones(6)), "water3d", "missing 'position'"),
             (dict(position=pos), "water3d", "missing 'particle_type'"),
             (dict(position=pos[0], particle_type=np.ones(6)), "water3d", r"\[T,n,3\]"),
             (dict(position=pos[..., :2], particle_type=np.ones(6)), "water3d", r"\[T>=1, n>=1, 3\]"),
             (dict(position=pos, particle_type=np.ones(5)), "water3d", r"must be \[6\]"),
             (dict(position=pos, viscosity=np.ones(6), mass=np.ones(6)), "largefluid", "needs velocities"),
             (dict(position=pos, velocity=pos[:3], viscosity=np.ones(6), mass=np.ones(6)), "largefluid", "velocity shape"),
             (dict(position=pos, particle_type=np.ones(6)), "largefluid", "missing 'viscosity'")]
    for k, (arrays, recipe, msg) in enumerate(cases):
        p = str(tmp_path / f"bad{k}.npz")
        np.savez(p, **arrays)
        with pytest.raises(ValueError, match=msg):
            load_scenes([p], recipe)
    with pytest.raises(ValueError, match="unknown recipe"):
        load_scenes(_water(tmp_path, [5]), "protein")
    d = _nbody(tmp_path)
    np.save(os.path.join(d, "charges_train_charged100_0_0_1.npy"), np.ones((4, 4, 1), np.float32))
    with pytest.raises(ValueError, match="charges"):
        load_nbody(d)


def test_stored_npz_members_are_memory_mapped(tmp_path):
    traj = load_scenes(_water(tmp_path, [7]), "water3d")
    assert isinstance(traj.scenes[0].position, np.memmap)
    p = str(tmp_path / "packed.npz")
    rng = np.random.default_rng(0)
    pos = _walk(rng, 3, 4)
    np.savez_compressed(p, position=pos, particle_type=np.arange(4))
    sc = load_scenes([p], "water3d").scenes[0]
    assert np.array_equal(sc.position, pos) and np.array_equal(sc.static[:, 0], np.arange(4, dtype=np.float32))


def test_complete_graph_is_the_reference_list():
    for n in (1, 2, 5):
        assert torch.equal(complete_graph_edges(n), fo.complete_edges(n))


def test_random_partition_is_split_large_graphs_chunking(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=0, max_samples=4, delta_t=1, frames_per_scene=1, max_frame=5)
    for P in (2, 3):
        loaders = [FrameLoader(traj, samples, world_size=P, rank=r, seed=11) for r in range(P)]
        for i, (s, _) in enumerate(samples):
            n = traj.scenes[s].n_nodes
            want = fo.sample("water3d", *_scene_tensors(traj, s), samples[i][1], 1, 0.2, world_size=P,
                             generator=loaders[0].sample_generator(i))
            got = [ld.partition(i) for ld in loaders]
            for r in range(P):
                assert torch.equal(got[r][0].long(), want[r]["index"])
                assert got[r][1] == [int(w["index"].numel()) for w in want]
            assert torch.equal(torch.sort(torch.cat([g[0] for g in got]).long())[0], torch.arange(n))
    tiny = load_scenes(_water(tmp_path, [2]), "water3d")
    with pytest.raises(ValueError, match="without nodes"):
        FrameLoader(tiny, [(0, 0)], world_size=3).partition(0)
    g = torch.Generator().manual_seed(5)
    chunks = node_chunks(10, 3, "random", generator=g)
    assert [c.numel() for c in chunks] == [3, 3, 4]
    assert torch.equal(torch.cat(chunks), torch.randperm(10, generator=torch.Generator().manual_seed(5)))


def _gloo_rank(rank, world, port, root, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        traj = load_scenes(sorted(os.path.join(root, f) for f in os.listdir(root) if f.startswith("water_")), "water3d")
        samples = sample_list(traj, seed=0, max_samples=6, delta_t=1, frames_per_scene=2, max_frame=5)
        ld = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=7, world_size=world, rank=rank)
        mine = dict(order=ld.batches(), parts=[ld.partition(i)[0].tolist() for i in range(len(samples))],
                    n=[traj.scenes[s].n_nodes for s, _ in samples])
        got = [None] * world
        dist.all_gather_object(got, mine)
        q.put((rank, got))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_walk_one_order_and_split_each_frame(tmp_path):
    _water(tmp_path, [40, 30, 50])
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_rank, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in procs]
    [p.join(timeout=60) for p in procs]
    got = res[0][1]
    assert got[0]["order"] == got[1]["order"] and len(got[0]["order"]) == 3
    for i, n in enumerate(got[0]["n"]):
        a, b = set(got[0]["parts"][i]), set(got[1]["parts"][i])
        assert not (a & b) and a | b == set(range(n)) and a and b


def test_abi_symbol_is_exported():
    import ctypes
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(lib, "distegnn_frames_assemble")
    assert _lib.load().distegnn_frames_assemble(7, 1, 0, 0, *([None] * 14)) == -1
    assert b"unknown recipe" in _lib.load().distegnn_last_error()


# ---- on the device ------------------------------------------------------------------------------------------------
def _ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    ia, ib = a.contiguous().view(torch.int32).long(), b.contiguous().view(torch.int32).long()
    same_sign = (a >= 0) == (b >= 0)
    assert bool(same_sign.all())
    return int((ia - ib).abs().max()) if a.numel() else 0


_NEAR = 1e-5


def _edge_set(ei):
    return set(zip(ei[0].tolist(), ei[1].tolist()))


def _check_batch(traj, loader, kwargs, extras, idx, recipe, radius, rate, P, rank):
    dev = kwargs["node_loc"].device
    g, ea = kwargs["edge_index"], kwargs["edge_attr"]
    loc, batch, B = kwargs["node_loc"], kwargs["data_batch"], len(idx)
    # the graph is the one radius_graph_csr / cutoff_edges_csr build on the assembled positions, bit for bit
    if radius is None:
        counts = extras["node_counts"]
        eis, off = [], 0
        for m in counts:
            eis.append(fo.complete_edges(m) + off)
            off += m
        cand, _ = CSRGraph.from_edge_index(torch.cat(eis, 1).to(dev), off)
        if rate > 0:
            from distegnn_b200 import cutoff_edges_csr
            wg, wea = cutoff_edges_csr(cand, loc, rate, batch, B)
        else:
            wg, wea = cand, None
    else:
        from distegnn_b200 import radius_graph_csr
        wg, wea = radius_graph_csr(loc, radius, batch, n_graphs=B, cutoff_rate=rate)
    E = int(g.rowptr[-1])
    assert torch.equal(g.rowptr, wg.rowptr) and torch.equal(g.col[:E], wg.col[:E])
    if wea is not None:
        assert torch.equal(ea[:E], wea[:E])
    row = g.rows()[:E].long().cpu()
    col = g.col[:E].long().cpu()
    ptr = extras["ptr"]
    assert extras["n_graphs"] == B and extras["node_counts"] == [ptr[b + 1] - ptr[b] for b in range(B)]
    for b, i in enumerate(idx):
        s, f = loader.samples[i]
        pos_t, vel_t, static = _scene_tensors(traj, s)
        want = fo.sample(recipe, pos_t, vel_t, static, f, loader.delta_t, radius, rate, world_size=P,
                         split_mode=loader.split_mode, generator=loader.sample_generator(i))[rank]
        lo, hi = ptr[b], ptr[b + 1]
        got = {k: kwargs[k][lo:hi].cpu() for k in ("node_loc", "node_vel", "node_attr", "node_feat")}
        assert torch.equal(got["node_loc"], want["pos"])
        assert torch.equal(got["node_vel"], want["vel"])
        assert torch.equal(got["node_attr"], want["attr"])
        assert torch.equal(extras["target"][lo:hi].cpu(), want["target"])
        assert torch.equal(kwargs["data_batch"][lo:hi].cpu(), torch.full((hi - lo,), b, dtype=torch.int64))
        if recipe == "largefluid":
            assert torch.equal(got["node_feat"][:, :2], want["x"][:, :2])
            assert _ulps(got["node_feat"][:, 2], want["x"][:, 2]) <= 1
        else:
            assert _ulps(got["node_feat"], want["x"]) <= 1
        whole = pos_t[f].double().mean(0)
        lm = kwargs["loc_mean"][b].cpu().double()
        assert float((lm - whole).abs().max()) <= 1e-6 * max(float(whole.abs().max()), 1e-30)
        # edges of this graph, in graph-local ids, against the oracle's.  Candidates may differ only for pairs within
        # _NEAR·r of r; kept sets only among edges tied with the longest kept one (the reference's order among equal
        # lengths is torch.sort's, the device's is CSR position — DESIGN §16)
        m = (row >= lo) & (row < hi)
        mine = _edge_set(torch.stack([row[m] - lo, col[m] - lo]))
        theirs = _edge_set(want["edge_index"])
        diff = mine ^ theirs
        if diff:
            p = want["pos"]
            d = torch.stack([(p[a] - p[c]).norm() for a, c in diff])
            if rate == 0:
                assert radius is not None
                assert bool(((d.double() - radius).abs() <= _NEAR * radius).all()), "edges differ away from the radius"
            else:
                ei = want["edge_index"]
                thr = (p[ei[0]] - p[ei[1]]).norm(dim=1).max()
                assert bool(((d - thr).abs() <= 1e-6 * thr).all()), f"{len(diff)} kept edges differ beyond ties"


CASES = [("nbody", None, 0.0, 1, "random"), ("nbody", None, 0.5, 1, "random"), ("nbody", 0.6, 0.3, 1, "random"),
         ("water3d", 0.2, 0.5, 1, "random"), ("water3d", 0.2, 0.0, 2, "random"), ("water3d", 0.25, 0.0, 2, "kmeans"),
         ("largefluid", 0.2, 0.0, 1, "random"), ("largefluid", 0.2, 0.0, 3, "random"),
         ("largefluid", 0.25, 0.0, 2, "kmeans")]


@pytest.mark.gpu
@pytest.mark.parametrize("recipe,radius,rate,P,split", CASES)
def test_assembly_matches_the_reference_lines(tmp_path, recipe, radius, rate, P, split):
    dev = torch.device("cuda:0")
    traj = _traj(tmp_path, recipe)
    dt = 3 if recipe == "nbody" else 2
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=dt, frames_per_scene=2, max_frame=4, frame_0=1)
    for rank in range(P):
        ld = FrameLoader(traj, samples, delta_t=dt, radius=radius, batch_size=2, shuffle=True, seed=5, device=dev,
                         world_size=P, rank=rank, split_mode=split, cutoff_rate=rate)
        order = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=5).batches()
        n = 0
        for (kwargs, extras), idx in zip(ld, order):
            _check_batch(traj, ld, kwargs, extras, idx, recipe, radius, rate, P, rank)
            n += 1
        assert n == len(order) == 2


@pytest.mark.gpu
@pytest.mark.parametrize("split", ["random", "kmeans"])
def test_partitions_equal_split_large_graph(tmp_path, split):
    from distegnn_b200 import split_large_graph
    dev = torch.device("cuda:0")
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=2, max_samples=3, delta_t=1, frames_per_scene=1, max_frame=4)
    P = 3
    loaders = [FrameLoader(traj, samples, radius=0.2, device=dev, world_size=P, rank=r, split_mode=split,
                           prefetch=0) for r in range(P)]
    outs = [list(ld) for ld in loaders]
    for i, (s, f) in enumerate(samples):
        pos_t, vel_t, static = _scene_tensors(traj, s)
        x = torch.zeros(pos_t.shape[1], 2)
        ref = split_large_graph(pos_t[f].to(dev), x.to(dev), pos_t[f + 1].to(dev), vel_t.to(dev) if vel_t is not None
                                else pos_t[f].to(dev), None, 0.2, P, split_mode=split,
                                generator=loaders[0].sample_generator(i))
        for r in range(P):
            kwargs, extras = outs[r][i]
            assert torch.equal(kwargs["node_loc"], ref[r]["pos"])
            assert torch.equal(kwargs["edge_index"].rowptr, ref[r]["edge_index"].rowptr)
            assert torch.equal(kwargs["edge_index"].col, ref[r]["edge_index"].col)


@pytest.mark.gpu
def test_mixed_sizes_one_node_scenes_and_p_close_to_n(tmp_path):
    dev = torch.device("cuda:0")
    traj = load_scenes(_water(tmp_path, [1, 5, 17, 1, 4]), "water3d")
    samples = [(0, 0), (1, 2), (2, 1), (3, 3), (4, 0)]
    ld = FrameLoader(traj, samples, delta_t=2, radius=0.4, batch_size=5, device=dev, cutoff_rate=0.5)
    (kwargs, extras), = list(ld)
    assert extras["node_counts"] == [1, 5, 17, 1, 4]
    _check_batch(traj, ld, kwargs, extras, list(range(5)), "water3d", 0.4, 0.5, 1, 0)
    P = 4                                                    # P = n − 1 on the 5-node scene
    sub = [(1, 2), (4, 0)]
    for rank in range(P):
        ld = FrameLoader(traj, sub, delta_t=2, radius=0.4, batch_size=2, device=dev, world_size=P, rank=rank)
        (kwargs, extras), = list(ld)
        assert min(extras["node_counts"]) >= 1
        _check_batch(traj, ld, kwargs, extras, [0, 1], "water3d", 0.4, 0.0, P, rank)


@pytest.mark.gpu
def test_nbody_candidates_are_the_reference_list(tmp_path):
    dev = torch.device("cuda:0")
    traj = _traj(tmp_path, "nbody")
    ld = FrameLoader(traj, sample_list(traj, delta_t=2), delta_t=2, radius=-1, batch_size=2, device=dev)
    (kwargs, _), _ = list(ld)
    cand = ld._complete[(5, 5)]
    want, _ = CSRGraph.from_edge_index(torch.cat([fo.complete_edges(5), fo.complete_edges(5) + 5], 1).to(dev), 10)
    assert torch.equal(cand.rowptr, want.rowptr) and torch.equal(cand.col, want.col) and torch.equal(cand.row, want.row)
    assert kwargs["edge_index"] is cand


def _train_step(model, kwargs, target, node_counts):
    from distegnn_b200 import train_loss
    model.zero_grad()
    torch.manual_seed(0)
    loc_pred, X = model(**kwargs)
    loss, _ = train_loss(loc_pred, target, X, kwargs["data_batch"], world_size=1, mmd_samples=8,
                         loc_mean=kwargs["loc_mean"], node_counts=node_counts)
    loss.backward()
    return float(loss), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


@pytest.mark.gpu
@pytest.mark.parametrize("recipe,radius,rate", [("water3d", 0.2, 0.0), ("largefluid", 0.2, 0.0), ("nbody", None, 0.5)])
def test_training_step_equals_the_shard_fed_step(tmp_path, recipe, radius, rate):
    """Cases without ties at the cutoff: a fully connected 5-node graph keeps whole pairs at rate 0.5 (k = 10 of 20), so
    the kept edges are the oracle's; a radius cutoff may split a mirrored pair, whose two edges have one length.  The
    targets lie O(1) away from the inputs: the two batches order each row's edges differently, and fp32 sums in another
    order move the predictions by ~1e-7, which a displacement near that scale would amplify in the MSE."""
    from distegnn_b200 import FastEGNN
    from distegnn_b200.shards import shard_from_forward_inputs, write_shard
    from oracle import fastegnn_oracle as orc
    dev = torch.device("cuda:0")
    dt = 2
    if recipe == "nbody":
        traj = _traj(tmp_path, recipe)
        samples = sample_list(traj, seed=0, max_samples=2, delta_t=dt, frame_0=1)
    else:
        paths = (_water if recipe == "water3d" else _fluid)(tmp_path, [40, 30], step=0.5)
        traj, samples = load_scenes(paths, recipe), [(0, 0), (1, 0)]
    F, Na = traj.recipe.node_feat_nf, traj.recipe.node_attr_nf
    paths = []
    for i, (s, f) in enumerate(samples):
        w = fo.sample(recipe, *_scene_tensors(traj, s), f, dt, radius, rate)[0]
        n = w["pos"].shape[0]
        inp = dict(node_feat=w["x"], node_loc=w["pos"], node_vel=w["vel"], loc_mean=w["loc_mean"],
                   data_batch=torch.zeros(n, dtype=torch.int64), edge_index=w["edge_index"], edge_attr=w["edge_attr"],
                   node_attr=w["attr"])
        paths.append(str(tmp_path / f"s{i}.shard"))
        write_shard(paths[-1], shard_from_forward_inputs(inp, target=w["target"]))
    sd = orc.init_state_dict(F, Na, 2, 64, 3, 2, seed=1, coord_gain=0.05)
    m = FastEGNN(node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=2, hidden_nf=64, virtual_channels=3, world_size=1,
                 n_layers=2)
    m.load_state_dict(sd)
    m = m.to(dev).train()
    (kf, ef), = list(FrameLoader(traj, samples, delta_t=dt, radius=radius, batch_size=2, device=dev, cutoff_rate=rate))
    (ks, es), = list(ShardLoader(paths, batch_size=2, device=dev))
    assert ef["node_counts"] == es["node_counts"]
    lf, gf = _train_step(m, kf, ef["target"], ef["node_counts"])
    ls, gs = _train_step(m, ks, es["target"], es["node_counts"])
    assert abs(lf - ls) <= 1e-6 * abs(ls)
    # against the model's gradient scale: some tensors' gradients (layer 0's virtual coordinate MLP) are ~1e-6 of it
    # and carry only summation-order noise
    scale = max(float(g.abs().max()) for g in gs.values())
    for k in gs:
        assert float((gf[k] - gs[k]).abs().max()) <= 1e-5 * scale, k


@pytest.mark.gpu
@pytest.mark.parametrize("split", ["random", "kmeans"])
def test_capacity_mode_epoch_never_synchronises(tmp_path, split):
    dev = torch.device("cuda:0")
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=0, max_samples=8, delta_t=1, frames_per_scene=2, max_frame=5)
    ld = FrameLoader(traj, samples, radius=0.2, batch_size=2, shuffle=True, device=dev, world_size=2, rank=1,
                     split_mode=split, capacity=20000, cutoff_rate=0.5 if split == "random" else 0.0)
    first = [kw["node_loc"].sum() for kw, _ in ld]           # caches the k-means labels, warms the allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steady = [(kw["node_loc"] * 2).sum() for kw, _ in ld]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(first) == len(steady) == 4
    ld.check()
    over = FrameLoader(traj, samples, radius=0.2, batch_size=2, device=dev, capacity=8)
    list(over)
    with pytest.raises(RuntimeError, match="outgrew the capacity 8"):
        over.check()
    ld.check()


@pytest.mark.gpu
def test_main_trains_and_evaluates_on_raw_frames(tmp_path):
    import subprocess
    import sys
    import yaml
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for part, sizes, seed in (("train", [60, 50], 1), ("valid", [40], 3)):
        (tmp_path / part).mkdir()
        _fluid(tmp_path / part, sizes, seed=seed)
    with open(os.path.join(root, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(inner_radius=0.3, max_samples=4, split_mode="random")
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    r = subprocess.run([sys.executable, os.path.join(root, "main.py"), "--config_path", str(p), "--trajectory",
                        str(tmp_path), "--train_steps", "3"], capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "3 train steps on raw frames" in r.stdout and "evaluation over 4 batches (valid)" in r.stdout, r.stdout
