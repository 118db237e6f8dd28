"""FrameLoader's training noise (DESIGN §22): the generator against an independent numpy Philox4x32-10 and float64
Box–Muller, its statistics, the noisy assembly restated bit for bit from the testing hook's ε, its invariance to how the
samples are split and batched, and `main.py --train_noise`."""
import ctypes as C
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from distegnn_b200 import _lib
from distegnn_b200.frames import FrameLoader, load_scenes, sample_list
from oracle import frames_oracle as fo
from tests.test_frames import CASES, _NEAR, _edge_set, _fluid, _scene_tensors, _traj, _ulps, _water

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M32 = np.uint64(0xFFFFFFFF)


# ---- numpy oracle of the generator --------------------------------------------------------------------------------
def philox4x32_10(ctr, key):
    """Random123's Philox4x32-10: ctr uint32 [..., 4], key uint32 [..., 2] (broadcast) -> uint32 [..., 4]."""
    ctr, key = np.broadcast_arrays(np.asarray(ctr, np.uint32)[..., :, None], np.asarray(key, np.uint32)[..., None, :])
    c = [ctr[..., i, 0].astype(np.uint64) for i in range(4)]
    k0, k1 = key[..., 0, 0].astype(np.uint64), key[..., 0, 1].astype(np.uint64)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & M32]
    return np.stack(c, -1).astype(np.uint32)


def raw_words(seed, epoch, sample, nodes, q):
    """The four Philox words of (nodes, stream q) of `sample` in `epoch` under `seed` (frames_noise.cuh's counter)."""
    nodes = np.asarray(nodes, np.uint64)
    ctr = np.stack([nodes.astype(np.uint32), np.full(nodes.shape, q, np.uint32), np.full(nodes.shape, sample, np.uint32),
                    np.full(nodes.shape, epoch, np.uint32)], -1)
    return philox4x32_10(ctr, [seed & 0xFFFFFFFF, seed >> 32])


def uniforms(o):
    """fp32 (o >> 8)·2^-24 + 2^-25, each operation in fp32."""
    return (o >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24) + np.float32(2.0 ** -25)


def box_muller64(o):
    """float64 Box–Muller of the fp32 uniforms of words o [..., 4]: (z [..., 3], radius of each component [..., 3])."""
    u = uniforms(o).astype(np.float64)
    r01, r23 = np.sqrt(-2 * np.log(u[..., 0])), np.sqrt(-2 * np.log(u[..., 2]))
    z = np.stack([r01 * np.cos(2 * np.pi * u[..., 1]), r01 * np.sin(2 * np.pi * u[..., 1]),
                  r23 * np.cos(2 * np.pi * u[..., 3])], -1)
    return z, np.stack([r01, r01, r23], -1)


# ---- host side (no GPU) ---------------------------------------------------------------------------------------------
def test_numpy_philox_matches_random123_known_answers():
    kat = [([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
           ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
           ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
            [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])]
    for ctr, key, want in kat:
        assert philox4x32_10(ctr, key).tolist() == want
    o = np.array([0, 0xffffffff, 0x80000000, 0xff], np.uint32)
    u = uniforms(o)
    assert u[0] == np.float32(2.0 ** -25) and u[3] == u[0] and 0 < u.min() and u.max() <= 1
    z, _ = box_muller64(np.array([[0, 0, 0, 0]], np.uint32))
    assert np.all(np.abs(z) <= math.sqrt(50 * math.log(2)))


def test_loader_rejects_bad_noise_arguments(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = [(0, 0), (1, 1)]
    for bad in [(-1e-3, 0.0), (0.0, -1.0), (float("nan"), 0.0), (0.0, float("inf")), (1e-3,), (1e-3, 1e-3, 1e-3),
                1e-3, "ab", ("a", 1.0)]:
        with pytest.raises(ValueError, match="noise"):
            FrameLoader(traj, samples, noise=bad)
    for seed in (-1, 1 << 64):
        with pytest.raises(ValueError, match="noise_seed"):
            FrameLoader(traj, samples, noise=(1e-3, 1e-3), noise_seed=seed)
    assert FrameLoader(traj, samples, noise=(0, 0)).noise is None and FrameLoader(traj, samples).noise is None
    ld = FrameLoader(traj, samples, noise=np.array([1e-3, 2e-3]), seed=9)
    assert ld.noise == (1e-3, 2e-3) and ld.noise_seed == 9
    assert FrameLoader(traj, samples, noise=(1e-3, 0), seed=9, noise_seed=(1 << 64) - 1).noise_seed == (1 << 64) - 1
    FrameLoader(traj, samples, seed=-1)                      # a sampler seed the noise cannot use is fine without noise
    FrameLoader(traj, samples, seed=-1, noise=(0, 0))
    with pytest.raises(ValueError, match="noise_seed"):
        FrameLoader(traj, samples, seed=-1, noise=(1e-3, 1e-3))


def _noise_call(**over):
    a = dict(recipe=_lib.FRAMES_WATER3D, B=1, n_frame=0, n_out=0, K=1, ptrs=[None] * 5, outs=[None] * 6 + [1, 1],
             ids=1, seed=0, epoch=0, sx=0.0, sv=0.0)
    a.update(over)
    return _lib.load().distegnn_frames_assemble_noise(a["recipe"], a["B"], a["n_frame"], a["n_out"], a["K"], *a["ptrs"],
                                                      *a["outs"], a["ids"], a["seed"], a["epoch"], a["sx"], a["sv"],
                                                      None)


def test_c_abi_rejects_bad_noise_arguments_before_launching():
    lib = _lib.load()
    # valid apart from the argument under test, with sizes that launch nothing but the (deviceless) scene kernel: every
    # rejection below returns before that launch
    cases = [(dict(sx=-1.0), b"sigma"), (dict(sv=float("nan")), b"sigma"), (dict(sx=float("inf")), b"sigma"),
             (dict(K=0), b"horizon"), (dict(ids=None), b"sample_ids"), (dict(recipe=7), b"unknown recipe"),
             (dict(B=0), b"bad size"), (dict(n_out=3), b"n_out == n_frame_nodes"),
             (dict(outs=[None] * 8), b"null pointer")]
    for over, msg in cases:
        assert _noise_call(**over) == -1, over
        err = lib.distegnn_last_error()
        assert msg in err and err.startswith(b"distegnn_frames_assemble_noise"), (over, err)
    # the testing hook: sample and node ids outside [0, 2^32), bad σ
    t = C.CDLL(os.path.join(os.path.dirname(_lib.LIB_PATH), "libdistegnn_b200_testing.so"))
    f = t.distegnn_testing_frames_noise
    f.argtypes = [C.c_uint64, C.c_uint32, C.c_int64, C.c_int64, C.c_int64, C.c_float, C.c_float] + [C.c_void_p] * 4
    assert f(0, 0, 1 << 32, 0, 1, 0.0, 0.0, None, None, None, None) == -1
    assert f(0, 0, -1, 0, 1, 0.0, 0.0, None, None, None, None) == -1
    assert f(0, 0, 0, (1 << 32) - 1, 2, 0.0, 0.0, None, None, None, None) == -1
    assert f(0, 0, 0, 0, 1, -1.0, 0.0, None, None, None, None) == -1
    assert f(0, 0, 0, 0, 0, 1.0, 1.0, None, None, None, None) == 0        # nothing to do


def test_epoch_counts_batches_calls_and_is_fixed_per_iteration(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=0, max_samples=6, delta_t=1, frames_per_scene=2, max_frame=5)
    ld = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=7, noise=(1e-3, 1e-3))
    assert ld.epoch == 0
    ld.batches()
    ld.batches()
    assert ld.epoch == 2
    host = ld._host_batch([3, 1], epoch=5)
    assert host["epoch"] == 5 and host["meta"][-2:].tolist() == [3, 1]
    assert FrameLoader(traj, samples)._host_batch([3, 1])["meta"].numel() == 2 * 2 + 2    # no ids without noise


def _gloo_rank(rank, world, port, root, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        traj = load_scenes(sorted(os.path.join(root, f) for f in os.listdir(root) if f.startswith("water_")), "water3d")
        samples = sample_list(traj, seed=0, max_samples=6, delta_t=1, frames_per_scene=2, max_frame=5)
        ld = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=7, world_size=world, rank=rank,
                         noise=(1e-3, 1e-3))
        mine = []
        for _ in range(3):
            e = ld.epoch
            mine.append((e, ld.batches()))
        got = [None] * world
        dist.all_gather_object(got, mine)
        q.put((rank, got))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_count_the_same_epochs(tmp_path):
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
    assert got[0] == got[1]
    assert [e for e, _ in got[0]] == [0, 1, 2]


def _main(args, timeout=600):
    return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), *args], capture_output=True, text=True,
                          timeout=timeout, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))


def test_main_rejects_bad_train_noise_before_cuda_work(tmp_path):
    cfg = os.path.join(ROOT, "config", "largefluid_distegnn.yaml")
    for bad, msg in (("1e-3", "two comma-separated"), ("a,b", "two comma-separated"), ("1,2,3", "two comma-separated"),
                     ("-1e-3,0", "finite and >= 0"), ("nan,0", "finite and >= 0")):
        r = _main(["--config_path", cfg, "--trajectory", str(tmp_path), f"--train_noise={bad}"])
        assert r.returncode == 2 and f"--train_noise {bad!r}: must be {msg}" in r.stdout, (bad, r.stdout, r.stderr)
        assert "CUDA" not in r.stderr
    r = _main(["--config_path", cfg, "--train_noise", "1e-3,1e-3"])
    assert r.returncode == 2 and "used with --trajectory" in r.stdout, r.stdout


def test_main_gives_the_noise_to_the_train_loader_only(tmp_path):
    import yaml
    import main
    for part, sizes, seed in (("train", [60, 50], 1), ("valid", [40], 3)):
        (tmp_path / part).mkdir()
        _fluid(tmp_path / part, sizes, seed=seed)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(inner_radius=0.3, max_samples=4, split_mode="random")
    dev = torch.device("cuda", 0)
    _, lds = main.frame_loaders(str(tmp_path), cfg, 1, 0, dev, None, noise=(1e-3, 2e-3))
    assert lds["train"].noise == (1e-3, 2e-3) and lds["valid"].noise is None
    _, lds = main.frame_loaders(str(tmp_path), cfg, 1, 0, dev, None, horizon=2, parts=("valid",))   # the rollout's
    assert lds["valid"].noise is None
    _, lds = main.frame_loaders(str(tmp_path), cfg, 1, 0, dev, None)
    assert lds["train"].noise is None


# ---- on the device ------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def hook(seed, epoch, sample, first, n, sx, sv, raw=False):
    """(eps_x, eps_v, raw words or None) of scene nodes first .. first + n − 1 from the testing library."""
    t = C.CDLL(os.path.join(os.path.dirname(_lib.LIB_PATH), "libdistegnn_b200_testing.so"))
    f = t.distegnn_testing_frames_noise
    f.argtypes = [C.c_uint64, C.c_uint32, C.c_int64, C.c_int64, C.c_int64, C.c_float, C.c_float] + [C.c_void_p] * 4
    ex = torch.empty(n, 3, device=_dev())
    ev = torch.empty(n, 3, device=_dev())
    w = torch.empty(n, 2, 4, dtype=torch.int32, device=_dev()) if raw else None
    rc = f(seed, epoch, sample, first, n, sx, sv, ex.data_ptr(), ev.data_ptr(), w.data_ptr() if raw else None,
           torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.load().distegnn_last_error()
    torch.cuda.synchronize()
    return ex.cpu(), ev.cpu(), None if w is None else w.cpu().numpy().view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("seed,epoch,sample,first", [(0, 0, 0, 0), (0xDEADBEEFCAFEF00D, 7, 123456, 1 << 20),
                                                     ((1 << 64) - 1, 0xFFFFFFFF, 0xFFFFFFFF, (1 << 32) - (1 << 20))])
def test_generator_equals_numpy_philox_and_box_muller(seed, epoch, sample, first):
    n = 1 << 20
    sx, sv = 0.37, 2.5e-3
    ex, ev, w = hook(seed, epoch, sample, first, n, sx, sv, raw=True)
    nodes = np.arange(first, first + n, dtype=np.uint64)
    for q, eps, sig in ((0, ex, sx), (1, ev, sv)):
        want = raw_words(seed, epoch, sample, nodes, q)
        assert np.array_equal(w[:, q], want), f"stream {q}: raw words differ"
        z, r = box_muller64(want)
        ulp = np.spacing(np.float32(sig * r).astype(np.float32)).astype(np.float64)
        err = np.abs(eps.numpy().astype(np.float64) - sig * z)
        assert np.all(err <= 4 * ulp), f"stream {q}: worst {float((err / ulp).max()):.2f} ulps"


@pytest.mark.gpu
def test_noise_statistics():
    from scipy import stats
    n = 1 << 20
    sx, sv = 0.5, 2.0
    ex, ev, _ = hook(12345, 3, 17, 0, n, sx, sv)
    ex1, _, _ = hook(12345, 4, 17, 0, n, sx, sv)
    bound = 5 / math.sqrt(n)
    for eps, sig in ((ex, sx), (ev, sv)):
        z = eps.double().numpy() / sig
        assert np.all(np.abs(z) <= 5.9)
        for d in range(3):
            assert abs(z[:, d].mean()) <= bound
            assert abs(z[:, d].var() - 1) <= 0.01
            assert stats.kstest(z[:, d], "norm").pvalue > 1e-4
        c = np.corrcoef(z.T)
        assert np.all(np.abs(c[np.triu_indices(3, 1)]) <= bound)                     # between axes
        for d in range(3):
            assert abs(np.corrcoef(z[:-1, d], z[1:, d])[0, 1]) <= bound               # consecutive node ids
    zx, zv, z1 = ex.double().numpy() / sx, ev.double().numpy() / sv, ex1.double().numpy() / sx
    for d in range(3):
        assert abs(np.corrcoef(zx[:, d], zv[:, d])[0, 1]) <= bound                    # between the streams
        assert abs(np.corrcoef(zx[:, d], z1[:, d])[0, 1]) <= bound                    # between epochs


def _noisy_fields(recipe, pos_t, vel_t, f, dt, ex, ev, K=1):
    """The assembly's noisy fields over the whole scene, restated on the CPU with the fp32 rules of DESIGN §22."""
    x = pos_t[f] + ex
    v = (pos_t[f + 1] - pos_t[f] if recipe == "water3d" else vel_t[f]) + ev
    speed = torch.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    targets = torch.stack([pos_t[f + t * dt] + ex for t in range(1, K + 1)])
    return x, v, speed, targets


def _check_noisy_batch(traj, ld, kwargs, extras, idx, epoch, recipe, radius, rate, P, rank):
    from distegnn_b200 import cutoff_edges_csr, radius_graph_csr
    from distegnn_b200.shards import CSRGraph
    dev = _dev()
    g, ea = kwargs["edge_index"], kwargs["edge_attr"]
    loc, batch, B = kwargs["node_loc"], kwargs["data_batch"], len(idx)
    sx, sv = ld.noise
    if radius is None:
        eis, off = [], 0
        for m in extras["node_counts"]:
            eis.append(fo.complete_edges(m) + off)
            off += m
        cand, _ = CSRGraph.from_edge_index(torch.cat(eis, 1).to(dev), off)
        wg, wea = cutoff_edges_csr(cand, loc, rate, batch, B) if rate > 0 else (cand, None)
    else:
        wg, wea = radius_graph_csr(loc, radius, batch, n_graphs=B, cutoff_rate=rate)
    E = int(g.rowptr[-1])
    assert torch.equal(g.rowptr, wg.rowptr) and torch.equal(g.col[:E], wg.col[:E])
    if wea is not None:
        assert torch.equal(ea[:E], wea[:E])
    row, col = g.rows()[:E].long().cpu(), g.col[:E].long().cpu()
    ptr = extras["ptr"]
    K = extras["targets"].shape[0]
    for b, i in enumerate(idx):
        s, f = ld.samples[i]
        pos_t, vel_t, static = _scene_tensors(traj, s)
        n = pos_t.shape[1]
        ex, ev, _ = hook(ld.noise_seed, epoch, i, 0, n, sx, sv)
        x, v, speed, targets = _noisy_fields(recipe, pos_t, vel_t, f, ld.delta_t, ex, ev, K)
        clean = fo.sample(recipe, pos_t, vel_t, static, f, ld.delta_t, radius, rate, world_size=P,
                          split_mode=ld.split_mode, generator=ld.sample_generator(i))[rank]
        ch = clean["index"]                                   # the split is the clean frame's
        lo, hi = ptr[b], ptr[b + 1]
        assert torch.equal(kwargs["node_loc"][lo:hi].cpu(), x[ch])
        assert torch.equal(kwargs["node_vel"][lo:hi].cpu(), v[ch])
        assert torch.equal(kwargs["node_attr"][lo:hi].cpu(), clean["attr"])
        assert torch.equal(extras["target"][lo:hi].cpu(), targets[0][ch])
        for t in range(K):
            assert torch.equal(extras["targets"][t, lo:hi].cpu(), targets[t][ch])
        assert torch.equal(kwargs["data_batch"][lo:hi].cpu(), torch.full((hi - lo,), b, dtype=torch.int64))
        feat = kwargs["node_feat"][lo:hi].cpu()
        sc = 2 if recipe == "largefluid" else 0
        assert _ulps(feat[:, sc], speed[ch]) <= 1
        other = [c for c in range(feat.shape[1]) if c != sc]
        if recipe == "largefluid":
            assert torch.equal(feat[:, other], clean["x"][:, other])
        else:                                                 # s / max s: as in test_frames' assembly test
            assert _ulps(feat[:, other], clean["x"][:, other]) <= 1
        whole = x.double().mean(0)
        lm = kwargs["loc_mean"][b].cpu().double()
        assert float((lm - whole).abs().max()) <= 1e-6 * max(float(whole.abs().max()), 1e-30)
        m = (row >= lo) & (row < hi)
        mine = _edge_set(torch.stack([row[m] - lo, col[m] - lo]))
        p = x[ch]
        ei = fo.complete_edges(p.shape[0]) if radius is None else fo.radius_edges(p, radius)
        if rate > 0:
            ei = fo.cutoff_edge(ei, p, rate)
        diff = mine ^ _edge_set(ei)
        if diff:
            d = torch.stack([(p[a] - p[c]).norm() for a, c in diff])
            if rate == 0:
                assert bool(((d.double() - radius).abs() <= _NEAR * radius).all()), "edges differ away from the radius"
            else:
                thr = (p[ei[0]] - p[ei[1]]).norm(dim=1).max()
                assert bool(((d - thr).abs() <= 1e-6 * thr).all()), f"{len(diff)} kept edges differ beyond ties"


@pytest.mark.gpu
@pytest.mark.parametrize("recipe,radius,rate,P,split", CASES)
def test_noisy_assembly_is_the_restated_rules_bit_for_bit(tmp_path, recipe, radius, rate, P, split):
    traj = _traj(tmp_path, recipe)
    dt = 2
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=dt, frames_per_scene=2, max_frame=3, frame_0=1)
    sig = (2e-3, 5e-2) if recipe != "nbody" else (2e-2, 5e-2)
    for rank in range(P):
        ld = FrameLoader(traj, samples, delta_t=dt, radius=radius, batch_size=2, shuffle=True, seed=5, device=_dev(),
                         world_size=P, rank=rank, split_mode=split, cutoff_rate=rate, horizon=2, noise=sig,
                         noise_seed=77)
        order = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=5)
        for epoch in range(2):                                # the second epoch checks the epoch number too
            n = 0
            for (kwargs, extras), idx in zip(ld, order.batches()):
                _check_noisy_batch(traj, ld, kwargs, extras, idx, epoch, recipe, radius, rate, P, rank)
                n += 1
            assert n == 2


def _all_nodes(ld, seed):
    """{(sample, scene node): (loc, vel, targets)} and {sample: loc_mean} over one epoch of `ld` (sampler seed `seed`)."""
    nodes, means = {}, {}
    for (kw, ex), idx in zip(ld, FrameLoader(ld.traj, ld.samples, batch_size=ld.batch_size, shuffle=ld.shuffle,
                                             seed=seed).batches()):
        ptr = ex["ptr"]
        for b, i in enumerate(idx):
            part, _ = ld.partition(i)
            ids = range(ptr[b + 1] - ptr[b]) if part is None else part.tolist()
            loc, vel = kw["node_loc"][ptr[b]:ptr[b + 1]].cpu(), kw["node_vel"][ptr[b]:ptr[b + 1]].cpu()
            tg = ex["targets"][:, ptr[b]:ptr[b + 1]].cpu()
            for r, j in enumerate(ids):
                nodes[(i, j)] = torch.cat([loc[r], vel[r], tg[:, r].reshape(-1)])
            means[i] = kw["loc_mean"][b].cpu()
    return nodes, means


@pytest.mark.gpu
def test_noise_is_a_function_of_seed_epoch_sample_and_node_only(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=1, max_samples=6, delta_t=1, frames_per_scene=2, max_frame=4)
    base = dict(delta_t=1, radius=0.2, device=_dev(), noise=(1e-2, 3e-2), noise_seed=5, horizon=2)
    runs = []
    for P, split, bs, shuffle in ((1, "random", 1, False), (2, "random", 2, True), (3, "random", 3, True),
                                  (2, "kmeans", 2, False)):
        nodes, means = {}, []
        for rank in range(P):
            ld = FrameLoader(traj, samples, batch_size=bs, shuffle=shuffle, seed=P, world_size=P, rank=rank,
                             split_mode=split, **base)
            got, m = _all_nodes(ld, P)
            nodes.update(got)
            means.append(m)
        for m in means[1:]:                                   # loc_mean: bitwise equal on every rank
            assert m.keys() == means[0].keys() and all(torch.equal(m[k], means[0][k]) for k in m)
        runs.append((nodes, means[0]))
    n0, m0 = runs[0]
    for nodes, means in runs[1:]:
        assert nodes.keys() == n0.keys()
        assert all(torch.equal(nodes[k], n0[k]) for k in nodes)
        assert all(torch.equal(means[k], m0[k]) for k in means)


def _launches(monkeypatch, ld):
    """(outputs of one epoch, names of the library calls it made)."""
    real = _lib.load()
    calls = []

    class Spy:
        def __getattr__(self, name):
            calls.append(name)
            return getattr(real, name)

    monkeypatch.setattr(_lib, "load", lambda: Spy())
    try:
        out = [(kw, ex) for kw, ex in ld]
        torch.cuda.synchronize()
    finally:
        monkeypatch.setattr(_lib, "load", lambda: real)
    return out, calls


def _same_outputs(a, b):
    for (ka, ea), (kb, eb) in zip(a, b):
        for k in ("node_feat", "node_loc", "node_vel", "loc_mean", "data_batch", "edge_attr", "node_attr"):
            assert torch.equal(ka[k], kb[k]), k
        assert torch.equal(ka["edge_index"].rowptr, kb["edge_index"].rowptr)
        assert torch.equal(ka["edge_index"].col, kb["edge_index"].col)
        assert torch.equal(ea["targets"], eb["targets"])


@pytest.mark.gpu
def test_zero_noise_is_no_noise(tmp_path, monkeypatch):
    traj = _traj(tmp_path, "largefluid")
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=1, frames_per_scene=2, max_frame=4)
    kw = dict(delta_t=1, radius=0.2, batch_size=2, shuffle=True, seed=3, device=_dev(), world_size=2, rank=1, horizon=3)
    clean, calls = _launches(monkeypatch, FrameLoader(traj, samples, **kw))
    for noise in (None, (0, 0), (0.0, 0.0)):
        out, c = _launches(monkeypatch, FrameLoader(traj, samples, noise=noise, **kw))
        assert c == calls
        _same_outputs(out, clean)
    assert "distegnn_frames_assemble_noise" not in calls
    # the entry point itself at σ = 0: the outputs of assemble + targets (a −0.0 coordinate may come back +0.0)
    ld = FrameLoader(traj, samples, **kw)
    host = ld._host_batch([2, 0])
    kc, ec = ld._to_device(host)
    ld.noise = (0.0, 0.0)
    host = ld._host_batch([2, 0])
    kn, en = ld._to_device(host)
    torch.cuda.synchronize()
    for k in ("node_feat", "node_loc", "node_vel", "loc_mean", "node_attr", "data_batch"):
        assert torch.equal(kn[k], kc[k]), k
    assert torch.equal(en["targets"], ec["targets"]) and torch.equal(en["scene_max"], ec["scene_max"])


@pytest.mark.gpu
def test_reproducible_across_loaders_epochs_streams_and_graph_replay(tmp_path):
    traj = _traj(tmp_path, "water3d", sizes=(400, 300))
    samples = sample_list(traj, seed=1, max_samples=2, delta_t=1, frames_per_scene=1, max_frame=4)
    kw = dict(delta_t=1, radius=0.2, batch_size=2, seed=3, device=_dev(), noise=(1e-3, 1e-3), noise_seed=11, horizon=2)
    a, b = FrameLoader(traj, samples, **kw), FrameLoader(traj, samples, **kw)
    ea = [list(a)[0][0]["node_loc"], list(a)[0][0]["node_loc"]]
    eb = [list(b)[0][0]["node_loc"], list(b)[0][0]["node_loc"]]
    assert torch.equal(ea[0], eb[0]) and torch.equal(ea[1], eb[1])
    clean = list(FrameLoader(traj, samples, **dict(kw, noise=None)))[0][0]["node_loc"]
    moved0, moved1 = (ea[0] - clean).abs().sum(1), (ea[1] - ea[0]).abs().sum(1)
    assert float((moved1 > 0).double().mean()) >= 0.999 and bool((moved0 > 0).all())
    # the entry point on a side stream and under CUDA-graph replay
    ld = FrameLoader(traj, samples, **kw)
    host = ld._host_batch([0, 1], epoch=4)
    ref = ld._to_device(host)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        on_side = ld._to_device(host)
    torch.cuda.synchronize()
    _same_outputs([on_side], [ref])
    B, M = 2, sum(host["node_counts"])
    dev = _dev()
    frames, statics, meta = (host[k].to(dev) for k in ("frames", "statics", "meta"))
    f32 = dict(dtype=torch.float32, device=dev)
    outs = dict(feat=torch.full((M, 2), -1.0, **f32), loc=torch.full((M, 3), -1.0, **f32),
                vel=torch.full((M, 3), -1.0, **f32), attr=torch.full((M, 1), -1.0, **f32),
                targets=torch.full((2, M, 3), -1.0, **f32), batch=torch.full((M,), -1, dtype=torch.int64, device=dev),
                loc_mean=torch.full((B, 3), -1.0, **f32), scene_max=torch.full((B,), -1.0, **f32))

    def call():
        p = lambda t: t.data_ptr()
        rc = _lib.load().distegnn_frames_assemble_noise(
            _lib.FRAMES_WATER3D, B, host["n_frame"], M, 2, p(frames), p(statics), p(meta[:B + 1]),
            p(meta[B + 1:2 * B + 2]), None, *(p(outs[k]) for k in ("feat", "loc", "vel", "attr", "targets", "batch",
                                                                   "loc_mean", "scene_max")),
            p(meta[2 * B + 2:]), 11, 4, 1e-3, 1e-3, torch.cuda.current_stream().cuda_stream)
        assert rc == 0
    call()
    torch.cuda.synchronize()
    for t in outs.values():
        t.fill_(-1)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            call()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    k0 = ref[0]
    assert torch.equal(outs["loc"], k0["node_loc"]) and torch.equal(outs["vel"], k0["node_vel"])
    assert torch.equal(outs["feat"], k0["node_feat"]) and torch.equal(outs["loc_mean"], k0["loc_mean"])
    assert torch.equal(outs["targets"], ref[1]["targets"]) and torch.equal(outs["batch"], k0["data_batch"])


@pytest.mark.gpu
def test_sample_id_outside_32_bits_gives_nan_in_that_sample_only(tmp_path):
    """The ids are device data, so the entry point cannot reject them without synchronising: an id outside [0, 2^32)
    makes every noisy value of its sample NaN and leaves the other samples and the noise-free fields alone."""
    traj = _traj(tmp_path, "largefluid", sizes=(40, 30))
    ld = FrameLoader(traj, [(0, 1), (1, 2)], delta_t=1, batch_size=2, device=_dev(), world_size=2, rank=0,
                     noise=(1e-2, 1e-2), horizon=2)
    host = ld._host_batch([0, 1], epoch=3)
    B, M, dev = 2, sum(host["node_counts"]), _dev()
    frames, statics, index = (host[k].to(dev) for k in ("frames", "statics", "index"))
    f32 = dict(dtype=torch.float32, device=dev)

    def run(ids):
        meta = host["meta"].clone()
        meta[2 * B + 2:] = torch.tensor(ids)
        meta = meta.to(dev)
        o = dict(feat=torch.empty(M, 3, **f32), loc=torch.empty(M, 3, **f32), vel=torch.empty(M, 3, **f32),
                 attr=torch.empty(M, 2, **f32), targets=torch.empty(2, M, 3, **f32),
                 batch=torch.empty(M, dtype=torch.int64, device=dev), loc_mean=torch.empty(B, 3, **f32),
                 scene_max=torch.empty(B, **f32))
        p = lambda t: t.data_ptr()
        rc = _lib.load().distegnn_frames_assemble_noise(
            _lib.FRAMES_LARGEFLUID, B, host["n_frame"], M, 2, p(frames), p(statics), p(meta[:B + 1]),
            p(meta[B + 1:2 * B + 2]), p(index), *(p(o[k]) for k in ("feat", "loc", "vel", "attr", "targets", "batch",
                                                                     "loc_mean", "scene_max")),
            p(meta[2 * B + 2:]), 5, 3, 1e-2, 1e-2, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _lib.load().distegnn_last_error()
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in o.items()}

    good = run([0, 1])
    c = host["node_counts"][0]
    for bad in (1 << 32, -1):
        out = run([bad, 1])
        for k in ("loc", "vel"):
            assert bool(out[k][:c].isnan().all()) and torch.equal(out[k][c:], good[k][c:]), (bad, k)
        assert bool(out["targets"][:, :c].isnan().all()) and torch.equal(out["targets"][:, c:], good["targets"][:, c:])
        assert bool(out["feat"][:c, 2].isnan().all()) and torch.equal(out["feat"][c:], good["feat"][c:])
        assert torch.equal(out["feat"][:, :2], good["feat"][:, :2])
        assert bool(out["loc_mean"][0].isnan().all()) and torch.equal(out["loc_mean"][1], good["loc_mean"][1])
        for k in ("attr", "batch", "scene_max"):
            assert torch.equal(out[k], good[k]), (bad, k)
    assert not any(bool(v.double().isnan().any()) for v in good.values())


@pytest.mark.gpu
def test_capacity_mode_epoch_with_noise_never_synchronises(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=0, max_samples=8, delta_t=1, frames_per_scene=2, max_frame=5)
    ld = FrameLoader(traj, samples, radius=0.2, batch_size=2, shuffle=True, device=_dev(), world_size=2, rank=1,
                     capacity=20000, cutoff_rate=0.5, noise=(1e-3, 1e-3), horizon=2)
    first = [kw["node_loc"].sum() for kw, _ in ld]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steady = [(kw["node_loc"] * 2).sum() for kw, _ in ld]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(first) == len(steady) == 4
    ld.check()


@pytest.mark.gpu
def test_main_trains_with_noise_and_rolls_out(tmp_path):
    import yaml
    for part, sizes, seed in (("train", [60, 50], 1), ("valid", [40], 3)):
        (tmp_path / part).mkdir()
        _fluid(tmp_path / part, sizes, seed=seed)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(inner_radius=0.3, max_samples=4, split_mode="random")
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--config_path", str(p), "--trajectory",
                        str(tmp_path), "--train_steps", "2", "--train_noise", "1e-3,1e-3", "--rollout_steps", "2",
                        "--rollout_tau", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "2 train steps on raw frames" in r.stdout, r.stdout
    mses = [float(line.rsplit("MSE", 1)[1].split()[0].rstrip(",")) for line in r.stdout.splitlines() if "MSE" in line]
    assert len(mses) == 4 and all(math.isfinite(v) for v in mses), r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("noise", [None, "1e-3,1e-3"])
def test_main_evaluates_on_the_train_split_when_valid_has_no_batch(tmp_path, noise):
    """A valid split with fewer samples than batch_size yields no batch (drop_last): the evaluation falls back to the
    train split, as without --train_noise, and with it on a loader without the noise."""
    import yaml
    for part, sizes, seed in (("train", [60, 50], 1), ("valid", [40], 3)):
        (tmp_path / part).mkdir()
        _fluid(tmp_path / part, sizes, seed=seed)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(inner_radius=0.3, max_samples=20, batch_size=18, split_mode="random")   # valid: 16 samples
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    extra = [] if noise is None else ["--train_noise", noise]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--config_path", str(p), "--trajectory",
                        str(tmp_path), "--train_steps", "1", *extra], capture_output=True, text=True, timeout=600,
                       cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    line = [ln for ln in r.stdout.splitlines() if "evaluation over" in ln]
    assert len(line) == 1 and "evaluation over 1 batches (train)" in line[0], r.stdout
    assert math.isfinite(float(line[0].rsplit("MSE", 1)[1])) and float(line[0].rsplit("MSE", 1)[1]) > 0, r.stdout
