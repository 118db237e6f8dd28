"""Rotated and translated evaluation splits in FrameLoader (DESIGN §23): the transform's generator against an independent
numpy Philox4x32-10 and a float64 restatement, its distribution (Haar rotations, Gaussian translations), the transformed
assembly restated bit for bit from the testing hook's R and t, its invariance to how the samples are split and batched,
the model's equivariance on a Fluid113K-sized scene, and `main.py --eval_rotate / --eval_translate`."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from distegnn_b200 import _lib
from distegnn_b200.frames import FrameLoader, sample_list
from oracle import frames_oracle as fo
from tests.test_frames import _NEAR, _edge_set, _fluid, _scene_tensors, _traj, _ulps
from tests.test_frames_noise import _all_nodes, _launches, _same_outputs, philox4x32_10, uniforms
from tests.test_rollout_eval import _nbody, _water

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = (1 << 64) - 1


# ---- numpy oracle of the transform ------------------------------------------------------------------------------------
def transform_words(seed, samples, q):
    """The four Philox words of counter (0, q, sample, 0) under `seed` (frames_transform.cuh), uint32 [n, 4]."""
    samples = np.asarray(samples, np.uint64)
    z = np.zeros(samples.shape, np.uint32)
    ctr = np.stack([z, np.full(samples.shape, q, np.uint32), samples.astype(np.uint32), z], -1)
    return philox4x32_10(ctr, [seed & 0xFFFFFFFF, seed >> 32])


def normals64(o):
    """float64 Box–Muller of the fp32 uniforms of words o [..., 4]: four normals [..., 4] and each one's radius."""
    u = uniforms(o).astype(np.float64)
    r01, r23 = np.sqrt(-2 * np.log(u[..., 0])), np.sqrt(-2 * np.log(u[..., 2]))
    z = np.stack([r01 * np.cos(2 * np.pi * u[..., 1]), r01 * np.sin(2 * np.pi * u[..., 1]),
                  r23 * np.cos(2 * np.pi * u[..., 3]), r23 * np.sin(2 * np.pi * u[..., 3])], -1)
    return z, np.stack([r01, r01, r23, r23], -1)


def rotation64(o):
    """float64 R [..., 3, 3] of the unit quaternion of the rotation counter's words."""
    q, _ = normals64(o)
    w, x, y, z = np.moveaxis(q / np.linalg.norm(q, axis=-1, keepdims=True), -1, 0)
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def rigid(R, t, x, position):
    """((R_a0·x0 + R_a1·x1) + R_a2·x2) (+ t_a) in fp32, one rounding per operation: the kernels' expression."""
    o = [(R[a, 0] * x[:, 0] + R[a, 1] * x[:, 1]) + R[a, 2] * x[:, 2] for a in range(3)]
    if position:
        o = [o[a] + t[a] for a in range(3)]
    return torch.stack(o, 1)


# ---- host side (no GPU) ---------------------------------------------------------------------------------------------
def test_loader_rejects_bad_transform_arguments(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = [(0, 0), (1, 1)]
    for bad in (-1.0, float("nan"), float("inf"), "1", None, (1.0,), True):
        with pytest.raises(ValueError, match="translate"):
            FrameLoader(traj, samples, translate=bad)
    for bad in (1, 0, "yes", None):
        with pytest.raises(ValueError, match="rotate"):
            FrameLoader(traj, samples, rotate=bad)
    for seed in (-1, 1 << 64):
        with pytest.raises(ValueError, match="transform_seed"):
            FrameLoader(traj, samples, rotate=True, transform_seed=seed)
    with pytest.raises(ValueError, match="cannot be combined"):
        FrameLoader(traj, samples, rotate=True, noise=(1e-3, 1e-3))
    with pytest.raises(ValueError, match="cannot be combined"):
        FrameLoader(traj, samples, translate=0.5, noise=(1e-3, 0))
    assert FrameLoader(traj, samples).transform is None
    assert FrameLoader(traj, samples, rotate=False, translate=0).transform is None
    assert FrameLoader(traj, samples, rotate=False, translate=0.0, noise=(1e-3, 1e-3)).noise == (1e-3, 1e-3)
    ld = FrameLoader(traj, samples, rotate=np.bool_(True), translate=np.float32(0.5), seed=9)
    assert ld.transform == (True, 0.5) and ld.transform_seed == 9
    assert FrameLoader(traj, samples, translate=2, transform_seed=U64).transform == (False, 2.0)
    FrameLoader(traj, samples, seed=-1)                      # a seed the transform cannot use is fine without one
    with pytest.raises(ValueError, match="transform_seed"):
        FrameLoader(traj, samples, seed=-1, rotate=True)
    host = FrameLoader(traj, samples, rotate=True)._host_batch([1, 0])
    assert host["meta"][-2:].tolist() == [1, 0]              # the sample ids ride in the pinned meta block


def _transform_call(**over):
    a = dict(recipe=_lib.FRAMES_WATER3D, B=1, n_frame=0, n_out=0, K=1, ptrs=[None] * 5, outs=[None] * 6 + [1, 1],
             ids=1, seed=0, rotate=1, translate=0.0)
    a.update(over)
    return _lib.load().distegnn_frames_assemble_transform(a["recipe"], a["B"], a["n_frame"], a["n_out"], a["K"],
                                                          *a["ptrs"], *a["outs"], a["ids"], a["seed"], a["rotate"],
                                                          a["translate"], None)


def _hook_fn():
    t = C.CDLL(os.path.join(os.path.dirname(_lib.LIB_PATH), "libdistegnn_b200_testing.so"))
    f = t.distegnn_testing_frames_transform
    f.argtypes = [C.c_uint64, C.c_int64, C.c_int64, C.c_int, C.c_float] + [C.c_void_p] * 4
    return f


def test_c_abi_rejects_bad_transform_arguments_before_launching():
    lib = _lib.load()
    # valid apart from the argument under test, with sizes that launch nothing but the (deviceless) scene kernel: every
    # rejection below returns before that launch
    cases = [(dict(translate=-1.0), b"translate"), (dict(translate=float("nan")), b"translate"),
             (dict(translate=float("inf")), b"translate"), (dict(rotate=2), b"rotate"), (dict(rotate=-1), b"rotate"),
             (dict(K=0), b"horizon"), (dict(ids=None), b"sample_ids"), (dict(recipe=7), b"unknown recipe"),
             (dict(B=0), b"bad size"), (dict(n_out=3), b"n_out == n_frame_nodes"),
             (dict(outs=[None] * 8), b"null pointer")]
    for over, msg in cases:
        assert _transform_call(**over) == -1, over
        err = lib.distegnn_last_error()
        assert msg in err and err.startswith(b"distegnn_frames_assemble_transform"), (over, err)
    f = _hook_fn()
    assert f(0, 1 << 32, 1, 1, 0.0, None, None, None, None) == -1
    assert f(0, -1, 1, 1, 0.0, None, None, None, None) == -1
    assert f(0, (1 << 32) - 1, 2, 1, 0.0, None, None, None, None) == -1
    assert f(0, 0, 1, 2, 0.0, None, None, None, None) == -1
    assert f(0, 0, 1, 1, -1.0, None, None, None, None) == -1
    assert f(0, 0, 1, 1, float("nan"), None, None, None, None) == -1
    assert f(0, 0, 0, 1, 1.0, None, None, None, None) == 0          # nothing to do


def _main(args, timeout=600):
    return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), *args], capture_output=True, text=True,
                          timeout=timeout, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))


def test_main_rejects_bad_eval_transform_before_cuda_work(tmp_path):
    cfg = os.path.join(ROOT, "config", "largefluid_distegnn.yaml")
    for bad, msg in (("a", "a number"), ("-1", "finite and >= 0"), ("nan", "finite and >= 0"),
                     ("inf", "finite and >= 0")):
        r = _main(["--config_path", cfg, "--trajectory", str(tmp_path), "--eval_rotate", f"--eval_translate={bad}"])
        assert r.returncode == 2 and f"--eval_translate {bad!r}: must be {msg}" in r.stdout, (bad, r.stdout, r.stderr)
        assert "CUDA" not in r.stderr
    r = _main(["--config_path", cfg, "--eval_rotate"])
    assert r.returncode == 2 and "--eval_rotate: must be used with --trajectory" in r.stdout, r.stdout
    r = _main(["--config_path", cfg, "--eval_translate", "1"])
    assert r.returncode == 2 and "used with --trajectory" in r.stdout, r.stdout


# ---- on the device ------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def hook(seed, first, n, rotate=True, translate=1.0, raw=False):
    """(R [n,3,3], t [n,3], raw words [n,2,4] or None) of sample ids first .. first + n − 1 from the testing library."""
    f = _hook_fn()
    R = torch.empty(n, 3, 3, device=_dev())
    t = torch.empty(n, 3, device=_dev())
    w = torch.empty(n, 2, 4, dtype=torch.int32, device=_dev()) if raw else None
    rc = f(seed, first, n, int(rotate), translate, R.data_ptr(), t.data_ptr(), w.data_ptr() if raw else None,
           torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.load().distegnn_last_error()
    torch.cuda.synchronize()
    return R.cpu(), t.cpu(), None if w is None else w.cpu().numpy().view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("seed,first", [(0, 0), (0x0123456789ABCDEF, 1 << 31), (U64, (1 << 32) - (1 << 16))])
def test_generator_equals_numpy_philox_and_float64_rotation(seed, first):
    n, tr = 1 << 16, 0.75
    R, t, w = hook(seed, first, n, translate=tr, raw=True)
    ids = np.arange(first, first + n, dtype=np.uint64)
    for q, k in ((2, 0), (3, 1)):
        assert np.array_equal(w[:, k], transform_words(seed, ids, q)), f"counter q={q}: raw words differ"
    Rd = R.double().numpy()
    eye = np.eye(3)
    assert np.abs(np.einsum("nji,njk->nik", Rd, Rd) - eye).max() <= 1e-6                  # orthonormal
    assert np.abs(np.linalg.det(Rd) - 1).max() <= 1e-6                                    # a rotation, not a reflection
    want = rotation64(w[:, 0])
    err = np.abs(Rd - want) / np.spacing(np.float32(1))                                    # ulps of the matrix's scale
    assert err.max() <= 4, f"R: worst {err.max():.2f} ulps"
    z, r = normals64(w[:, 1])
    ulp = np.spacing((np.float32(tr) * r[:, :3]).astype(np.float32)).astype(np.float64)
    err = np.abs(t.double().numpy() - np.float32(tr) * z[:, :3]) / ulp
    assert err.max() <= 4, f"t: worst {err.max():.2f} ulps"
    R0, t0, _ = hook(seed, first, 4, rotate=False, translate=0.0)                        # rotate=False: the identity
    assert torch.equal(R0, torch.eye(3).expand(4, 3, 3)) and bool((t0 == 0).all())


@pytest.mark.gpu
def test_rotations_are_haar_and_translations_gaussian():
    from scipy import stats
    n, tr = 1 << 16, 2.5
    R, t, _ = hook(987654321, 0, n, translate=tr)
    Rd = R.double().numpy()
    cos = np.clip((np.trace(Rd, axis1=1, axis2=2) - 1) / 2, -1, 1)
    theta = np.arccos(cos)
    assert stats.kstest(theta, lambda x: (x - np.sin(x)) / np.pi).pvalue > 1e-4           # density (1 − cos θ)/π
    bound = 5 / math.sqrt(n)
    assert np.abs(Rd.mean(0)).max() <= bound                                               # E[R] = 0
    assert np.abs((Rd ** 2).mean(0) - 1 / 3).max() <= 0.01                                 # every entry: variance 1/3
    z = t.double().numpy() / tr
    assert np.abs(z.mean(0)).max() <= bound and np.abs(z.var(0) - 1).max() <= 0.02
    for d in range(3):
        assert stats.kstest(z[:, d], "norm").pvalue > 1e-4
    c = np.corrcoef(np.concatenate([z, Rd.reshape(n, 9)], 1).T)                            # t independent of R
    assert np.abs(c[:3, 3:]).max() <= bound


def _transformed_fields(recipe, pos_t, vel_t, f, dt, R, t, K=1):
    """The assembly's transformed fields over the whole scene, restated on the CPU with the fp32 rules of DESIGN §23."""
    x = rigid(R, t, pos_t[f], True)
    v = rigid(R, t, pos_t[f + 1], True) - x if recipe == "water3d" else rigid(R, t, vel_t[f], False)
    speed = torch.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    targets = torch.stack([rigid(R, t, pos_t[f + k * dt], True) for k in range(1, K + 1)])
    return x, v, speed, targets


def _check_transformed_batch(traj, ld, kwargs, extras, idx, recipe, radius, rate, P, rank):
    from distegnn_b200 import cutoff_edges_csr, radius_graph_csr
    from distegnn_b200.shards import CSRGraph
    dev = _dev()
    g, ea = kwargs["edge_index"], kwargs["edge_attr"]
    loc, batch, B = kwargs["node_loc"], kwargs["data_batch"], len(idx)
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
    rotate, tr = ld.transform
    for b, i in enumerate(idx):
        s, f = ld.samples[i]
        pos_t, vel_t, static = _scene_tensors(traj, s)
        R, t, _ = hook(ld.transform_seed, i, 1, rotate, tr)
        x, v, speed, targets = _transformed_fields(recipe, pos_t, vel_t, f, ld.delta_t, R[0], t[0], K)
        plain = fo.sample(recipe, pos_t, vel_t, static, f, ld.delta_t, radius, rate, world_size=P,
                          split_mode=ld.split_mode, generator=ld.sample_generator(i))[rank]
        ch = plain["index"]                                   # the split is the untransformed frame's
        lo, hi = ptr[b], ptr[b + 1]
        assert torch.equal(kwargs["node_loc"][lo:hi].cpu(), x[ch])
        assert torch.equal(kwargs["node_vel"][lo:hi].cpu(), v[ch])
        assert torch.equal(kwargs["node_attr"][lo:hi].cpu(), plain["attr"])
        assert torch.equal(extras["target"][lo:hi].cpu(), targets[0][ch])
        for k in range(K):
            assert torch.equal(extras["targets"][k, lo:hi].cpu(), targets[k][ch])
        assert torch.equal(kwargs["data_batch"][lo:hi].cpu(), torch.full((hi - lo,), b, dtype=torch.int64))
        feat = kwargs["node_feat"][lo:hi].cpu()
        sc = 2 if recipe == "largefluid" else 0
        assert _ulps(feat[:, sc], speed[ch]) <= 1
        other = [c for c in range(feat.shape[1]) if c != sc]
        if recipe == "largefluid":
            assert torch.equal(feat[:, other], plain["x"][:, other])
        else:                                                 # s / max s: as in test_frames' assembly test
            assert _ulps(feat[:, other], plain["x"][:, other]) <= 1
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


# (recipe, radius, cutoff rate, world size, split, horizon, rotate, translate)
XF_CASES = [("nbody", None, 0.0, 1, "random", 3, True, 0.5), ("nbody", 0.6, 0.3, 1, "random", 1, True, 2.0),
            ("water3d", 0.2, 0.5, 1, "random", 3, True, 0.5), ("water3d", 0.2, 0.0, 2, "random", 1, True, 0.0),
            ("water3d", 0.25, 0.0, 2, "kmeans", 3, False, 1.5),
            ("largefluid", 0.2, 0.0, 1, "random", 1, True, 0.5), ("largefluid", 0.2, 0.0, 2, "random", 3, True, 3.0),
            ("largefluid", 0.25, 0.0, 2, "kmeans", 1, True, 0.5)]


@pytest.mark.gpu
@pytest.mark.parametrize("recipe,radius,rate,P,split,K,rotate,translate", XF_CASES)
def test_transformed_assembly_is_the_restated_rules_bit_for_bit(tmp_path, recipe, radius, rate, P, split, K, rotate,
                                                                translate):
    traj = _traj(tmp_path, recipe)
    dt = 1
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=dt, frames_per_scene=2, max_frame=3, frame_0=1)
    for rank in range(P):
        ld = FrameLoader(traj, samples, delta_t=dt, radius=radius, batch_size=2, shuffle=True, seed=5, device=_dev(),
                         world_size=P, rank=rank, split_mode=split, cutoff_rate=rate, horizon=K, rotate=rotate,
                         translate=translate, transform_seed=77)
        order = FrameLoader(traj, samples, batch_size=2, shuffle=True, seed=5)
        n = 0
        for (kwargs, extras), idx in zip(ld, order.batches()):
            _check_transformed_batch(traj, ld, kwargs, extras, idx, recipe, radius, rate, P, rank)
            n += 1
        assert n == 2


@pytest.mark.gpu
def test_transform_is_a_function_of_seed_and_sample_only(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=1, max_samples=6, delta_t=1, frames_per_scene=2, max_frame=4)
    base = dict(delta_t=1, radius=0.2, device=_dev(), rotate=True, translate=0.7, transform_seed=5, horizon=2)
    runs = []
    for P, split, bs, shuffle in ((1, "random", 1, False), (2, "random", 2, True), (3, "random", 3, True),
                                  (2, "kmeans", 2, False)):
        nodes, means = {}, []
        for rank in range(P):
            ld = FrameLoader(traj, samples, batch_size=bs, shuffle=shuffle, seed=P, world_size=P, rank=rank,
                             split_mode=split, **base)
            for epoch in range(2):                            # the transform does not depend on the epoch
                got, m = _all_nodes(ld, P) if epoch == 0 else _all_nodes_epoch1(ld, P)
                if epoch == 0:
                    first, first_m = got, m
                else:
                    assert got.keys() == first.keys() and all(torch.equal(got[k], first[k]) for k in got)
                    assert all(torch.equal(m[k], first_m[k]) for k in m)
            nodes.update(first)
            means.append(first_m)
        for m in means[1:]:                                   # loc_mean: bitwise equal on every rank
            assert m.keys() == means[0].keys() and all(torch.equal(m[k], means[0][k]) for k in m)
        runs.append((nodes, means[0]))
    n0, m0 = runs[0]
    for nodes, means in runs[1:]:
        assert nodes.keys() == n0.keys()
        assert all(torch.equal(nodes[k], n0[k]) for k in nodes)
        assert all(torch.equal(means[k], m0[k]) for k in means)


def _all_nodes_epoch1(ld, seed):
    """_all_nodes of the loader's second epoch: the order is that of a sampler that has drawn one epoch already."""
    order = FrameLoader(ld.traj, ld.samples, batch_size=ld.batch_size, shuffle=ld.shuffle, seed=seed)
    order.batches()
    nodes, means = {}, {}
    for (kw, ex), idx in zip(ld, order.batches()):
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
def test_no_transform_is_todays_loader(tmp_path, monkeypatch):
    traj = _traj(tmp_path, "largefluid")
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=1, frames_per_scene=2, max_frame=4)
    kw = dict(delta_t=1, radius=0.2, batch_size=2, shuffle=True, seed=3, device=_dev(), world_size=2, rank=1, horizon=3)
    plain, calls = _launches(monkeypatch, FrameLoader(traj, samples, **kw))
    for rotate, translate in ((False, 0), (False, 0.0)):
        out, c = _launches(monkeypatch, FrameLoader(traj, samples, rotate=rotate, translate=translate, **kw))
        assert c == calls
        _same_outputs(out, plain)
    assert "distegnn_frames_assemble_transform" not in calls
    out, c = _launches(monkeypatch, FrameLoader(traj, samples, rotate=True, **kw))
    assert "distegnn_frames_assemble_transform" in c and "distegnn_frames_assemble" not in c


@pytest.mark.gpu
def test_reproducible_across_loaders_streams_and_graph_replay(tmp_path):
    traj = _traj(tmp_path, "water3d", sizes=(400, 300))
    samples = sample_list(traj, seed=1, max_samples=2, delta_t=1, frames_per_scene=1, max_frame=4)
    kw = dict(delta_t=1, radius=0.2, batch_size=2, seed=3, device=_dev(), rotate=True, translate=1.0,
              transform_seed=11, horizon=2)
    a, b = FrameLoader(traj, samples, **kw), FrameLoader(traj, samples, **kw)
    ea = [list(a)[0][0]["node_loc"], list(a)[0][0]["node_loc"]]
    eb = [list(b)[0][0]["node_loc"], list(b)[0][0]["node_loc"]]
    assert torch.equal(ea[0], eb[0]) and torch.equal(ea[1], eb[1]) and torch.equal(ea[0], ea[1])
    ld = FrameLoader(traj, samples, **kw)
    host = ld._host_batch([0, 1])
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
        rc = _lib.load().distegnn_frames_assemble_transform(
            _lib.FRAMES_WATER3D, B, host["n_frame"], M, 2, p(frames), p(statics), p(meta[:B + 1]),
            p(meta[B + 1:2 * B + 2]), None, *(p(outs[k]) for k in ("feat", "loc", "vel", "attr", "targets", "batch",
                                                                   "loc_mean", "scene_max")),
            p(meta[2 * B + 2:]), 11, 1, 1.0, torch.cuda.current_stream().cuda_stream)
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
    traj = _traj(tmp_path, "largefluid", sizes=(40, 30))
    ld = FrameLoader(traj, [(0, 1), (1, 2)], delta_t=1, batch_size=2, device=_dev(), world_size=2, rank=0,
                     rotate=True, translate=1.0, horizon=2)
    host = ld._host_batch([0, 1])
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
        rc = _lib.load().distegnn_frames_assemble_transform(
            _lib.FRAMES_LARGEFLUID, B, host["n_frame"], M, 2, p(frames), p(statics), p(meta[:B + 1]),
            p(meta[B + 1:2 * B + 2]), p(index), *(p(o[k]) for k in ("feat", "loc", "vel", "attr", "targets", "batch",
                                                                     "loc_mean", "scene_max")),
            p(meta[2 * B + 2:]), 5, 1, 1.0, torch.cuda.current_stream().cuda_stream)
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
        assert bool(out["loc_mean"][0].isnan().all()) and torch.equal(out["loc_mean"][1], good["loc_mean"][1])
        for k in ("attr", "batch", "scene_max"):
            assert torch.equal(out[k], good[k]), (bad, k)
    assert not any(bool(v.double().isnan().any()) for v in good.values())


@pytest.mark.gpu
def test_capacity_mode_epoch_with_transform_never_synchronises(tmp_path):
    traj = _traj(tmp_path, "water3d")
    samples = sample_list(traj, seed=0, max_samples=8, delta_t=1, frames_per_scene=2, max_frame=5)
    ld = FrameLoader(traj, samples, radius=0.2, batch_size=2, shuffle=True, device=_dev(), world_size=2, rank=1,
                     capacity=20000, cutoff_rate=0.5, rotate=True, translate=1.0, horizon=2)
    first = [kw["node_loc"].sum() for kw, _ in ld]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steady = [(kw["node_loc"] * 2).sum() for kw, _ in ld]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(first) == len(steady) == 4
    ld.check()


# ---- equivariance at Fluid113K size -----------------------------------------------------------------------------------
def equivariance_at_scale(tmp, dev, scales=(0.0, 1.0, 10.0), seed=0):
    """A randomly initialised FastEGNN (C = 8) on the 113,140-node random-walk scene of scripts/bench_frames.py, plain
    and with the loader's rigid transform at translations of `scales` scene extents.  The transformed forward runs on the
    plain batch's graph (edge_attr from the transformed positions), so both see the same edges.  Returns per scale the
    residuals |pred' − (R·pred + t)| and |X' − (R·X + t)|, the gate 1e-4·max(1, displacement scale), the edges that
    differ between the plain and the transformed radius graph with their largest float64 distance from r (relative to
    r), and the fp32 spacing of the largest transformed coordinate (the rounding of x' moves lengths by about that)."""
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    from bench_frames import write_scene
    from distegnn_b200 import FastEGNN, synth
    from distegnn_b200.frames import load_scenes
    from distegnn_b200._lib import check, ptr
    w = synth.WORKLOADS["fluid113k"]
    n = w.n_nodes
    path = os.path.join(tmp, "equivariance.npz")
    write_scene(path, w, n, seed=n)
    traj = load_scenes([path], "largefluid")
    pos0 = np.array(traj.scenes[0].position[0], dtype=np.float64)
    extent = float((pos0.max(0) - pos0.min(0)).max())
    torch.manual_seed(seed)
    model = FastEGNN(node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2, hidden_nf=64, virtual_channels=8, world_size=1,
                     n_layers=4).to(dev)
    kw = dict(delta_t=1, radius=w.radius, device=dev)
    (kp, _), = list(FrameLoader(traj, [(0, 0)], **kw))
    with torch.no_grad():
        pred, X = model(**kp)
    disp = float((pred - kp["node_loc"]).abs().max())
    gate = 1e-4 * max(1.0, disp)
    g = kp["edge_index"]
    E = int(g.rowptr[-1])
    rows32 = g.rows()[:E].contiguous()
    rows, cols = rows32.long().cpu().numpy(), g.col[:E].long().cpu().numpy()
    plain_keys = rows * n + cols
    out = dict(nodes=n, edges=E, radius=w.radius, extent=extent, displacement_scale=disp, gate=gate, scales={})
    for s in scales:
        (kt, _), = list(FrameLoader(traj, [(0, 0)], rotate=True, translate=s * extent, **kw))
        R, t, _ = hook(0, 0, 1, True, s * extent)
        Rd, td = R[0].to(dev), t[0].to(dev)
        ea = torch.empty(E, 2, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(_lib.load().distegnn_edge_lengths_csr(E, 2, ptr(rows32), ptr(g.col), ptr(kt["node_loc"]), None,
                                                        ptr(ea), _lib.stream_ptr(dev)), "edge_lengths_csr")
        with torch.no_grad():
            pred_t, X_t = model(**dict(kt, edge_index=g, edge_attr=ea))
        res = float((pred_t - (pred @ Rd.T + td)).abs().max())
        res_x = float((X_t.permute(0, 2, 1) - (X.permute(0, 2, 1) @ Rd.T + td)).abs().max())
        gt = kt["edge_index"]
        Et = int(gt.rowptr[-1])
        tkeys = gt.rows()[:Et].long().cpu().numpy() * n + gt.col[:Et].long().cpu().numpy()
        flipped = np.setxor1d(plain_keys, tkeys)
        a, c = flipped // n, flipped % n
        dist = np.sqrt(((pos0[a] - pos0[c]) ** 2).sum(1)) if flipped.size else np.zeros(0)
        coord = float(kt["node_loc"].abs().max())
        out["scales"][str(s)] = dict(translate=s * extent, residual=res, residual_virtual=res_x, max_coordinate=coord,
                                     coordinate_spacing=float(np.spacing(np.float32(coord))),
                                     passes=res <= gate and res_x <= gate, flipped_edges=int(flipped.size),
                                     flipped_max_rel_from_r=float(np.abs(dist - w.radius).max() / w.radius)
                                     if flipped.size else 0.0)
    return out


@pytest.mark.gpu
def test_model_is_equivariant_on_a_fluid113k_scene(tmp_path):
    """The gate holds at 0, 1 and 10 scene extents.  Edges flip between the plain and the transformed graph only at the
    boundary: within 1e-5·r of r up to 1 extent; at 10 extents the coordinates reach ~27, whose fp32 spacing (1.9e-6)
    is already 2.5e-5·r, so there the bound is four spacings of the largest transformed coordinate."""
    res = equivariance_at_scale(str(tmp_path), _dev())
    print(res)
    r_ = res["radius"]
    for s, r in res["scales"].items():
        band = 1e-5 if s in ("0.0", "1.0") else 4 * r["coordinate_spacing"] / r_
        assert r["flipped_max_rel_from_r"] <= band, (s, r)    # flipped edges only at the boundary
    assert res["displacement_scale"] > 1e-4                   # the model really moves the particles
    for s, r in res["scales"].items():
        assert r["residual"] <= res["gate"] and r["residual_virtual"] <= res["gate"], (s, r, res["gate"])


# ---- main.py end to end ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_main_evaluates_plain_and_transformed_splits(tmp_path):
    import yaml

    def run(cfg, data, *extra):
        p = tmp_path / "cfg.yaml"
        with open(p, "w") as f:
            yaml.safe_dump(cfg, f)
        return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--config_path", str(p), "--trajectory",
                               str(data), "--train_steps", "1", "--eval_rotate", "--eval_translate", "0.5",
                               "--rollout_steps", "3", *extra], capture_output=True, text=True, timeout=600, cwd=ROOT)

    def check_out(r, batches):
        assert r.returncode == 0, r.stderr[-3000:]
        out = r.stdout
        assert f"evaluation over {batches} batches (valid): mean MSE" in out, out
        line = [ln for ln in out.splitlines() if "(valid, rotated and translated by 0.5): mean MSE" in ln]
        assert len(line) == 1 and "relative difference" in line[0], out
        assert math.isfinite(float(line[0].rsplit("relative difference", 1)[1]))
        assert f"rollout evaluation over {batches} batches (valid), 3 steps" in out, out
        assert f"rollout evaluation over {batches} batches (valid, rotated and translated by 0.5), 3 steps" in out, out
        for t in (1, 2, 3):
            assert f"rollout step {t}: MSE" in out and f"rollout step {t} (rotated and translated by 0.5): MSE" in out

    data = tmp_path / "water"
    for part, sizes, seed in (("train", [60, 50], 1), ("valid", [40, 45], 3)):
        (data / part).mkdir(parents=True)
        _water(data / part, sizes, T=10, seed=seed)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"].update(node_feat_nf=2, node_attr_nf=1)
    cfg["data"].update(dataset_name="Water3D", inner_radius=0.3, max_samples=4, split_mode="random", delta_t=2)
    check_out(run(cfg, data, "--rollout_chamfer"), 4)
    data = tmp_path / "nbody"
    _nbody(data, "train", S=4, T=10)
    _nbody(data, "valid", S=2, T=10, seed=5)
    with open(os.path.join(ROOT, "config", "nbody_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(batch_size=2, frame_0=1, frame_T=3, cutoff_rate=0.5)
    check_out(run(cfg, data, "--rollout_tau", "0.5"), 1)
