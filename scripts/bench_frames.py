"""Cost of building training batches from raw frames on the device (distegnn_b200.frames.FrameLoader), on one GPU.

    python scripts/bench_frames.py [--reps 10] [--steps 10] [--out result.json]

Sizes: a Fluid113K-sized scene (113,140 nodes, r = 0.075) at P = 1 and one rank's share at P = 2 (random split), and
config 5 (1M nodes, r = 0.075).  Scenes are seeded random walks around synth.make_points, written as .npz in the
loader's input layout to a temporary directory (Fluid113K recipe: position, velocity, viscosity, mass).

Per size:
(1) ms per batch (batch_size 1) of the loader with prefetch 0 — host staging from the memory-mapped scene, H2D,
    assembly, radius graph — in exact mode (counts read back) and capacity mode (no host synchronisation); wall clock
    around each batch after a device synchronise, median / min / max of `--reps` after a warm-up.  The assembly kernel
    alone and the graph build alone between CUDA events.
(2) PCIe bytes per batch from the shapes: the loader's staging (three frames of the whole scene, the static columns, the
    node index list at 4 B per node of this rank) against a shard of the same sample (node arrays, CSR, edge_attr).
(3) One training step (forward + fused loss + backward) fed by FrameLoader (prefetch 2) against one fed by ShardLoader
    (prefetch 2) over shards written from the loader's own batch: ms per step over `--steps` steps, after a warm-up epoch.
(4) Training noise (DESIGN §22, σ = NOISE): the batch time in capacity mode with noise, and the noisy assembly
    (distegnn_frames_assemble_noise, horizon 1) between CUDA events beside the assembly without noise.
Reports the card name and power limit read in the same run.  Prints one JSON line; `--out` also writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from distegnn_b200 import FastEGNN, synth, train_loss  # noqa: E402
from distegnn_b200.frames import FrameLoader, load_scenes  # noqa: E402
from distegnn_b200.loader import ShardLoader  # noqa: E402
from distegnn_b200.partition import radius_graph_csr  # noqa: E402
from distegnn_b200.shards import write_shard  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402

T_FRAMES = 4
NOISE = (3e-4, 3e-4)


def stats(v):
    return dict(median=statistics.median(v), min=min(v), max=max(v))


def write_scene(path, w, n, seed):
    pts = synth.make_points(w, seed, n)
    rng = np.random.default_rng(seed)
    steps = rng.normal(0.0, 0.002, (T_FRAMES, n, 3))
    steps[0] = pts["pos"]
    pos = np.cumsum(steps, 0).astype(np.float32)
    np.savez(path, position=pos, velocity=rng.normal(0, 1, (T_FRAMES, n, 3)).astype(np.float32),
             viscosity=rng.random(n).astype(np.float32), mass=rng.random(n).astype(np.float32))


def loader_batch_ms(make, reps):
    ld = make()
    times = []
    for _ in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        (kw, ex), = list(ld)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    ld.check()
    return stats(times[1:]), kw, ex


def event_ms(fn, reps):
    fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return stats(out)


def shard_arrays(kw, ex):
    g = kw["edge_index"]
    E = int(g.rowptr[-1])
    return dict(node_feat=kw["node_feat"].cpu().numpy(), node_loc=kw["node_loc"].cpu().numpy(),
                node_vel=kw["node_vel"].cpu().numpy(), loc_mean=kw["loc_mean"].cpu().numpy(),
                data_batch=kw["data_batch"].cpu().numpy().astype(np.int32), rowptr=g.rowptr.cpu().numpy(),
                col=g.col[:E].cpu().numpy(), edge_attr=kw["edge_attr"][:E].cpu().numpy(),
                node_attr=kw["node_attr"].cpu().numpy(), target=ex["target"].cpu().numpy())


def train_ms(model, loader, steps):
    model.train()
    times = []
    for epoch in range(2):                                       # the first epoch warms up
        it = iter(loader)
        for _ in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            kw, ex = next(it)
            model.zero_grad(set_to_none=True)
            pred, X = model(**kw)
            loss, _ = train_loss(pred, ex["target"], X, kw["data_batch"], world_size=1, loc_mean=kw["loc_mean"],
                                 node_counts=ex["node_counts"])
            loss.backward()
            torch.cuda.synchronize()
            if epoch:
                times.append((time.perf_counter() - t0) * 1e3)
        for _ in it:
            pass
    return stats(times)


def run_size(name, n, P, reps, steps, tmp, dev):
    w = synth.WORKLOADS["fluid113k"]
    path = os.path.join(tmp, f"{name}.npz")
    write_scene(path, w, n, seed=n)
    traj = load_scenes([path], "largefluid")
    one = [(0, 0)]
    kw_ = dict(delta_t=1, radius=w.radius, device=dev, prefetch=0, world_size=P, rank=0)
    exact, kw, ex = loader_batch_ms(lambda: FrameLoader(traj, one, **kw_), reps)
    M, E = kw["node_loc"].shape[0], int(kw["edge_index"].rowptr[-1])
    cap = int(1.25 * E)
    capm, _, _ = loader_batch_ms(lambda: FrameLoader(traj, one, capacity=cap, **kw_), reps)
    ld = FrameLoader(traj, one, capacity=cap, **kw_)
    host = ld._host_batch([0])
    host = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    from distegnn_b200 import _lib
    from distegnn_b200._lib import check, ptr
    f32 = dict(dtype=torch.float32, device=dev)
    outs = [torch.empty(M, 3, **f32), torch.empty(M, 3, **f32), torch.empty(M, 3, **f32), torch.empty(M, 2, **f32),
            torch.empty(M, 3, **f32), torch.empty(M, dtype=torch.int64, device=dev), torch.empty(1, 3, **f32),
            torch.empty(1, **f32)]
    feat, loc, vel, attr, target, batch, lm, smax = outs

    def assemble():
        check(_lib.load().distegnn_frames_assemble(
            _lib.FRAMES_LARGEFLUID, 1, n, M, ptr(host["frames"]), ptr(host["statics"]), ptr(host["meta"][:2]),
            ptr(host["meta"][2:]), ptr(host.get("index")), ptr(feat), ptr(loc), ptr(vel), ptr(attr), ptr(target),
            ptr(batch), ptr(lm), ptr(smax), _lib.stream_ptr(dev)), "frames_assemble")

    t_asm = event_ms(assemble, reps)
    noisy, _, _ = loader_batch_ms(lambda: FrameLoader(traj, one, capacity=cap, noise=NOISE, **kw_), reps)
    ids = torch.zeros(1, dtype=torch.int64, device=dev)

    def assemble_noise():
        check(_lib.load().distegnn_frames_assemble_noise(
            _lib.FRAMES_LARGEFLUID, 1, n, M, 1, ptr(host["frames"]), ptr(host["statics"]), ptr(host["meta"][:2]),
            ptr(host["meta"][2:]), ptr(host.get("index")), ptr(feat), ptr(loc), ptr(vel), ptr(attr), ptr(target),
            ptr(batch), ptr(lm), ptr(smax), ptr(ids), 0, 0, NOISE[0], NOISE[1], _lib.stream_ptr(dev)),
            "frames_assemble_noise")

    t_asm_noise = event_ms(assemble_noise, reps)
    t_graph = event_ms(lambda: radius_graph_csr(loc, w.radius, batch, capacity=cap, n_graphs=1), reps)
    staged = 3 * n * 3 * 4 + n * 2 * 4 + 4 * 8 + (4 * M if P > 1 else 0)
    arrays = shard_arrays(kw, ex)
    shard_bytes = sum(a.nbytes for a in arrays.values())
    # a training step fed by each loader (the shard holds this very batch)
    spath = os.path.join(tmp, f"{name}.shard")
    write_shard(spath, arrays)
    model = FastEGNN(node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2, hidden_nf=64, virtual_channels=w.virtual_channels,
                     world_size=1, n_layers=4).to(dev)
    t_frames = train_ms(model, FrameLoader(traj, one * steps, delta_t=1, radius=w.radius, device=dev, world_size=P,
                                           rank=0, capacity=cap), steps)
    t_shard = train_ms(model, ShardLoader([spath] * steps, device=dev), steps)
    return dict(nodes_scene=n, world_size=P, nodes_rank=M, edges=E, capacity=cap,
                batch_ms=dict(exact=exact, capacity=capm, capacity_noise=noisy), assembly_kernel_ms=t_asm,
                assembly_noise_kernel_ms=t_asm_noise, radius_graph_ms=t_graph,
                pcie_bytes=dict(frames=staged, shard=shard_bytes, ratio=staged / shard_bytes),
                train_step_ms=dict(frame_loader=t_frames, shard_loader=t_shard))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--sizes", default="fluid113k_p1,fluid113k_p2,config5")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sizes = dict(fluid113k_p1=(113_140, 1), fluid113k_p2=(113_140, 2), config5=(1_000_000, 1))
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), reps=args.reps, steps=args.steps,
               noise=NOISE)
    tmp = tempfile.mkdtemp(prefix="bench_frames_")
    try:
        for name in args.sizes.split(","):
            n, P = sizes[name]
            res[name] = run_size(name, n, P, args.reps, args.steps, tmp, dev)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
