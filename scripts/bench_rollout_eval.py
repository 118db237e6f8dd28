"""Cost of evaluating rollouts against recorded trajectories (DESIGN §19) on one GPU.

    python scripts/bench_rollout_eval.py [--steps 20] [--reps 3] [--out result.json]

(1) Rollout ms/step with and without `targets`, at BASELINE config 5 (synth1m: one 1M-node graph, r = 0.075) and at
    Fluid113K size (113,140 nodes), eager with a fixed capacity, the two runs ALTERNATING `--reps` times in one process
    (host clock around a device synchronise).
(2) The error kernel alone (distegnn_rollout_sq_err): CUDA events around each of `--steps` launches, and its share of a
    step without targets.
(3) FrameLoader batch time (staging + assembly + targets + graph, capacity mode) and the PCIe bytes staged per batch for
    horizon 1 against horizon K, on a random-walk Fluid113K scene.
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

from distegnn_b200 import FastEGNN, rollout, synth  # noqa: E402
from distegnn_b200.frames import FrameLoader, load_scenes  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402


def stats(v):
    return dict(median=statistics.median(v), min=min(v), max=max(v), all=v)


def rollout_size(name, n, K, reps, dev):
    import bench
    w = synth.WORKLOADS[name]
    pts = synth.make_points(w, 0, n)
    N = int(pts["pos"].shape[0])
    model = FastEGNN(hidden_nf=64, world_size=1, **bench.model_dims(w))
    model.load_state_dict(bench.make_state_dict(w))
    model = model.to(dev).eval()
    t = lambda a: torch.from_numpy(a).to(dev)
    node = dict(node_feat=t(pts["feat"]), node_loc=t(pts["pos"]), node_vel=t(pts["vel"]),
                loc_mean=t(pts["pos"].mean(axis=0, keepdims=True)), data_batch=torch.zeros(N, dtype=torch.int64, device=dev),
                node_attr=t(pts["attr"]) if pts["attr"].shape[1] else None)
    g = torch.Generator(device=dev).manual_seed(0)
    targets = node["node_loc"] + 1e-3 * torch.randn(K, N, 3, device=dev, generator=g)
    cap = rollout(model, **node, steps=K, radius=w.radius, speed_col=0).capacity      # warm-up, sizes the capacity
    runs = dict(plain=dict(), targets=dict(targets=targets))
    for kw in runs.values():
        rollout(model, **node, steps=K, radius=w.radius, speed_col=0, capacity=cap, **kw)
    times = {k: [] for k in runs}
    for _ in range(reps):
        for k, kw in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = rollout(model, **node, steps=K, radius=w.radius, speed_col=0, capacity=cap, **kw)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3 / K)
    mse = res.mse.tolist()
    # the error kernel alone, on the rollout's final state, every launch timed
    be = model._get_backend(dev)
    counter = torch.zeros(8, dtype=torch.int32, device=dev)
    sq = torch.zeros(K, 1, dtype=torch.float64, device=dev)
    ws = be.rollout_sq_err_workspace(N, dev)
    pred = res.node_loc
    be.rollout_sq_err(pred, targets, None, counter, sq, ws)
    kern = []
    for s in range(K):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        be.rollout_sq_err(pred, targets, None, counter, sq, ws)
        b.record()
        torch.cuda.synchronize()
        kern.append(a.elapsed_time(b))
    plain = statistics.median(times["plain"])
    return dict(nodes=N, radius=w.radius, steps=K, capacity=cap,
                ms_per_step={k: stats(v) for k, v in times.items()},
                sq_err_kernel_ms=stats(kern), sq_err_kernel_share_of_step=statistics.median(kern) / plain,
                step_overhead=statistics.median(times["targets"]) / plain - 1.0, mse_first_last=[mse[0], mse[-1]])


def loader_size(n, horizons, reps, tmp, dev):
    w = synth.WORKLOADS["fluid113k"]
    T = 2 + max(horizons)
    pts = synth.make_points(w, n, n)
    rng = np.random.default_rng(n)
    steps = rng.normal(0.0, 0.002, (T, n, 3))
    steps[0] = pts["pos"]
    path = os.path.join(tmp, f"scene_{n}.npz")
    np.savez(path, position=np.cumsum(steps, 0).astype(np.float32),
             velocity=rng.normal(0, 1, (T, n, 3)).astype(np.float32), viscosity=rng.random(n).astype(np.float32),
             mass=rng.random(n).astype(np.float32))
    traj = load_scenes([path], "largefluid")
    (kw, _), = list(FrameLoader(traj, [(0, 0)], radius=w.radius, device=dev))
    cap = int(1.25 * int(kw["edge_index"].rowptr[-1]))
    out = {}
    for K in horizons:
        ld = FrameLoader(traj, [(0, 0)], radius=w.radius, device=dev, prefetch=0, capacity=cap, horizon=K)
        times = []
        for _ in range(reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            (kw, ex), = list(ld)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        ld.check()
        host = ld._host_batch([0])
        staged = sum(v.numel() * v.element_size() for v in host.values() if isinstance(v, torch.Tensor))
        out[f"horizon_{K}"] = dict(batch_ms=stats(times[1:]), pcie_bytes=staged, frames_staged=int(host["frames"].shape[0]))
    return dict(nodes=n, capacity=cap, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), steps=args.steps, reps=args.reps)
    res["rollout_config5"] = rollout_size("synth1m", synth.WORKLOADS["synth1m"].n_nodes, args.steps, args.reps, dev)
    res["rollout_fluid113k"] = rollout_size("fluid113k", 113_140, args.steps, args.reps, dev)
    tmp = tempfile.mkdtemp(prefix="bench_rollout_eval_")
    try:
        res["frame_loader_fluid113k"] = loader_size(113_140, (1, 5, args.steps), 2 * args.reps + 1, tmp, dev)
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
