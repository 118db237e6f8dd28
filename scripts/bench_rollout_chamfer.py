"""Cost of the rollout's per-step Chamfer distance (DESIGN §20) on one GPU.

    python scripts/bench_rollout_chamfer.py [--steps 20] [--reps 3] [--out result.json]

(1) Rollout ms/step with `targets` alone and with `targets` and `chamfer=True`, at BASELINE config 5 (synth1m: one
    1M-node graph, r = 0.075) and at Fluid113K size (113,140 nodes): eager, a fixed capacity, the two runs ALTERNATING
    `--reps` times in one process (host clock around a device synchronise).
(2) The Chamfer launches alone (distegnn_rollout_chamfer, seven kernels and a cub scan): CUDA events around each of
    `--steps` calls on the rollout's final state against its targets, and their share of a step with targets alone.
Reports the card name and power limit read in the same run.  Prints one JSON line; `--out` also writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from distegnn_b200 import FastEGNN, rollout, synth  # noqa: E402
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
    runs = dict(targets=dict(targets=targets), chamfer=dict(targets=targets, chamfer=True))
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
    ch = res.chamfer_mse.tolist()
    mse = res.mse.tolist()
    # the Chamfer launches alone, on the rollout's final state, every call timed
    be = model._get_backend(dev)
    counter = torch.zeros(8, dtype=torch.int32, device=dev)
    out = torch.zeros(K, 1, 2, dtype=torch.float64, device=dev)
    ws = be.rollout_chamfer_workspace(N, 1, dev)
    pred = res.node_loc
    be.rollout_chamfer(pred, targets, None, counter, out, ws)
    kern = []
    for s in range(K):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        be.rollout_chamfer(pred, targets, None, counter, out, ws)
        b.record()
        torch.cuda.synchronize()
        kern.append(a.elapsed_time(b))
    base = statistics.median(times["targets"])
    return dict(nodes=N, radius=w.radius, steps=K, capacity=cap, workspace_bytes=ws.numel(),
                ms_per_step={k: stats(v) for k, v in times.items()},
                chamfer_ms=stats(kern), chamfer_share_of_step=statistics.median(kern) / base,
                step_overhead=statistics.median(times["chamfer"]) / base - 1.0,
                mse_first_last=[mse[0], mse[-1]], chamfer_mse_first_last=[ch[0], ch[-1]])


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
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
