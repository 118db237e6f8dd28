"""Cost of the differentiable Chamfer distance (DESIGN §21) on one GPU.

    python scripts/bench_chamfer_grad.py [--calls 20] [--reps 3] [--noise 0.1] [--out result.json]

At BASELINE config 5 (synth1m: one 1M-node graph, r = 0.075) and at Fluid113K size (113,140 nodes), on two clouds:
  "noise":   the initial positions against themselves plus Gaussian noise of `--noise`·r per coordinate;
  "rollout": the final state of a 20-step random-weight rollout (as scripts/bench_rollout_chamfer.py) against its
             targets.
(1) CUDA-event times of `--calls` calls each of the rollout's evaluation (distegnn_rollout_chamfer), the forward with
    nearest ids (distegnn_chamfer_distance, alternated with the evaluation call) and the backward
    (distegnn_chamfer_distance_bwd, both gradients), and the workspace bytes of both.
(2) One differentiable_rollout step: the time of loss.backward() with an MSE loss against the record and with a Chamfer
    loss (host clock around a device synchronise), alternated `--reps` times.
Reports the card name and power limit read in the same run, medians with min and max.  Prints one JSON line; `--out` also
writes it to a file.
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

from distegnn_b200 import FastEGNN, chamfer_distance, differentiable_rollout, rollout, synth  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402


def stats(v):
    return dict(median=statistics.median(v), min=min(v), max=max(v))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def kernels(be, pred, tg, calls, dev):
    """(1) on one pair of clouds (one graph)."""
    N = int(pred.shape[0])
    counter = torch.zeros(8, dtype=torch.int32, device=dev)
    ev = torch.empty(1, 1, 2, dtype=torch.float64, device=dev)
    out = torch.empty(1, 2, dtype=torch.float64, device=dev)
    nearest = torch.empty(2 * N, dtype=torch.int32, device=dev)
    ws = be.rollout_chamfer_workspace(N, 1, dev)
    ws_b = be.chamfer_distance_bwd_workspace(N, dev)
    g = torch.ones(1, 2, dtype=torch.float64, device=dev)
    gp, gt = torch.empty_like(pred), torch.empty_like(tg)
    tg1 = tg[None].contiguous()
    run_ev = lambda: be.rollout_chamfer(pred, tg1, None, counter, ev, ws)
    run_fwd = lambda: be.chamfer_distance(pred, tg, None, out, nearest, ws)
    run_bwd = lambda: be.chamfer_distance_bwd(pred, tg, None, nearest, g, gp, gt, ws_b)
    for f in (run_ev, run_fwd, run_bwd):                       # warm-up
        f()
    torch.cuda.synchronize()
    t = dict(eval=[], forward=[], backward=[])
    for _ in range(calls):
        t["eval"].append(timed(run_ev))
        t["forward"].append(timed(run_fwd))
    for _ in range(calls):
        t["backward"].append(timed(run_bwd))
    same = bool(torch.equal(ev[0], out))
    outliers = float((nearest[:N].long() != torch.arange(N, device=dev)).float().mean())
    return dict(ms={k: stats(v) for k, v in t.items()}, sums_equal_eval=same, chamfer=out[0].tolist(),
                share_of_ids_not_the_matched_node=outliers, workspace_bytes=dict(forward=ws.numel(), backward=ws_b.numel()))


def one_size(name, n, steps, calls, reps, noise, dev):
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
    gen = torch.Generator(device=dev).manual_seed(0)
    targets = node["node_loc"] + 1e-3 * torch.randn(steps, N, 3, device=dev, generator=gen)
    res = rollout(model, **node, steps=steps, radius=w.radius, speed_col=0, targets=targets)
    be = model._get_backend(dev)
    x0 = node["node_loc"].contiguous()
    noisy = (x0 + noise * w.radius * torch.randn(N, 3, device=dev, generator=gen)).contiguous()
    out = dict(nodes=N, radius=w.radius, noise_of_r=noise,
               noise=kernels(be, x0, noisy, calls, dev),
               rollout=kernels(be, res.node_loc.contiguous(), targets[-1].contiguous(), calls, dev))
    # (2) one differentiable_rollout step: MSE against Chamfer
    cap = 2 * res.capacity
    model.train()
    batch, tg = node["data_batch"], targets[0]
    losses = dict(mse=lambda tr: ((tr[0] - tg) ** 2).mean(), chamfer=lambda tr: chamfer_distance(tr[0], tg, batch, 1).sum() / (3 * N))
    times = {k: [] for k in losses}
    for rep in range(reps + 1):                                # the first round warms up
        for k, f in losses.items():
            model.zero_grad(set_to_none=True)
            r = differentiable_rollout(model, **node, steps=1, radius=w.radius, speed_col=0, capacity=cap)
            loss = f(r.trajectory)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loss.backward()
            torch.cuda.synchronize()
            if rep:
                times[k].append((time.perf_counter() - t0) * 1e3)
    out["differentiable_rollout_step_backward_ms"] = {k: stats(v) for k, v in times.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--noise", type=float, default=0.1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), calls=args.calls, reps=args.reps)
    res["config5"] = one_size("synth1m", synth.WORKLOADS["synth1m"].n_nodes, args.steps, args.calls, args.reps,
                              args.noise, dev)
    res["fluid113k"] = one_size("fluid113k", 113_140, args.steps, args.calls, args.reps, args.noise, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
