"""Cost of training through a K-step rollout (`differentiable_rollout`) at BASELINE config 5 (1M nodes, r = 0.075).

    python scripts/bench_rollout_grad.py [--nodes 1000000] [--steps 4 8] [--reps 3] [--out result.json]

For every K in `--steps`, ALTERNATING the Ks `--reps` times in one process: forward (`differentiable_rollout`) and
backward (`.backward()` of a loss on every step's positions and virtual coordinates), each timed with the host clock
around a device synchronise, reported per step; the peak of `max_memory_allocated` over forward + backward above what was
allocated before.  The backward's parts (graph rebuild, recomputed forward, advance backward, the model's backward
kernels, edge-length backward) come from CUDA events in the backward of each timed repetition.  Then, once per K, the same
for the hand-written loop (`model.input_grads = True`, `radius_graph_csr` per step, edge_attr and the advance in torch)
when it fits in memory.  Also one training step of the model alone, for its peak memory.  Reports the card name and power
limit read in the same run.  Prints one JSON line; `--out` also writes it to a file.
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

from distegnn_b200 import FastEGNN, differentiable_rollout, radius_graph_csr, synth  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=None, help="default: the full config-5 graph (synth1m)")
    ap.add_argument("--steps", type=int, nargs="+", default=[4, 8])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import importlib

    import bench
    R = importlib.import_module("distegnn_b200.rollout")        # the module (the package exports a function of that name)

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    w = synth.WORKLOADS["synth1m"]
    pts = synth.make_points(w, 0, args.nodes or w.n_nodes)
    N = int(pts["pos"].shape[0])
    model = FastEGNN(hidden_nf=64, world_size=1, **bench.model_dims(w))
    model.load_state_dict(bench.make_state_dict(w))
    model = model.to(dev).train()
    t = lambda a: torch.from_numpy(a).to(dev)
    node = dict(node_feat=t(pts["feat"]), node_loc=t(pts["pos"]), node_vel=t(pts["vel"]),
                loc_mean=t(pts["pos"].mean(axis=0, keepdims=True)), data_batch=torch.zeros(N, dtype=torch.int64, device=dev),
                node_attr=t(pts["attr"]) if pts["attr"].shape[1] else None)
    r = w.radius
    leaves = lambda: {k: (v.clone().requires_grad_(True) if (v is not None and v.is_floating_point()) else v)
                      for k, v in node.items()}

    def measured(fn):
        """(forward ms, backward ms, peak bytes above the start) of fn() -> loss."""
        model.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        loss = fn()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        loss.backward()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        peak = torch.cuda.max_memory_allocated() - base
        del loss
        return (t1 - t0) * 1e3, (t2 - t1) * 1e3, peak

    cap = {}

    def diff(K):
        def run():
            lf = leaves()
            res = differentiable_rollout(model, **lf, steps=K, radius=r, speed_col=0, capacity=cap.get("c"))
            cap["c"] = res.capacity
            return res.trajectory.square().mean() + res.virtual_locs.square().mean()
        return run

    def hand(K):
        def run():
            model.input_grads = True
            try:
                lf = leaves()
                x, v, f, lm = lf["node_loc"], lf["node_vel"], lf["node_feat"], lf["loc_mean"]
                loss = 0
                for _ in range(K):
                    g, _ = radius_graph_csr(x.detach(), r)
                    e = g.edge_index()
                    a = (x[e[0]] - x[e[1]]).norm(dim=1, keepdim=True).expand(-1, w.edge_attr_nf).contiguous()
                    out, X = model(f, x, v, lm, g, lf["data_batch"], a, lf["node_attr"])
                    loss = loss + out.square().mean() + X.square().mean()
                    v = out - x
                    f = torch.cat([v.norm(dim=1, keepdim=True), f[:, 1:]], 1)
                    lm = out.mean(0, keepdim=True)
                    x = out
                return loss
            finally:
                model.input_grads = False
        return run

    def one_step():
        g, ea = radius_graph_csr(node["node_loc"], r)
        out, X = model(node["node_feat"], node["node_loc"], node["node_vel"], node["loc_mean"], g, node["data_batch"], ea,
                       node["node_attr"])
        return out.square().mean() + X.square().mean()

    measured(one_step)                                          # warm-up
    step_fwd, step_bwd, step_peak = measured(one_step)
    for K in args.steps:                                        # warm-up of every shape
        measured(diff(K))
    times = {K: dict(fwd=[], bwd=[], peak=[]) for K in args.steps}
    parts = {K: {} for K in args.steps}
    for _ in range(args.reps):
        for K in args.steps:
            R._bwd_timing = marks = []
            fwd, bwd, peak = measured(diff(K))
            R._bwd_timing = None
            times[K]["fwd"].append(fwd / K)
            times[K]["bwd"].append(bwd / K)
            times[K]["peak"].append(peak)
            by_step = {}
            for s, name, ev in marks:
                by_step.setdefault(s, []).append((name, ev))
            for s, evs in by_step.items():
                for (name, a), (_, b) in zip(evs, evs[1:]):
                    parts[K].setdefault(name, []).append(a.elapsed_time(b))
    hand_res = {}
    for K in args.steps:
        try:
            measured(hand(K))                                   # warm-up
            fwd, bwd, peak = measured(hand(K))
            hand_res[K] = dict(fwd_ms_per_step=fwd / K, bwd_ms_per_step=bwd / K, peak_gb=peak / 2**30)
        except torch.cuda.OutOfMemoryError:
            hand_res[K] = "out of memory"
        model.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
    med = statistics.median
    out = dict(config="synth1m (BASELINE config 5)", nodes=N, radius=r, n_layers=model.n_layers, reps=args.reps,
               gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), capacity=cap.get("c"),
               one_training_step=dict(fwd_ms=step_fwd, bwd_ms=step_bwd, peak_gb=step_peak / 2**30),
               differentiable_rollout={K: dict(fwd_ms_per_step=dict(median=med(v["fwd"]), all=v["fwd"]),
                                               bwd_ms_per_step=dict(median=med(v["bwd"]), all=v["bwd"]),
                                               peak_gb=max(v["peak"]) / 2**30,
                                               bwd_part_ms_per_step={k: med(a) for k, a in parts[K].items()})
                                       for K, v in times.items()},
               hand_written_loop=hand_res)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
