"""Cost of a K-step rollout at BASELINE config 5 (1M nodes, r = 0.075) on one GPU.

    python scripts/bench_rollout.py [--nodes 1000000] [--steps 20] [--reps 3] [--out result.json]

Times three loops of `--steps` steps each, ALTERNATING them `--reps` times in one process, host clock around a device
synchronise:
  (a) hand-written: exact `radius_graph_csr` (one host read of the edge count per step), `model(...)`, torch advance;
  (b) `rollout` eager (capacity from step 0, one overflow check at the end);
  (c) `rollout` with `model.cuda_graph = True`.
Then, in a separate pass, CUDA events around the three parts of the rollout step (radius-graph build, forward, advance)
over `--steps` steps.  Reports the card name and power limit read in the same run.  Prints one JSON line; `--out` also
writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from distegnn_b200 import FastEGNN, radius_graph_csr, rollout, synth  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:                       # noqa: BLE001 — reported as unknown, the timing is still valid
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=None, help="default: the full config-5 graph (synth1m)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bench
    from distegnn_b200.rollout import _Rollout

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    w = synth.WORKLOADS["synth1m"]
    pts = synth.make_points(w, 0, args.nodes or w.n_nodes)
    N = int(pts["pos"].shape[0])
    model = FastEGNN(hidden_nf=64, world_size=1, **bench.model_dims(w))
    model.load_state_dict(bench.make_state_dict(w))
    model = model.to(dev).eval()
    t = lambda a: torch.from_numpy(a).to(dev)
    node = dict(node_feat=t(pts["feat"]), node_loc=t(pts["pos"]), node_vel=t(pts["vel"]),
                loc_mean=t(pts["pos"].mean(axis=0, keepdims=True)), data_batch=torch.zeros(N, dtype=torch.int64, device=dev),
                node_attr=t(pts["attr"]) if pts["attr"].shape[1] else None)
    K, r = args.steps, w.radius

    def hand():
        x, v, f, lm = node["node_loc"].clone(), node["node_vel"].clone(), node["node_feat"].clone(), node["loc_mean"]
        with torch.no_grad():
            for _ in range(K):
                g, ea = radius_graph_csr(x, r)
                out, _ = model(f, x, v, lm, g, node["data_batch"], ea, node["node_attr"])
                v = out - x
                f[:, 0] = v.norm(dim=1)
                lm = out.mean(0, keepdim=True)
                x = out
        return x

    cap = {}

    def eager():
        model.cuda_graph = False
        res = rollout(model, **node, steps=K, radius=r, speed_col=0, capacity=cap.get("c"))
        cap["c"] = res.capacity
        return res.node_loc

    def graphed():
        model.cuda_graph = True
        res = rollout(model, **node, steps=K, radius=r, speed_col=0, capacity=cap.get("c"))
        model.cuda_graph = False
        return res.node_loc

    loops = dict(hand=hand, eager=eager, graphed=graphed)
    outs = {k: f() for k, f in loops.items()}                  # warm-up of every shape
    times = {k: [] for k in loops}
    for _ in range(args.reps):
        for k, f in loops.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outs[k] = f()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3 / K)
    diff = {k: float((outs[k] - outs["hand"]).abs().max()) for k in ("eager", "graphed")}

    # per-component times of the rollout step (CUDA events, eager)
    be = model._get_backend(dev)
    with torch.no_grad():
        ro = _Rollout(model, be, dev, node["node_feat"], node["node_loc"], node["node_vel"], node["loc_mean"],
                      node["data_batch"], node["node_attr"], steps=K, radius=r, graph=None, loop=False, tau=1.0,
                      speed_col=0, cutoff_rate=0.0)
        ro.set_capacity(cap["c"])
        comp = {"graph_build": [], "forward": [], "advance": []}
        for s in range(K):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            ro.graph_at(ro.loc)
            ev[1].record()
            model._forward(be, ro.pk, ro.dims, ro.model_args(ro.feat, ro.loc, ro.vel), ro.ws, init_centroid=s > 0)
            ev[2].record()
            be.rollout_advance(0, 1.0, ro.ws["out"], ro.loc, ro.vel, ro.feat, None, ro.edge_count, ro.overflow,
                               ro.n_edges, ro.counter)
            ev[3].record()
            torch.cuda.synchronize()
            for i, k in enumerate(comp):
                comp[k].append(ev[i].elapsed_time(ev[i + 1]))
        n_edges = ro.n_edges.tolist()
    med = lambda a: statistics.median(a)
    res = dict(config="synth1m (BASELINE config 5)", nodes=N, radius=r, steps=K, reps=args.reps,
               gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), capacity=cap["c"],
               edges_per_step=dict(first=n_edges[0], last=n_edges[-1], mean=sum(n_edges) / len(n_edges)),
               ms_per_step={k: dict(median=med(v), all=v) for k, v in times.items()},
               component_ms={k: dict(median=med(v), min=min(v), max=max(v)) for k, v in comp.items()},
               max_abs_vs_hand_written=diff)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
