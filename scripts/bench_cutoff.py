"""Cost of the edge cutoff (FastEGNN's cutoff_edges mode) and what it buys, on one GPU.

    python scripts/bench_cutoff.py [--nodes 1000000] [--reps 5] [--steps 10] [--out result.json]

(1) `cutoff_edges_csr` per call at BASELINE config 5 (1M nodes, r = 0.075, ~20.6M candidates) for rates 0.25 / 0.5 /
    0.75, next to the capacity-mode radius build it follows; and the same for the reference's N-body batch (250 fully
    connected 100-node graphs, 9,900 candidates each).  CUDA events around each call; the calls of one rep are
    ALTERNATED (radius build, then every rate) and every number is the median of `--reps` reps after a warm-up, with
    min and max.
(2) config 5: the inference forward and `rollout` ms/step with and without `cutoff_rate=0.5`, alternated.
(3) peak memory of a rollout step with and without the cutoff.
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

from distegnn_b200 import FastEGNN, cutoff_edges_csr, radius_graph_csr, rollout, synth  # noqa: E402
from distegnn_b200.partition import RadiusGraphBuffers  # noqa: E402
from distegnn_b200.shards import CSRGraph  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402

RATES = (0.25, 0.5, 0.75)


def stats(v):
    return dict(median=statistics.median(v), min=min(v), max=max(v))


def time_calls(calls, reps):
    """calls: name -> fn; each rep runs all of them once, in turn, each between two CUDA events."""
    for f in calls.values():
        f()
    out = {k: [] for k in calls}
    for _ in range(reps):
        for k, f in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            torch.cuda.synchronize()
            out[k].append(a.elapsed_time(b))
    return {k: stats(v) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=None, help="default: the full config-5 graph (synth1m)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bench

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), reps=args.reps)

    # ---- (1a) config 5: radius build and the cutoff that follows it ----
    w = synth.WORKLOADS["synth1m"]
    pts = synth.make_points(w, 0, args.nodes or w.n_nodes)
    N = int(pts["pos"].shape[0])
    t = lambda a: torch.from_numpy(a).to(dev)
    x = t(pts["pos"])
    g0, _ = radius_graph_csr(x, w.radius, edge_attr_nf=0)
    E = g0.num_edges
    cap = int(1.25 * E)
    cand = RadiusGraphBuffers(N, cap, 0, dev)
    outs = {r: RadiusGraphBuffers(N, cap, 2, dev) for r in RATES}
    calls = {"radius_build": lambda: radius_graph_csr(x, w.radius, edge_attr_nf=0, out=cand)}
    calls["radius_build"]()
    for r in RATES:
        calls[f"cutoff_{r}"] = (lambda r=r: cutoff_edges_csr(cand.graph, x, r, out=outs[r]))
    res["config5"] = dict(nodes=N, candidates=E, capacity=cap, ms=time_calls(calls, args.reps),
                          kept={str(r): int(outs[r].info[0]) for r in RATES})

    # ---- (1b) the reference N-body batch: 250 fully connected 100-node graphs ----
    B, n = 250, 100
    gen = torch.Generator().manual_seed(0)
    xp = torch.randn(B * n, 3, generator=gen).to(dev)
    i, j = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    keep = i != j
    ei = torch.cat([torch.stack([i[keep], j[keep]]) + n * b for b in range(B)], 1).to(dev)
    gb, _ = CSRGraph.from_edge_index(ei, B * n)
    batch = torch.arange(B, device=dev).repeat_interleave(n)
    nb_out = {r: RadiusGraphBuffers(B * n, gb.num_edges, 2, dev) for r in RATES}
    calls = {f"cutoff_{r}": (lambda r=r: cutoff_edges_csr(gb, xp, r, batch, B, out=nb_out[r])) for r in RATES}
    res["nbody250x100"] = dict(candidates=gb.num_edges, ms=time_calls(calls, args.reps))
    del cand, outs, nb_out

    # ---- (2) config 5 forward and rollout, with and without the cutoff ----
    model = FastEGNN(hidden_nf=64, world_size=1, **bench.model_dims(w))
    model.load_state_dict(bench.make_state_dict(w))
    model = model.to(dev).eval()
    node = dict(node_feat=t(pts["feat"]), node_loc=x, node_vel=t(pts["vel"]),
                loc_mean=t(pts["pos"].mean(axis=0, keepdims=True)), data_batch=torch.zeros(N, dtype=torch.int64, device=dev),
                node_attr=t(pts["attr"]) if pts["attr"].shape[1] else None)
    graphs = {0.0: radius_graph_csr(x, w.radius), 0.5: radius_graph_csr(x, w.radius, cutoff_rate=0.5)}

    def fwd(rate):
        g, ea = graphs[rate]
        with torch.no_grad():
            model(node["node_feat"], x, node["node_vel"], node["loc_mean"], g, node["data_batch"], ea, node["node_attr"])

    res["forward_ms"] = {str(k): v for k, v in time_calls({0.0: lambda: fwd(0.0), 0.5: lambda: fwd(0.5)},
                                                          args.reps).items()}
    res["forward_edges"] = {str(k): g.num_edges for k, (g, _) in graphs.items()}
    del graphs
    K = args.steps
    caps = {}

    def ro(rate):
        r = rollout(model, **node, steps=K, radius=w.radius, speed_col=0, capacity=caps.get(rate), cutoff_rate=rate)
        caps[rate] = r.capacity
        return r

    for rate in (0.0, 0.5):
        ro(rate)
    times, peaks = {0.0: [], 0.5: []}, {}
    for _ in range(max(1, args.reps // 2)):
        for rate in (0.0, 0.5):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            t0 = time.perf_counter()
            r = ro(rate)
            torch.cuda.synchronize()
            times[rate].append((time.perf_counter() - t0) * 1e3 / K)
            peaks[rate] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
            edges = r.n_edges.double().mean().item()
            res.setdefault("rollout_edges_per_step", {})[str(rate)] = edges
    res["rollout_ms_per_step"] = {str(k): stats(v) for k, v in times.items()}
    res["rollout_peak_gib"] = {str(k): v for k, v in peaks.items()}
    res["steps"] = K
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
