"""The METIS partitioner (split_mode="metis", DESIGN §10) on one GPU and its host.

    python scripts/bench_metis.py [--reps 5] [--out profiles/metis_h100.json]

Clouds are synth's Water-3D-like 10k points (r = 0.035) and Fluid113K-like 113,140 points (r = 0.075), split into
P = 2, 4 and 8 parts with outer_radius = inner_radius = r, as the reference's configs do.  For each cloud:
(1) the device half between CUDA events: the outer-radius graph (`radius_graph_csr`, exact mode: it reads its edge
    count back once) plus the row sort (`csr_sorted_i64`), and the sort alone;
(2) for each P, the host METIS call (`metis_recursive`, wall clock) and the whole `metis_labels` (wall clock from a
    synchronised start to a synchronised end), medians of `--reps` with min–max;
(3) for each P, the edges of the radius graph each split mode keeps (both ends on one rank) out of all of them:
    random (synth's seeded randperm), kmeans, spectral and metis.
Reports the card name and power limit and the host CPU read in the same run.  Prints one JSON line and writes `--out`.
"""
from __future__ import annotations

import argparse
import json
import os
import platform
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from distegnn_b200 import kmeans_labels, metis_labels, radius_graph_csr, spectral_labels, synth  # noqa: E402
from distegnn_b200.partition import csr_sorted_i64, metis_recursive  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402


def stats(ts):
    return dict(median=float(np.median(ts)), min=float(np.min(ts)), max=float(np.max(ts)))


def cpu_name() -> str:
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor()


def events_ms(fn, reps):
    ts = []
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts[1:]                                                # the first call is the warm-up


def wall_s(fn, reps):
    fn()                                                         # warm-up
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return ts


def kept_edges(row, col, labels):
    """Undirected edges of the graph with both ends in one part."""
    return int((labels[row] == labels[col]).sum().item()) // 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "metis_h100.json"))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), cpu=cpu_name(),
               cpu_count=os.cpu_count(), reps=args.reps, clouds={})
    for name in ("water3d_10k", "fluid113k"):
        w = synth.WORKLOADS[name]
        n, r = w.n_nodes, w.radius
        pos_np = synth.make_points(w, seed=0)["pos"]
        pos = torch.from_numpy(pos_np).to(dev)
        g, _ = radius_graph_csr(pos, r, edge_attr_nf=0)
        E = g.num_edges
        row, col = g.rows().to(torch.int64), g.col.to(torch.int64)
        out = dict(nodes=n, radius=r, directed_edges=E,
                   graph_and_sort_ms=stats(events_ms(lambda: csr_sorted_i64(radius_graph_csr(pos, r, edge_attr_nf=0)[0]),
                                                     args.reps)),
                   sort_ms=stats(events_ms(lambda: csr_sorted_i64(g), args.reps)), parts={})
        xadj, adjncy = csr_sorted_i64(g)
        xadj_h, adj_h = xadj.cpu().numpy(), adjncy.cpu().numpy()
        for P in (2, 4, 8):
            host = wall_s(lambda: metis_recursive(xadj_h, adj_h, P), args.reps)
            total = wall_s(lambda: metis_labels(pos, P, r), args.reps)
            labels = dict(random=torch.empty(n, dtype=torch.int64),
                          kmeans=kmeans_labels(pos, P), spectral=spectral_labels(pos, P), metis=metis_labels(pos, P, r))
            for i, idx in enumerate(synth.random_partition(n, P, seed=0)):
                labels["random"][torch.from_numpy(idx)] = i
            kept = {k: kept_edges(row, col, v.to(dev)) for k, v in labels.items()}
            sizes = torch.bincount(labels["metis"], minlength=P)
            out["parts"][str(P)] = dict(metis_host_s=stats(host), metis_labels_s=stats(total),
                                        undirected_edges=E // 2, edges_kept=kept,
                                        metis_sizes=[int(sizes.min()), int(sizes.max())])
            print(name, P, out["parts"][str(P)], flush=True)
        print(name, {k: out[k] for k in ("graph_and_sort_ms", "sort_ms")}, flush=True)
        res["clouds"][name] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
