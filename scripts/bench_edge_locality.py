"""Time the edge kernel (distegnn_edge_layer_fwd) at config 5 (synth1m: 1M nodes, ~20.6M edges, C = 8, the seeded graph of
bench.py) on two row orders of the same graph: id order (distegnn_build_csr) and the cell order the model caches
(distegnn_build_csr_cells, DESIGN §3).

    python scripts/bench_edge_locality.py [--launches 60] [--out result.json]

Each launch is timed with CUDA events after a 256 MiB L2 flush; the two orders alternate launch by launch, for both
values of FLAG_LAST, so that clock and neighbour changes hit both alike.  The outputs of the two orders are compared.
The GPU name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from distegnn_b200 import FastEGNN, _lib, synth  # noqa: E402
from distegnn_b200.backend import CudaBackend  # noqa: E402
from oracle import fastegnn_oracle as orc  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60, help="timed launches per order and FLAG_LAST value")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")

    w = synth.WORKLOADS["synth1m"]
    host = synth.make_partitions(w, seed=0)[0]
    N, E = int(host["node_loc"].shape[0]), int(host["edge_index"].shape[1])
    A = w.edge_attr_nf
    be = CudaBackend()
    ei = host["edge_index"].to(dev)
    pos = host["node_loc"].to(dev)
    orders = {"id": be.build_csr(ei, N), "cell": be.build_csr_cells(ei, N, pos, None, 1)}
    ea_dev = host["edge_attr"].to(dev)
    graphs = {k: (row, col, be.gather_rows(ea_dev, perm)) for k, (_, row, col, perm) in orders.items()}
    sd = orc.init_state_dict(w.node_feat_nf, w.node_attr_nf, A, 64, w.virtual_channels, 1, seed=0, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=w.node_feat_nf, node_attr_nf=w.node_attr_nf,
                 edge_attr_nf=A, virtual_channels=w.virtual_channels, n_layers=1)
    m.load_state_dict(sd)
    lp = m.to(dev)._packed_params(dev)["layers"][0]
    g = torch.Generator().manual_seed(0)
    P, Q = torch.randn(N, 64, generator=g).to(dev), torch.randn(N, 64, generator=g).to(dev)
    x4 = torch.zeros(N, 4, device=dev)
    x4[:, :3] = pos
    agg_m = {k: torch.zeros(N, 64, device=dev) for k in graphs}
    agg_x = {k: torch.zeros(N, 4, device=dev) for k in graphs}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def launch(k, flags):
        row, col, ea = graphs[k]
        be.edge_layer((N, E, A, w.virtual_channels, w.node_attr_nf), flags, row, col, ea, x4, P, Q, lp, agg_m[k],
                      agg_x[k])

    result = {"gpu_before": gpu_info(), "N": N, "E": E, "A": A, "launches": args.launches, "flags": {}}
    for flags, name in ((0, "layer"), (_lib.FLAG_LAST, "last_layer")):
        for k in graphs:                                           # warm-up, then one clean run for the output check
            for _ in range(3):
                launch(k, flags)
            agg_m[k].zero_()
            agg_x[k].zero_()
            launch(k, flags)
        torch.cuda.synchronize()
        outs = {k: (agg_m[k].clone(), agg_x[k].clone()) for k in graphs}
        times = {k: [] for k in graphs}
        for _ in range(args.launches):
            for k in graphs:
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                launch(k, flags)
                e.record()
                times[k].append((s, e))
        torch.cuda.synchronize()
        entry = {}
        for k in graphs:
            ms = [s.elapsed_time(e) for s, e in times[k]]
            entry[k] = {"mean_ms": statistics.fmean(ms), "median_ms": statistics.median(ms), "min_ms": min(ms),
                        "max_ms": max(ms), "stdev_ms": statistics.stdev(ms)}
        entry["speedup_mean"] = entry["id"]["mean_ms"] / entry["cell"]["mean_ms"]
        ref_m, ref_x = outs["id"]
        entry["cell_vs_id_rel_diff"] = {
            "agg_x": float((outs["cell"][1] - ref_x).abs().max() / ref_x.abs().max()),
            "agg_m": None if flags else float((outs["cell"][0] - ref_m).abs().max() / ref_m.abs().max())}
        result["flags"][name] = entry
    result["gpu_after"] = gpu_info()
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
