"""Time the real<->virtual kernel alone (distegnn_virtual_layer_fwd) on the config-5 shapes of bench.py: 1M nodes, C = 8,
one graph, seeded inputs.

    python scripts/bench_virtual_kernel.py [--lib A.so [--lib B.so]] [--launches 60] [--out result.json]

Each launch is timed with CUDA events after a 256 MiB L2 flush, for both values of FLAG_LAST.  With two libraries the
launches alternate between them (A, B, A, B, ...), so that clock and neighbour changes hit both alike, and the outputs of
the two are compared.  TFLOP/s uses bench.py's logical FLOP count for the kernel, N·C·(3·2·64·64 + 2·2·64).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from distegnn_b200 import FastEGNN, _lib, synth  # noqa: E402
from distegnn_b200._lib import ptr  # noqa: E402
from oracle import fastegnn_oracle as orc  # noqa: E402

_i64, _i32, _u32, _vp = C.c_int64, C.c_int, C.c_uint, C.c_void_p


def load(path):
    lib = C.CDLL(path)
    fn = lib.distegnn_virtual_layer_fwd
    fn.argtypes = [_i64, _i32, _i32, _i32, _i32, _u32] + [_vp] * 10
    fn.restype = C.c_int
    return fn


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def virtual_kernel_flops(n_nodes: int, channels: int) -> int:
    """bench.py's logical FLOP of one real<->virtual launch."""
    return n_nodes * channels * (3 * 2 * 64 * 64 + 2 * 2 * 64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="library to time (repeat for two; default: the package's)")
    ap.add_argument("--launches", type=int, default=60, help="timed launches per library and FLAG_LAST value (>= 50)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    libs = args.lib or [_lib.LIB_PATH]
    fns = [load(p) for p in libs]
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")

    w = synth.WORKLOADS["synth1m"]
    host = synth.make_partitions(w, seed=0)[0]
    N = int(host["node_loc"].shape[0])
    Cn, A, B = w.virtual_channels, w.edge_attr_nf, 1
    sd = orc.init_state_dict(w.node_feat_nf, w.node_attr_nf, A, 64, Cn, 1, seed=0, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=w.node_feat_nf, node_attr_nf=w.node_attr_nf,
                 edge_attr_nf=A, virtual_channels=Cn, n_layers=1)
    m.load_state_dict(sd)
    lp = m.to(dev)._packed_params(dev)["layers"][0]
    g = torch.Generator().manual_seed(0)
    batch = torch.zeros(N, dtype=torch.int32, device=dev)
    x4 = torch.zeros(N, 4, device=dev)
    x4[:, :3] = host["node_loc"].to(dev)
    Hn = torch.randn(N, 64, generator=g).to(dev)
    Xv = (x4[:, :3].mean(0)[None, :, None] + torch.randn(B, 3, Cn, generator=g).to(dev))
    G = torch.randn(B, Cn, 64, generator=g).to(dev)
    K = 4 + 3 * Cn + 64 * Cn
    agg_v = [torch.zeros(N, 64, device=dev) for _ in fns]
    trans_v = [torch.zeros(N, 4, device=dev) for _ in fns]
    vsum = [torch.zeros(B, K, device=dev) for _ in fns]
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def launch(i, flags):
        rc = fns[i](N, B, A, Cn, w.node_attr_nf, flags, ptr(batch), ptr(x4), ptr(Hn), ptr(Xv), ptr(G), ptr(lp),
                    ptr(agg_v[i]), ptr(trans_v[i]), ptr(vsum[i]), stream)
        assert rc == 0, f"{libs[i]}: distegnn_virtual_layer_fwd returned {rc}"

    flops = virtual_kernel_flops(N, Cn)
    result = {"gpu": gpu_info(), "N": N, "C": Cn, "B": B, "flop_per_launch": flops, "launches": args.launches,
              "libs": libs, "flags": {}}
    for flags, name in ((0, "layer"), (_lib.FLAG_LAST, "last_layer")):
        for i in range(len(fns)):                                  # warm-up, then one clean run for the output check
            for _ in range(3):
                launch(i, flags)
            agg_v[i].zero_()
            trans_v[i].zero_()
            vsum[i].zero_()
            launch(i, flags)
        torch.cuda.synchronize()
        outs = [(agg_v[i].clone(), trans_v[i].clone(), vsum[i].clone()) for i in range(len(fns))]
        times = [[] for _ in fns]
        for _ in range(args.launches):
            for i in range(len(fns)):
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                launch(i, flags)
                e.record()
                times[i].append((s, e))
        torch.cuda.synchronize()
        entry = {}
        for i, p in enumerate(libs):
            ms = [s.elapsed_time(e) for s, e in times[i]]
            mean = statistics.fmean(ms)
            entry[p] = {"mean_ms": mean, "median_ms": statistics.median(ms), "stdev_ms": statistics.stdev(ms),
                        "min_ms": min(ms), "max_ms": max(ms), "TFLOPs": flops / (mean * 1e-3) / 1e12}
        if len(fns) == 2:
            diff = {}
            for k, nm in enumerate(("agg_v", "trans_v", "vsum")):
                if nm == "agg_v" and flags:
                    continue
                ref = outs[0][k]
                diff[nm] = float((outs[1][k] - ref).abs().max() / ref.abs().max())
            entry["output_rel_diff"] = diff
            entry["speedup"] = entry[libs[0]]["mean_ms"] / entry[libs[1]]["mean_ms"]
        result["flags"][name] = entry
    result["gpu_after"] = gpu_info()
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
