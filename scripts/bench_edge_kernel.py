"""Time the edge kernel alone (distegnn_edge_layer_fwd) on the config-5 shapes of bench.py: 1M nodes, ~20.6M edges,
edge_attr_nf = 2, C = 8, the same seeded graph.

    python scripts/bench_edge_kernel.py [--lib A.so [--lib B.so]] [--launches 60] [--out result.json]

Each launch is timed with CUDA events after a 256 MiB L2 flush, for both values of FLAG_LAST.  With two libraries the
launches alternate between them (A, B, A, B, ...), so that clock and neighbour changes hit both alike, and the outputs of
the two are compared: the default mode's as a relative difference (float atomics add in arrival order), the
deterministic mode's (distegnn_edge_layer_fwd_det, then distegnn_edge_combine_det) bit for bit.  GB/s uses bench.py's
byte count for the kernel, E·284 + N·536, against the H100 SXM data-sheet HBM bandwidth of 3.35 TB/s.
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
from distegnn_b200.backend import CudaBackend  # noqa: E402
from oracle import fastegnn_oracle as orc  # noqa: E402

PEAK_GBS = 3350.0
_i64, _i32, _u32, _vp = C.c_int64, C.c_int, C.c_uint, C.c_void_p


def load(path):
    lib = C.CDLL(path)
    for name, argtypes in (("distegnn_edge_layer_fwd", [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 11),
                           ("distegnn_edge_layer_fwd_det", [_i64, _i64, _i32, _i32, _i32, _u32] + [_vp] * 11 + [_i64, _vp]),
                           ("distegnn_edge_combine_det", [_i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
                           ("distegnn_deterministic_workspace_bytes", [_i64, _i64, _i32, _vp])):
        getattr(lib, name).argtypes = argtypes
        getattr(lib, name).restype = C.c_int
    return lib


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="library to time (repeat for two; default: the package's)")
    ap.add_argument("--launches", type=int, default=60, help="timed launches per library and FLAG_LAST value (>= 50)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    libs = args.lib or [_lib.LIB_PATH]
    dets = [load(p) for p in libs]
    fns = [lib.distegnn_edge_layer_fwd for lib in dets]
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")

    w = synth.WORKLOADS["synth1m"]
    host = synth.make_partitions(w, seed=0)[0]
    N, E = int(host["node_loc"].shape[0]), int(host["edge_index"].shape[1])
    A = w.edge_attr_nf
    be = CudaBackend()
    ei = host["edge_index"].to(dev)
    rowptr, row, col, perm = be.build_csr(ei, N)
    ea = be.gather_rows(host["edge_attr"].to(dev), perm)
    sd = orc.init_state_dict(w.node_feat_nf, w.node_attr_nf, A, 64, w.virtual_channels, 1, seed=0, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=w.node_feat_nf, node_attr_nf=w.node_attr_nf,
                 edge_attr_nf=A, virtual_channels=w.virtual_channels, n_layers=1)
    m.load_state_dict(sd)
    lp = m.to(dev)._packed_params(dev)["layers"][0]
    g = torch.Generator().manual_seed(0)
    P, Q = torch.randn(N, 64, generator=g).to(dev), torch.randn(N, 64, generator=g).to(dev)
    x4 = torch.zeros(N, 4, device=dev)
    x4[:, :3] = host["node_loc"].to(dev)
    agg_m = [torch.zeros(N, 64, device=dev) for _ in fns]
    agg_x = [torch.zeros(N, 4, device=dev) for _ in fns]
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def launch(i, flags):
        rc = fns[i](N, E, A, w.virtual_channels, w.node_attr_nf, flags, ptr(row), ptr(col), ptr(ea), ptr(x4), ptr(P),
                    ptr(Q), ptr(lp), ptr(agg_m[i]), ptr(agg_x[i]), None, stream)
        assert rc == 0, f"{libs[i]}: distegnn_edge_layer_fwd returned {rc}"

    ws_bytes = C.c_int64(0)
    assert dets[0].distegnn_deterministic_workspace_bytes(N, E, w.virtual_channels, C.byref(ws_bytes)) == 0
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)

    def deterministic(i, flags):
        """One deterministic-mode edge stage (kernel, then combine) of library i: (agg_m or None, agg_x)."""
        m = None if flags & _lib.FLAG_LAST else torch.zeros(N, 64, device=dev)
        x = torch.zeros(N, 4, device=dev)
        lib = dets[i]
        rc = lib.distegnn_edge_layer_fwd_det(N, E, A, w.virtual_channels, w.node_attr_nf, flags, ptr(row), ptr(col),
                                             ptr(ea), ptr(x4), ptr(P), ptr(Q), ptr(lp), ptr(m), ptr(x), None, ptr(ws),
                                             ws.numel(), stream)
        assert rc == 0, f"{libs[i]}: distegnn_edge_layer_fwd_det returned {rc}"
        rc = lib.distegnn_edge_combine_det(N, E, w.virtual_channels, ptr(row), None, ptr(m), ptr(x), ptr(ws), ws.numel(),
                                           stream)
        assert rc == 0, f"{libs[i]}: distegnn_edge_combine_det returned {rc}"
        torch.cuda.synchronize()
        return m, x

    nbytes = E * 284 + N * 536
    result = {"gpu": gpu_info(), "N": N, "E": E, "A": A, "bytes_per_launch": nbytes, "peak_GBps": PEAK_GBS,
              "launches": args.launches, "libs": libs, "flags": {}}
    for flags, name in ((0, "layer"), (_lib.FLAG_LAST, "last_layer")):
        for i in range(len(fns)):                                  # warm-up, then one clean run for the output check
            for _ in range(3):
                launch(i, flags)
            agg_m[i].zero_()
            agg_x[i].zero_()
            launch(i, flags)
        torch.cuda.synchronize()
        outs = [(agg_m[i].clone(), agg_x[i].clone()) for i in range(len(fns))]
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
            entry[p] = {"mean_ms": mean, "median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms),
                        "stdev_ms": statistics.stdev(ms),
                        "GBps": nbytes / (mean * 1e-3) / 1e9, "frac_of_peak": nbytes / (mean * 1e-3) / 1e9 / PEAK_GBS}
        if len(fns) == 2:
            ref_m, ref_x = outs[0]
            entry["output_rel_diff"] = {
                "agg_x": float((outs[1][1] - ref_x).abs().max() / ref_x.abs().max()),
                "agg_m": None if flags else float((outs[1][0] - ref_m).abs().max() / ref_m.abs().max())}
            entry["speedup"] = entry[libs[0]]["mean_ms"] / entry[libs[1]]["mean_ms"]
            (m0, x0), (m1, x1) = deterministic(0, flags), deterministic(1, flags)
            entry["deterministic_bitwise_equal"] = {"agg_x": bool(torch.equal(x0, x1)),
                                                    "agg_m": None if flags else bool(torch.equal(m0, m1))}
        result["flags"][name] = entry
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
