"""Time the node-stage kernels alone (distegnn_node_layer_fwd and distegnn_embed_fwd) on the config-5 shapes of bench.py:
1M nodes, C = 8, Na = 2, F = 3, one graph, seeded inputs.

    python scripts/bench_node_kernel.py [--lib A.so [--lib B.so]] [--launches 60] [--out result.json]

Three launches are timed, each alone:
  layer       distegnn_node_layer_fwd with FLAG_ZERO_AGG (as FastEGNN's layer loop passes it) and a separate next-layer
              parameter block
  last_layer  the same with FLAG_LAST
  embed       distegnn_embed_fwd
h' and x' are written out of place, so the inputs stay the same from launch to launch.  Before each timed launch agg_m and
agg_x are restored from saved copies (the kernel clears them) and a 256 MiB buffer is cleared to flush L2; neither is inside
the CUDA events.  With two libraries the launches alternate between them (A, B, A, B, ...), so that clock and neighbour
changes hit both alike, and every output of the two is compared row by row.  GB/s uses the bytes each launch must move at
the least (node_bytes / embed_bytes below).
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

HBM_TBPS = 3.35        # H100 SXM data-sheet HBM3 bandwidth


def load(path):
    lib = C.CDLL(path)
    fns = {}
    for name in ("distegnn_node_layer_fwd", "distegnn_embed_fwd"):
        fn = getattr(lib, name)
        fn.argtypes = _lib.SIGNATURES[name]
        fn.restype = C.c_int
        fns[name] = fn
    return fns


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def node_bytes(n_nodes: int, Na: int, last: bool) -> int:
    """Least HBM traffic of one node-layer launch: every input row read once, every output row written once (int32 ids)."""
    rows64, rows4 = 64 * 4, 4 * 4
    if last:
        reads = rows64 + 3 * rows4 + 12 + 8 + 4                 # h | x4, agg_x, trans_v | vel | rowptr | batch
        writes = rows4 + 12 + rows4                             # x4' | loc | zeroed agg_x
    else:
        reads = 3 * rows64 + 3 * rows4 + 12 + 4 * Na + 8 + 4    # h, agg_m, agg_v | x4, agg_x, trans_v | vel | attr | ...
        writes = 4 * rows64 + rows64 + rows4 + rows4            # h', P, Q, Hn | zeroed agg_m | x4' | zeroed agg_x
    return n_nodes * (reads + writes)


def embed_bytes(n_nodes: int, F: int) -> int:
    reads = 4 * F + 12 + 8                                      # feat | loc | int64 data_batch
    writes = 4 * 64 * 4 + 16 + 4                                # h, P, Q, Hn | x4 | batch32
    return n_nodes * (reads + writes)


def rowwise_rel_diff(ref: torch.Tensor, out: torch.Tensor) -> float:
    """max over rows of max|out - ref| / max|ref| of the row (0 where both rows are all zero)."""
    ref, out = ref.double().reshape(ref.shape[0], -1), out.double().reshape(out.shape[0], -1)
    d = (out - ref).abs().amax(1)
    s = ref.abs().amax(1)
    rel = torch.where(d == 0, torch.zeros_like(d), d / s.clamp_min(1e-300))
    return float(rel.max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="library to time (repeat for two; default: the package's)")
    ap.add_argument("--launches", type=int, default=60, help="timed launches per library and kernel (>= 50)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert args.launches >= 50, "take at least 50 launches"
    libs = args.lib or [_lib.LIB_PATH]
    fns = [load(p) for p in libs]
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    info_before = gpu_info()

    w = synth.WORKLOADS["synth1m"]
    N, F, Na, A, Cn, B = w.n_nodes, w.node_feat_nf, w.node_attr_nf, w.edge_attr_nf, w.virtual_channels, 1
    sd = orc.init_state_dict(F, Na, A, 64, Cn, 2, seed=0, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=Cn,
                 n_layers=2).to(dev)
    m.load_state_dict(sd)
    layers = m._packed_params(dev)["layers"]
    lp, lp_next = layers[0], layers[1]
    emb_wt = m.embedding_in.weight.detach().t().contiguous()
    emb_b = m.embedding_in.bias.detach().contiguous()

    g = torch.Generator().manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g).to(dev)  # noqa: E731
    deg = torch.randint(10, 32, (N,), generator=g, dtype=torch.int32)          # mean 20.5: 20.5M edges
    rowptr = torch.cat([torch.zeros(1, dtype=torch.int32), deg.cumsum(0, dtype=torch.int32)]).to(dev)
    batch32 = torch.zeros(N, dtype=torch.int32, device=dev)
    batch64 = torch.zeros(N, dtype=torch.int64, device=dev)
    h = rn(N, 64)
    x4 = torch.zeros(N, 4, device=dev)
    x4[:, :3] = rn(N, 3)
    vel, attr, feat, loc = rn(N, 3), rn(N, Na), rn(N, F), rn(N, 3)
    agg_m0, agg_v = rn(N, 64) * 20.0, rn(N, 64) * 0.3
    agg_x0, trans_v = torch.zeros(N, 4, device=dev), torch.zeros(N, 4, device=dev)
    agg_x0[:, :3] = rn(N, 3) * 0.1
    trans_v[:, :3] = rn(N, 3) * 0.01
    agg_m, agg_x = agg_m0.clone(), agg_x0.clone()
    K = 4 + 3 * Cn + 64 * Cn
    mk = lambda *s: [torch.zeros(*s, device=dev) for _ in fns]  # noqa: E731
    h_out, x4_out, P, Q, Hn, loc_out, vsum = mk(N, 64), mk(N, 4), mk(N, 64), mk(N, 64), mk(N, 64), mk(N, 3), mk(B, K)
    b32_out = [torch.zeros(N, dtype=torch.int32, device=dev) for _ in fns]
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def launch(i, kind):
        if kind == "embed":
            rc = fns[i]["distegnn_embed_fwd"](N, B, F, A, Cn, Na, ptr(feat), ptr(loc), ptr(batch64), ptr(emb_wt),
                                              ptr(emb_b), ptr(lp), ptr(h_out[i]), ptr(x4_out[i]), ptr(b32_out[i]),
                                              ptr(P[i]), ptr(Q[i]), ptr(Hn[i]), ptr(vsum[i]), None, stream)
        else:
            last = kind == "last_layer"
            flags = _lib.FLAG_ZERO_AGG | (_lib.FLAG_LAST if last else 0)
            nl = (lambda t: None if last else t)
            rc = fns[i]["distegnn_node_layer_fwd"](
                N, B, A, Cn, Na, flags, ptr(rowptr), ptr(batch32), ptr(h), ptr(x4), ptr(vel), ptr(attr), ptr(nl(agg_m)),
                ptr(agg_x), ptr(nl(agg_v)), ptr(trans_v), ptr(lp), ptr(nl(lp_next)), ptr(nl(h_out[i])), ptr(x4_out[i]),
                ptr(nl(P[i])), ptr(nl(Q[i])), ptr(nl(Hn[i])), ptr(loc_out[i]) if last else None, ptr(vsum[i]), stream)
        assert rc == 0, f"{libs[i]}: {kind} returned {rc}"

    def restore():
        agg_m.copy_(agg_m0)
        agg_x.copy_(agg_x0)

    outputs = {"layer": ("h_out", "x4_out", "P", "Q", "Hn", "vsum"), "last_layer": ("x4_out", "loc_out", "vsum"),
               "embed": ("h", "x4", "batch32", "P", "Q", "Hn", "vsum")}
    bufs = {"h_out": h_out, "h": h_out, "x4_out": x4_out, "x4": x4_out, "P": P, "Q": Q, "Hn": Hn, "loc_out": loc_out,
            "vsum": vsum, "batch32": b32_out}
    nbytes = {"layer": node_bytes(N, Na, False), "last_layer": node_bytes(N, Na, True), "embed": embed_bytes(N, F)}
    result = {"gpu": info_before, "N": N, "C": Cn, "Na": Na, "F": F, "B": B, "launches": args.launches, "libs": libs,
              "kernels": {}}
    for kind in ("layer", "last_layer", "embed"):
        for i in range(len(fns)):                                  # warm-up, then one clean run for the output check
            for _ in range(3):
                restore()
                launch(i, kind)
            for t in (h_out[i], x4_out[i], P[i], Q[i], Hn[i], loc_out[i], vsum[i], b32_out[i]):
                t.zero_()
            restore()
            launch(i, kind)
        torch.cuda.synchronize()
        outs = [{nm: bufs[nm][i].clone() for nm in outputs[kind]} for i in range(len(fns))]
        if kind != "embed":
            assert not agg_x.any() and (kind == "last_layer" or not agg_m.any()), "FLAG_ZERO_AGG left agg_m / agg_x"
        times = [[] for _ in fns]
        for _ in range(args.launches):
            for i in range(len(fns)):
                restore()
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                launch(i, kind)
                e.record()
                times[i].append((s, e))
        torch.cuda.synchronize()
        entry = {"bytes_per_launch": nbytes[kind]}
        for i, p in enumerate(libs):
            ms = [s.elapsed_time(e) for s, e in times[i]]
            mean = statistics.fmean(ms)
            gbs = nbytes[kind] / (mean * 1e-3) / 1e9
            entry[p] = {"mean_ms": mean, "median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms),
                        "GBps": gbs, "share_of_3.35TBps": gbs / (HBM_TBPS * 1e3)}
        if len(fns) == 2:
            entry["output_rowwise_rel_diff"] = {nm: rowwise_rel_diff(outs[0][nm], outs[1][nm]) for nm in outputs[kind]}
            entry["speedup"] = entry[libs[0]]["mean_ms"] / entry[libs[1]]["mean_ms"]
        result["kernels"][kind] = entry
    result["gpu_after"] = gpu_info()
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
