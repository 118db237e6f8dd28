"""Cost of the deterministic mode (model.deterministic, DESIGN §17) on the config-5 shapes of bench.py: 1M nodes, one
graph, radius graph of ~21M edges, C = 8, A = 2, 4 layers, seeded inputs.

    python scripts/bench_deterministic.py [--reps 5] [--steps 20] [--out result.json]

- forward: default and deterministic alternated, `reps` timed forwards of each (CUDA events around each forward, after a
  warm-up of each mode), stage times from the model's own event marks (edge = edge kernel [+ its combine], node = node
  kernel [+ the vsum combine]);
- per-kernel times from one torch.profiler pass of one forward per mode (a separate run: tracing slows the host);
- peak memory of one forward per mode (torch.cuda.max_memory_allocated, from fresh workspaces), and the size of the
  deterministic workspace;
- a `steps`-step radius-graph rollout per mode, ms per step;
- the count of output elements that differ between two forwards, and between two rollouts, of the same mode.
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

from distegnn_b200 import FastEGNN, _lib, rollout, synth  # noqa: E402
from oracle import fastegnn_oracle as orc  # noqa: E402

MODES = (("default", False), ("deterministic", True))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed forwards per mode (alternated), >= 3")
    ap.add_argument("--steps", type=int, default=20, help="rollout steps per mode")
    ap.add_argument("--nodes", type=int, default=None, help="override the node count (default: config 5's 1M)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    w = synth.WORKLOADS["synth1m"]
    host = synth.make_partitions(w, seed=0, **({"n_nodes": args.nodes} if args.nodes else {}))[0]
    inp = {k: (v.to(dev) if v is not None else None) for k, v in host.items()}
    N, E = int(inp["node_loc"].shape[0]), int(inp["edge_index"].shape[1])
    L = 4
    sd = orc.init_state_dict(w.node_feat_nf, w.node_attr_nf, w.edge_attr_nf, 64, w.virtual_channels, L, seed=0,
                             coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=w.node_feat_nf, node_attr_nf=w.node_attr_nf,
                 edge_attr_nf=w.edge_attr_nf, virtual_channels=w.virtual_channels, n_layers=L, normalize=w.normalize)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    res = {"gpu": gpu_info(), "workload": f"synth1m: N={N} E={E} C={w.virtual_channels} A={w.edge_attr_nf} L={L}",
           "reps": args.reps, "forward": {}, "stages_ms": {}, "kernels_ms": {}, "peak_mem_MiB": {}, "rollout": {},
           "differing_elements": {}}

    def fwd():
        with torch.no_grad():
            return m(**inp)

    outs = {}
    for name, det in MODES:                                     # warm-up (workspaces, CSR cache) and output pairs
        m.deterministic = det
        fwd()
        a = fwd()
        b = fwd()
        torch.cuda.synchronize()
        outs[name] = a
        res["differing_elements"][name + "_forward"] = int((a[0] != b[0]).sum() + (a[1] != b[1]).sum())
    res["forward_max_abs_diff_default_vs_deterministic"] = float((outs["default"][0] - outs["deterministic"][0]).abs().max())

    times = {n: [] for n, _ in MODES}
    stages = {n: [] for n, _ in MODES}
    for _ in range(args.reps):
        for name, det in MODES:
            m.deterministic = det
            m._timing = []
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fwd()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e))
            st = {"edge": 0.0, "virtual": 0.0, "node": 0.0, "update": 0.0}
            for (_, t0, t1, t2, t3, t4) in m._timing:
                st["edge"] += t0.elapsed_time(t1)
                st["virtual"] += t1.elapsed_time(t2)
                st["node"] += t2.elapsed_time(t3)
                st["update"] += t3.elapsed_time(t4)
            stages[name].append(st)
            m._timing = None
    for name, _ in MODES:
        ms = times[name]
        res["forward"][name] = {"mean_ms": statistics.fmean(ms), "median_ms": statistics.median(ms), "min_ms": min(ms),
                                "max_ms": max(ms), "all_ms": ms}
        res["stages_ms"][name] = {k: statistics.median([s[k] for s in stages[name]]) for k in stages[name][0]}
    res["forward"]["slowdown"] = res["forward"]["deterministic"]["median_ms"] / res["forward"]["default"]["median_ms"]

    for name, det in MODES:                                     # per kernel, one traced forward
        m.deterministic = det
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fwd()
            torch.cuda.synchronize()
        k = {}
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA and getattr(ev, "device_time_total", 0) > 0:
                k[ev.key[:120]] = {"ms": ev.device_time_total / 1e3, "calls": ev.count}
        res["kernels_ms"][name] = dict(sorted(k.items(), key=lambda kv: -kv[1]["ms"]))

    res["det_workspace_MiB"] = _lib.deterministic_workspace_bytes(N, E, w.virtual_channels) / 2 ** 20
    for name, det in MODES:                                     # each mode's forward allocates its own workspace here
        m.deterministic = det
        m._workspaces.clear()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        fwd()
        torch.cuda.synchronize()
        res["peak_mem_MiB"][name] = torch.cuda.max_memory_allocated(dev) / 2 ** 20

    node = {k: v for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
    for name, det in MODES:
        m.deterministic = det
        m.cuda_graph = True
        runs = []
        for rep in range(2):
            with torch.no_grad():
                torch.cuda.synchronize()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                r = rollout(m, **node, steps=args.steps, radius=w.radius, capacity=int(E * 1.3), check_every=0,
                            return_trajectory=True)
                e.record()
                torch.cuda.synchronize()
                r.check()
            runs.append((r, s.elapsed_time(e)))
        res["rollout"][name] = {"steps": args.steps, "ms_per_step_first": runs[0][1] / args.steps,
                                "ms_per_step_second": runs[1][1] / args.steps}
        a, b = runs[0][0], runs[1][0]
        res["differing_elements"][name + "_rollout_trajectory"] = int((a.trajectory != b.trajectory).sum())
        res["differing_elements"][name + "_rollout_virtual_loc"] = int((a.virtual_loc != b.virtual_loc).sum())
        m.cuda_graph = False
        del runs, a, b, r
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
