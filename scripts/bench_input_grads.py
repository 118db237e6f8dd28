"""Cost of the input gradients (`model.input_grads = True`) on the training step, at BASELINE config 5 on one GPU.

    python scripts/bench_input_grads.py [--nodes 1000000] [--steps 6] [--out result.json]

Times the training step (forward + backward, no optimizer; the loss of bench.py's train leg) with the flag off and with it
on and all six floating inputs requiring grad, ALTERNATING the two in one process, CUDA events per step, bench.py's L2 flush
(256 MiB written) before every timed step.  Reports the median and spread of each, the peak memory of one step of each,
the per-launch time of the three backward kernels the flag changes (edge, node, embed), and the card name and power limit
read in the same run.  Prints one JSON line; `--out` also writes it to a file (outside the source tree).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from distegnn_b200 import FastEGNN, synth  # noqa: E402

INPUTS = ["node_feat", "node_loc", "node_vel", "loc_mean", "edge_attr", "node_attr"]


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
    ap.add_argument("--steps", type=int, default=6, help="timed steps per mode")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import bench
    from distegnn_b200.backend import cuda_backend

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    w = synth.WORKLOADS["synth1m"]
    host = synth.make_partitions(w, seed=0, n_nodes=args.nodes or w.n_nodes)[0]
    N, E = int(host["node_loc"].shape[0]), int(host["edge_index"].shape[1])
    model = FastEGNN(hidden_nf=64, world_size=1, **bench.model_dims(w))
    model.load_state_dict(bench.make_state_dict(w))
    model = model.to(dev).train()
    inp = {k: (v.to(dev) if v is not None else None) for k, v in host.items()}
    leaf = {k: (v.clone().requires_grad_(True) if (k in INPUTS and v is not None) else v) for k, v in inp.items()}
    target = (inp["node_loc"] + 0.01 * inp["node_vel"]).detach()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def step(on):
        model.input_grads = on
        o, xv = model(**(leaf if on else inp))
        loss = torch.nn.functional.mse_loss(o, target) + 1e-3 * xv.square().mean()
        loss.backward()

    def clear():
        for t in list(model.parameters()) + [leaf[k] for k in INPUTS if leaf.get(k) is not None]:
            t.grad = None

    # per-launch time of the changed backward kernels: events around each call during one extra step per mode
    be = cuda_backend()
    kernel_ms = {}
    originals = {n: getattr(be, n) for n in ("edge_layer_bwd", "node_layer_bwd", "embed_bwd")}

    def timed(name, fn, sink):
        def call(*a, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn(*a, **k)
            e.record()
            sink.append((name, s, e))
        return call

    for on in (False, True):
        step(on)                                            # warm-up (lazy smem opt-ins, graph cache)
        clear()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        sink = []
        for n, fn in originals.items():
            setattr(be, n, timed(n, fn, sink))
        step(on)
        torch.cuda.synchronize()
        for n in originals:
            delattr(be, n)
        peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
        per = {}
        for n, s, e in sink:
            per.setdefault(n, []).append(s.elapsed_time(e))
        kernel_ms["on" if on else "off"] = {"peak_mem_gb": round(peak, 3), **{
            n: {"launches": len(v), "ms_per_launch_median": round(statistics.median(v), 4), "ms_total": round(sum(v), 3)}
            for n, v in per.items()}}
        clear()

    times = {"off": [], "on": []}
    for i in range(args.steps):
        for on in ((False, True) if i % 2 == 0 else (True, False)):
            clear()
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            step(on)
            e.record()
            torch.cuda.synchronize()
            times["on" if on else "off"].append(s.elapsed_time(e))

    def summary(v):
        return {"median_ms": round(statistics.median(v), 2), "min_ms": round(min(v), 2), "max_ms": round(max(v), 2),
                "spread_pct": round(100 * (max(v) - min(v)) / statistics.median(v), 2), "steps": len(v)}

    line = {
        "metric": "train_step_ms_input_grads", "workload": f"synth1m (BASELINE config 5): {N} nodes, {E} edges, "
                                                          f"L={bench.N_LAYERS}, C={w.virtual_channels}, A={w.edge_attr_nf}",
        "gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
        "flag_off": summary(times["off"]), "flag_on_all_inputs": summary(times["on"]),
        "overhead_pct": round(100 * (statistics.median(times["on"]) / statistics.median(times["off"]) - 1), 2),
        "per_mode": kernel_ms,
        "method": "alternating flag off / on in one process; CUDA events per step; 256 MiB L2 flush before each step; "
                  "forward + backward, no optimizer; per-kernel times from events around each call in one extra step",
    }
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
