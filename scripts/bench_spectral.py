"""The spectral partitioner (split_mode="spectral", DESIGN §10) on one GPU.

    python scripts/bench_spectral.py [--reps 5] [--out profiles/spectral_h100.json]

Clouds are synth's Fluid113K points (r = 0.075 density) at 10k, 113,140 and 1M nodes.
(1) The block product S·X (distegnn_spectral_apply) between CUDA events, k = 16 and k = 1 (the degree pass), medians of
    `--reps` with min–max, and the achieved exponentials per second against the ex2 issue rate of the card
    (16 per SM per clock at the maximum SM clock).
(2) The whole `spectral_labels` per frame (σ, degrees, eigensolver, ten k-means runs) at 10k and 113,140 nodes, P = 8,
    with the eigensolver's block products.
(3) sklearn's SpectralClustering by the reference's recipe on the host, at growing N until one call takes over
    `--sklearn-budget` seconds (N doubling from 2000); the largest N done and its time.  The parts can run in separate
    processes (`--skip-sklearn`, `--skip-device`); `--merge` adds a file's parts to this run's result.
Reports the card name and power limit read in the same run.  Prints one JSON line; `--out` also writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from distegnn_b200 import synth  # noqa: E402
from distegnn_b200.spectral import SpectralOperator, rbf_gamma, spectral_embedding, spectral_labels  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402


def max_sm_clock_mhz() -> float:
    out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return float(out[0]) if out else float("nan")


def stats(ts):
    return dict(median=float(np.median(ts)), min=float(np.min(ts)), max=float(np.max(ts)))


def time_apply(op, x, scale, reps):
    ts = []
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        op.apply(x, scale)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts[1:]                                                # the first call is the warm-up


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--label-reps", type=int, default=7)
    ap.add_argument("--sklearn-budget", type=float, default=60.0)
    ap.add_argument("--skip-device", action="store_true", help="only the sklearn part (3)")
    ap.add_argument("--skip-sklearn", action="store_true", help="only the device parts (1), (2)")
    ap.add_argument("--merge", default=None, help="a result file whose parts this run did not measure are kept")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    w = synth.WORKLOADS["fluid113k"]
    props = torch.cuda.get_device_properties(dev)
    clk = max_sm_clock_mhz()
    peak = 16 * props.multi_processor_count * clk * 1e6     # ex2 per second
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), sms=props.multi_processor_count,
               max_sm_clock_mhz=clk, ex2_issue_rate_per_s=peak, reps=args.reps, block_product={}, labels={})
    for n in (() if args.skip_device else (10_000, 113_140, 1_000_000)):
        pos = torch.from_numpy(synth.make_points(w, seed=0, n_nodes=n)["pos"]).to(dev)
        op = SpectralOperator(pos, rbf_gamma(pos.cpu().numpy()))
        reps = args.reps if n < 1_000_000 else max(1, args.reps // 2)
        x = torch.randn(n, 16, dtype=torch.float64, device=dev)
        s = torch.rand(n, dtype=torch.float64, device=dev) + 0.5
        t16 = time_apply(op, x, s, reps)
        t1 = time_apply(op, None, None, reps)
        res["block_product"][str(n)] = dict(
            k16_ms=stats(t16), k1_ms=stats(t1),
            k16_ex2_per_s=n * n / (np.median(t16) * 1e-3), k1_ex2_per_s=n * n / (np.median(t1) * 1e-3),
            k16_fraction_of_ex2_rate=n * n / (np.median(t16) * 1e-3) / peak,
            k1_fraction_of_ex2_rate=n * n / (np.median(t1) * 1e-3) / peak)
        print(n, res["block_product"][str(n)], flush=True)
        del op, x, s
        torch.cuda.empty_cache()
    for n in (() if args.skip_device else (10_000, 113_140)):
        pos = torch.from_numpy(synth.make_points(w, seed=0, n_nodes=n)["pos"]).to(dev)
        _, info = spectral_embedding(pos, 8)
        spectral_labels(pos, 8)                                  # warm-up
        ts = []
        for _ in range(args.label_reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            lab = spectral_labels(pos, 8)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t)
        res["labels"][str(n)] = dict(P=8, seconds=stats(ts), block_products=int(info["products"]),
                                     eigenvalues=[float(v) for v in info["eigenvalues"]],
                                     sizes=torch.bincount(lab, minlength=8).tolist())
        print(n, res["labels"][str(n)], flush=True)
    done, n = None, 2000
    while not args.skip_sklearn:                                 # doubling N until one call exceeds the budget
        X = synth.make_points(w, seed=0, n_nodes=n)["pos"]
        t = time.perf_counter()
        synth.spectral_partition(X, 8)
        dt = time.perf_counter() - t
        done = dict(nodes=n, P=8, seconds=dt)
        print("sklearn", done, flush=True)
        if dt > args.sklearn_budget:
            break
        n *= 2
    res["sklearn_largest"] = done
    if args.merge:
        with open(args.merge) as f:
            for k, v in json.load(f).items():
                if res.get(k) in (None, {}):
                    res[k] = v
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
