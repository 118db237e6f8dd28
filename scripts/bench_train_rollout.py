"""Cost of `--train_rollout K` (DESIGN §26): one optimiser step on a K-step rollout against the one-step path.

    python scripts/bench_train_rollout.py [--steps 1 2 4 8] [--reps 5] [--out result.json]

Two workloads, both through main.py's own loaders and loss functions, each from a seed and written to a temporary
directory: a Fluid113K-sized synthetic trajectory (one .npz scene of ~113k particles, radius graph r = 0.075, config
largefluid_distegnn.yaml) and nbody_100 at batch 250 (`distegnn_b200.nbody`, config nbody_fastegnn.yaml, fully connected).
For every workload one FrameLoader batch of horizon max(K) is assembled once; then, ALTERNATING the variants `--reps`
times in one process, one optimiser step (zero_grad, loss, backward, clip 0.3, Adam) of the one-step path
(`trajectory_loss`) and of every K (`trajectory_rollout_loss`), each timed with the host clock around a device
synchronise; the peak of `max_memory_allocated` above what was allocated before.  Medians are reported.  Also, per K,
K separate one-step `train_loss` calls (forward and backward) against one stepped call on the same inputs, default
samples (the K·B host draws are in both).  Reports the card name and power limit read in the same run.  Prints one JSON
line; `--out` also writes it to a file."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import main  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402
from distegnn_b200 import synth, train_loss  # noqa: E402


def fluid_data(path, seed=0, frames=12):
    """One Fluid113K-sized scene: synth's fluid113k points moving with their velocities plus a seeded jitter."""
    w = synth.WORKLOADS["fluid113k"]
    pts = synth.make_points(w, seed, w.n_nodes)
    rng = np.random.default_rng(seed)
    x0, v = pts["pos"].astype(np.float32), 0.002 * rng.standard_normal(pts["pos"].shape).astype(np.float32)
    pos = np.stack([x0 + t * v + 1e-4 * t * rng.standard_normal(x0.shape).astype(np.float32) for t in range(frames)])
    os.makedirs(os.path.join(path, "train"))
    n = x0.shape[0]
    np.savez(os.path.join(path, "train", "scene_0.npz"), position=pos, velocity=np.broadcast_to(v, pos.shape).copy(),
             viscosity=np.full(n, 0.1, np.float32), mass=np.ones(n, np.float32))
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"]["max_samples"] = 1
    return cfg, None, 1.0                                       # distribute mode (no cutoff), tau 1


def nbody_data(path, Kmax):
    from distegnn_b200 import nbody
    nbody.generate_dataset(path, num_train=250, num_valid=0, num_test=0, length=100 * (Kmax + 1), n_isolated=100,
                           seed=43)
    with open(os.path.join(ROOT, "config", "nbody_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(frame_0=0, frame_T=1)
    return cfg, float(cfg["data"].get("cutoff_rate", 0.0)), nbody.meta_rollout_tau(path, 1)


def run(name, path, cfg, rate, tau, steps, reps, dev):
    recipe = main.recipe_of_config(cfg)[0]
    torch.manual_seed(0)
    model = main.get_model(cfg, 1).to(dev).train()
    ld = main.frame_loaders(path, cfg, 1, 0, dev, rate, horizon=max(steps), parts=("train",))[1]["train"]
    kw, ex = next(iter(ld))
    opt = torch.optim.Adam(model.parameters(), lr=1e-6)
    variants = {"one_step": main.trajectory_loss(cfg, model, 1, False)}
    for K in steps:
        variants[f"K={K}"] = main.trajectory_rollout_loss(cfg, model, 1, False, ld, recipe, tau, K)
    exK = {K: dict(ex, targets=ex["targets"][:K].contiguous()) for K in steps}

    def one(label):
        e = ex if label == "one_step" else exK[int(label[2:])]
        opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        loss, _ = variants[label](kw, e, 1)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
        opt.step()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, torch.cuda.max_memory_allocated() - base

    for label in variants:                                      # warm-up: every shape, module loads
        one(label)
    ms = {k: [] for k in variants}
    peak = {k: 0 for k in variants}
    for _ in range(reps):
        for label in variants:
            t, p = one(label)
            ms[label].append(t)
            peak[label] = max(peak[label], p)
    out = {"nodes": int(kw["node_loc"].shape[0]), "graphs": int(ex["n_graphs"]), "variants": {}}
    base = statistics.median(ms["one_step"])
    for label in variants:
        m = statistics.median(ms[label])
        out["variants"][label] = dict(ms_per_optimiser_step=round(m, 3), min_ms=round(min(ms[label]), 3),
                                      vs_one_step=round(m / base, 3), peak_mib=round(peak[label] / 2 ** 20, 1))
    out["loss_calls"] = loss_calls(cfg, kw, ex, steps, reps, dev)
    return out


def loss_calls(cfg, kw, ex, steps, reps, dev):
    """K one-step train_loss calls against one stepped call: forward + backward, default samples."""
    mmd = (cfg.get("train") or {}).get("mmd") or {}
    C = int(cfg["model"]["virtual_channels"])
    N, B = int(kw["node_loc"].shape[0]), int(ex["n_graphs"])
    g = torch.Generator(device=dev).manual_seed(0)
    args = dict(mmd_samples=int(mmd.get("samples", 50)), mmd_sigma=float(mmd.get("sigma", 3)),
                mmd_weight=float(mmd.get("weight", 0.01)), node_counts=ex["node_counts"], loc_mean=kw["loc_mean"])
    out = {}
    for K in steps:
        pred = torch.randn(K, N, 3, device=dev, generator=g).requires_grad_(True)
        Xv = torch.randn(K, B, 3, C, device=dev, generator=g).requires_grad_(True)
        tgt = ex["targets"][:K].contiguous()

        def separate():
            loss = sum(train_loss(pred[t], tgt[t], Xv[t], kw["data_batch"], **args)[0] for t in range(K)) / K
            loss.backward()

        def stepped():
            train_loss(pred, tgt, Xv, kw["data_batch"], **args)[0].backward()
        res = {}
        for fn in (separate, stepped):
            fn()
        ts = {"separate": [], "stepped": []}
        for _ in range(reps):
            for label, fn in (("separate", separate), ("stepped", stepped)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(10):
                    fn()
                torch.cuda.synchronize()
                ts[label].append((time.perf_counter() - t0) * 1e2)  # ms per call
        for label in ts:
            res[f"{label}_ms"] = round(statistics.median(ts[label]), 3)
        out[f"K={K}"] = res
    return out


def main_():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", nargs="+", default=["fluid113k", "nbody_100"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_train_rollout needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    result = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "reps": args.reps,
              "steps": args.steps, "timing": "median of host clock around a device synchronise, one optimiser step",
              "workloads": {}}
    for wl in args.workloads:
        with tempfile.TemporaryDirectory() as tmp:
            if wl == "fluid113k":
                cfg, rate, tau = fluid_data(tmp)
                desc = "Fluid113K-sized synthetic scene, r = 0.075, batch 1"
            else:
                cfg, rate, tau = nbody_data(tmp, max(args.steps))
                desc = "nbody_100 (distegnn_b200.nbody), batch 250, fully connected"
            r = run(wl, tmp, cfg, rate, tau, args.steps, args.reps, dev)
            result["workloads"][wl] = dict(description=desc, **r)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(result, indent=1) + "\n")


if __name__ == "__main__":
    main_()
