"""Cost of the epoch loop (`main.fit`, DESIGN §24) against the `--train_steps` loop on the same batches, on one GPU.

    python scripts/bench_fit.py [--reps 3] [--out result.json]

Data: one Fluid113K-sized scene (113,140 nodes) per split, seeded random walks around synth.make_points written as .npz
to a temporary directory (Fluid113K recipe, delta_t 1, 16 samples per split, batch size 1, r = 0.075), the model of
config/largefluid_distegnn.yaml.  Both loops run with accumulation 1 and the clip on (dataset_name LargeFluid), so they
do the same work per batch: forward, fused loss, backward, clip, Adam step.

Per repetition, alternating:
(1) steps: one pass over the train loader through `--trajectory --train_steps`'s loop (main.trajectory_run), restated
    here without its prints: wall clock around the pass, ending in a device synchronise.
(2) fit, train only: `main.fit` for one epoch with log.test_interval beyond it (no evaluation, no checkpoint; one host
    read of the epoch loss and the log.json write).
(3) fit, full epoch: `main.fit` for one epoch with test_interval 1: train, valid and test passes, best and last
    checkpoints.  The torch.save calls are timed one by one (each ends in the copy of the state to the host).  The ms
    per eval batch is derived: (full − train only − checkpoint writes) / eval batches.
Reports medians over the repetitions and the card name and power limit read in the same run.  Prints one JSON line;
`--out` also writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
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
from distegnn_b200 import synth  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402

N_NODES = 113_140
T_FRAMES = 6


def write_scene(path, w, n, seed):
    pts = synth.make_points(w, seed, n)
    rng = np.random.default_rng(seed)
    steps = rng.normal(0.0, 0.002, (T_FRAMES, n, 3))
    steps[0] = pts["pos"]
    np.savez(path, position=np.cumsum(steps, 0).astype(np.float32),
             velocity=rng.normal(0, 1, (T_FRAMES, n, 3)).astype(np.float32),
             viscosity=rng.random(n).astype(np.float32), mass=rng.random(n).astype(np.float32))


def steps_pass(model, opt, loader, loss_of):
    """One pass of trajectory_run's --train_steps loop."""
    model.train()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for kw, ex in loader:
        opt.zero_grad()
        loss, _ = loss_of(kw, ex)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
        opt.step()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def fit_pass(model, opt, loaders, loss_of, cfg, interval, out_dir):
    cfg = json.loads(json.dumps(cfg))
    cfg["log"]["test_interval"] = interval
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with open(os.devnull, "w") as quiet:
        stdout, sys.stdout = sys.stdout, quiet
        try:
            main.fit(model, opt, None, loaders, loss_of, cfg, 1, out_dir=out_dir)
        finally:
            sys.stdout = stdout
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main_():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fit measures on a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(dataset_name="LargeFluid", delta_t=1, max_samples=16, split_mode="random", batch_size=1)
    cfg["train"] = {"accumulation_steps": 1}
    tmp = tempfile.mkdtemp(prefix="bench_fit_")
    real_save = torch.save
    try:
        w = synth.WORKLOADS["fluid113k"]
        for k, part in enumerate(("train", "valid", "test")):
            os.makedirs(os.path.join(tmp, part))
            write_scene(os.path.join(tmp, part, "scene.npz"), w, N_NODES, seed=k)
        cfg["log"] = {"log_dir": tmp, "test_interval": 1}
        _, loaders = main.frame_loaders(tmp, cfg, 1, 0, dev, None, parts=("train", "valid", "test"))
        torch.manual_seed(0)
        model = main.get_model(cfg, 1).to(dev)
        opt = torch.optim.Adam(model.parameters(), lr=5e-4, weight_decay=1e-12)
        loss_of = main.trajectory_loss(cfg, model, 1, False)
        n_train, n_eval = len(loaders["train"]), len(loaders["valid"]) + len(loaders["test"])

        saves = []

        def timed_save(obj, path, *a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            real_save(obj, path, *a, **k)
            saves.append(time.perf_counter() - t0)
        torch.save = timed_save                            # main.fit's checkpoint writes; restored below

        steps_pass(model, opt, loaders["train"], loss_of)   # warm-up: every shape, the allocator, the first draws
        fit_pass(model, opt, loaders, loss_of, cfg, 1, os.path.join(tmp, "warm"))
        saves.clear()
        t_steps, t_train, t_full, t_saves = [], [], [], []
        for r in range(args.reps):
            t_steps.append(steps_pass(model, opt, loaders["train"], loss_of))
            t_train.append(fit_pass(model, opt, loaders, loss_of, cfg, 10 ** 6, os.path.join(tmp, f"t{r}")))
            saves.clear()
            t_full.append(fit_pass(model, opt, loaders, loss_of, cfg, 1, os.path.join(tmp, f"f{r}")))
            t_saves.append(list(saves))
            saves.clear()
        ckpt_bytes = os.path.getsize(os.path.join(tmp, f"f{args.reps - 1}", "state_dict", "last_model.pth"))
        ms = lambda v, n: [x / n * 1e3 for x in v]
        eval_ms = [(f - t - sum(s)) / n_eval * 1e3 for f, t, s in zip(t_full, t_train, t_saves)]
        res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), reps=args.reps,
                   nodes=N_NODES, train_batches=n_train, eval_batches=n_eval,
                   steps_loop_ms_per_train_batch=ms(t_steps, n_train),
                   fit_ms_per_train_batch=ms(t_train, n_train),
                   fit_ms_per_eval_batch=eval_ms,
                   checkpoint_write_ms=[[x * 1e3 for x in s] for s in t_saves],
                   checkpoint_bytes=ckpt_bytes)
        res["median"] = {k: statistics.median(res[k]) for k in ("steps_loop_ms_per_train_batch",
                                                                 "fit_ms_per_train_batch", "fit_ms_per_eval_batch")}
        res["median"]["checkpoint_write_ms"] = statistics.median(x for s in res["checkpoint_write_ms"] for x in s)
    finally:
        torch.save = real_save
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main_()
