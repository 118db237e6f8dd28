#!/usr/bin/env python
"""torchrun entry point with the reference's CLI (reference main.py:95-163) for the accelerated hot path.

    python main.py --config_path config.yaml [--model_name FastEGNN --batch_size 1 --split_mode random
                                              --virtual_channels 8 --checkpoint best_model.pth --seed 0]
    torchrun --nproc_per_node=P --master_addr=127.0.0.1 --master_port=29500 main.py --config_path ...

It reads the reference's YAML layout (sections `model`, `data`, `seed`; e.g. config/largefluid_distegnn.yaml),
takes the same command-line overrides, initialises `torch.distributed` exactly as the reference does
(`init_process_group("nccl")`, rank = LOCAL_RANK, one process per GPU, main.py:143-163), builds
`distegnn_b200.FastEGNN` through the same `get_model` switch (main.py:58-62), wraps it in
`DistributedDataParallel(..., find_unused_parameters=True)` (main.py:196), optionally loads a reference checkpoint
(`{'model_state_dict': ...}` with or without DDP's `module.` prefix, main.py:208-220, train.py:235-259) and runs the
DistEGNN forward over graph partitions.

What it does NOT do: the reference's datasets are not redistributable and its data pipeline needs PyG/h5py/
MDAnalysis, so inputs are the seeded synthetic restatement of the configured dataset (`distegnn_b200/synth.py`:
same node/edge statistics, `radius`/`split_mode` semantics of datasets/distribute_graphs.py) with a synthetic
target (constant-velocity step).  It evaluates `--eval_steps` forward passes (graph-steps/s, edges/s) and, with
`--train_steps K`, runs K optimisation steps of the reference's training step (utils/train.py:98-158: node-count
weighted MSE x world_size, MMD regulariser on the virtual coordinates, gradient clipping 0.3, Adam) through the
fused forward AND backward kernels under DDP — the epoch loop, loaders, checkpoints and wandb logging of
utils/train.py stay with the reference (out of scope).

`--trajectory PATH` trains and evaluates on real frames instead (distegnn_b200.frames.FrameLoader, DESIGN §18): the
config's recipe (N-body, Water-3D, Fluid113K), radius / inner_radius, delta_t (N-body: frame_0, frame_T), split_mode and
cutoff_rate; every batch is assembled on the device from the raw trajectories as it is needed.  With `--rollout_steps K`
it then rolls the trained model out K steps from every validation batch and prints the per-step MSE against the recorded
frames f + Δ .. f + KΔ (DESIGN §19; `--rollout_tau` sets the velocity's time step, Water-3D defaults to Δ);
`--rollout_chamfer` adds both directions of the normalised Chamfer distance to every step's line (DESIGN §20).  Without the
flag the synthetic path below runs unchanged.

`data.accelerate_mode: cutoff_edges` (FastEGNN, e.g. config/nbody_fastegnn.yaml) is the reference's single-device mode:
`batch_size` synthetic graphs in one batch, the candidate graph fully connected for `radius: -1` (N-body) or a radius
graph, then `data.cutoff_rate` (`--cutoff_rate` overrides it, reference main.py:133-134) drops the longest edges of
every graph on the device (`distegnn_b200.cutoff_edges_csr`, datasets/process_dataset.py:103,300-305).  The evaluation,
`--train_steps` and `--rollout_steps` all run on the cut graph; a rollout re-selects the kept edges every step.  Under
torchrun with more than one rank this mode exits with a message.  In `distribute` mode `--cutoff_rate` is ignored, as
the reference ignores it there.
"""
from __future__ import annotations

import argparse
import os
import re
import sys
import time

import torch
import torch.distributed as dist
import yaml
from torch.nn.parallel import DistributedDataParallel

from distegnn_b200 import FastEGNN, synth


class Cfg(dict):
    """Attribute access over nested dicts (stand-in for easydict.EasyDict, which the reference uses)."""

    def __getattr__(self, k):
        v = self[k]
        return Cfg(v) if isinstance(v, dict) else v

    __setattr__ = dict.__setitem__


DATASET_TO_WORKLOAD = {"nbody": "nbody100", "water3d": "water3d_10k", "water-3d": "water3d_10k",
                       "fluid113k": "fluid113k", "largefluid": "fluid113k", "synth1m": "synth1m"}


def get_model(cfg: Cfg, world_size: int) -> torch.nn.Module:
    """reference main.py:58-92 — only the DistEGNN family lives here."""
    m = cfg["model"]
    if m["model_name"] != "FastEGNN":
        raise NotImplementedError(f"model_name={m['model_name']!r}: only FastEGNN (DistEGNN) is accelerated here")
    return FastEGNN(node_feat_nf=m["node_feat_nf"], node_attr_nf=m["node_attr_nf"], edge_attr_nf=m["edge_attr_nf"],
                    hidden_nf=m["hidden_nf"], virtual_channels=m["virtual_channels"], world_size=world_size,
                    n_layers=m["n_layers"], normalize=m["normalize"])


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--config_path", type=str, required=True, help="path to config yaml file")
    p.add_argument("--wandb", action="store_true")
    p.add_argument("--lr", type=float, default=None)
    p.add_argument("--seed", type=int, default=None)
    p.add_argument("--model_name", type=str, default=None)
    p.add_argument("--batch_size", type=int, default=None)
    p.add_argument("--split_mode", type=str, default=None)
    p.add_argument("--early_stop", type=int, default=None)
    p.add_argument("--checkpoint", type=str, default=None)
    p.add_argument("--cutoff_rate", type=float, default=None)
    p.add_argument("--outer_radius", type=float, default=None)
    p.add_argument("--inner_radius", type=float, default=None)
    p.add_argument("--virtual_channels", type=int, default=None)
    p.add_argument("--eval_steps", type=int, default=10, help="(new) forward passes to time")
    p.add_argument("--nodes", type=int, default=None, help="(new) override the synthetic node count")
    p.add_argument("--rollout_steps", type=int, default=0, help="(new) K-step rollout from the synthetic state "
                   "(distegnn_b200.rollout): graph rebuilt on the device every step; prints ms/step and edges/step")
    p.add_argument("--train_steps", type=int, default=0, help="(new) optimisation steps of the reference's training "
                   "step (utils/train.py:98-158) on the synthetic target")
    p.add_argument("--trajectory", type=str, default=None, help="(new) train and evaluate on raw frames under this "
                   "directory (distegnn_b200.frames): N-body .npy files, or train/ and valid/ folders of .npz scenes; "
                   "with --rollout_steps K also a K-step rollout from every validation batch against the recorded frames")
    p.add_argument("--rollout_chamfer", action="store_true", help="(new) with --trajectory and --rollout_steps: also "
                   "print each step's Chamfer distance to the recorded frame (prediction -> record, record -> "
                   "prediction), normalised like the MSE; independent of particle identity")
    p.add_argument("--rollout_tau", type=float, default=None, help="(new) time step of a --trajectory rollout's "
                   "velocity v = (x' − x)/tau; default Δ for Water-3D (one-frame differences), required for N-body and "
                   "Fluid113K (physical velocities; the frame time is not in the files)")
    return p.parse_args()


def main():
    args = parse()
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    cfg.setdefault("data", {})
    if args.seed is not None:
        cfg["seed"] = args.seed
    if args.model_name is not None:
        cfg["model"]["model_name"] = args.model_name
    if args.batch_size is not None:
        cfg["data"]["batch_size"] = args.batch_size
    if args.split_mode is not None:
        cfg["data"]["split_mode"] = args.split_mode
    if args.checkpoint is not None:
        cfg["model"]["checkpoint"] = args.checkpoint
    if args.inner_radius is not None:
        cfg["data"]["inner_radius"] = args.inner_radius
    if args.virtual_channels is not None:
        cfg["model"]["virtual_channels"] = args.virtual_channels

    # FastEGNN's cutoff_edges mode (reference README.md:30-33): the cutoff rate applies; in distribute mode it does not
    cutoff_mode = str(cfg["data"].get("accelerate_mode", "distribute")) == "cutoff_edges"
    rate = None
    if cutoff_mode:
        rate = float(args.cutoff_rate if args.cutoff_rate is not None else cfg["data"].get("cutoff_rate", 0.0))
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            if int(os.environ.get("LOCAL_RANK", "0")) == 0:
                print("accelerate_mode=cutoff_edges (FastEGNN) is a single-device mode, as in the reference; run it "
                      "without torchrun or with one process (use accelerate_mode=distribute for several GPUs)", flush=True)
            sys.exit(2)
    # options of the reference CLI that belong to its data pipeline / epoch loop (out of scope here): say so, loudly
    ignored = [n for n, v in (("--wandb", args.wandb), ("--early_stop", args.early_stop),
                              ("--cutoff_rate", None if cutoff_mode else args.cutoff_rate),
                              ("--outer_radius", args.outer_radius)) if v]
    if ignored and int(os.environ.get("LOCAL_RANK", "0")) == 0:
        print(f"WARNING: {', '.join(ignored)} accepted for CLI compatibility but NOT used: logging, early stopping and "
              "the cutoff / outer-radius edge pruning live in the reference's data pipeline and epoch loop "
              "(utils/train.py, datasets/process_dataset.py), which this entry point does not replace", flush=True)

    assert torch.cuda.is_available(), "distegnn_b200 needs CUDA devices (there is no CPU path)"
    distributed = "LOCAL_RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world_size = int(os.environ["WORLD_SIZE"]) if distributed else 1
    torch.cuda.set_device(local_rank)
    if distributed:                                            # reference main.py:159-163
        dist.init_process_group("nccl", rank=local_rank, world_size=world_size)
    if local_rank == 0:
        print(f"Use {world_size} GPUs!")
    torch.manual_seed(cfg.get("seed", 0))

    model = get_model(cfg, world_size).to(local_rank)
    ck = cfg["model"].get("checkpoint")
    if ck:
        state = torch.load(ck, map_location=f"cuda:{local_rank}")
        sd = state.get("model_state_dict", state)
        sd = {k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}
        model.load_state_dict(sd)
    if distributed:                                            # reference main.py:194-196
        model = DistributedDataParallel(model, device_ids=[local_rank], find_unused_parameters=True)
    model.eval()
    if args.trajectory:
        trajectory_run(args, cfg, model, world_size, local_rank, distributed, rate)
        if distributed:
            dist.destroy_process_group()
        return

    # ---- inputs: synthetic restatement of the configured dataset, partitioned like datasets/distribute_graphs.py ----
    d = cfg["data"]
    ds = str(d.get("dataset_name", "fluid113k")).lower()
    name = DATASET_TO_WORKLOAD.get(ds)
    if name is None and cutoff_mode:                           # the FastEGNN configs name sized sets: nbody_100, ...
        name = DATASET_TO_WORKLOAD.get(re.split(r"[_\-]", ds)[0])
    base = synth.WORKLOADS[name or "fluid113k"]
    m = cfg["model"]
    radius = d.get("inner_radius", d.get("radius", base.radius))
    if cutoff_mode and radius is not None and radius < 0:     # radius: -1 = fully connected (process_dataset.py:97-98)
        radius = None
    w = synth.Workload(base.name, args.nodes or base.n_nodes, radius,
                       base.degree, m["node_feat_nf"], m["node_attr_nf"], m["edge_attr_nf"], m["virtual_channels"],
                       m["normalize"])
    split = d.get("split_mode", "random")
    if world_size > 1 and split not in ("random", "kmeans"):
        if local_rank == 0:
            print(f"split_mode={split!r} needs METIS/spectral partitioners of the reference's data pipeline; "
                  "using 'random' for the synthetic graph")
        split = "random"
    cut = None
    if cutoff_mode:
        inp, cut = cutoff_inputs(w, int(d.get("batch_size", 1)), cfg.get("seed", 0), rate, local_rank)
        n_r, e_r = inp["node_loc"].shape[0], cut["kept"]
    else:
        part = synth.make_partitions(w, world_size=world_size, split_mode=split, seed=cfg.get("seed", 0),
                                     only_rank=local_rank)[local_rank]
        inp = {k: (v.to(local_rank) if v is not None else None) for k, v in part.items()}
        n_r, e_r = inp["node_loc"].shape[0], inp["edge_index"].shape[1]

    def forward():                                             # positional call as in utils/train.py:63-71
        node_attr = inp["node_attr"] if m["node_attr_nf"] > 0 else None
        return model(inp["node_feat"], inp["node_loc"], inp["node_vel"], inp["loc_mean"], inp["edge_index"],
                     inp["data_batch"], inp["edge_attr"], node_attr)

    with torch.no_grad():
        for _ in range(3):
            out, X = forward()
        torch.cuda.synchronize()
        if distributed:
            dist.barrier()
        t0 = time.perf_counter()
        for _ in range(args.eval_steps):
            out, X = forward()
        torch.cuda.synchronize()
        if distributed:
            dist.barrier()
        dt = (time.perf_counter() - t0) / args.eval_steps
        # node-count weighted MSE across ranks, as utils/train.py:98-110 weights the loss
        se = ((out - inp["node_loc"]) ** 2).sum()
        cnt = torch.tensor([float(n_r), float(e_r)], device=local_rank)
        if distributed:
            dist.all_reduce(se)
            dist.all_reduce(cnt)
    if local_rank == 0:
        print(f"[{w.name}] world_size={world_size} split={split if world_size > 1 else 'none'} nodes={int(cnt[0])} "
              f"edges(sum over partitions)={int(cnt[1])}  forward {dt * 1e3:.3f} ms  "
              f"{1.0 / dt:.2f} graph-steps/s  {cnt[1].item() / dt / 1e6:.1f} M edges/s  "
              f"mean squared displacement {se.item() / (3 * cnt[0].item()):.4e}  virtual_loc {tuple(X.shape)}")
    if cut is not None and local_rank == 0:
        print(f"[{w.name}] cutoff_edges: cutoff_rate={rate} kept {cut['kept']} of {cut['candidates']} candidate edges "
              f"({cut['graphs']} graphs)")
    if args.rollout_steps > 0:
        rollout_steps(args, model, inp, w, world_size, local_rank, distributed, cut)
    if args.train_steps > 0:
        train_steps(args, cfg, model, inp, forward, world_size, local_rank, distributed, cut)
    if distributed:
        dist.destroy_process_group()


def recipe_of_config(cfg):
    """(recipe name, frame_0, Δ) of the config's dataset (N-body: frame_T − frame_0; else data.delta_t)."""
    d = cfg["data"]
    ds = str(d.get("dataset_name", "")).lower()
    recipe = "nbody" if ds.startswith("nbody") else "water3d" if ds.startswith("water") else "largefluid"
    if recipe == "nbody":
        frame_0, frame_T = int(d.get("frame_0", 30)), int(d.get("frame_T", 40))
        return recipe, frame_0, frame_T - frame_0
    return recipe, 0, int(d.get("delta_t", 1))


def frame_loaders(path, cfg, world_size, rank, device, rate, horizon=1, parts=("train", "valid")):
    """FrameLoaders over the raw trajectories under `path` with the config's recipe (datasets/process_dataset.py):
    N-body (`dataset_name: nbody*`, the reference's loc_/vel_/charges_ .npy files, frame_0 / frame_T), Water-3D or
    Fluid113K (`path`/train/*.npz, `path`/valid/*.npz).  cutoff_edges mode: one graph per sample, radius = data.radius
    (−1 fully connected; Water-3D: the reference's hard-coded 0.035, :264), then the cutoff.  distribute mode: the
    sample split over the ranks by split_mode (metis / spectral fall back to random), a radius graph per partition with
    inner_radius.  `horizon` K: every sample holds frames f + Δ .. f + KΔ (the frame draw is capped for that; a fixed
    N-body frame_0 that cannot hold them exits with a message).  Returns (recipe name, {part: loader or None})."""
    import glob
    from distegnn_b200.frames import FrameLoader, load_nbody, load_scenes, sample_list
    d = cfg["data"]
    recipe, frame_0, delta = recipe_of_config(cfg)
    cutoff_mode = rate is not None
    if cutoff_mode:
        radius = 0.035 if recipe == "water3d" else d.get("radius", -1)
    else:
        radius = d.get("inner_radius")
    split = str(d.get("split_mode", "random"))
    if split not in ("random", "kmeans"):
        split = "random"
    seed, bs = int(cfg.get("seed", 0)), int(d.get("batch_size", 1))
    out = {}
    for part in parts:
        if recipe == "nbody":
            if not os.path.exists(os.path.join(path, f"loc_{part}_charged100_0_0_1.npy")):
                out[part] = None
                continue
            traj = load_nbody(path, part)
        else:
            files = sorted(glob.glob(os.path.join(path, part, "*.npz")))
            if not files:
                out[part] = None
                continue
            traj = load_scenes(files, recipe)
        kw = {}
        if recipe != "nbody":
            shortest = min(sc.n_frames for sc in traj.scenes)
            kw["max_frame"] = min(traj.recipe.max_frame, shortest - 1 - max(horizon * delta, 1))
            if horizon > 1 and kw["max_frame"] < 0:
                raise SystemExit(f"--trajectory {path}/{part}: the shortest scene has {shortest} frames; it cannot hold "
                                 f"{horizon} step(s) of delta_t={delta} frames after any frame")
        samples = sample_list(traj, seed=seed, max_samples=d.get("max_samples"), delta_t=delta, frame_0=frame_0, **kw)
        out[part] = FrameLoader(traj, samples, delta_t=delta, radius=radius, batch_size=bs, shuffle=part == "train",
                                seed=seed, device=device, world_size=world_size, rank=rank, split_mode=split,
                                cutoff_rate=rate or 0.0, horizon=horizon)
    if "train" in parts and out["train"] is None:
        raise SystemExit(f"--trajectory {path}: no training data for recipe {recipe!r}")
    return recipe, out


def trajectory_run(args, cfg, model, world_size, local_rank, distributed, rate):
    """--trajectory: `--train_steps` optimisation steps (at least one epoch's worth if 0 is given: one pass) of the
    reference's training step on batches from FrameLoader, then the mean MSE over the validation batches."""
    from distegnn_b200 import train_loss
    recipe, _, delta = recipe_of_config(cfg)
    K = args.rollout_steps
    tau = args.rollout_tau if args.rollout_tau is not None else (float(delta) if recipe == "water3d" else None)
    if K > 0 and tau is None:                                  # before any training: the rollout could not run
        if local_rank == 0:
            print(f"--rollout_steps with --trajectory on {recipe!r} needs --rollout_tau: its velocities are physical and "
                  "the frame time is not in the files (Water-3D defaults to delta_t)", flush=True)
        sys.exit(2)
    recipe, loaders = frame_loaders(args.trajectory, cfg, world_size, local_rank, torch.device("cuda", local_rank), rate)
    tc = cfg.get("train", {}) or {}
    mmd = tc.get("mmd", {}) or {}
    lr = args.lr if args.lr is not None else float(tc.get("learning_rate", tc.get("lr", 5e-4)))
    opt = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=float(tc.get("weight_decay", 1e-12)))
    inner = model.module if distributed else model
    use_attr = cfg["model"]["node_attr_nf"] > 0

    def forward(kw):                                           # positional call as in utils/train.py:63-71
        return model(kw["node_feat"], kw["node_loc"], kw["node_vel"], kw["loc_mean"], kw["edge_index"],
                     kw["data_batch"], kw["edge_attr"], kw["node_attr"] if use_attr else None)

    def loss_of(kw, ex):
        pred, X = forward(kw)
        return train_loss(pred, ex["target"], X, kw["data_batch"], world_size=world_size,
                          mmd_samples=int(mmd.get("samples", 50)), mmd_sigma=float(mmd.get("sigma", 3)),
                          mmd_weight=float(mmd.get("weight", 0.01)), loc_mean=kw["loc_mean"],
                          node_counts=ex["node_counts"], model=inner)

    steps = args.train_steps or len(loaders["train"])
    model.train()
    done, t0 = 0, time.perf_counter()
    while done < steps:
        for kw, ex in loaders["train"]:
            opt.zero_grad()
            loss, info = loss_of(kw, ex)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
            opt.step()
            done += 1
            if local_rank == 0 and (done % 10 == 0 or done == steps):
                print(f"[{recipe}] train step {done}: MSE {info['logged'].item():.6e}", flush=True)
            if done == steps:
                break
    torch.cuda.synchronize()
    if local_rank == 0:
        print(f"[{recipe}] {steps} train steps on raw frames: {(time.perf_counter() - t0) / steps * 1e3:.2f} ms/step")
    ev = loaders["valid"] or loaders["train"]
    model.eval()
    tot, n = 0.0, 0
    with torch.no_grad():
        for kw, ex in ev:
            _, info = loss_of(kw, ex)
            tot, n = tot + float(info["logged"]), n + 1
    if local_rank == 0:
        print(f"[{recipe}] evaluation over {n} batches ({'valid' if loaders['valid'] else 'train'}): mean MSE "
              f"{tot / max(n, 1):.6e}")
    if K > 0:
        rollout_eval(args, cfg, model, world_size, local_rank, rate, recipe, tau)


# the |v| column of each recipe's node features (distegnn_b200/frames.py): N-body, Water-3D [‖v‖, ·], Fluid113K [·, ·, ‖v‖]
SPEED_COL = {"nbody": 0, "water3d": 0, "largefluid": 2}


def rollout_eval(args, cfg, model, world_size, local_rank, rate, recipe, tau):
    """--trajectory with --rollout_steps K: a K-step `rollout(targets=...)` from every batch of the valid split (the
    train split without one), through a FrameLoader with horizon K and the config's radius and cutoff rate; prints the
    per-step MSE averaged over the batches, each weighted by its graph count (utils/train.py:112-114, 166).  With
    --rollout_chamfer each line also carries the two directions of `chamfer_mse`, averaged the same way."""
    from distegnn_b200 import rollout
    K = args.rollout_steps
    dev = torch.device("cuda", local_rank)
    part = "valid"
    try:
        _, lds = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, horizon=K, parts=(part,))
        if lds[part] is None:
            part = "train"
            _, lds = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, horizon=K, parts=(part,))
    except ValueError as e:                                    # a sample that cannot hold K steps
        if local_rank == 0:
            print(f"--rollout_steps {K}: {e}", flush=True)
        sys.exit(2)
    ld = lds[part]
    use_attr = cfg["model"]["node_attr_nf"] > 0
    tot, graphs, n = torch.zeros(K, dtype=torch.float64, device=dev), 0, 0
    ch_tot = torch.zeros(K, 2, dtype=torch.float64, device=dev)
    t0 = time.perf_counter()
    for kw, ex in ld:
        if ld.radius is not None:
            g = dict(radius=ld.radius)
        else:                                                  # fully connected: the candidates, cut again every step
            g = dict(graph=ld.complete_graph(tuple(ex["node_counts"])) if ld.cutoff_rate > 0 else kw["edge_index"])
        res = rollout(model, kw["node_feat"], kw["node_loc"], kw["node_vel"], kw["loc_mean"], kw["data_batch"],
                      kw["node_attr"] if use_attr else None, steps=K, tau=tau, speed_col=SPEED_COL[recipe],
                      cutoff_rate=ld.cutoff_rate, targets=ex["targets"], chamfer=args.rollout_chamfer, **g)
        tot += res.mse * ex["n_graphs"]
        if args.rollout_chamfer:
            ch_tot += res.chamfer_mse * ex["n_graphs"]
        graphs, n = graphs + ex["n_graphs"], n + 1
    mse = (tot / max(graphs, 1)).tolist()
    ch = (ch_tot / max(graphs, 1)).tolist()
    dt = time.perf_counter() - t0
    if local_rank == 0:
        print(f"[{recipe}] rollout evaluation over {n} batches ({part}), {K} steps, tau={tau:g}: "
              f"{dt / max(n * K, 1) * 1e3:.2f} ms/step", flush=True)
        for t, v in enumerate(mse):
            extra = f", Chamfer pred->rec {ch[t][0]:.6e}, rec->pred {ch[t][1]:.6e}" if args.rollout_chamfer else ""
            print(f"[{recipe}] rollout step {t + 1}: MSE {v:.6e}{extra}", flush=True)


def cutoff_inputs(w, batch_size, seed, rate, device):
    """`batch_size` synthetic graphs of the workload in one batch, their candidate graph as CSR, and its cut: FastEGNN's
    cutoff_edges data (datasets/process_dataset.py:96-104, one cut per graph).  Returns (forward inputs, cut info)."""
    from distegnn_b200 import cutoff_edges_csr
    from distegnn_b200.shards import CSRGraph
    parts = [synth.make_partitions(w, seed=seed + b)[0] for b in range(batch_size)]
    cat = lambda k: None if parts[0][k] is None else torch.cat([p[k] for p in parts]).to(device)
    n = [int(p["node_loc"].shape[0]) for p in parts]
    off = [sum(n[:b]) for b in range(batch_size)]
    ei = torch.cat([p["edge_index"] + off[b] for b, p in enumerate(parts)], 1).to(device)
    batch = torch.arange(batch_size, device=device).repeat_interleave(torch.tensor(n, device=device))
    inp = dict(node_feat=cat("node_feat"), node_loc=cat("node_loc"), node_vel=cat("node_vel"), node_attr=cat("node_attr"),
               loc_mean=torch.stack([p["node_loc"].mean(0) for p in parts]).to(device), data_batch=batch)
    cand, _ = CSRGraph.from_edge_index(ei, sum(n))
    g, ea = cutoff_edges_csr(cand, inp["node_loc"], rate, batch, batch_size, w.edge_attr_nf)
    inp["edge_index"], inp["edge_attr"] = g, ea
    return inp, dict(candidates=cand.num_edges, kept=g.num_edges, graphs=batch_size, graph=cand, rate=rate,
                     node_counts=n)


def rollout_steps(args, model, inp, w, world_size, local_rank, distributed, cut=None):
    """K steps of `distegnn_b200.rollout` from the partition's state (radius graph rebuilt every step, or the fully
    connected graph kept when the dataset has no radius); ms/step from a host clock around a device synchronise, after
    one untimed rollout that also fixes the edge capacity."""
    from distegnn_b200 import rollout
    from distegnn_b200.shards import CSRGraph
    node = {k: inp[k] for k in ("node_feat", "node_loc", "node_vel", "loc_mean", "data_batch")}
    node["node_attr"] = inp["node_attr"] if w.node_attr_nf > 0 else None
    if cut is not None:                                        # the candidates; each step keeps its shortest edges
        kw = dict(radius=w.radius) if w.radius is not None else dict(graph=cut["graph"])
        kw["cutoff_rate"] = cut["rate"]
    else:
        kw = dict(radius=w.radius) if w.radius is not None else \
            dict(graph=CSRGraph.from_edge_index(inp["edge_index"], inp["node_loc"].shape[0])[0])
    K = args.rollout_steps
    # the synthetic features stand for the datasets' (|v|, ...) columns: column 0 is the speed, one frame per step
    kw.update(speed_col=0, tau=1.0)
    res = rollout(model, **node, steps=K, **kw)                # warm-up; sizes the capacity
    torch.cuda.synchronize()
    if distributed:
        dist.barrier()
    t0 = time.perf_counter()
    res = rollout(model, **node, steps=K, capacity=res.capacity, **kw)
    torch.cuda.synchronize()
    if distributed:
        dist.barrier()
    dt = (time.perf_counter() - t0) / K
    edges = res.n_edges.double().mean().reshape(1)
    if distributed:
        dist.all_reduce(edges)
    if local_rank == 0:
        print(f"[{w.name}] rollout {K} steps, world_size={world_size}: {dt * 1e3:.3f} ms/step, "
              f"{edges.item():.0f} edges/step (sum over partitions), capacity {res.capacity}")


def train_steps(args, cfg, model, inp, forward, world_size, local_rank, distributed, cut=None):
    """utils/train.py:98-158 on one (partitioned) synthetic graph: loss = n_r/Σn · MSE_r · world_size (DDP averages the
    gradients, the reference wants their sum) + MMD between the virtual coordinates and sampled target positions."""
    tc = cfg.get("train", {}) or {}
    mmd = tc.get("mmd", {}) or {}
    sigma, mmd_w, samples = float(mmd.get("sigma", 3)), float(mmd.get("weight", 0.01)), int(mmd.get("samples", 50))
    # the reference's YAML key is `learning_rate` (config/largefluid_distegnn.yaml:26); `--lr` overrides it (main.py:118-119)
    lr = args.lr if args.lr is not None else float(tc.get("learning_rate", tc.get("lr", 5e-4)))
    C = cfg["model"]["virtual_channels"]
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=float(tc.get("weight_decay", 1e-12)))
    target = inp["node_loc"] + 0.01 * inp["node_vel"]          # synthetic: one constant-velocity step
    from distegnn_b200 import train_loss
    inner = model.module if distributed else model
    n_nodes = [int(target.shape[0])]                           # batch_size 1: one graph per rank
    if cut is not None:                                        # cutoff_edges: batch_size graphs in one batch
        n_nodes = cut["node_counts"]

    t_step = []
    for step in range(args.train_steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        opt.zero_grad()
        loc_pred, X = forward()
        # utils/train.py:98-147 fused (csrc/loss.cu): node-count weighted MSE x world_size + MMD regulariser, the three
        # per-step collectives folded into one packed all-reduce (through the model's peer-memory communicator)
        loss, info = train_loss(loc_pred, target, X, inp["data_batch"], world_size=world_size, mmd_samples=samples,
                                mmd_sigma=sigma, mmd_weight=mmd_w, loc_mean=inp["loc_mean"], node_counts=n_nodes,
                                model=inner)
        logged = info["logged"]
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
        opt.step()
        torch.cuda.synchronize()
        t_step.append(time.perf_counter() - t0)
        if local_rank == 0:
            print(f"train step {step}: MSE {logged.item():.6e}  ({t_step[-1] * 1e3:.1f} ms)")
    if local_rank == 0 and len(t_step) > 2:
        print(f"train step time (median of {len(t_step)}): {sorted(t_step)[len(t_step) // 2] * 1e3:.2f} ms")


if __name__ == "__main__":
    main()
