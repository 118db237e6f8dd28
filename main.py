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
fused forward AND backward kernels under DDP.  The synthetic path has no splits, so its epoch loop is `--trajectory`'s
(below); wandb logging stays with the reference (out of scope).

`--trajectory PATH` trains and evaluates on real frames instead (distegnn_b200.frames.FrameLoader, DESIGN §18): the
config's recipe (N-body, Water-3D, Fluid113K, protein: DESIGN §27), radius / inner_radius, delta_t (N-body: frame_0,
frame_T), split_mode and cutoff_rate; every batch is assembled on the device from the raw trajectories as it is needed.  With `--rollout_steps K`
it then rolls the trained model out K steps from every validation batch and prints the per-step MSE against the recorded
frames f + Δ .. f + KΔ (DESIGN §19; `--rollout_tau` sets the velocity's time step, Water-3D defaults to Δ);
`--rollout_chamfer` adds both directions of the normalised Chamfer distance to every step's line (DESIGN §20).
`--train_noise SX,SV` trains on noisy input states (FrameLoader's `noise`, DESIGN §22); the evaluation and the rollout stay
noise-free.  `--eval_rotate` and / or `--eval_translate S` evaluate (and roll out) the validation split twice, as recorded
and with every sample rotated and translated (FrameLoader's `rotate` / `translate`, DESIGN §23), and print the relative
difference of the two mean MSEs: an equivariant model's error does not depend on the frame.  Without the flags the
synthetic path below runs unchanged.

`--trajectory PATH --epochs E` trains to convergence instead (`fit`, DESIGN §24): the reference's epoch loop
(utils/train.py:17-289) over the train, valid and test splits, with `train.accumulation_steps`, `train.scheduler: cosine`,
`train.early_stop` (`--early_stop` overrides it) and `log.test_interval`; `best_model.pth`, `last_model.pth` and
`log.json` under `log.log_dir`/exp_name.  `--checkpoint` of such a file resumes the run after its epoch (optimiser,
scheduler and the train loader's order included).  After the loop the best checkpoint's weights are restored and
`--eval_rotate` / `--eval_translate` / `--rollout_steps` run on them.

`--train_rollout K` (with --trajectory, in both loops) trains on K-step rollouts instead (DESIGN §26): a train loader of
horizon K, `differentiable_rollout` from every batch and the stepped `train_loss`, the mean of the K one-step losses;
with several ranks `rollout_grad_sum` adds the parameter gradients up before the clip.  Valid, test and the evaluations
stay one-step.

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
import json
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
                   "directory (distegnn_b200.frames): N-body .npy files, the protein's PSF and DCD, or train/ and valid/ "
                   "folders of .npz scenes; "
                   "with --rollout_steps K also a K-step rollout from every validation batch against the recorded frames")
    p.add_argument("--rollout_chamfer", action="store_true", help="(new) with --trajectory and --rollout_steps: also "
                   "print each step's Chamfer distance to the recorded frame (prediction -> record, record -> "
                   "prediction), normalised like the MSE; independent of particle identity")
    p.add_argument("--rollout_tau", type=float, default=None, help="(new) time step of a --trajectory rollout's "
                   "velocity v = (x' − x)/tau; default Δ for Water-3D (one-frame differences); for N-body "
                   "files written by `python -m distegnn_b200.nbody` Δ·sample_freq·dt from their meta file; required "
                   "otherwise for N-body and Fluid113K (physical velocities; the frame time is not in the files)")
    p.add_argument("--train_noise", type=str, default=None, help="(new) with --trajectory: SX,SV, the standard deviations "
                   "of the training noise on positions (and targets) and on velocities (FrameLoader's noise, DESIGN §22); "
                   "the train loader only, the evaluation and the rollout stay noise-free")
    p.add_argument("--eval_rotate", action="store_true", help="(new) with --trajectory: evaluate (and roll out) the "
                   "validation split a second time with every sample rotated, Haar-uniform (FrameLoader's rotate, "
                   "DESIGN §23), and print the relative difference of the mean MSEs")
    p.add_argument("--eval_translate", type=str, default=None, help="(new) with --trajectory: S >= 0, the scale of the "
                   "second evaluation's per-sample translation S·N(0, I) (FrameLoader's translate, DESIGN §23)")
    p.add_argument("--epochs", type=int, default=None, help="(new) with --trajectory: E >= 1 epochs of the reference's "
                   "epoch loop (utils/train.py) over train/valid/test, with best/last checkpoints, early stopping and "
                   "resume from --checkpoint (DESIGN §24)")
    p.add_argument("--train_rollout", type=int, default=None, help="(new) with --trajectory: train on K-step rollouts "
                   "(differentiable_rollout and the stepped train_loss, the mean of the K one-step losses against the "
                   "recorded frames, DESIGN §26); valid, test and the evaluations stay one-step")
    return p.parse_args()


def nbody_tag(cfg):
    """The N-body file tag, without its leading underscore: the config's `data.nbody_tag` (e.g. charged0_5_0_1 for
    files written by `nbody.generate_dataset(n_isolated=0, n_stick=5)`), by default charged100_0_0_1."""
    return str((cfg.get("data") or {}).get("nbody_tag", "charged100_0_0_1"))


def split_files(path, recipe, part, tag="charged100_0_0_1"):
    """The files of split `part` under `path`: N-body's loc_`part`_`tag`.npy, the protein trajectory in `path` (one PSF
    and one DCD, or one .npz: `protein.find_files`; the same files for every split), or `path`/`part`/*.npz; [] if
    missing."""
    import glob
    if recipe == "protein":
        from distegnn_b200.protein import find_files
        return find_files(path)
    if recipe == "nbody":
        f = os.path.join(path, f"loc_{part}_{tag}.npy")
        return [f] if os.path.exists(f) else []
    return sorted(glob.glob(os.path.join(path, part, "*.npz")))


def epochs_of(args, cfg):
    """--epochs E, or None; exits with a message when it cannot run: no --trajectory, --train_steps given, E < 1, or
    the trajectory has no valid or no test split."""
    if args.epochs is None:
        return None
    msg = None
    if not args.trajectory:
        msg = "used with --trajectory"
    elif args.train_steps:
        msg = "used without --train_steps (the epochs set the number of steps)"
    elif args.epochs < 1:
        msg = ">= 1"
    else:
        recipe = recipe_of_config(cfg)[0]
        missing = [part for part in ("valid", "test") if not split_files(args.trajectory, recipe, part, nbody_tag(cfg))]
        if missing:
            msg = f"used with a trajectory that has valid and test splits ({args.trajectory} has no {' or '.join(missing)})"
    if msg is not None:
        if int(os.environ.get("LOCAL_RANK", "0")) == 0:
            print(f"--epochs {args.epochs}: must be {msg}", flush=True)
        sys.exit(2)
    return args.epochs


def train_noise_of(args):
    """--train_noise SX,SV as (σ_x, σ_v), or None; exits with a message on a malformed or negative value."""
    if args.train_noise is None:
        return None
    import math
    msg = None
    try:
        sx, sv = (float(v) for v in args.train_noise.split(","))
    except ValueError:
        msg = "two comma-separated numbers SX,SV"
    else:
        if not (math.isfinite(sx) and math.isfinite(sv) and sx >= 0 and sv >= 0):
            msg = "finite and >= 0"
    if msg is None and not args.trajectory:
        msg = "used with --trajectory"
    if msg is not None:
        if int(os.environ.get("LOCAL_RANK", "0")) == 0:
            print(f"--train_noise {args.train_noise!r}: must be {msg}", flush=True)
        sys.exit(2)
    return sx, sv


def eval_transform_of(args):
    """--eval_rotate / --eval_translate S as (rotate, translate), or None; exits with a message on a malformed or
    negative scale."""
    if not args.eval_rotate and args.eval_translate is None:
        return None
    import math
    msg, t = None, 0.0
    if args.eval_translate is not None:
        try:
            t = float(args.eval_translate)
        except ValueError:
            msg = "a number"
        else:
            if not (math.isfinite(t) and t >= 0):
                msg = "finite and >= 0"
    if msg is None and not args.trajectory:
        msg = "used with --trajectory"
    if msg is not None:
        if int(os.environ.get("LOCAL_RANK", "0")) == 0:
            what = f"--eval_translate {args.eval_translate!r}" if args.eval_translate is not None else "--eval_rotate"
            print(f"{what}: must be {msg}", flush=True)
        sys.exit(2)
    return bool(args.eval_rotate), t


def split_samples(path, cfg, part, horizon=1):
    """(trajectories, (scene, frame) samples) of split `part` under `path` with the config's recipe, or None without
    files.  Water-3D / Fluid113K: the frame draw is capped so that every sample holds `horizon` steps of delta_t frames;
    SystemExit with a message when the shortest scene cannot hold them."""
    from distegnn_b200.frames import load_nbody, load_scenes, sample_list
    d = cfg["data"]
    recipe, frame_0, delta = recipe_of_config(cfg)
    files = split_files(path, recipe, part, nbody_tag(cfg))
    if not files:
        return None
    if recipe == "protein":                                    # every frame of the split's fixed range
        from distegnn_b200.protein import load_protein
        traj = load_protein(files, backbone=bool(d.get("backbone", True)))
        return traj, sample_list(traj, delta_t=delta, split=part)
    traj = load_nbody(path, part, nbody_tag(cfg)) if recipe == "nbody" else load_scenes(files, recipe)
    kw = {}
    if recipe != "nbody":
        shortest = min(sc.n_frames for sc in traj.scenes)
        kw["max_frame"] = min(traj.recipe.max_frame, shortest - 1 - max(horizon * delta, 1))
        if horizon > 1 and kw["max_frame"] < 0:
            raise SystemExit(f"--trajectory {path}/{part}: the shortest scene has {shortest} frames; it cannot hold "
                             f"{horizon} step(s) of delta_t={delta} frames after any frame")
    return traj, sample_list(traj, seed=int(cfg.get("seed", 0)), max_samples=d.get("max_samples"), delta_t=delta,
                             frame_0=frame_0, **kw)


def protein_test_transform(path, cfg):
    """FrameLoader's rotate / translate keywords for the protein recipe's test split: `data.test_rot` a Haar-uniform
    rotation per sample, `data.test_trans` a translation S·N(0, I) with S half the edge of the DCD's cubic unit cell
    (the reference's randn(3)·box/2, process_dataset.py:162-174).  ValueError when test_trans is set and the trajectory
    has no single cubic cell over the test frames."""
    from distegnn_b200.frames import PROTEIN_SPLITS
    from distegnn_b200.protein import cubic_edge, read_dcd
    d = cfg["data"]
    rot, trans = bool(d.get("test_rot", False)), bool(d.get("test_trans", False))
    out = dict(rotate=True) if rot else {}
    if trans:
        dcd = [f for f in split_files(path, "protein", "test") if f.endswith(".dcd")]
        if not dcd:
            raise ValueError(f"data.test_trans needs a DCD with a cubic unit cell (the translation is box/2·N(0, I)); "
                             f"{path} has none")
        try:                                                   # the cell of every sample's frame t
            out["translate"] = cubic_edge(read_dcd(dcd[0]), range(*PROTEIN_SPLITS["test"])) / 2
        except ValueError as e:
            raise ValueError(f"data.test_trans needs a cubic unit cell (the translation is box/2·N(0, I)): {e}") from None
    return out


def protein_check(args, cfg):
    """The protein recipe with --trajectory: exits with code 2 and a message, before any CUDA work, when the trajectory
    is missing, cannot hold every sample of the three splits (delta_t frames after the last), or cannot give the test
    split's translation (`protein_test_transform`)."""
    if not args.trajectory or recipe_of_config(cfg)[0] != "protein":
        return
    from distegnn_b200.frames import check_samples
    msg = None
    try:
        if not split_files(args.trajectory, "protein", "train"):
            msg = (f"--trajectory {args.trajectory}: no protein trajectory (one .psf and one .dcd, or one .npz with "
                   "position and charges)")
        else:
            for part in ("train", "valid", "test"):
                traj, samples = split_samples(args.trajectory, cfg, part)
                check_samples(traj, samples, recipe_of_config(cfg)[2])
            protein_test_transform(args.trajectory, cfg)
    except (OSError, ValueError) as e:
        msg = f"--trajectory {args.trajectory}: {e}"
    if msg is not None:
        if int(os.environ.get("LOCAL_RANK", "0")) == 0:
            print(msg, flush=True)
        sys.exit(2)


def train_rollout_of(args, cfg):
    """--train_rollout K, or None; exits with code 2 and a message, before any CUDA work, when it cannot run: K < 1, no
    --trajectory, a train split whose samples cannot hold K steps (frame_loaders' horizon check), or no rollout time
    step (rollout_args' rule)."""
    K = args.train_rollout
    if K is None:
        return None
    msg = None
    if K < 1:
        msg = ">= 1"
    elif not args.trajectory:
        msg = "used with --trajectory (the synthetic path has no recorded frames to train against)"
    else:
        from distegnn_b200.frames import check_samples
        try:
            found = split_samples(args.trajectory, cfg, "train", horizon=K)
            if found is not None:
                check_samples(found[0], found[1], recipe_of_config(cfg)[2], K)
        except (SystemExit, ValueError) as e:
            msg = f"used with a train split whose samples hold {K} step(s): {e}"
    if msg is not None:
        if int(os.environ.get("LOCAL_RANK", "0")) == 0:
            print(f"--train_rollout {K}: must be {msg}", flush=True)
        sys.exit(2)
    rollout_args(args, cfg, int(os.environ.get("LOCAL_RANK", "0")), K, "--train_rollout")
    return K


def main():
    args = parse()
    noise = train_noise_of(args)
    transform = eval_transform_of(args)
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
    if args.outer_radius is not None:                          # the METIS split's graph radius (reference main.py)
        cfg["data"]["outer_radius"] = args.outer_radius
    if args.virtual_channels is not None:
        cfg["model"]["virtual_channels"] = args.virtual_channels
    protein_check(args, cfg)
    epochs = epochs_of(args, cfg)
    train_rollout = train_rollout_of(args, cfg)

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
    ignored = [n for n, v in (("--wandb", args.wandb), ("--early_stop", None if epochs else args.early_stop),
                              ("--cutoff_rate", None if cutoff_mode else args.cutoff_rate),
                              ("--outer_radius", None if cfg["data"].get("split_mode") == "metis" else args.outer_radius))
               if v]
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
    ck, state = cfg["model"].get("checkpoint"), None
    if ck:
        state = torch.load(ck, map_location=f"cuda:{local_rank}")
        sd = state.get("model_state_dict", state)
        sd = {k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}
        model.load_state_dict(sd)
    if distributed:                                            # reference main.py:194-196
        model = DistributedDataParallel(model, device_ids=[local_rank], find_unused_parameters=True)
    model.eval()
    if args.trajectory:
        if epochs:
            trajectory_fit(args, cfg, model, world_size, local_rank, distributed, rate, noise, transform, state,
                           train_rollout)
        else:
            trajectory_run(args, cfg, model, world_size, local_rank, distributed, rate, noise, transform, train_rollout)
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
    if world_size > 1 and split == "metis":
        outer = metis_outer_radius(d, local_rank)
        if local_rank == 0:
            print(f"split_mode='metis': METIS (recursive bisection) on the graph of outer_radius={outer}")
    cut = None
    if cutoff_mode:
        inp, cut = cutoff_inputs(w, int(d.get("batch_size", 1)), cfg.get("seed", 0), rate, local_rank)
        n_r, e_r = inp["node_loc"].shape[0], cut["kept"]
    else:
        part = synth.make_partitions(w, world_size=world_size, split_mode=split, seed=cfg.get("seed", 0),
                                     only_rank=local_rank, device=torch.device("cuda", local_rank),
                                     outer_radius=d.get("outer_radius"))[local_rank]
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
    recipe = "nbody" if ds.startswith("nbody") else "water3d" if ds.startswith("water") else \
        "protein" if ds.startswith("protein") else "largefluid"
    if recipe == "nbody":
        frame_0, frame_T = int(d.get("frame_0", 30)), int(d.get("frame_T", 40))
        return recipe, frame_0, frame_T - frame_0
    return recipe, 0, int(d.get("delta_t", 1))


def frame_loaders(path, cfg, world_size, rank, device, rate, horizon=1, parts=("train", "valid"), noise=None,
                  transform=None):
    """FrameLoaders over the raw trajectories under `path` with the config's recipe (datasets/process_dataset.py):
    N-body (`dataset_name: nbody*`, the reference's loc_/vel_/charges_ .npy files, frame_0 / frame_T), Water-3D or
    Fluid113K (`path`/train/*.npz, `path`/valid/*.npz, `path`/test/*.npz).  Only the train loader shuffles (the
    reference's same-seed sampler); a split without files gives None.  cutoff_edges mode: one graph per sample, radius = data.radius
    (−1 fully connected; Water-3D: the reference's hard-coded 0.035, :264), then the cutoff.  distribute mode: the
    sample split over the ranks by split_mode (metis on the graph of data.outer_radius), a radius graph per partition
    with inner_radius.  `horizon` K: every sample holds frames f + Δ .. f + KΔ (the frame draw is capped for that; a fixed
    N-body frame_0 that cannot hold them exits with a message).  `noise` (σ_x, σ_v) goes to the train loader only;
    `transform` (rotate, translate) to every loader built (the same samples as without it: a rotated and translated
    copy of the split); without it the protein recipe's test loader takes data.test_rot / data.test_trans
    (`protein_test_transform`).  Returns (recipe name, {part: loader or None})."""
    from distegnn_b200.frames import FrameLoader
    d = cfg["data"]
    recipe, _, delta = recipe_of_config(cfg)
    cutoff_mode = rate is not None
    if cutoff_mode:
        radius = 0.035 if recipe == "water3d" else d.get("radius", -1)
    else:
        radius = d.get("inner_radius")
    split = str(d.get("split_mode", "random"))
    outer = metis_outer_radius(d, rank) if split == "metis" and world_size > 1 else None
    seed, bs = int(cfg.get("seed", 0)), int(d.get("batch_size", 1))
    xf = {} if transform is None else dict(rotate=transform[0], translate=transform[1])
    out = {}
    for part in parts:
        found = split_samples(path, cfg, part, horizon)
        if found is None:
            out[part] = None
            continue
        traj, samples = found
        if recipe == "protein" and part == "test" and transform is None:
            xf = protein_test_transform(path, cfg)
        out[part] = FrameLoader(traj, samples, delta_t=delta, radius=radius, batch_size=bs, shuffle=part == "train",
                                seed=seed, device=device, world_size=world_size, rank=rank, split_mode=split,
                                cutoff_rate=rate or 0.0, horizon=horizon, noise=noise if part == "train" else None,
                                outer_radius=outer, **xf)
    if "train" in parts and out["train"] is None:
        raise SystemExit(f"--trajectory {path}: no training data for recipe {recipe!r}")
    return recipe, out


def metis_outer_radius(d, rank):
    """data.outer_radius (or --outer_radius), the radius of the graph the metis split partitions; exits with code 2 and
    a message when it is missing or not > 0."""
    r = d.get("outer_radius")
    if r is None or not float(r) > 0:
        if rank == 0:
            print(f"split_mode='metis' needs data.outer_radius > 0 (or --outer_radius), the radius of the graph METIS "
                  f"partitions (got {r!r})", flush=True)
        sys.exit(2)
    return float(r)


def rollout_args(args, cfg, local_rank, K=None, flag="--rollout_steps"):
    """(recipe, K, tau) of `--rollout_steps K` (or of `flag` with K steps) on the trajectory; exits with a message before
    any training when the rollout could not run (no `--rollout_tau` for a recipe with physical velocities)."""
    recipe, _, delta = recipe_of_config(cfg)
    K = args.rollout_steps if K is None else K
    tau = args.rollout_tau if args.rollout_tau is not None else \
        (float(delta) if recipe in ("water3d", "protein") else None)
    if tau is None and recipe == "nbody" and args.trajectory:   # files written by distegnn_b200.nbody record their dt
        from distegnn_b200.nbody import meta_rollout_tau
        tau = meta_rollout_tau(args.trajectory, delta, "_" + nbody_tag(cfg))
    if K > 0 and tau is None:
        if local_rank == 0:
            print(f"{flag} with --trajectory on {recipe!r} needs --rollout_tau: its velocities are physical and "
                  "the frame time is not in the files (Water-3D defaults to delta_t; N-body files written by "
                  "distegnn_b200.nbody default to delta_t·sample_freq·dt from their meta file)", flush=True)
        sys.exit(2)
    return recipe, K, tau


def trajectory_loss(cfg, model, world_size, distributed):
    """loss_of(kw, ex, accumulation_steps=1) -> (loss, info) of one FrameLoader batch: the model's positional call
    (utils/train.py:63-71) and the fused `train_loss` with the config's MMD settings (utils/train.py:98-150)."""
    from distegnn_b200 import train_loss
    mmd = (cfg.get("train", {}) or {}).get("mmd", {}) or {}
    inner = model.module if distributed else model
    use_attr = cfg["model"]["node_attr_nf"] > 0

    def loss_of(kw, ex, accumulation_steps=1):
        pred, X = model(kw["node_feat"], kw["node_loc"], kw["node_vel"], kw["loc_mean"], kw["edge_index"],
                        kw["data_batch"], kw["edge_attr"], kw["node_attr"] if use_attr else None)
        return train_loss(pred, ex["target"], X, kw["data_batch"], world_size=world_size,
                          mmd_samples=int(mmd.get("samples", 50)), mmd_sigma=float(mmd.get("sigma", 3)),
                          mmd_weight=float(mmd.get("weight", 0.01)), accumulation_steps=accumulation_steps,
                          loc_mean=kw["loc_mean"], node_counts=ex["node_counts"], model=inner)
    return loss_of


def trajectory_rollout_loss(cfg, model, world_size, distributed, train_loader, recipe, tau, steps):
    """loss_of(kw, ex, accumulation_steps=1) -> (loss, info) of `--train_rollout K` (DESIGN §26).  With gradients
    enabled: a K-step `differentiable_rollout` from the batch's state, with `rollout_eval`'s graph arguments (the train
    loader's radius, or its complete graph and cutoff rate) and `tau`, then the stepped `train_loss` of the trajectory
    and the virtual coordinates against ex["targets"] [K,M,3]: the mean over the steps of the one-step loss.  Under
    no_grad (fit's valid and test passes, the evaluations): `trajectory_loss`'s one-step loss, so that those losses mean
    what they mean without the flag.  With several ranks the parameter gradients are this rank's only: `rollout_grad_sum`
    adds them up once per optimiser step."""
    from distegnn_b200 import differentiable_rollout, train_loss
    one_step = trajectory_loss(cfg, model, world_size, distributed)
    mmd = (cfg.get("train", {}) or {}).get("mmd", {}) or {}
    inner = model.module if distributed else model
    use_attr = cfg["model"]["node_attr_nf"] > 0
    ld = train_loader

    def loss_of(kw, ex, accumulation_steps=1):
        if not torch.is_grad_enabled():
            return one_step(kw, ex, accumulation_steps)
        if ld.radius is not None:
            g = dict(radius=ld.radius)
        else:                                                  # fully connected: the candidates, cut again every step
            g = dict(graph=ld.complete_graph(tuple(ex["node_counts"])) if ld.cutoff_rate > 0 else kw["edge_index"])
        res = differentiable_rollout(model, kw["node_feat"], kw["node_loc"], kw["node_vel"], kw["loc_mean"],
                                     kw["data_batch"], kw["node_attr"] if use_attr else None, steps=steps, tau=tau,
                                     speed_col=SPEED_COL[recipe], cutoff_rate=ld.cutoff_rate, **g)
        return train_loss(res.trajectory, ex["targets"], res.virtual_locs, kw["data_batch"], world_size=world_size,
                          mmd_samples=int(mmd.get("samples", 50)), mmd_sigma=float(mmd.get("sigma", 3)),
                          mmd_weight=float(mmd.get("weight", 0.01)), accumulation_steps=accumulation_steps,
                          loc_mean=kw["loc_mean"], node_counts=ex["node_counts"], model=inner)
    return loss_of


def rollout_grad_sum(model, world_size):
    """A callable that sums the parameter gradients over the ranks in one all-reduce, each divided by world_size first:
    what DDP's reducer does for the one-step path, which it cannot do for a differentiable rollout (it never sees that
    call).  Run once per optimiser step, after the last accumulated backward and before clipping; with the train
    loss's world·n_r/Σn weighting, K = 1 then gives the one-step path's gradients."""
    params = list(model.parameters())

    def grad_sum():
        have = [p for p in params if p.grad is not None]       # the same set on every rank: the same model and steps
        if not have:
            return
        flat = torch.cat([p.grad.reshape(-1) for p in have]).div_(world_size)
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        off = 0
        for p in have:
            p.grad.copy_(flat[off:off + p.numel()].view_as(p.grad))
            off += p.numel()
    return grad_sum


def trajectory_run(args, cfg, model, world_size, local_rank, distributed, rate, noise=None, transform=None,
                   train_rollout=None):
    """--trajectory: `--train_steps` optimisation steps (at least one epoch's worth if 0 is given: one pass) of the
    reference's training step on batches from FrameLoader (with `noise` on its inputs), then `trajectory_eval`.  With
    `train_rollout` K every step trains on a K-step rollout (`trajectory_rollout_loss`) from a train loader of horizon K;
    the evaluation stays one-step."""
    recipe, K, tau = rollout_args(args, cfg, local_rank)
    dev = torch.device("cuda", local_rank)
    recipe, loaders = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, noise=noise)
    tc = cfg.get("train", {}) or {}
    lr = args.lr if args.lr is not None else float(tc.get("learning_rate", tc.get("lr", 5e-4)))
    opt = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=float(tc.get("weight_decay", 1e-12)))
    loss_of = trajectory_loss(cfg, model, world_size, distributed)
    train_ld, train_of, grad_sum, what = loaders["train"], loss_of, None, "MSE"
    if train_rollout is not None:                              # the one-step train loader stays for the evaluation
        _, _, r_tau = rollout_args(args, cfg, local_rank, train_rollout, "--train_rollout")
        train_ld = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, horizon=train_rollout,
                                 parts=("train",), noise=noise)[1]["train"]
        train_of = trajectory_rollout_loss(cfg, model, world_size, distributed, train_ld, recipe, r_tau, train_rollout)
        grad_sum = rollout_grad_sum(model, world_size) if distributed else None
        what = f"{train_rollout}-step rollout mean MSE"

    steps = args.train_steps or len(train_ld)
    model.train()
    done, t0 = 0, time.perf_counter()
    while done < steps:
        for kw, ex in train_ld:
            opt.zero_grad()
            loss, info = train_of(kw, ex)
            loss.backward()
            if grad_sum is not None:
                grad_sum()
            torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
            opt.step()
            done += 1
            if local_rank == 0 and (done % 10 == 0 or done == steps):
                print(f"[{recipe}] train step {done}: {what} {info['logged'].item():.6e}", flush=True)
            if done == steps:
                break
    torch.cuda.synchronize()
    if local_rank == 0:
        print(f"[{recipe}] {steps} train steps on raw frames: {(time.perf_counter() - t0) / steps * 1e3:.2f} ms/step")
    trajectory_eval(args, cfg, model, world_size, local_rank, rate, loaders, loss_of, noise, transform)


def trajectory_eval(args, cfg, model, world_size, local_rank, rate, loaders, loss_of, noise=None, transform=None):
    """The mean MSE over the validation batches (noise-free; the train split without a valid batch); with `transform`
    (rotate, translate) also over the same batches rigidly transformed, and the relative difference of the two; with
    `--rollout_steps K` the rollout evaluation (`rollout_eval`), plain and transformed."""
    recipe, K, tau = rollout_args(args, cfg, local_rank)
    dev = torch.device("cuda", local_rank)
    ev = loaders["valid"]
    if not ev:                                                 # no valid split or no batch in it: the train split, clean
        ev = loaders["train"] if noise is None else \
            frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, parts=("train",))[1]["train"]
    model.eval()
    part = "valid" if loaders["valid"] else "train"

    def mean_mse(ld):
        tot, n = 0.0, 0
        with torch.no_grad():
            for kw, ex in ld:
                _, info = loss_of(kw, ex)
                tot, n = tot + float(info["logged"]), n + 1
        return tot / max(n, 1), n

    plain, n = mean_mse(ev)
    if local_rank == 0:
        print(f"[{recipe}] evaluation over {n} batches ({part}): mean MSE {plain:.6e}")
    if transform is not None:                                  # the same samples, batches and split, transformed
        moved, n = mean_mse(frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, parts=(part,),
                                          transform=transform)[1][part])
        if local_rank == 0:
            rel = (moved - plain) / plain if plain != 0 else float("nan")
            print(f"[{recipe}] evaluation over {n} batches ({part}, {transform_label(transform)}): mean MSE "
                  f"{moved:.6e}, relative difference {rel:+.3e}", flush=True)
    if K > 0:
        rollout_eval(args, cfg, model, world_size, local_rank, rate, recipe, tau)
        if transform is not None:
            rollout_eval(args, cfg, model, world_size, local_rank, rate, recipe, tau, transform)


def reference_clips(cfg, world_size):
    """The reference's clip condition (utils/train.py:153): FastEGNN with several ranks, or the dataset named exactly
    `LargeFluid` (the shipped Fluid113K config is not, so one GPU does not clip it)."""
    return (world_size > 1 or cfg["data"].get("dataset_name") == "LargeFluid") and \
        cfg["model"].get("model_name") == "FastEGNN"


def exp_name_of(cfg, world_size, rate=None):
    """The reference's experiment name (main.py:147-157, the FastEGNN branches) with a local-time suffix."""
    d, m = cfg["data"], cfg["model"]
    suffix = time.strftime("%Y-%m-%d_%H-%M-%S", time.localtime(time.time()))
    if rate is None:                                           # accelerate_mode: distribute
        return (f"{d.get('dataset_name')}_{d.get('split_mode')}_{m['model_name']}_{d.get('outer_radius')}_"
                f"{d.get('inner_radius')}_{world_size}_{m['virtual_channels']}_{suffix}")
    return f"{d.get('dataset_name')}_{m['model_name']}_{d.get('radius')}_{rate:.3f}_{m['virtual_channels']}_{world_size}_{suffix}"


def fit(model, opt, scheduler, loaders, loss_of, cfg, epochs, start_epoch=0, world_size=1, rank=0, out_dir=".",
        before_step=None, train_note=""):
    """The reference's epoch loop (utils/train.py:17-289, DESIGN §24): epochs start_epoch + 1 .. `epochs`, each a train
    pass, and every `log.test_interval` epochs a valid and a test pass; `best_model.pth` (strictly lower valid loss),
    `last_model.pth` (every evaluation epoch) and `log/log.json` under `out_dir`, written by rank 0 only.

    loaders     {"train", "valid", "test"}: iterables of (forward kwargs, extras with "n_graphs") with len(); the train
                loader as constructed (its epoch 0): a resumed run calls its `batches()` `start_epoch` times first, so
                its order (and FrameLoader's noise, keyed by the loader's epoch) continues as without the interruption
    loss_of     (kw, ex, accumulation_steps) -> (loss, info), info["logged"] a 0-dim tensor: the batch's logged MSE
    cfg         the run's config (a plain dict, stored in every checkpoint and in log.json): train.accumulation_steps
                (1), train.early_stop (None: never), log.test_interval (1), and the clip condition `reference_clips`
    before_step None, or a callable run once per optimiser step after the last accumulated backward and before the
                clip and the step (`rollout_grad_sum`: the rank sum of a differentiable rollout's gradients)
    train_note  appended to every train pass's loss line (what the train loss is, when it is not the one-step MSE)
    Returns (best_log_dict, log_dict) on rank 0, (None, None) on the others."""
    tc, lc = cfg.get("train") or {}, cfg.get("log") or {}
    A, interval = int(tc.get("accumulation_steps", 1)), int(lc.get("test_interval", 1))
    early_stop = tc.get("early_stop")
    clip = reference_clips(cfg, world_size)
    dev = next(model.parameters()).device
    for _ in range(start_epoch):
        loaders["train"].batches()
    if rank == 0:
        log_dict = {"epochs": [], "loss": [], "loss_train": []}
        best = {"epoch_index": 0, "loss_valid": 1e8, "loss_test": 1e8, "loss_train": 1e8}
        log_dir, sd_dir = os.path.join(out_dir, "log"), os.path.join(out_dir, "state_dict")
        os.makedirs(log_dir, exist_ok=True)
        os.makedirs(sd_dir, exist_ok=True)
        print(f"logs and checkpoints: {out_dir}", flush=True)
        t0 = time.perf_counter()
    stop = torch.zeros((), dtype=torch.int64, device=dev)

    def one_pass(tag, epoch):                                  # train.py:17-168
        train = tag == "train"
        if train:
            model.train()
            opt.zero_grad()
        else:
            model.eval()
        tot, graphs = torch.zeros((), dtype=torch.float64, device=dev), 0
        with torch.set_grad_enabled(train):
            for step, (kw, ex) in enumerate(loaders[tag]):
                loss, info = loss_of(kw, ex, A if train else 1)
                tot += info["logged"].double() * ex["n_graphs"]
                graphs += ex["n_graphs"]
                if train:
                    loss.backward()
                    if (step + 1) % A == 0:
                        if before_step is not None:
                            before_step()
                        if clip:
                            torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
                        opt.step()
                        if scheduler is not None:
                            scheduler.step()
                        opt.zero_grad()
        value = float(tot) / graphs if graphs else float("nan")    # the one host read of the pass
        if rank == 0:
            print(f"{'' if train else '==> '}{tag} epoch: {epoch}, avg loss: {value:.5f}{train_note if train else ''}",
                  flush=True)
        return value

    for epoch in range(start_epoch + 1, epochs + 1):
        loss_train = one_pass("train", epoch)
        if rank == 0:
            log_dict["loss_train"].append(loss_train)
        if epoch % interval == 0:
            loss_valid, loss_test = one_pass("valid", epoch), one_pass("test", epoch)
            if rank == 0:
                log_dict["epochs"].append(epoch)
                log_dict["loss"].append(loss_test)
                state = {"epoch": epoch, "model_state_dict": model.state_dict(),
                         "optimizer_state_dict": opt.state_dict(),
                         "scheduler_state_dict": None if scheduler is None else scheduler.state_dict(),
                         "loss_train": loss_train, "loss_valid": loss_valid, "loss_test": loss_test, "config": cfg}
                if loss_valid < best["loss_valid"]:
                    best = {"epoch_index": epoch, "loss_valid": loss_valid, "loss_test": loss_test,
                            "loss_train": loss_train}
                    torch.save(state, os.path.join(sd_dir, "best_model.pth"))
                print(best_line(best), flush=True)
                torch.save(state, os.path.join(sd_dir, "last_model.pth"))
                if early_stop is not None and epoch - best["epoch_index"] >= early_stop:
                    best["early_stop"] = epoch
                    print(f"Early stopped! Epoch: {epoch}", flush=True)
                    stop.fill_(1)
            if world_size > 1:                                 # every rank leaves at rank 0's epoch
                import torch.distributed as dist
                dist.all_reduce(stop, op=dist.ReduceOp.MAX)
        if rank == 0:
            best["time_cost"] = time.perf_counter() - t0
            with open(os.path.join(log_dir, "log.json"), "w") as f:
                f.write(json.dumps([best, log_dict, cfg], indent=4))
        if epoch % interval == 0 and int(stop):
            break
    return (best, log_dict) if rank == 0 else (None, None)


def best_line(best):
    return (f"*** Best Valid Loss: {best['loss_valid']:.5f} | Best Test Loss: {best['loss_test']:.5f} | "
            f"Best Epoch Index: {best['epoch_index']}")


def optimizer_of(model, cfg, epochs, n_batches):
    """The reference's Adam (train.learning_rate, train.weight_decay) and, for train.scheduler: cosine, its
    CosineAnnealingLR over the run's optimiser steps, T_max = epochs·n_batches // accumulation_steps, eta_min 1e-8
    (main.py:197-202); any other scheduler value: None."""
    tc = cfg.get("train") or {}
    lr = float(tc.get("learning_rate", tc.get("lr", 5e-4)))
    opt = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=float(tc.get("weight_decay", 1e-12)))
    if tc.get("scheduler") != "cosine":
        return opt, None
    t_max = epochs * n_batches // int(tc.get("accumulation_steps", 1))
    return opt, torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=t_max, eta_min=1e-8)


def trajectory_fit(args, cfg, model, world_size, local_rank, distributed, rate, noise=None, transform=None, state=None,
                   train_rollout=None):
    """--trajectory with --epochs E: `fit` on FrameLoader's train (with `noise`), valid and test splits, the reference's
    Adam and optional cosine schedule (main.py:197-202); `state`, a checkpoint with an `epoch` key, resumes after that
    epoch (main.py:208-220).  Then the best checkpoint's weights, and `trajectory_eval` on them.  With `train_rollout` K
    the train passes run on K-step rollouts from a train loader of horizon K (`trajectory_rollout_loss`, the ranks'
    gradients summed by `rollout_grad_sum`); valid and test stay one-step, and K goes into the config as
    train.train_rollout."""
    recipe, _, _ = rollout_args(args, cfg, local_rank)
    dev = torch.device("cuda", local_rank)
    _, loaders = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, parts=("train", "valid", "test"),
                               noise=noise)
    if train_rollout is not None:
        loaders["train"] = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, horizon=train_rollout,
                                         parts=("train",), noise=noise)[1]["train"]
    for part, ld in loaders.items():
        if not ld:
            if local_rank == 0:
                print(f"--epochs: the {part} split of {args.trajectory} has fewer samples than batch_size "
                      f"{ld.batch_size}: no batch", flush=True)
            sys.exit(2)
    cfg = json.loads(json.dumps(cfg))                          # a plain dict: the checkpoints' and log.json's config
    tc = cfg["train"] = dict(cfg.get("train") or {})
    if args.lr is not None:
        tc["learning_rate"] = args.lr
    if args.early_stop is not None:
        tc["early_stop"] = args.early_stop
    tc["epochs"] = args.epochs
    if train_rollout is not None:
        tc["train_rollout"] = train_rollout
    cfg["data"]["world_size"] = world_size
    opt, scheduler = optimizer_of(model, cfg, args.epochs, len(loaders["train"]))
    start = 0
    if state is not None and "epoch" in state:
        start = int(state["epoch"])
        opt.load_state_dict(state["optimizer_state_dict"])
        if scheduler is not None:
            scheduler.load_state_dict(state["scheduler_state_dict"])
        if local_rank == 0:
            print(f"resuming after epoch {start} of {args.checkpoint}", flush=True)
    name = [exp_name_of(cfg, world_size, rate)]
    if distributed:                                            # one directory: rank 0's clock
        dist.broadcast_object_list(name, src=0)
    cfg["log"] = dict(cfg.get("log") or {}, exp_name=name[0])
    out_dir = os.path.join(cfg["log"].get("log_dir", "./logs"), name[0])
    loss_of = trajectory_loss(cfg, model, world_size, distributed)
    extra = {}
    if train_rollout is not None:
        _, _, r_tau = rollout_args(args, cfg, local_rank, train_rollout, "--train_rollout")
        extra = dict(train_note=f" (mean over {train_rollout} rollout steps)",
                     before_step=rollout_grad_sum(model, world_size) if distributed else None)
        train_of = trajectory_rollout_loss(cfg, model, world_size, distributed, loaders["train"], recipe, r_tau,
                                           train_rollout)
    else:
        train_of = loss_of
    best, _ = fit(model, opt, scheduler, loaders, train_of, cfg, args.epochs, start, world_size, local_rank, out_dir,
                  **extra)
    if distributed:
        dist.barrier()
    path = os.path.join(out_dir, "state_dict", "best_model.pth")
    if not os.path.exists(path):
        if local_rank == 0:
            print(f"[{recipe}] no evaluation epoch in {start + 1} .. {args.epochs}: no best model", flush=True)
        return
    model.load_state_dict(torch.load(path, map_location=dev)["model_state_dict"])
    if local_rank == 0:
        print(f"[{recipe}] best model restored: {best_line(best)}", flush=True)
    if transform is not None or args.rollout_steps > 0:
        trajectory_eval(args, cfg, model, world_size, local_rank, rate, loaders, loss_of, noise, transform)


def transform_label(transform):
    rotate, translate = transform
    return " and ".join((["rotated"] if rotate else []) + ([f"translated by {translate:g}"] if translate else [])) \
        or "untransformed"


# the |v| column of each recipe's node features (distegnn_b200/frames.py): N-body, Water-3D, protein [‖v‖, ·],
# Fluid113K [·, ·, ‖v‖]
SPEED_COL = {"nbody": 0, "water3d": 0, "largefluid": 2, "protein": 0}


def rollout_eval(args, cfg, model, world_size, local_rank, rate, recipe, tau, transform=None):
    """--trajectory with --rollout_steps K: a K-step `rollout(targets=...)` from every batch of the valid split (the
    train split without one), through a FrameLoader with horizon K and the config's radius and cutoff rate; prints the
    per-step MSE averaged over the batches, each weighted by its graph count (utils/train.py:112-114, 166).  With
    --rollout_chamfer each line also carries the two directions of `chamfer_mse`, averaged the same way.  `transform`
    (rotate, translate): the split rigidly transformed (its targets too), lines marked with the transform."""
    from distegnn_b200 import rollout
    K = args.rollout_steps
    dev = torch.device("cuda", local_rank)
    part = "valid"
    try:
        _, lds = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, horizon=K, parts=(part,),
                               transform=transform)
        if lds[part] is None:
            part = "train"
            _, lds = frame_loaders(args.trajectory, cfg, world_size, local_rank, dev, rate, horizon=K, parts=(part,),
                                   transform=transform)
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
        which = part if transform is None else f"{part}, {transform_label(transform)}"
        print(f"[{recipe}] rollout evaluation over {n} batches ({which}), {K} steps, tau={tau:g}: "
              f"{dt / max(n * K, 1) * 1e3:.2f} ms/step", flush=True)
        tag = "" if transform is None else f" ({transform_label(transform)})"
        for t, v in enumerate(mse):
            extra = f", Chamfer pred->rec {ch[t][0]:.6e}, rec->pred {ch[t][1]:.6e}" if args.rollout_chamfer else ""
            print(f"[{recipe}] rollout step {t + 1}{tag}: MSE {v:.6e}{extra}", flush=True)


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
