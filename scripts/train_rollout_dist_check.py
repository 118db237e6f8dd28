"""Two-rank check of `--train_rollout` (DESIGN §26), run under torchrun with 2 processes on 2 GPUs:

    python -m torch.distributed.run --nproc-per-node 2 scripts/train_rollout_dist_check.py

Every rank writes the same seeded Water-3D-style scenes to its own temporary directory and takes its partition of the
first train batch.  (1) K = 1: the rollout loss's gradients after `rollout_grad_sum` against the one-step path's under
DistributedDataParallel, same weights and MMD samples: within 1e-5 relative, in the norm over all parameters.  (2) K = 3:
after one optimiser step (rank sum, clip 0.3, Adam) both ranks hold the same parameters, bit for bit.  Prints
TRAIN_ROLLOUT_DIST PASS on rank 0."""
from __future__ import annotations

import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist
import yaml
from torch.nn.parallel import DistributedDataParallel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import main  # noqa: E402


def scenes(path):
    rng = np.random.default_rng(0)
    os.makedirs(os.path.join(path, "train"))
    for k, n in enumerate([300, 260]):
        x0 = rng.uniform(0.2, 0.8, (1, n, 3))
        pos = (x0 + np.cumsum(0.01 * rng.standard_normal((14, n, 3)), 0)).astype(np.float32)
        np.savez(os.path.join(path, "train", f"water_{k}.npz"), position=pos, particle_type=rng.integers(1, 9, n))


def grads(model):
    return [p.grad.detach().clone() for p in model.parameters() if p.grad is not None]


def main_():
    rank, world = int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    assert world == 2
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    dev = torch.device("cuda", rank)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"].update(node_feat_nf=2, node_attr_nf=1)
    cfg["data"].update(dataset_name="Water3D", inner_radius=0.3, max_samples=4, split_mode="random", delta_t=2,
                       batch_size=2)
    ok = True
    with tempfile.TemporaryDirectory() as tmp:
        scenes(tmp)
        torch.manual_seed(0)
        model = DistributedDataParallel(main.get_model(cfg, world).to(dev), device_ids=[rank],
                                        find_unused_parameters=True)
        model.train()
        ld = main.frame_loaders(tmp, cfg, world, rank, dev, None, horizon=3, parts=("train",))[1]["train"]
        kw, ex = next(iter(ld))
        one = main.trajectory_loss(cfg, model, world, True)
        model.zero_grad()
        torch.manual_seed(7)
        one(kw, ex, 1)[0].backward()
        g_ddp = grads(model)
        grad_sum = main.rollout_grad_sum(model, world)
        roll1 = main.trajectory_rollout_loss(cfg, model, world, True, ld, "water3d", 2.0, 1)
        model.zero_grad()
        torch.manual_seed(7)
        roll1(kw, dict(ex, targets=ex["targets"][:1].contiguous()), 1)[0].backward()
        grad_sum()
        g_roll = grads(model)
        a, b = (torch.cat([g.double().reshape(-1) for g in gs]) for gs in (g_ddp, g_roll))
        rel = float((a - b).norm() / a.norm())
        print(f"rank {rank}: K = 1 after the rank sum vs DDP one-step: {rel:.2e} relative (norm over all parameters)",
              flush=True)
        ok &= len(g_ddp) == len(g_roll) and rel <= 1e-5
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)
        roll3 = main.trajectory_rollout_loss(cfg, model, world, True, ld, "water3d", 2.0, 3)
        model.zero_grad()
        roll3(kw, ex, 1)[0].backward()
        grad_sum()
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
        opt.step()
        flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
        both = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(both, flat)
        same = bool(torch.equal(both[0], both[1]))
        print(f"rank {rank}: K = 3 parameters identical on both ranks after a step: {same}", flush=True)
        ok &= same
    flag = torch.tensor([0 if ok else 1], device=dev)
    dist.all_reduce(flag)
    if rank == 0 and int(flag) == 0:
        print("TRAIN_ROLLOUT_DIST PASS", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if int(flag) == 0 else 1)


if __name__ == "__main__":
    main_()
