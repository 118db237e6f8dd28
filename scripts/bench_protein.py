"""Cost of the protein recipe on one GPU: FrameLoader batches read from a DCD and a PSF, and FastEGNN's train and eval
steps on them, at config/protein_fastegnn.yaml's settings (batch 5, r = 10 Å, backbone atoms, C = 3).

    python scripts/bench_protein.py [--reps 20] [--out result.json]

The trajectory is synthetic, of the AdK shape: 3,341 atoms in 214 residues (855 backbone atoms), uniform in a ball of
20 Å radius (about 0.1 atoms per Å³, a protein's density with its hydrogens), each frame a small seeded displacement of
the last; written as a PSF and a DCD to a temporary directory and read back by distegnn_b200.protein.  An r = 10 Å graph
on these atoms is dense (about 75 neighbours per backbone atom), so the edge count is reported beside every time; the
real AdK's count depends on its fold and is not measured here.

(1) ms per batch of the loader with prefetch 0 (host gather of the 855 atoms from the memory-mapped DCD, H2D, assembly,
    radius graph, exact mode), wall clock after a device synchronise, median / min / max of `--reps` after a warm-up;
    the edges of each batch.
(2) ms per train step (forward, main.py's fused loss with the config's MMD, backward, clip, Adam) and per eval step
    (no_grad forward and loss) on batches assembled beforehand, after a warm-up.
(3) The same train step fed by the loader (prefetch 2), so the loader's cost that is not hidden shows.
Reports the card name and power limit read in the same run.  Prints one JSON line; `--out` also writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import struct
import sys
import tempfile
import time

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import main as entry  # noqa: E402
from distegnn_b200.frames import FrameLoader  # noqa: E402
from distegnn_b200.protein import find_files, load_protein  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402

SIDE = ["HA", "CB", "HB1", "HB2", "CG", "HG1", "HG2", "CD", "HD1", "HD2"]


def stats(v):
    return dict(median=statistics.median(v), min=min(v), max=max(v))


def write_adk_shape(d, T, seed=0):
    """prot.psf and prot.dcd in `d`: 214 residues of N HN CA <10 side atoms> C O, the first 130 with one more side
    atom, the last ending in OT1 OT2: 3,341 atoms, 855 backbone."""
    names, resn = [], []
    for k in range(214):
        atoms = ["N", "HN", "CA"] + SIDE + (["HZ"] if k < 130 else []) + (["C", "OT1", "OT2"] if k == 213 else ["C", "O"])
        names += atoms
        resn += [("GLY", "HSD", "LYS", "ALA")[k % 4]] * len(atoms)
    n = len(names)
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3))
    x0 = v / np.linalg.norm(v, axis=1, keepdims=True) * 20.0 * rng.random((n, 1)) ** (1 / 3)
    pos = (x0[None] + np.cumsum(rng.normal(0, 0.05, (T, n, 3)), 0)).astype(np.float32)
    charges = rng.uniform(-0.6, 0.6, n).round(3)
    with open(os.path.join(d, "prot.psf"), "w") as f:
        f.write(f"PSF\n\n       1 !NTITLE\n* AdK-shaped\n\n{n:8d} !NATOM\n")
        for k, (a, r, q) in enumerate(zip(names, resn, charges)):
            f.write(f"{k + 1:8d} ADK  {k // 16 + 1:<4d} {r:<4s} {a:<4s} {a:<4s} {q:14.6f}{12.011:14.4f}{0:12d}\n")

    def rec(b):
        return struct.pack("<i", len(b)) + b + struct.pack("<i", len(b))
    with open(os.path.join(d, "prot.dcd"), "wb") as f:
        f.write(rec(b"CORD" + struct.pack("<9i", T, 0, 1, T, 0, 0, 0, 0, 0) + struct.pack("<f", 0.0489) +
                    struct.pack("<10i", *([0] * 9 + [24]))))
        f.write(rec(struct.pack("<i", 1) + b"REMARKS AdK-shaped".ljust(80)))
        f.write(rec(struct.pack("<i", n)))
        for t in range(T):
            for c in range(3):
                f.write(rec(pos[t, :, c].astype("<f4").tobytes()))
    return n


def step_ms(fn, batches, reps):
    for kw, ex in batches[:2]:
        fn(kw, ex)
    torch.cuda.synchronize()
    out = []
    for k in range(reps):
        kw, ex = batches[k % len(batches)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(kw, ex)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return stats(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    with open(os.path.join(ROOT, "config", "protein_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    d, B, r, dt = cfg["data"], cfg["data"]["batch_size"], float(cfg["data"]["radius"]), int(cfg["data"]["delta_t"])
    tmp = tempfile.mkdtemp(prefix="bench_protein_")
    try:
        frames = B * (args.reps + 1) + dt + 1                   # one pass of the loader gives reps + 1 batches
        n_atoms = write_adk_shape(tmp, frames)
        t0 = time.perf_counter()
        traj = load_protein(find_files(tmp), backbone=d["backbone"])
        open_ms = (time.perf_counter() - t0) * 1e3
        samples = [(0, t) for t in range(frames - dt - 1)]
        it = iter(FrameLoader(traj, samples, delta_t=dt, radius=r, batch_size=B, device=dev, prefetch=0))
        times, edges, batches = [], [], []
        for _ in range(args.reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            kw, ex = next(it)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
            edges.append(int(kw["edge_index"].rowptr[-1]))
            batches.append((kw, ex))
        batch_ms = stats(times[1:])
        torch.manual_seed(0)
        model = entry.get_model(cfg, 1).to(dev)
        loss_of = entry.trajectory_loss(cfg, model, 1, False)
        opt = torch.optim.Adam(model.parameters(), lr=float(cfg["train"]["learning_rate"]),
                               weight_decay=float(cfg["train"]["weight_decay"]))

        def train(kw, ex):
            model.train()
            opt.zero_grad()
            loss, _ = loss_of(kw, ex)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=0.3)
            opt.step()

        def evaluate(kw, ex):
            model.eval()
            with torch.no_grad():
                loss_of(kw, ex)

        train_ms = step_ms(train, batches, args.reps)
        eval_ms = step_ms(evaluate, batches, args.reps)
        fed = FrameLoader(traj, samples, delta_t=dt, radius=r, batch_size=B, device=dev, prefetch=2)
        fed_times = []
        for epoch in range(2):                                   # the first pass warms up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            k = 0
            for kw, ex in fed:
                train(kw, ex)
                k += 1
            torch.cuda.synchronize()
            if epoch:
                fed_times.append((time.perf_counter() - t0) * 1e3 / k)
        res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), reps=args.reps,
                   trajectory=dict(atoms=n_atoms, backbone_atoms=traj.scenes[0].n_nodes, frames=frames,
                                   open_psf_dcd_ms=open_ms),
                   batch=dict(graphs=B, nodes=B * traj.scenes[0].n_nodes, radius=r, delta_t=dt),
                   edges_per_batch=stats(edges), edges_per_node=statistics.median(edges) / (B * traj.scenes[0].n_nodes),
                   loader_batch_ms=batch_ms, train_step_ms=train_ms, eval_step_ms=eval_ms,
                   train_step_fed_by_loader_ms=fed_times[0])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=2) + "\n")


if __name__ == "__main__":
    main()
