"""Rotated and translated evaluation splits (FrameLoader's rotate / translate, DESIGN §23) at full size, on one GPU.

    python scripts/bench_frames_transform.py [--reps 10] [--out result.json]

Scenes are the seeded random walks of scripts/bench_frames.py (Fluid113K recipe, r = 0.075): 113,140 nodes and config
5's 1M nodes.
(1) Cost: the assembly (distegnn_frames_assemble, horizon 1) and the transformed assembly
    (distegnn_frames_assemble_transform, rotate, translate = 1) between CUDA events, medians of `--reps` with min–max;
    the loader's batch time in capacity mode with and without the transform.
(2) Bit for bit at 113k nodes, horizon 3, world sizes 1 and 2 (both ranks, random split): node_loc, node_vel and every
    targets row against the CPU restatement fed the testing hook's R and t; the speed column within 1 ulp; loc_mean
    against the float64 mean of the transformed scene; the graph against radius_graph_csr on the transformed positions;
    the same bits for every node and the same loc_mean at both world sizes.
(3) Equivariance of a randomly initialised FastEGNN (C = 8) at translations of 0, 1 and 10 scene extents, on the plain
    batch's graph, and the edges that flip between the plain and the transformed radius graph
    (tests/test_frames_transform.py: equivariance_at_scale).
(4) The mean MSE of the same model over the 113k-node sample, plain and transformed (rotate, translate = 1 extent), and
    the per-step MSE of a 3-step rollout against the recorded frames for both, with their relative differences.
Reports the card name and power limit read in the same run.  Prints one JSON line; `--out` also writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from distegnn_b200 import FastEGNN, _lib, rollout, synth, train_loss  # noqa: E402
from distegnn_b200._lib import check, ptr  # noqa: E402
from distegnn_b200.frames import FrameLoader, load_scenes  # noqa: E402
from distegnn_b200.partition import radius_graph_csr  # noqa: E402
from bench_frames import event_ms, loader_batch_ms, write_scene  # noqa: E402
from bench_rollout import power_limit_w  # noqa: E402
from tests.test_frames_transform import equivariance_at_scale, hook, rigid  # noqa: E402


def cost(traj, n, reps, dev, radius):
    kw_ = dict(delta_t=1, radius=radius, device=dev, prefetch=0)
    one = [(0, 0)]
    exact, kw, _ = loader_batch_ms(lambda: FrameLoader(traj, one, **kw_), reps)
    cap = int(1.25 * int(kw["edge_index"].rowptr[-1]))
    plain_b, _, _ = loader_batch_ms(lambda: FrameLoader(traj, one, capacity=cap, **kw_), reps)
    moved_b, _, _ = loader_batch_ms(lambda: FrameLoader(traj, one, capacity=cap, rotate=True, translate=1.0, **kw_),
                                    reps)
    host = FrameLoader(traj, one, rotate=True, **kw_)._host_batch([0])
    host = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    f32 = dict(dtype=torch.float32, device=dev)
    feat, loc, vel, attr, target = (torch.empty(n, c, **f32) for c in (3, 3, 3, 2, 3))
    batch, lm, smax = torch.empty(n, dtype=torch.int64, device=dev), torch.empty(1, 3, **f32), torch.empty(1, **f32)
    meta = host["meta"]

    def assemble():
        check(_lib.load().distegnn_frames_assemble(
            _lib.FRAMES_LARGEFLUID, 1, n, n, ptr(host["frames"]), ptr(host["statics"]), ptr(meta[:2]), ptr(meta[2:4]),
            None, ptr(feat), ptr(loc), ptr(vel), ptr(attr), ptr(target), ptr(batch), ptr(lm), ptr(smax),
            _lib.stream_ptr(dev)), "frames_assemble")

    def assemble_transform():
        check(_lib.load().distegnn_frames_assemble_transform(
            _lib.FRAMES_LARGEFLUID, 1, n, n, 1, ptr(host["frames"]), ptr(host["statics"]), ptr(meta[:2]),
            ptr(meta[2:4]), None, ptr(feat), ptr(loc), ptr(vel), ptr(attr), ptr(target), ptr(batch), ptr(lm),
            ptr(smax), ptr(meta[4:]), 0, 1, 1.0, _lib.stream_ptr(dev)), "frames_assemble_transform")

    rows = []
    for _ in range(3):                                           # alternate the two, three rounds each
        rows.append((event_ms(assemble, reps), event_ms(assemble_transform, reps)))
    return dict(nodes=n, assembly_kernel_ms=[r[0] for r in rows], assembly_transform_kernel_ms=[r[1] for r in rows],
                batch_ms=dict(exact=exact, capacity=plain_b, capacity_transform=moved_b))


def bitwise(traj, dev, radius, K=3, rotate=True, translate=1.0, seed=3):
    """Check (2) on one sample; returns the findings (the script fails on none of them, it reports them)."""
    sc = traj.scenes[0]
    pos = torch.from_numpy(np.array(sc.position[:K + 1]))
    vel = torch.from_numpy(np.array(sc.velocity[0]))
    R, t, _ = hook(seed, 0, 1, rotate, translate)
    R, t = R[0], t[0]
    x = rigid(R, t, pos[0], True)
    v = rigid(R, t, vel, False)
    speed = torch.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    targets = torch.stack([rigid(R, t, pos[k], True) for k in range(1, K + 1)])
    whole = x.double().mean(0)
    out, per_node = {}, {}
    for P in (1, 2):
        nodes, means = {}, []
        for rank in range(P):
            ld = FrameLoader(traj, [(0, 0)], delta_t=1, radius=radius, device=dev, world_size=P, rank=rank, horizon=K,
                             rotate=rotate, translate=translate, transform_seed=seed)
            (kw, ex), = list(ld)
            part, _ = ld.partition(0)
            idx = torch.arange(x.shape[0]) if part is None else part.long()
            loc, vl, tg = kw["node_loc"].cpu(), kw["node_vel"].cpu(), ex["targets"].cpu()
            ia = speed[idx].view(torch.int32).long()
            ib = kw["node_feat"][:, 2].cpu().contiguous().view(torch.int32).long()
            lm = kw["loc_mean"][0].cpu().double()
            g = kw["edge_index"]
            wg, _ = radius_graph_csr(kw["node_loc"], radius, kw["data_batch"], n_graphs=1)
            E = int(g.rowptr[-1])
            out[f"P{P}_rank{rank}"] = dict(
                node_loc=torch.equal(loc, x[idx]), node_vel=torch.equal(vl, v[idx]),
                targets=all(torch.equal(tg[k], targets[k][idx]) for k in range(K)),
                speed_max_ulps=int((ia - ib).abs().max()),
                loc_mean_rel_err=float((lm - whole).abs().max() / whole.abs().max()),
                graph_equal=bool(torch.equal(g.rowptr, wg.rowptr) and torch.equal(g.col[:E], wg.col[:E])))
            means.append(kw["loc_mean"][0].cpu())
            full = torch.cat([loc, vl, tg.permute(1, 0, 2).reshape(-1, 3 * K)], 1)
            for r, j in enumerate(idx.tolist()):
                nodes[j] = r, full
        per_node[P] = (nodes, means)
    n1, m1 = per_node[1]
    n2, m2 = per_node[2]
    same = all(torch.equal(n1[j][1][n1[j][0]], n2[j][1][n2[j][0]]) for j in n1)
    out["same_bits_world_1_and_2"] = bool(same and len(n1) == len(n2))
    out["loc_mean_equal_on_all_ranks"] = bool(torch.equal(m1[0], m2[0]) and torch.equal(m2[0], m2[1]))
    return out


def mse_plain_and_transformed(traj, dev, radius, extent, K=3):
    torch.manual_seed(0)
    model = FastEGNN(node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2, hidden_nf=64, virtual_channels=8, world_size=1,
                     n_layers=4).to(dev).eval()
    res = {}
    for name, xf in (("plain", {}), ("transformed", dict(rotate=True, translate=extent))):
        ld = FrameLoader(traj, [(0, 0)], delta_t=1, radius=radius, device=dev, horizon=K, **xf)
        (kw, ex), = list(ld)
        with torch.no_grad():
            pred, X = model(**kw)
            _, info = train_loss(pred, ex["target"], X, kw["data_batch"], world_size=1, loc_mean=kw["loc_mean"],
                                 node_counts=ex["node_counts"])
            r = rollout(model, kw["node_feat"], kw["node_loc"], kw["node_vel"], kw["loc_mean"], kw["data_batch"],
                        kw["node_attr"], steps=K, radius=radius, tau=1.0, speed_col=2, targets=ex["targets"])
        res[name] = dict(mse=float(info["logged"]), rollout_mse=[float(v) for v in r.mse.flatten().tolist()])
    p, m = res["plain"], res["transformed"]
    res["relative_difference"] = (m["mse"] - p["mse"]) / p["mse"]
    res["rollout_relative_difference"] = [(b - a) / a for a, b in zip(p["rollout_mse"], m["rollout_mse"])]
    res["translate"] = extent
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    w = synth.WORKLOADS["fluid113k"]
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), reps=args.reps)
    tmp = tempfile.mkdtemp(prefix="bench_frames_transform_")
    try:
        trajs = {}
        for name, n in (("fluid113k", 113_140), ("config5", 1_000_000)):
            path = os.path.join(tmp, f"{name}.npz")
            write_scene(path, w, n, seed=n)
            trajs[name] = load_scenes([path], "largefluid")
            res[name] = dict(cost=cost(trajs[name], n, args.reps, dev, w.radius))
        pos0 = np.array(trajs["fluid113k"].scenes[0].position[0], dtype=np.float64)
        extent = float((pos0.max(0) - pos0.min(0)).max())
        res["fluid113k"]["bitwise"] = bitwise(trajs["fluid113k"], dev, w.radius)
        res["fluid113k"]["equivariance"] = equivariance_at_scale(tmp, dev)
        res["fluid113k"]["mse"] = mse_plain_and_transformed(trajs["fluid113k"], dev, w.radius, extent)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
