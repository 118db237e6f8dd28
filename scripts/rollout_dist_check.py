"""Multi-GPU rollout check: run under torchrun with 2 ranks (one per GPU).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29547 \
        scripts/rollout_dist_check.py [--nodes 12000] [--steps 3]

Every rank rolls its random partition of one fluid graph out for `--steps` steps with `model.cuda_graph = True`; rank 0
starts with half the edge capacity its graph needs, so it alone regrows while both ranks roll back, rerun and recapture.
Rank 0 gathers every rank's trajectory and checks each step against `oracle.forward_partitions` in float64 on the state
the rollout produced (each partition's graph rebuilt from its x_t, the global loc_mean of x_t), the velocity / speed /
loc_mean rules, and that loc_mean and virtual_loc are bit-identical on the ranks.  With `--deterministic` the model runs in
deterministic mode and every rank rolls out twice: the two runs (regrowth and rerun included) must be bitwise equal on
each rank.  Prints one JSON line and `ROLLOUT_DIST PASS|FAIL`.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KW = dict(node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2, virtual_channels=5, n_layers=4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=12000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--deterministic", action="store_true",
                    help="model.deterministic = True; roll out twice and require bitwise equal runs on every rank")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    from distegnn_b200 import FastEGNN, radius_graph_csr, rollout, synth
    from oracle import fastegnn_oracle as orc
    w = synth.WORKLOADS["fluid113k"]
    parts = synth.make_partitions(w, world_size=world, split_mode="random", seed=0, n_nodes=args.nodes)
    sd = orc.init_state_dict(3, 2, 2, 64, 5, 4, seed=1, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=world, normalize=w.normalize, **KW)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    m.cuda_graph = True
    m.deterministic = args.deterministic
    mine = {k: (v.to(dev) if v is not None else None) for k, v in parts[rank].items() if k not in ("edge_index", "edge_attr")}
    cap = int(parts[rank]["edge_index"].shape[1]) // 2 if rank == 0 else None
    K = args.steps
    res = rollout(m, **mine, steps=K, radius=w.radius, speed_col=0, capacity=cap, check_every=K, return_trajectory=True)
    repeat_equal = None
    if args.deterministic:
        again = rollout(m, **mine, steps=K, radius=w.radius, speed_col=0, capacity=cap, check_every=K,
                        return_trajectory=True)
        repeat_equal = all(torch.equal(getattr(res, k), getattr(again, k))
                           for k in ("trajectory", "node_vel", "node_feat", "loc_mean", "virtual_loc", "n_edges"))
    got = dict(traj=res.trajectory.cpu(), vel=res.node_vel.cpu(), feat=res.node_feat.cpu(), loc_mean=res.loc_mean.cpu(),
               X=res.virtual_loc.cpu(), n_edges=res.n_edges.cpu(), regrowths=res.regrowths, replays=res.replays,
               peer=bool(m._comm), repeat_equal=repeat_equal)
    allg = [None] * world
    dist.all_gather_object(allg, got)
    ok, report = True, {}
    if rank == 0:
        sd64 = {k: v.to(dev).double() for k, v in sd.items()}
        x = [p["node_loc"].to(dev).double() for p in parts]
        v = [p["node_vel"].to(dev).double() for p in parts]
        f = [p["node_feat"].to(dev).double() for p in parts]
        lm = parts[0]["loc_mean"].to(dev).double()
        worst, worst_rel = 0.0, 0.0
        for t in range(K):
            pin = []
            for r in range(world):
                g, _ = radius_graph_csr(x[r].float().contiguous(), w.radius)
                ok &= int(allg[r]["n_edges"][t]) == g.num_edges
                ei = g.edge_index()
                ea = (x[r][ei[0]] - x[r][ei[1]]).norm(dim=1, keepdim=True).expand(-1, 2).contiguous()
                pin.append(dict(node_feat=f[r], node_loc=x[r], node_vel=v[r], edge_index=ei,
                                data_batch=torch.zeros(x[r].shape[0], dtype=torch.int64, device=dev), edge_attr=ea,
                                node_attr=parts[r]["node_attr"].to(dev).double()))
            outs, X = orc.forward_partitions(sd64, pin, lm, normalize=w.normalize)
            for r in range(world):
                out = allg[r]["traj"][t].to(dev).double()
                e = float((out - outs[r]).abs().max())
                den = float((outs[r] - x[r]).abs().max())
                worst, worst_rel = max(worst, e), max(worst_rel, e / max(den, 1e-30))
                ok &= e <= 1e-5 * max(1.0, float(outs[r].abs().max())) and e <= 1e-4 * den
                xd = out
                v[r] = xd - x[r]
                f[r] = f[r].clone()
                f[r][:, 0] = v[r].norm(dim=1)
                x[r] = xd
            lm = torch.cat(x).mean(0, keepdim=True)
        eX = float((allg[0]["X"].to(dev).double() - X).abs().max())
        elm = float((allg[0]["loc_mean"].to(dev).double() - lm).abs().max())
        ev = max(float((allg[r]["vel"].to(dev).double() - v[r]).abs().max()) for r in range(world))
        ef = max(float((allg[r]["feat"].to(dev).double() - f[r]).abs().max()) for r in range(world))
        same = all(torch.equal(allg[r]["loc_mean"], allg[0]["loc_mean"]) and torch.equal(allg[r]["X"], allg[0]["X"])
                   for r in range(world))
        regrow = bool(allg[0]["regrowths"]) and not any(allg[r]["regrowths"] for r in range(1, world))
        # steps 1..K-1 replayed twice on every rank: the overflowed attempt and the rerun after rank 0 regrew
        graphed = all(a["replays"] == 2 * (K - 1) for a in allg) if all(a["peer"] for a in allg) else None
        repeats = [a["repeat_equal"] for a in allg]
        ok &= eX <= 1e-5 * max(1.0, float(X.abs().max())) and elm <= 1e-6 and ev <= 1e-5 and ef <= 1e-5 and same \
            and regrow and graphed is not False and (not args.deterministic or all(repeats))
        report = dict(world=world, nodes=args.nodes, steps=K, max_abs=worst, max_rel_disp=worst_rel, virtual_loc=eX,
                      loc_mean=elm, vel=ev, feat=ef, bit_identical=same, rank0_regrew=regrow,
                      regrowths=[a["regrowths"] for a in allg], peer_exchange=[a["peer"] for a in allg],
                      replays=[a["replays"] for a in allg], deterministic=args.deterministic,
                      repeat_bitwise_equal=repeats, pass_=bool(ok))
        print(json.dumps(report), flush=True)
        print("ROLLOUT_DIST", "PASS" if ok else "FAIL", flush=True)
    flag = torch.tensor([int(ok)], device=dev)
    dist.broadcast(flag, 0)
    dist.barrier()
    m.release_comm()
    dist.destroy_process_group()
    if not int(flag.item()):
        sys.exit(1)


if __name__ == "__main__":
    main()
