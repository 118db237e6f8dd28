"""Generate INPUT-GRADIENT fixtures (tests/golden/*.input_grads.npz) by running the UNMODIFIED reference module under autograd.

Run where the reference is available (it is not needed to use the fixtures):

    python oracle/make_golden_input_grads.py

Same cases, inputs, weights and cotangents as oracle/make_golden_grads.py (inputs and weights read back from the committed
forward fixtures; cotangents seed 7, per rank 100+r and 99 for the virtual output), but here every floating input of the
reference ``FastEGNN.forward`` (node_feat, node_loc, node_vel, loc_mean, edge_attr, node_attr) is an autograd leaf and the
fixture holds d L / d input, in float64.  For the 2-partition case the reference's real ``world_size=2`` branch runs under
gloo (``torch.Tensor.cuda`` patched to the identity), each rank back-propagating its own L_r into its own inputs.

Test infrastructure; not imported by the product.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_golden import OUT, import_reference  # noqa: E402
from make_golden_grads import cotangents  # noqa: E402
from tests.helpers import DIST_CASE, SINGLE_CASES, golden_inputs, load_golden  # noqa: E402

FLOAT_INPUTS = ["node_feat", "node_loc", "node_vel", "loc_mean", "edge_attr", "node_attr"]


def reference_input_grads(FastEGNN, kw, sd, inp, cot_out, cot_X, world_size=1):
    model = FastEGNN(hidden_nf=64, world_size=world_size, **kw)
    model.load_state_dict(sd)
    model = model.to(torch.float64)
    leaf = {k: inp[k].to(torch.float64).clone().requires_grad_(True) for k in FLOAT_INPUTS if inp.get(k) is not None}
    out, X = model(leaf["node_feat"], leaf["node_loc"], leaf["node_vel"], leaf["loc_mean"], inp["edge_index"],
                   inp["data_batch"], leaf["edge_attr"], leaf.get("node_attr"))
    loss = (out * cot_out).sum() + (X * cot_X).sum()
    loss.backward()
    return {k: (t.grad if t.grad is not None else torch.zeros_like(t)).detach().clone() for k, t in leaf.items()}, \
        float(loss.detach())


def _rank_main(rank, world, port, kw, sd, parts, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.Tensor.cuda = lambda self, *a, **k: self          # reference hard-codes .cuda()
    FastEGNN = import_reference()
    n, B, C = parts[rank]["node_loc"].shape[0], parts[rank]["loc_mean"].shape[0], kw["virtual_channels"]
    cot_out, _ = cotangents(100 + rank, n, B, C, torch.float64)
    _, cot_X = cotangents(99, n, B, C, torch.float64)       # the virtual output is identical on every rank
    grads, loss = reference_input_grads(FastEGNN, kw, sd, parts[rank], cot_out, cot_X, world_size=world)
    q.put((rank, {k: v.numpy() for k, v in grads.items()}, loss))
    dist.barrier()
    dist.destroy_process_group()


def main():
    FastEGNN = import_reference()
    for name in SINGLE_CASES:
        z, kw, sd = load_golden(name)
        inp = golden_inputs(z)
        n, B, C = inp["node_loc"].shape[0], inp["loc_mean"].shape[0], kw["virtual_channels"]
        cot_out, cot_X = cotangents(7, n, B, C, torch.float64)
        grads, loss = reference_input_grads(FastEGNN, kw, sd, inp, cot_out, cot_X)
        blob = {"ig." + k: v.numpy() for k, v in grads.items()}
        blob.update({"cot.out": cot_out.numpy(), "cot.X": cot_X.numpy(), "loss": np.array(loss)})
        np.savez_compressed(os.path.join(OUT, name + ".input_grads.npz"), **blob)
        print(name, "loss", loss, {k: float(v.abs().max()) for k, v in grads.items()})

    import torch.multiprocessing as mp
    z, kw, sd = load_golden(DIST_CASE)
    parts = [golden_inputs(z, f"in{r}.") for r in range(2)]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, 29614, kw, sd, parts, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get() for _ in procs], key=lambda t: t[0])
    [p.join() for p in procs]
    blob = {}
    for r, grads, loss in res:
        blob.update({f"ig{r}." + k: v for k, v in grads.items()})
        blob[f"loss{r}"] = np.array(loss)
    np.savez_compressed(os.path.join(OUT, DIST_CASE + ".input_grads.npz"), **blob)
    print(DIST_CASE, "losses", [r[2] for r in res])


if __name__ == "__main__":
    main()
