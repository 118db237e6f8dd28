"""Gradients with respect to the model's inputs (`model.input_grads = True`): node_feat, node_loc, node_vel, loc_mean,
edge_attr and node_attr receive what the reference module's autograd gives them.

CPU: (1) the oracle's fp64 autograd w.r.t. the inputs is pinned to fixtures from the unmodified reference
(oracle/make_golden_input_grads.py); (2) the host orchestration with the kernels replaced by a torch stand-in reproduces
them; (3) the same under gloo with world_size=2, with one extra backward exchange only when node_loc needs a gradient;
(4) the flag changes nothing when no input needs a gradient, and frozen weights still give input gradients.
GPU: each changed kernel against float64 autograd of its stage restatement, the whole model against the fixtures and the
oracle, a two-step rollout, and size-independent properties on a 200k-node graph.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from distegnn_b200 import _lib
from oracle import fastegnn_oracle as orc
from tests.helpers import DIST_CASE, GOLDEN, SINGLE_CASES, golden_inputs, load_golden
from tests.shadow_backend import ShadowBackend

INPUTS = ["node_feat", "node_loc", "node_vel", "loc_mean", "edge_attr", "node_attr"]
H = 64


def load_input_grads(name):
    return np.load(os.path.join(GOLDEN, name + ".input_grads.npz"))


def rel_err(mine, ref):
    ref = torch.as_tensor(ref).double()
    return float((mine.detach().cpu().double() - ref).abs().max() / ref.abs().max().clamp(min=1e-30))


def leaves(inp, dtype=None, device=None):
    """The inputs with every floating one a fresh autograd leaf."""
    out = {}
    for k, v in inp.items():
        if isinstance(v, torch.Tensor) and v.is_floating_point():
            v = v.to(dtype=dtype or v.dtype, device=device or v.device).clone().requires_grad_(True)
        elif isinstance(v, torch.Tensor) and device is not None:
            v = v.to(device)
        out[k] = v
    return out


def check_inputs(leaf, zi, prefix, tol):
    errs = {}
    for k in INPUTS:
        if leaf.get(k) is None or prefix + k not in zi.files:
            continue
        ref = torch.from_numpy(zi[prefix + k])
        g = leaf[k].grad
        assert g is not None, k
        assert g.dtype == leaf[k].dtype and g.device == leaf[k].device, k
        if float(ref.abs().max()) == 0.0:
            assert float(g.abs().max()) == 0.0, k
            continue
        errs[k] = rel_err(g, ref)
    worst = max(errs, key=errs.get)
    assert errs[worst] <= tol, errs
    return errs


# ---- the torch stand-in, extended by the keyword outputs of the input gradients -------------------------------------------
class InputGradShadowBackend(ShadowBackend):
    """ShadowBackend plus the input-gradient outputs of CudaBackend (g_ea, g_vel / g_attr, g_feat / g_loc, inverse
    gather), by torch.autograd through the stage restatements; counts every call for the launch-sequence checks."""

    def __init__(self):
        super().__init__()
        self.calls = []
        for name in [n for n in dir(self) if not n.startswith("_")]:
            fn = getattr(self, name)
            if callable(fn):
                setattr(self, name, self._counted(name, fn))

    def _counted(self, name, fn):
        def call(*a, **k):
            self.calls.append((name, tuple(sorted(key for key, v in k.items() if v is not None))))
            return fn(*a, **k)
        return call

    def gather_rows(self, src, perm, inverse=False):
        if not inverse:
            return super().gather_rows(src, perm)
        dst = torch.empty_like(src)
        dst[perm.long()] = src
        return dst

    def edge_layer_bwd(self, dims, flags, row, col, ea, x4, P, Q, lp, g_agg_m, g_agg_x, g_P, g_Q, g_x4, g_lp,
                       n_edges_dev=None, g_ea=None):
        if g_ea is None:
            return super().edge_layer_bwd(dims, flags, row, col, ea, x4, P, Q, lp, g_agg_m, g_agg_x, g_P, g_Q, g_x4, g_lp,
                                          n_edges_dev)
        from tests import shadow_autograd as sa
        N, E, A, C, Na = dims
        with torch.enable_grad():
            Pl, Ql, xl, lpl, eal = (t.detach().clone().requires_grad_(True) for t in (P, Q, x4[:, :3], lp, ea))
            am, ax = sa.edge_stage(dims, flags, row, col, eal, xl, Pl, Ql, lpl)
            loss = (ax * g_agg_x[:, :3]).sum()
            if g_agg_m is not None and not flags & _lib.FLAG_LAST:
                loss = loss + (am * g_agg_m).sum()
            gP, gQ, gx, glp, gea = torch.autograd.grad(loss, (Pl, Ql, xl, lpl, eal), allow_unused=True)
        g_P += gP
        g_Q += gQ
        g_x4[:, :3] += gx
        g_lp += glp
        g_ea += gea

    def node_layer_bwd(self, dims, flags, rowptr, batch32, h, vel, attr, agg_m, agg_v, lp, lp_next, g_x_out, g_vsum,
                       g_h_out, g_P, g_Q, g_Hn, g_h, g_x, g_agg_x, g_trans_v, g_agg_m, g_agg_v, g_lp, g_lp_next,
                       g_vel=None, g_attr=None):
        from tests import dense_stages as ds
        N, B, A, C, Na = dims
        last = bool(flags & _lib.FLAG_LAST)
        deg = (rowptr[1:] - rowptr[:-1]).clamp(min=1).to(h.dtype).unsqueeze(1)
        leaf = lambda t: t.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            hl, lpl, vl = leaf(h), leaf(lp), leaf(vel)
            al = leaf(attr) if Na else None
            xl, axl, tvl = (torch.zeros(N, 3, dtype=h.dtype, device=h.device).requires_grad_(True) for _ in range(3))
            aml, avl, lpn = (None, None, None) if last else (leaf(agg_m), leaf(agg_v), leaf(lp_next))
            xn, hn, Pn, Qn, Hnn = ds.node_stage(hl, xl, vl, al, aml, axl, avl, tvl, deg, ds.field_views(lpl, A, C, Na),
                                                None if last else ds.field_views(lpn, A, C, Na))
            gx = g_x_out if g_vsum is None else g_x_out + g_vsum[batch32.long(), 0:3]
            outs, gouts = [xn], [gx]
            for o, g in ((hn, g_h_out), (Pn, g_P), (Qn, g_Q), (Hnn, g_Hn)):
                if o is not None and g is not None:
                    outs.append(o)
                    gouts.append(g)
            ins = [hl, xl, axl, tvl, lpl, vl] + ([al] if al is not None else []) + ([] if last else [aml, avl, lpn])
            r = torch.autograd.grad(outs, ins, gouts, allow_unused=True)
            r = [torch.zeros_like(i) if g is None else g for g, i in zip(r, ins)]
        g_h.copy_(r[0])
        g_x.copy_(r[1])
        g_agg_x.zero_(); g_agg_x[:, :3] = r[2]
        g_trans_v.zero_(); g_trans_v[:, :3] = r[3]
        g_lp += r[4]
        if g_vel is not None:
            g_vel += r[5]
        k = 6
        if al is not None:
            if g_attr is not None:
                g_attr += r[k]
            k += 1
        if not last:
            g_agg_m.copy_(r[k])
            g_agg_v.copy_(r[k + 1])
            g_lp_next += r[k + 2]

    def embed_bwd(self, dims, node_feat, h0, lp0, g_h, g_P, g_Q, g_Hn, g_emb_wt, g_emb_b, g_lp0, g_feat=None, g_loc=None,
                  emb_wt=None, batch32=None, g_x0=None, g_vsum0=None):
        from tests import dense_stages as ds
        super().embed_bwd(dims, node_feat, h0, lp0, g_h, g_P, g_Q, g_Hn, g_emb_wt, g_emb_b, g_lp0)
        N, B, Fn, A, C, Na = dims
        if g_feat is not None:
            with torch.enable_grad():
                fl = node_feat.detach().clone().requires_grad_(True)
                hh = fl @ emb_wt + (h0.detach() - node_feat @ emb_wt)
                P, Q, Hn = ds.projections(hh, ds.field_views(lp0, A, C, Na))
                (gf,) = torch.autograd.grad([hh, P, Q, Hn], [fl], [g_h, g_P, g_Q, g_Hn])
            g_feat.copy_(gf)
        if g_loc is not None:
            g_loc.copy_(g_x0 + (0 if g_vsum0 is None else g_vsum0[batch32.long(), 0:3]))


def stand_in_model(kw, sd, world_size=1):
    from distegnn_b200 import FastEGNN
    m = FastEGNN(hidden_nf=64, world_size=world_size, **kw)
    m.load_state_dict(sd)
    m._backend = InputGradShadowBackend()
    m.input_grads = True
    return m


# ---- 1. the oracle against the reference ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SINGLE_CASES)
def test_oracle_input_grads_match_reference(name):
    z, kw, sd = load_golden(name)
    zi = load_input_grads(name)
    inp = leaves(golden_inputs(z), dtype=torch.float64)
    sd64 = {k: v.double() for k, v in sd.items()}
    out, X = orc.forward(sd64, **inp, normalize=kw["normalize"])
    loss = (out * torch.from_numpy(zi["cot.out"])).sum() + (X * torch.from_numpy(zi["cot.X"])).sum()
    assert abs(float(loss) - float(zi["loss"])) <= 1e-10 * max(1.0, abs(float(zi["loss"])))
    loss.backward()
    print(name, check_inputs(inp, zi, "ig.", 1e-9))


# ---- 2. host orchestration with the stand-in --------------------------------------------------------------------------
@pytest.mark.parametrize("name", SINGLE_CASES)
def test_training_path_input_grads_match_reference(name):
    from tests.test_backward import check_against, load_grads
    z, kw, sd = load_golden(name)
    zi, zg = load_input_grads(name), load_grads(name)
    m = stand_in_model(kw, sd)
    inp = leaves(golden_inputs(z))
    out, X = m(**inp)
    loss = (out * torch.from_numpy(zi["cot.out"]).float()).sum() + (X * torch.from_numpy(zi["cot.X"]).float()).sum()
    loss.backward()
    errs = check_inputs(inp, zi, "ig.", 2e-4)
    dead = []
    check_against({k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in m.named_parameters()}, zg,
                  "grad.", 2e-4, dead)
    print(name, errs)


# ---- 3. two partitions under gloo ---------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        z, kw, sd = load_golden(DIST_CASE)
        zi = load_input_grads(DIST_CASE)
        zg = np.load(os.path.join(GOLDEN, DIST_CASE + ".grads.npz"))
        m = stand_in_model(kw, sd, world_size=world)
        calls = []
        orig = dist.all_reduce

        def counting(t, *a, **k):
            calls.append(tuple(t.shape))
            return orig(t, *a, **k)

        dist.all_reduce = counting
        res = []
        for with_loc in (True, False):
            inp = leaves(golden_inputs(z, f"in{rank}."))
            if not with_loc:
                inp["node_loc"] = inp["node_loc"].detach()
            del calls[:]
            out, X = m(**inp)
            n_fwd = len(calls)
            loss = (out * torch.from_numpy(zg[f"cot{rank}.out"])).sum() + (X * torch.from_numpy(zg["cot.X"])).sum()
            loss.backward()
            grads = {k: inp[k].grad.numpy() for k in INPUTS if inp.get(k) is not None and inp[k].grad is not None}
            res.append((grads, n_fwd, len(calls) - n_fwd))
        dist.all_reduce = orig
        q.put((rank, res, {k: zi[f"ig{rank}." + k] for k in INPUTS if f"ig{rank}." + k in zi.files}))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_partition_input_grads_match_reference_world_size_2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda t: t[0])
    [p.join(timeout=60) for p in procs]
    z, kw, sd = load_golden(DIST_CASE)
    L = kw["n_layers"]
    for r, runs, ref in res:
        (g_all, f1, b1), (g_noloc, f2, b2) = runs
        errs = {k: rel_err(torch.from_numpy(g_all[k]), torch.from_numpy(ref[k])) for k in ref}
        print("rank", r, errs)
        assert max(errs.values()) <= 5e-4, errs
        assert "node_loc" not in g_noloc
        for k in g_noloc:                                  # the other inputs do not depend on node_loc's grad
            assert rel_err(torch.from_numpy(g_noloc[k]), torch.from_numpy(ref[k])) <= 5e-4, k
        # forward L+1 packed collectives; backward L, plus one for the Σx term of the initial centroid with node_loc
        assert f1 == L + 1 and f2 == L + 1
        assert b1 == L + 1 and b2 == L


# ---- 4. flag semantics ------------------------------------------------------------------------------------------------
def test_flag_without_input_requiring_grad_changes_nothing():
    z, kw, sd = load_golden("fluid160_c5")
    zg = np.load(os.path.join(GOLDEN, "fluid160_c5.grads.npz"))
    inp = golden_inputs(z)
    cot, cotX = torch.from_numpy(zg["cot.out"]).float(), torch.from_numpy(zg["cot.X"]).float()
    runs = []
    for flag in (False, True):
        m = stand_in_model(kw, sd)
        m.input_grads = flag
        out, X = m(**inp)
        n_fwd = len(m._backend.calls)
        ((out * cot).sum() + (X * cotX).sum()).backward()
        runs.append((out.detach(), X.detach(), m._backend.calls[n_fwd:], {k: p.grad for k, p in m.named_parameters()}))
    (o0, X0, c0, g0), (o1, X1, c1, g1) = runs
    assert torch.equal(o0, o1) and torch.equal(X0, X1)
    assert c0 == c1                                       # same backward calls, none with an input-gradient output
    # the stand-in's CPU reductions are not bitwise reproducible from run to run (two flag-off runs differ by ~1e-9)
    assert all(rel_err(g1[k], g0[k]) <= 1e-6 for k in g0 if float(g0[k].abs().max()) > 0)


def test_frozen_parameters_still_give_input_grads():
    z, kw, sd = load_golden("fluid160_c5")
    zi = load_input_grads("fluid160_c5")
    m = stand_in_model(kw, sd)
    for p in m.parameters():
        p.requires_grad_(False)
    inp = golden_inputs(z)
    inp["node_loc"] = inp["node_loc"].clone().requires_grad_(True)
    out, X = m(**inp)
    assert out.requires_grad and out.grad_fn is not None          # the autograd path, not the inference path
    ((out * torch.from_numpy(zi["cot.out"]).float()).sum() + (X * torch.from_numpy(zi["cot.X"]).float()).sum()).backward()
    assert all(p.grad is None for p in m.parameters())
    assert rel_err(inp["node_loc"].grad, torch.from_numpy(zi["ig.node_loc"])) <= 2e-4
    m.input_grads = False                                        # flag off: frozen weights mean the inference path
    out2, _ = m(**golden_inputs(z))
    assert out2.grad_fn is None


# ======================================================================================================================
# GPU
# ======================================================================================================================
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def to_dev(inp):
    return {k: (v.to(dev()) if v is not None else None) for k, v in inp.items()}


def cuda_model(kw, sd, world_size=1):
    from distegnn_b200 import FastEGNN
    m = FastEGNN(hidden_nf=64, world_size=world_size, **kw)
    m.load_state_dict(sd)
    m.input_grads = True
    return m.to(dev())


def _close(a, b, tol=1e-5):
    """The weights-only and the *_inputs entry points run the same arithmetic, but the kernels accumulate with float
    atomics, so two launches agree to rounding, not bit for bit."""
    den = float(b.abs().max())
    return float((a - b).abs().max()) <= tol * den if den > 0 else float(a.abs().max()) == 0.0


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max() / b.detach().cpu().double().abs().max().clamp(min=1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, _lib.FLAG_NORMALIZE, _lib.FLAG_LAST])
@pytest.mark.parametrize("A", [0, 2, 8])
def test_edge_stage_input_backward(flags, A):
    """distegnn_edge_layer_bwd_inputs: g_edge_attr (accumulated) against float64 autograd; every other output equals the
    weights-only entry point to rounding."""
    from distegnn_b200 import synth
    from distegnn_b200.backend import cuda_backend
    from tests import shadow_autograd as sa
    be = cuda_backend()
    inp = to_dev(synth.make_partitions(synth.WORKLOADS["water3d_10k"], n_nodes=6_000, seed=21)[0])
    C, Na = 3, 0
    sd = orc.init_state_dict(2, Na, A, 64, C, 1, seed=5, coord_gain=1.0)
    m = cuda_model(dict(node_feat_nf=2, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=C, n_layers=1), sd)
    lp = m._packed_params(dev())["layers"][0]
    N, E = inp["node_loc"].shape[0], inp["edge_index"].shape[1]
    rowptr, row, col, perm = be.build_csr(inp["edge_index"], N)
    g = torch.Generator().manual_seed(6)
    ea = (torch.randn(E, A, generator=g) * 0.5).to(dev()) if A else None
    P, Q = torch.randn(N, 64, generator=g).to(dev()), torch.randn(N, 64, generator=g).to(dev())
    x4 = torch.zeros(N, 4, device=dev())
    x4[:, :3] = inp["node_loc"]
    g_m = torch.randn(N, 64, generator=g).to(dev())
    g_x = torch.zeros(N, 4, device=dev())
    g_x[:, :3] = torch.randn(N, 3, generator=g).to(dev())
    last = bool(flags & _lib.FLAG_LAST)
    outs = []
    for extra in (False, True):
        gP, gQ, gx4, glp = (torch.zeros_like(t) for t in (P, Q, x4, lp))
        g_ea = torch.full((E, A), 0.25, device=dev()) if (extra and A) else None       # accumulates onto what is there
        be.edge_layer_bwd((N, E, A, C, Na), flags, row, col, ea, x4, P, Q, lp, None if last else g_m, g_x, gP, gQ, gx4,
                          glp, None, g_ea)
        outs.append((gP, gQ, gx4, glp, g_ea))
    torch.cuda.synchronize()
    for a_, b_ in zip(outs[0][:4], outs[1][:4]):
        assert _close(b_, a_)
    if not A:
        return
    Pd, Qd, xd, lpd, ead = (t.double().requires_grad_(True) for t in (P, Q, x4[:, :3], lp, ea))
    am, ax = sa.edge_stage((N, E, A, C, Na), flags, row, col, ead, xd, Pd, Qd, lpd)
    loss = (ax * g_x[:, :3].double()).sum() + (0 if last else (am * g_m.double()).sum())
    (rea,) = torch.autograd.grad(loss, (ead,))
    e = _rel(outs[1][4] - 0.25, rea)
    print(f"edge stage input backward flags={flags} A={A}: g_edge_attr rel err {e:.1e}")
    assert e <= 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize("Na,last,N", [(0, False, 5_003), (2, False, 5_003), (8, False, 1_111), (2, True, 1_111),
                                       (8, False, 128)])
def test_node_stage_input_backward(Na, last, N):
    """distegnn_node_layer_bwd_inputs: g_node_vel / g_node_attr (accumulated) against float64 autograd of the stage; the
    other outputs equal the weights-only entry point to rounding.  N = 5003 / 1111 leave a ragged last tile."""
    from distegnn_b200.backend import cuda_backend
    be, sh = cuda_backend(), InputGradShadowBackend()
    A, C, B = 2, 3, 2
    g = torch.Generator().manual_seed(N + Na)
    sd = orc.init_state_dict(3, Na, A, 64, C, 2, seed=2, coord_gain=1.0)
    m = cuda_model(dict(node_feat_nf=3, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=C, n_layers=2), sd)
    pk = m._packed_params(dev())
    lp, lpn = pk["layers"][0], pk["layers"][1]
    K = 4 + 3 * C + 64 * C
    rnd = lambda *s: torch.randn(*s, generator=g)
    deg = torch.randint(0, 6, (N,), generator=g)
    rowptr = torch.zeros(N + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).to(torch.int32)
    batch32 = torch.sort(torch.randint(0, B, (N,), generator=g)).values.to(torch.int32)
    t = dict(h=rnd(N, 64), vel=rnd(N, 3), attr=rnd(N, Na) if Na else None, agg_m=rnd(N, 64) * 3, agg_v=rnd(N, 64),
             g_x=rnd(N, 3), g_vsum=rnd(B, K), g_h=rnd(N, 64), g_P=rnd(N, 64), g_Q=rnd(N, 64), g_Hn=rnd(N, 64))
    flags = _lib.FLAG_LAST if last else 0
    total = lp.numel()

    def run(backend, dt, device, extra):
        c = lambda v: None if v is None else v.to(device=device, dtype=dt)
        o = dict(g_h=torch.empty(N, 64, dtype=dt, device=device), g_x=torch.empty(N, 3, dtype=dt, device=device),
                 g_agg_x=torch.empty(N, 4, dtype=dt, device=device), g_trans_v=torch.empty(N, 4, dtype=dt, device=device),
                 g_agg_m=torch.zeros(N, 64, dtype=dt, device=device), g_agg_v=torch.zeros(N, 64, dtype=dt, device=device),
                 g_lp=torch.zeros(total, dtype=dt, device=device), g_lpn=torch.zeros(total, dtype=dt, device=device))
        kw = {}
        if extra:
            o["g_vel"] = torch.full((N, 3), 0.5, dtype=dt, device=device)
            o["g_attr"] = torch.full((N, Na), 0.5, dtype=dt, device=device) if Na else None
            kw = dict(g_vel=o["g_vel"], g_attr=o["g_attr"])
        backend.node_layer_bwd((N, B, A, C, Na), flags, rowptr.to(device), batch32.to(device), c(t["h"]), c(t["vel"]),
                               c(t["attr"]), None if last else c(t["agg_m"]), None if last else c(t["agg_v"]),
                               lp.to(device=device, dtype=dt), None if last else lpn.to(device=device, dtype=dt),
                               c(t["g_x"]), c(t["g_vsum"]), None if last else c(t["g_h"]), None if last else c(t["g_P"]),
                               None if last else c(t["g_Q"]), None if last else c(t["g_Hn"]), o["g_h"], o["g_x"],
                               o["g_agg_x"], o["g_trans_v"], None if last else o["g_agg_m"], None if last else o["g_agg_v"],
                               o["g_lp"], None if last else o["g_lpn"], **kw)
        return o
    plain, got = run(be, torch.float32, dev(), False), run(be, torch.float32, dev(), True)
    torch.cuda.synchronize()
    for k in plain:
        assert _close(got[k], plain[k]), k
    want = run(sh, torch.float64, torch.device("cpu"), True)
    errs = {"g_vel": _rel(got["g_vel"] - 0.5, want["g_vel"] - 0.5)}
    if Na:
        wa, ga = want["g_attr"] - 0.5, got["g_attr"] - 0.5
        if last:                                              # no node MLP in the last layer: nothing is added
            assert float(ga.abs().max()) == 0.0 and float(wa.abs().max()) == 0.0
        else:
            errs["g_attr"] = _rel(ga, wa)
    print(f"node stage input backward Na={Na} last={last} N={N}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) <= 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 3, 16])
@pytest.mark.parametrize("B", [1, 5])
def test_embed_input_backward(F, B):
    """distegnn_embed_bwd_inputs: g_node_feat = g_h0·emb_wtᵀ and g_node_loc = g_x0 + g_vsum0[batch, 0:3] against float64
    autograd of the embedding stage; the weight gradients equal the weights-only entry point to rounding."""
    from distegnn_b200.backend import cuda_backend
    be, sh = cuda_backend(), InputGradShadowBackend()
    A, C, Na, N = 2, 5, 0, 3_001
    K = 4 + 3 * C + 64 * C
    g = torch.Generator().manual_seed(F * 10 + B)
    sd = orc.init_state_dict(F, Na, A, 64, C, 1, seed=3)
    m = cuda_model(dict(node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=C, n_layers=1), sd)
    pk = m._packed_params(dev())
    lp0, emb_wt = pk["layers"][0], pk["emb_wt"].cpu()
    feat = torch.randn(N, F, generator=g)
    h0 = feat @ emb_wt + pk["emb_b"].cpu()
    gs = [torch.randn(N, 64, generator=g) for _ in range(4)]
    batch32 = torch.sort(torch.randint(0, B, (N,), generator=g)).values.to(torch.int32)
    g_x0, g_vsum0 = torch.randn(N, 3, generator=g), torch.randn(B, K, generator=g)

    def run(backend, dt, device, extra):
        c = lambda v: v.to(device=device, dtype=dt)
        o = [torch.zeros(F, 64, dtype=dt, device=device), torch.zeros(64, dtype=dt, device=device),
             torch.zeros(lp0.numel(), dtype=dt, device=device)]
        kw = {}
        if extra:
            kw = dict(g_feat=torch.empty(N, F, dtype=dt, device=device), g_loc=torch.empty(N, 3, dtype=dt, device=device),
                      emb_wt=c(emb_wt), batch32=batch32.to(device), g_x0=c(g_x0), g_vsum0=c(g_vsum0))
        backend.embed_bwd((N, B, F, A, C, Na), c(feat), c(h0), c(lp0), *[c(x) for x in gs], *o, **kw)
        return o + ([kw["g_feat"], kw["g_loc"]] if extra else [])
    plain, got = run(be, torch.float32, dev(), False), run(be, torch.float32, dev(), True)
    torch.cuda.synchronize()
    for a_, b_ in zip(plain, got):
        assert _close(b_, a_)
    want = run(sh, torch.float64, torch.device("cpu"), True)
    errs = dict(g_node_feat=_rel(got[3], want[3]), g_node_loc=_rel(got[4], want[4]))
    print(f"embed input backward F={F} B={B}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) <= 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", SINGLE_CASES)
def test_model_input_grads_against_reference_fixtures(name):
    z, kw, sd = load_golden(name)
    zi = load_input_grads(name)
    m = cuda_model(kw, sd).train()
    inp = leaves(golden_inputs(z), device=dev())
    out, X = m(**inp)
    loss = (out * torch.from_numpy(zi["cot.out"]).float().to(dev())).sum() + \
           (X * torch.from_numpy(zi["cot.X"]).float().to(dev())).sum()
    loss.backward()
    errs = check_inputs(inp, zi, "ig.", 2e-4)
    print(f"{name}: input gradients vs reference fp64: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))


def _oracle_input_grads(sd, host, cot_out, cot_X, normalize):
    sd64 = {k: v.double() for k, v in sd.items()}
    inp64 = leaves(host, dtype=torch.float64)
    o64, X64 = orc.forward(sd64, **inp64, normalize=normalize)
    ((o64 * cot_out.double()).sum() + (X64 * cot_X.double()).sum()).backward()
    return {k: inp64[k].grad for k in INPUTS if inp64.get(k) is not None}


@pytest.mark.gpu
@pytest.mark.parametrize("wname,n,normalize", [("fluid113k", 4000, False), ("water3d_10k", 3000, True)])
def test_model_input_grads_against_oracle_autograd(wname, n, normalize):
    from distegnn_b200 import synth
    w = synth.WORKLOADS[wname]
    host = synth.make_partitions(w, n_nodes=n, seed=31)[0]
    F, Na, A, C = w.node_feat_nf, w.node_attr_nf, 2, w.virtual_channels
    sd = orc.init_state_dict(F, Na, A, 64, C, 3, seed=12, coord_gain=0.05)
    kw = dict(node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=C, n_layers=3, normalize=normalize)
    g = torch.Generator().manual_seed(13)
    cot_out, cot_X = torch.randn(n, 3, generator=g), torch.randn(1, 3, C, generator=g)
    ref = _oracle_input_grads(sd, host, cot_out, cot_X, normalize)
    m = cuda_model(kw, sd).train()
    inp = leaves(host, device=dev())
    out, X = m(**inp)
    ((out * cot_out.to(dev())).sum() + (X * cot_X.to(dev())).sum()).backward()
    errs = {k: _rel(inp[k].grad, ref[k]) for k in ref if float(ref[k].abs().max()) > 0}
    print(f"{wname} n={n} normalize={normalize}: input gradients vs oracle fp64: "
          + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) <= 5e-4


@pytest.mark.gpu
def test_two_step_rollout_gradients_against_oracle():
    """The motivating use: step 1's prediction is step 2's position, vel = pos1 − pos0, edge_attr = ‖Δx‖ computed in torch
    from pos1; the loss is on step 2.  Gradients w.r.t. the parameters and pos0 against the fp64 oracle on the same
    rollout."""
    from distegnn_b200 import synth
    w = synth.WORKLOADS["fluid113k"]
    host = synth.make_partitions(w, n_nodes=3000, seed=17)[0]
    F, Na, A, C = w.node_feat_nf, w.node_attr_nf, 1, w.virtual_channels
    sd = orc.init_state_dict(F, Na, A, 64, C, 2, seed=19, coord_gain=0.05)
    kw = dict(node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=C, n_layers=2)
    ei = host["edge_index"]
    target = host["node_loc"] + 0.01 * torch.randn(host["node_loc"].shape, generator=torch.Generator().manual_seed(3))

    def rollout(fwd, pos0, vel0, t):
        ea0 = (pos0[ei[0]] - pos0[ei[1]]).norm(dim=1, keepdim=True)
        pos1, _ = fwd(pos0, vel0, pos0.mean(0, keepdim=True), ea0)
        ea1 = (pos1[ei[0]] - pos1[ei[1]]).norm(dim=1, keepdim=True)
        pos2, _ = fwd(pos1, pos1 - pos0, pos1.mean(0, keepdim=True), ea1)
        return ((pos2 - t) ** 2).sum()

    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    pos64 = host["node_loc"].double().requires_grad_(True)
    fo = lambda x, v, lm, ea: orc.forward(sd64, host["node_feat"].double(), x, v, lm, ei, host["data_batch"], ea,
                                          None if host["node_attr"] is None else host["node_attr"].double())
    l64 = rollout(fo, pos64, host["node_vel"].double(), target.double())
    keys = list(sd64)
    gr = torch.autograd.grad(l64, [pos64] + [sd64[k] for k in keys], allow_unused=True)
    ref_pos, ref_p = gr[0], dict(zip(keys, gr[1:]))

    m = cuda_model(kw, sd).train()
    d = to_dev(host)
    pos = d["node_loc"].clone().requires_grad_(True)
    fc = lambda x, v, lm, ea: m(d["node_feat"], x, v, lm, d["edge_index"], d["data_batch"], ea, d["node_attr"])
    ei = d["edge_index"]
    loss = rollout(fc, pos, d["node_vel"], target.to(dev()))
    loss.backward()
    errs = {"pos0": _rel(pos.grad, ref_pos)}
    for k, p in m.named_parameters():
        r = ref_p[k]
        if r is not None and float(r.abs().max()) > 0:
            errs[k] = _rel(p.grad, r)
    worst = max(errs, key=errs.get)
    print(f"two-step rollout: pos0 {errs['pos0']:.1e}, worst {worst} {errs[worst]:.1e}; loss {float(loss):.6e} vs "
          f"{float(l64):.6e}")
    assert errs[worst] <= 5e-4


def _rotation(seed):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return torch.from_numpy(q.astype(np.float32))


@pytest.mark.gpu
def test_input_grads_properties_at_200k_nodes():
    """Config-5 density at 200k nodes (≈4M edges): translation identity of the coordinate gradients, rotation behaviour of
    every input gradient, invariance of g_edge_attr to the edge order, and the CSRGraph path against the edge_index path."""
    from distegnn_b200 import synth
    from distegnn_b200.shards import CSRGraph
    w = synth.WORKLOADS["synth1m"]
    host = synth.make_partitions(w, n_nodes=200_000, seed=0)[0]
    sd = orc.init_state_dict(3, 2, 2, 64, 8, 4, seed=2, coord_gain=0.05)
    m = cuda_model(dict(node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2, virtual_channels=8, n_layers=4), sd).train()
    di = to_dev(host)
    N, B, C = di["node_loc"].shape[0], di["loc_mean"].shape[0], 8
    g = torch.Generator().manual_seed(4)
    cot, cotX = torch.randn(N, 3, generator=g).to(dev()), torch.randn(B, 3, C, generator=g).to(dev())

    def grads(inp, cot=cot, cotX=cotX):
        inp = leaves(inp)
        out, X = m(**inp)
        ((out * cot).sum() + (X * cotX).sum()).backward()
        return {k: inp[k].grad for k in INPUTS if inp.get(k) is not None}

    g0 = grads(di)
    # translation: out(x + t) = out(x) + t and X likewise, so Σ g_loc + Σ g_loc_mean = Σ cot_out + Σ_{b,c} cot_X
    lhs = g0["node_loc"].double().sum(0) + g0["loc_mean"].double().sum(0)
    rhs = cot.double().sum(0) + cotX.double().sum((0, 2))
    mag = g0["node_loc"].double().abs().sum(0) + g0["loc_mean"].double().abs().sum(0) + cot.double().abs().sum(0) \
        + cotX.double().abs().sum((0, 2))
    print("translation residual", (lhs - rhs).tolist(), "of", mag.tolist())
    assert float(((lhs - rhs).abs() / mag).max()) <= 1e-4
    # rotation: rotate the inputs and the cotangents; coordinate gradients rotate, the invariant ones stay
    R, t = _rotation(5).to(dev()), torch.tensor([0.3, -1.0, 2.0], device=dev())
    gr = grads({**di, "node_loc": di["node_loc"] @ R + t, "node_vel": di["node_vel"] @ R,
                "loc_mean": di["loc_mean"] @ R + t}, cot @ R, (cotX.permute(0, 2, 1) @ R).permute(0, 2, 1).contiguous())
    errs = {k: float((gr[k] - (g0[k] @ R if k in ("node_loc", "node_vel", "loc_mean") else g0[k])).abs().max()
                     / g0[k].abs().max()) for k in g0}
    print("rotation", errs)
    assert max(errs.values()) <= 1e-4
    # edge order: g_edge_attr follows its edge
    perm = torch.randperm(di["edge_index"].shape[1], generator=torch.Generator().manual_seed(1)).to(dev())
    gp = grads({**di, "edge_index": di["edge_index"][:, perm].contiguous(), "edge_attr": di["edge_attr"][perm].contiguous()})
    e_perm = float((gp["edge_attr"] - g0["edge_attr"][perm]).abs().max() / g0["edge_attr"].abs().max())
    # CSRGraph input: g_edge_attr comes back in the CSR order of the graph
    csr, ea_csr = CSRGraph.from_edge_index(di["edge_index"], N, di["edge_attr"])
    gc = grads({**di, "edge_index": csr, "edge_attr": ea_csr})
    order = torch.argsort(di["edge_index"][0], stable=True)
    e_csr = float((gc["edge_attr"] - g0["edge_attr"][order]).abs().max() / g0["edge_attr"].abs().max())
    print(f"edge-order {e_perm:.1e}, CSRGraph {e_csr:.1e}")
    assert e_perm <= 1e-5 and e_csr <= 1e-5
