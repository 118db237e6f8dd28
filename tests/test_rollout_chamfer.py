"""The rollout's per-step Chamfer distance against recorded frames (DESIGN §20): rollout(targets=..., chamfer=True) and
distegnn_rollout_chamfer.

CPU: the exported symbols and argument checks, the grid sizing's invariant through the testing library, rollout()'s
checks, and two gloo ranks with a torch stand-in for the kernels.  GPU: the kernel against float64 (per-node minima
bit for bit, per-graph sums against math.fsum, chamfer <= sq_err bit for bit), and inside rollouts: nothing else changes,
bitwise reproducibility across graph capture, capacities, an overflow rerun and a side stream, no host synchronisation,
a fixed launch count, and main.py."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from distegnn_b200 import _lib, rollout
from tests.test_rollout import FLUID, _cpu_case, _free_port
from tests.test_rollout_eval import (ErrStandIn, _fluid_batch, _model, _nbody, _node, _sq_err_kernel, _water, dev)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
INF, NAN, FLT_MAX = float("inf"), float("nan"), float(np.finfo(np.float32).max)


# ---- float64 reference: the same fp32 differences, squared and summed in fp64 in the same order -----------------------
def _d(p, q):
    """d(p, q) of every pair row by row: p [n,3], q [m,3] float32 -> float64 [n,m]."""
    dd = (p[:, None, :] - q[None, :, :]).astype(np.float64)      # fp32 differences, rounded to nearest
    return (dd[..., 0] * dd[..., 0] + dd[..., 1] * dd[..., 1]) + dd[..., 2] * dd[..., 2]


def _nearest(p, q):
    """min over q of d(p_i, q) for every row of p: brute force for small clouds, cKDTree candidates re-scored with the
    same expression for large ones."""
    if len(p) == 0:
        return np.zeros(0)
    if len(p) * len(q) <= 40_000_000:
        out = np.empty(len(p))
        step = max(1, 4_000_000 // len(q))
        for a in range(0, len(p), step):
            out[a:a + step] = _d(p[a:a + step], q).min(1)
        return out
    from scipy.spatial import cKDTree
    _, idx = cKDTree(q.astype(np.float64)).query(p.astype(np.float64), k=8, workers=-1)
    dd = (p[:, None, :] - q[idx]).astype(np.float64)
    return ((dd[..., 0] * dd[..., 0] + dd[..., 1] * dd[..., 1]) + dd[..., 2] * dd[..., 2]).min(1)


def ref_minima(pred, tg, batch, B):
    """float64 [2, N]: per-node minima prediction -> record and record -> prediction within each graph."""
    P, Q = pred.numpy().astype(F32), tg.numpy().astype(F32)
    b = np.zeros(len(P), np.int64) if batch is None else batch.numpy()
    out = np.zeros((2, len(P)))
    for g in range(B):
        i = np.nonzero(b == g)[0]
        out[0, i] = _nearest(P[i], Q[i])
        out[1, i] = _nearest(Q[i], P[i])
    return out


# ---- CPU: the C ABI ---------------------------------------------------------------------------------------------------
def test_abi_symbols_are_exported_and_arguments_checked():
    lib = _lib.load()
    assert lib.distegnn_abi_version() == 3
    for name in ("distegnn_rollout_chamfer", "distegnn_rollout_chamfer_workspace_bytes"):
        assert hasattr(lib, name)
    p = 256                                                    # never dereferenced: the checks return first
    nb = C.c_int64(0)
    assert lib.distegnn_rollout_chamfer_workspace_bytes(-1, 1, C.byref(nb)) == -1
    assert lib.distegnn_rollout_chamfer_workspace_bytes(10, 0, C.byref(nb)) == -1
    assert lib.distegnn_rollout_chamfer_workspace_bytes(1 << 29, 1, C.byref(nb)) == -1
    assert lib.distegnn_rollout_chamfer_workspace_bytes(10, 1, None) == -1
    assert lib.distegnn_rollout_chamfer(4, 2, 1, p, p, None, p, p, p, 1 << 20, None) == -1
    assert b"data_batch" in lib.distegnn_last_error()
    assert lib.distegnn_rollout_chamfer(4, 1, 0, p, p, None, p, p, p, 1 << 20, None) == -1     # steps
    assert lib.distegnn_rollout_chamfer(4, 1, 1, p, p, None, None, p, p, 1 << 20, None) == -1  # counter
    assert lib.distegnn_rollout_chamfer(4, 1, 1, p, p, None, p, p, p + 8, 1 << 20, None) == -1  # alignment
    assert lib.distegnn_rollout_chamfer(5000, 1, 1, p, p, None, p, p, p, 8, None) != 0         # workspace too small
    assert lib.distegnn_rollout_chamfer(0, 1, 1, None, None, None, p, p, None, 0, None) == 0   # nothing to do


# ---- CPU: grid sizing through the testing library -----------------------------------------------------------------------
def _grid_size(ext, budget):
    """distegnn_chamfer_grid_size (include/distegnn_b200_testing_grid.h) -> (cell, dims, ncell)."""
    from tests import twin_backend
    fn = twin_backend.load_testing().distegnn_chamfer_grid_size
    fn.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    fn.restype = C.c_int
    cell, dims, ncell = C.c_float(0), (C.c_int32 * 3)(), C.c_int64(0)
    e = (C.c_float * 3)(*ext)
    twin_backend.check(fn(C.addressof(e), int(budget), C.addressof(cell), C.addressof(dims), C.addressof(ncell)),
                       "chamfer_grid_size")
    return cell.value, list(dims), ncell.value


EXTENTS = [(1.0, 1.0, 1.0), (0.0, 0.0, 0.0), (30.0, 0.1, 0.1), (1e3, 1e3, 1e3), (1e4, 0.0, 2.0), (3e38, 3e38, 3e38),
           (3e38, 0.0, 0.0), (INF, 1.0, 1.0), (INF, INF, INF), (-INF, -INF, -INF), (NAN, 1.0, 2.0), (NAN, NAN, NAN),
           (1.0, -INF, NAN), (FLT_MAX, 1e-30, 7.0), (1e-40, 0.0, 0.0), (1e-30, 1e-30, 1e-30)]


@pytest.mark.parametrize("ext", EXTENTS)
def test_grid_size_keeps_every_key_inside_the_graph_cells(ext):
    """For any extent and budget: dims in [1, 1024], Πdims <= budget, a normal positive cell that covers the extent."""
    for budget in (1, 2, 3, 27, 100, 1001, 113_141, 2_000_001, 1 << 29):
        cell, dims, ncell = _grid_size(ext, budget)
        assert all(1 <= d <= 1024 for d in dims), (ext, budget, dims)
        assert ncell == dims[0] * dims[1] * dims[2] <= budget, (ext, budget, dims)
        assert np.isfinite(cell) and cell >= np.finfo(np.float32).tiny
        for e, d in zip(ext, dims):
            if np.isfinite(e) and e >= 0 and d > 1:
                assert e / cell < d + 1e-3                     # the grid covers the extent
            if not (np.isfinite(e) and e >= 0):
                assert d == 1                                  # a non-finite extent is one slab


def test_grid_size_holds_about_one_point_per_cell():
    for n in (100, 10_000, 1_000_000):
        _, dims, ncell = _grid_size((1.0, 1.0, 1.0), n + 1)
        assert (n + 1) / 1.25 ** 3 <= ncell <= n + 1
    _, dims, ncell = _grid_size((1.0, 0.0, 0.0), 1001)         # collinear: all cells on the one axis
    assert dims[1:] == [1, 1] and 800 <= dims[0] <= 1001
    assert _grid_size((FLT_MAX, FLT_MAX, FLT_MAX), 5)[1:] == ([1, 1, 1], 1)


# ---- CPU: rollout(chamfer=) ------------------------------------------------------------------------------------------
def _torch_chamfer(pred, tg, batch, B):
    m = ref_minima(pred.detach().cpu(), tg.detach().cpu(), None if batch is None else batch.cpu(), B)
    b = np.zeros(pred.shape[0], np.int64) if batch is None else batch.cpu().numpy()
    return torch.tensor([[math.fsum(m[k, b == g]) for k in (0, 1)] for g in range(B)], dtype=torch.float64)


class ChamferStandIn(ErrStandIn):
    """ErrStandIn plus the Chamfer sums in numpy (row counter[0], plain stores, the kernel's seven launches)."""

    def rollout_chamfer_workspace(self, n, B, device):
        return torch.zeros(16, dtype=torch.uint8, device=device)

    def rollout_chamfer(self, pred, targets, batch, counter, chamfer, ws):
        t = int(counter[0])
        if 0 <= t < chamfer.shape[0]:
            chamfer[t] = _torch_chamfer(pred, targets[t], batch, chamfer.shape[1])
        self.launches += 7


def test_rollout_chamfer_argument_checks():
    m, node, r, _ = _cpu_case(n=40)
    m._backend = be = ChamferStandIn()
    N = node["node_loc"].shape[0]
    good = node["node_loc"].float().expand(3, -1, -1).contiguous() + 0.01
    with pytest.raises(ValueError, match="chamfer=True needs targets"):
        rollout(m, **node, steps=3, radius=r, chamfer=True)
    for bad in (1, "yes", None):
        with pytest.raises(ValueError, match="chamfer"):
            rollout(m, **node, steps=3, radius=r, targets=good, chamfer=bad)
    assert be.launches == 0 and be.builds == []               # rejected before anything was enqueued
    res = rollout(m, **node, steps=3, radius=r, speed_col=0, targets=good, chamfer=True, return_trajectory=True)
    assert res.chamfer.shape == (3, 1, 2) and res.chamfer.dtype == torch.float64
    assert res.chamfer_mse.shape == (3, 2) and res.chamfer_mse.dtype == torch.float64
    want = torch.stack([_torch_chamfer(res.trajectory[t], good[t], None, 1) for t in range(3)])
    assert torch.equal(res.chamfer, want)
    assert torch.allclose(res.chamfer_mse, want[:, 0] / (3 * N), rtol=1e-15, atol=0)
    assert (res.chamfer_mse <= res.mse[:, None]).all()
    plain = rollout(m, **node, steps=3, radius=r, speed_col=0, targets=good)
    assert plain.chamfer is None and plain.chamfer_mse is None
    assert torch.equal(plain.sq_err, res.sq_err) and torch.equal(plain.node_loc, res.node_loc)


def _gloo_rank(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        m, node, r, _ = _cpu_case(n=240, world=2, rank=rank)
        N = node["node_loc"].shape[0]
        tg = node["node_loc"] + torch.randn(4, N, 3, generator=torch.Generator().manual_seed(rank)) * 0.01
        m._backend = ChamferStandIn()
        ref = rollout(m, **node, steps=4, radius=r, speed_col=0, check_every=4, targets=tg)
        m._backend = ChamferStandIn()
        calls = []
        orig = dist.all_reduce

        def counting(t, *a, **k):
            calls.append((tuple(t.shape), t.dtype))
            return orig(t, *a, **k)

        dist.all_reduce = counting
        res = rollout(m, **node, steps=4, radius=r, speed_col=0, check_every=4, capacity=ref.capacity, targets=tg,
                      chamfer=True, return_trajectory=True)
        dist.all_reduce = orig
        own = torch.stack([_torch_chamfer(res.trajectory[t], tg[t], None, 1) for t in range(4)])
        same = torch.equal(res.node_loc, ref.node_loc) and torch.equal(res.sq_err, ref.sq_err)
        q.put((rank, calls, own, res.chamfer, res.chamfer_mse, res.sq_err, N, same))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_ranks_sum_chamfer_in_the_final_reduction():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_rank, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in procs], key=lambda t: t[0])
    [p.join(timeout=60) for p in procs]
    L, Cv = FLUID["n_layers"], FLUID["virtual_channels"]
    K = 4 + 3 * Cv + 64 * Cv
    total = res[0][2] + res[1][2]
    n_all = res[0][6] + res[1][6]
    for rank, calls, own, ch, ch_mse, sq, N, same in res:
        assert same, f"rank {rank}: chamfer changed the rollout or sq_err"
        assert torch.equal(ch, total), f"rank {rank}: chamfer is not the sum of the partition-local sums"
        assert torch.allclose(ch_mse, total[:, 0] / (3 * n_all), rtol=1e-15, atol=0)
        assert (ch <= sq[:, :, None]).all()
        stats = [c for c in calls if c == ((1, K), torch.float32)]
        assert len(stats) == (L + 1) * 4                      # L+1 exchanges per step, as without chamfer
        assert calls.count(((1 * 4 + 4 * 1 + 4 * 1 * 2,), torch.float64)) == 1   # ONE end-of-rollout reduction
        assert calls.count(((1,), torch.int32)) == 1
        assert len(calls) == len(stats) + 2


# ---- GPU: the kernel against float64 ---------------------------------------------------------------------------------
def _al(x):
    return (x + 255) // 256 * 256


def _ws_minima(ws, N, B):
    """The per-node minima [2, N] in the workspace (csrc/chamfer.cu, chamfer_layout: bounds, flags, grids, keys, table,
    sorted points, then the minima)."""
    off = _al(24 * B) + _al(4 * B) + _al(40 * B) + _al(16 * N) + _al(4 * (2 * (N + B) + 1)) + _al(32 * N)
    return ws[off:off + 16 * N].view(torch.float64).view(2, N)


@pytest.mark.gpu
def test_workspace_size_and_a_too_small_workspace():
    lib = _lib.load()
    nb = C.c_int64(0)
    assert lib.distegnn_rollout_chamfer_workspace_bytes(1000, 3, C.byref(nb)) == 0 and nb.value >= 1000 * 72
    p = 256
    assert lib.distegnn_rollout_chamfer(1000, 3, 1, p, p, p, p, p, p, nb.value - 1, None) != 0
    assert b"workspace" in lib.distegnn_last_error()


def _chamfer_kernel(pred, tg, batch, B, t=1, steps=3):
    from distegnn_b200.backend import CudaBackend
    be = CudaBackend()
    N = pred.shape[0]
    full = torch.zeros(steps, N, 3, device=dev())
    full[t] = tg.to(dev())
    counter = torch.zeros(8, dtype=torch.int32, device=dev())
    counter[0] = t
    out = torch.full((steps, B, 2), -7.0, dtype=torch.float64, device=dev())
    ws = be.rollout_chamfer_workspace(N, B, dev())
    ws.fill_(0xA5)                                             # needs no initialisation
    be.rollout_chamfer(pred.to(dev()), full, None if batch is None else batch.to(dev()), counter, out, ws)
    torch.cuda.synchronize()
    return out.cpu(), _ws_minima(ws, N, B).cpu()


def _batch(sizes):
    return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))


def _noisy(sizes, seed=0, scale=1.0, noise=1e-2, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    N = sum(sizes)
    pred = torch.rand(N, 3, generator=g) * scale + offset
    tg = pred + torch.randn(N, 3, generator=g) * noise
    return pred, tg, _batch(sizes)


def _ring_boundaries():
    """Lattice points on cell faces, each graph's targets shifted along x by the ring-stop distance c·(1 − 2^-10), its
    fp32 neighbours, c and c/2; two shared corners fix every graph's box, so c is known in advance."""
    L = F32(8.0)
    n = 6 ** 3 + 2
    c = F32(_grid_size((L, L, L), n + 1)[0])
    ijk = np.stack(np.meshgrid(*[np.arange(6)] * 3, indexing="ij"), -1).reshape(-1, 3)
    lat = np.minimum((ijk * c).astype(F32), L)
    corners = np.array([[0, 0, 0], [L, L, L]], F32)
    bound = F32(c * F32(1 - 2 ** -10))
    P, Q, sizes = [], [], []
    for w in (bound, np.nextafter(bound, F32(0)), np.nextafter(bound, F32(10)), c, F32(c / 2)):
        q = lat.copy()
        q[:, 0] = np.minimum(q[:, 0] + w, L)
        P.append(np.concatenate([corners, lat]))
        Q.append(np.concatenate([corners, q]))
        sizes.append(n)
    return torch.from_numpy(np.concatenate(P)), torch.from_numpy(np.concatenate(Q)), _batch(sizes)


def _outliers():
    g = np.random.default_rng(3)
    dense = g.random((3000, 3), dtype=np.float32) * F32(0.01)
    sparse = g.random((20, 3), dtype=np.float32) * F32(10.0)
    far = np.array([[1e4, -1e4, 5e3]], F32)
    P = np.concatenate([dense, sparse, far])
    Q = np.concatenate([dense + g.normal(0, 1e-3, dense.shape).astype(F32), sparse[::-1], far * F32(0.5)])
    return torch.from_numpy(P), torch.from_numpy(Q), None


def _degenerate():
    """Flat, collinear and coincident clouds, and clouds of duplicates, one graph each."""
    g = torch.Generator().manual_seed(4)
    flat = torch.rand(500, 3, generator=g)
    flat[:, 2] = 0.25
    line = torch.zeros(400, 3)
    line[:, 0] = torch.rand(400, generator=g)
    same = torch.full((300, 3), 0.5)
    dup = torch.rand(50, 3, generator=g).repeat(6, 1)
    P = torch.cat([flat, line, same, dup])
    Q = torch.cat([flat.flip(0) + torch.randn(500, 3, generator=g) * 1e-3 * torch.tensor([1.0, 1.0, 0.0]),
                   line[torch.randperm(400, generator=g)] * 1.01, torch.full((300, 3), 0.75), dup.flip(0) + 1e-4])
    return P, Q, _batch([500, 400, 300, 300])


KERNEL_CASES = {
    "small graphs": lambda: _noisy([0, 1, 2, 31, 33, 255, 257]),
    "chunk boundaries": lambda: _noisy([2047, 1, 2049, 0, 4097, 6000], seed=1, noise=3e-2),
    "n-body 250x100": lambda: _noisy([100] * 250, seed=2, scale=5.0, noise=0.3),
    "offset 1e3": lambda: _noisy([700, 900], seed=5, offset=1e3),
    "offset -1e4": lambda: _noisy([800, 600], seed=6, offset=-1e4, noise=5e-3),
    "degenerate": _degenerate,
    "outliers": _outliers,
    "ring boundaries": _ring_boundaries,
}


def _check_case(pred, tg, batch):
    B = 1 if batch is None else int(batch.max()) + 1
    out, mins = _chamfer_kernel(pred, tg, batch, B)
    want = ref_minima(pred, tg, batch, B)
    assert np.array_equal(mins.numpy(), want), "per-node minima differ from the float64 reference"
    assert (out[[0, 2]] == -7.0).all(), "rows other than the counter's step were written"
    b = np.zeros(pred.shape[0], np.int64) if batch is None else batch.numpy()
    for g in range(B):
        for k in (0, 1):
            ref = math.fsum(want[k, b == g])
            got = float(out[1, g, k])
            assert abs(got - ref) <= 1e-12 * abs(ref), (g, k, got, ref)
    sq = _sq_err_kernel(pred.to(dev()), tg.to(dev()), None if batch is None else batch.to(dev()), B, 1, 3).cpu()
    assert (out[1] <= sq[1][:, None]).all(), "chamfer above sq_err"
    return out[1], sq[1]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(KERNEL_CASES))
def test_chamfer_kernel_against_float64(case):
    _check_case(*KERNEL_CASES[case]())


@pytest.mark.gpu
def test_chamfer_kernel_one_2m_node_graph():
    _check_case(*_noisy([2_000_000], seed=7, noise=2e-3))


@pytest.mark.gpu
def test_chamfer_of_a_permutation_is_zero():
    pred, _, batch = _noisy([1000, 3000, 17], seed=8)
    perm = torch.cat([torch.randperm(n, generator=torch.Generator().manual_seed(n)) + o
                      for n, o in ((1000, 0), (3000, 1000), (17, 4000))])
    out, mins = _chamfer_kernel(pred, pred[perm], batch, 3)
    assert (out[1] == 0).all() and (mins == 0).all()


@pytest.mark.gpu
def test_non_finite_graph_is_nan_and_its_neighbours_unaffected():
    pred, tg, batch = _noisy([300, 500, 400], seed=9)
    ref, _ = _chamfer_kernel(pred, tg, batch, 3)
    for cloud, bad in ((0, NAN), (1, INF), (0, -INF)):
        p2, t2 = pred.clone(), tg.clone()
        (p2 if cloud == 0 else t2)[300 + 250, 1] = bad
        out, _ = _chamfer_kernel(p2, t2, batch, 3)
        assert torch.isnan(out[1, 1]).all()
        assert torch.equal(out[1, [0, 2]], ref[1, [0, 2]])


@pytest.mark.gpu
def test_chamfer_kernel_outside_the_steps_writes_nothing():
    from distegnn_b200.backend import CudaBackend
    be = CudaBackend()
    pred, tg, batch = _noisy([500, 7000], seed=10)
    ws = be.rollout_chamfer_workspace(7500, 2, dev())
    want = _torch_chamfer(pred, tg, batch, 2)
    for t in (-1, 3, 2):
        counter = torch.tensor([t, 0, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=dev())
        o = torch.full((3, 2, 2), -7.0, dtype=torch.float64, device=dev())
        be.rollout_chamfer(pred.to(dev()), tg.to(dev()).expand(3, -1, -1).contiguous(), batch.to(dev()), counter, o, ws)
        o = o.cpu()
        if t == 2:                                             # the same workspace serves the next call
            assert ((o[2] - want).abs() <= 1e-12 * want.abs()).all() and (o[:2] == -7.0).all()
        else:
            assert (o == -7.0).all(), f"step {t} is outside [0, steps): nothing may be written"


# ---- GPU: rollouts ---------------------------------------------------------------------------------------------------
def _rollout_check(res, ex, kw):
    """chamfer <= sq_err bit for bit, and each step's sums against the float64 reference on the trajectory."""
    assert (res.chamfer <= res.sq_err[:, :, None]).all()
    assert (res.chamfer_mse <= res.mse[:, None]).all()
    for t in range(res.chamfer.shape[0]):
        want = _torch_chamfer(res.trajectory[t], ex["targets"][t], kw["data_batch"], 2)
        assert ((res.chamfer[t].cpu() - want).abs() <= 1e-12 * want.abs()).all(), t


@pytest.mark.gpu
def test_chamfer_changes_nothing_else_and_adds_a_fixed_launch_count(tmp_path):
    K = 5
    ld, kw, ex = _fluid_batch(tmp_path, K)
    m = _model(deterministic=True)
    be = m._get_backend(dev())
    common = dict(steps=K, radius=ld.radius, speed_col=2, tau=1.0, return_trajectory=True, targets=ex["targets"])
    cap = rollout(m, **_node(kw), **common).capacity
    n0 = be.launches
    plain = rollout(m, **_node(kw), capacity=cap, **common)
    n1 = be.launches
    res = rollout(m, **_node(kw), capacity=cap, chamfer=True, **common)
    n2 = be.launches
    assert (n2 - n1) - (n1 - n0) == 7 * K                      # seven launches per step (and the cub scan's)
    for k in ("node_loc", "node_vel", "node_feat", "loc_mean", "virtual_loc", "trajectory", "n_edges", "sq_err", "mse"):
        assert torch.equal(getattr(res, k), getattr(plain, k)), k
    _rollout_check(res, ex, kw)
    assert res.chamfer_mse.shape == (K, 2)
    want = res.chamfer.sum(1) / (3 * sum(ex["node_counts"]))
    assert torch.allclose(res.chamfer_mse, want, rtol=1e-15, atol=0)


@pytest.mark.gpu
def test_chamfer_is_bitwise_reproducible(tmp_path):
    """eager == graphed, two capacities, an overflow rerun == an ample capacity, and a rollout on a side stream while
    other work runs, all bit for bit (default mode: the Chamfer sums never depend on the order of any atomic)."""
    K = 6
    ld, kw, ex = _fluid_batch(tmp_path, K)
    m = _model()
    common = dict(steps=K, radius=ld.radius, speed_col=2, targets=ex["targets"], chamfer=True, return_trajectory=True)
    ref = rollout(m, **_node(kw), **common)
    cap = ref.capacity
    e0 = int(ref.n_edges.max())
    runs = {"eager, 2x capacity": rollout(m, **_node(kw), capacity=2 * cap, **common),
            "eager, 4x capacity": rollout(m, **_node(kw), capacity=4 * cap, **common)}
    m.cuda_graph = True
    runs["graphed"] = rollout(m, **_node(kw), capacity=2 * cap, **common)
    m.cuda_graph = False
    small = rollout(m, **_node(kw), capacity=max(1, e0 // 2), check_every=2, **common)
    assert small.regrowths
    runs["overflow rerun"] = small
    side = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device=dev())
    with torch.cuda.stream(side):
        runs["side stream"] = rollout(m, **_node(kw), capacity=2 * cap, **common)
    for _ in range(4):
        a = a @ a / 64.0                                       # work on the default stream meanwhile
    torch.cuda.synchronize()
    assert runs["graphed"].replays == K - 1
    _rollout_check(ref, ex, kw)
    for what, r in runs.items():
        # the trajectory itself may differ in default mode: compare chamfer with the reference of its own trajectory
        if torch.equal(r.trajectory, ref.trajectory):
            assert torch.equal(r.chamfer, ref.chamfer), what
            assert torch.equal(r.chamfer_mse, ref.chamfer_mse), what
        else:
            _rollout_check(r, ex, kw)


@pytest.mark.gpu
def test_chamfer_is_bitwise_reproducible_in_deterministic_mode(tmp_path):
    K = 4
    ld, kw, ex = _fluid_batch(tmp_path, K)
    m = _model(deterministic=True)
    common = dict(steps=K, radius=ld.radius, speed_col=2, targets=ex["targets"], chamfer=True)
    ref = rollout(m, **_node(kw), **common)
    cap = ref.capacity
    m.cuda_graph = True
    graphed = rollout(m, **_node(kw), capacity=3 * cap, **common)
    m.cuda_graph = False
    small = rollout(m, **_node(kw), capacity=max(1, int(ref.n_edges.max()) // 2), check_every=2, **common)
    assert small.regrowths
    for what, r in (("graphed", graphed), ("overflow rerun", small)):
        assert torch.equal(r.chamfer, ref.chamfer), what
        assert torch.equal(r.sq_err, ref.sq_err), what


@pytest.mark.gpu
def test_rollout_with_chamfer_never_synchronises(tmp_path):
    K = 4
    ld, kw, ex = _fluid_batch(tmp_path, K)
    m = _model()
    warm = rollout(m, **_node(kw), steps=K, radius=ld.radius, speed_col=2, targets=ex["targets"], chamfer=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = rollout(m, **_node(kw), steps=K, radius=ld.radius, speed_col=2, capacity=2 * warm.capacity,
                      check_every=0, targets=ex["targets"], chamfer=True, return_trajectory=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    res.check()
    _rollout_check(res, ex, kw)


@pytest.mark.gpu
def test_main_prints_chamfer_columns(tmp_path):
    import subprocess
    import yaml

    def run(cfg, data, K, *extra):
        p = tmp_path / "cfg.yaml"
        with open(p, "w") as f:
            yaml.safe_dump(cfg, f)
        return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--config_path", str(p), "--trajectory",
                               str(data), "--train_steps", "1", "--rollout_steps", str(K), *extra],
                              capture_output=True, text=True, timeout=600, cwd=ROOT)

    data = tmp_path / "water"
    for part, sizes, seed in (("train", [60, 50], 1), ("valid", [40, 45], 3)):
        (data / part).mkdir(parents=True)
        _water(data / part, sizes, T=10, seed=seed)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"].update(node_feat_nf=2, node_attr_nf=1)
    cfg["data"].update(dataset_name="Water3D", inner_radius=0.3, max_samples=4, split_mode="random", delta_t=2)
    r = run(cfg, data, 3, "--rollout_chamfer")
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [ln for ln in r.stdout.splitlines() if "rollout step" in ln]
    assert len(lines) == 3
    for ln in lines:
        mse = float(ln.split("MSE ")[1].split(",")[0])
        a = float(ln.split("pred->rec ")[1].split(",")[0])
        b = float(ln.split("rec->pred ")[1])
        assert 0 <= a <= mse and 0 <= b <= mse, ln
    r = run(cfg, data, 3)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [ln for ln in r.stdout.splitlines() if "rollout step" in ln]
    assert len(lines) == 3 and not any("Chamfer" in ln for ln in lines)
    assert all(ln.startswith(f"[water3d] rollout step {t + 1}: MSE ") and len(ln.split()) == 6
               for t, ln in enumerate(lines))
    data = tmp_path / "nbody"
    _nbody(data, "train", S=4, T=10)
    _nbody(data, "valid", S=2, T=10, seed=5)
    with open(os.path.join(ROOT, "config", "nbody_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(batch_size=2, frame_0=1, frame_T=3, cutoff_rate=0.5)
    r = run(cfg, data, 3, "--rollout_tau", "0.5", "--rollout_chamfer")
    assert r.returncode == 0, r.stderr[-3000:]
    assert "rollout step 3: MSE" in r.stdout and "rec->pred" in r.stdout, r.stdout
