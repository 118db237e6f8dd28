"""chamfer_distance(): the differentiable Chamfer distance (DESIGN §21) and its C ABI, distegnn_chamfer_distance and
distegnn_chamfer_distance_bwd.

CPU: the Python argument checks and the C-ABI argument checks.  GPU: the nearest ids against a numpy brute force with the
same distance and tie rule, the sums bit for bit against distegnn_rollout_chamfer, the gradient bit for bit against a
numpy restatement of the backward rule and against float64 autograd of a brute-force Chamfer loss, the special cases,
reproducibility (graph capture and a side stream included), no host synchronisation, and a Chamfer loss through
differentiable_rollout."""
import ctypes as C

import numpy as np
import pytest
import torch

from distegnn_b200 import _lib, chamfer_distance, differentiable_rollout, rollout
from tests.test_rollout_chamfer import KERNEL_CASES, _batch, _chamfer_kernel, _d, _noisy
from tests.test_rollout_eval import _fluid_batch, _model, _node, dev

F32 = np.float32
NAN = float("nan")


# ---- CPU: argument checks ---------------------------------------------------------------------------------------------
def test_python_argument_checks():
    good = torch.zeros(4, 3)
    b = torch.zeros(4, dtype=torch.int64)
    bad = [
        ((good.double(), good), "float32"),
        ((good, good.half()), "float32"),
        ((torch.zeros(4, 2), good), r"\[N,3\]"),
        ((torch.zeros(4, 3, 1), good), r"\[N,3\]"),
        ((good, torch.zeros(6, 3)[::2]), "contiguous"),
        ((good, torch.zeros(5, 3)), "same rows"),
        ((good, good, b.int()), "int64"),
        ((good, good, b[:3]), "int64"),
        ((good, good, torch.zeros(8, dtype=torch.int64)[::2]), "contiguous"),
        ((good, good, b, 0), "n_graphs"),
        ((good, good, b, True), "n_graphs"),
        ((good, good, b, 2.0), "n_graphs"),
        ((good, good, None, 2), "needs data_batch"),
        ((good, good), "CUDA"),
        ((good, good, b, 1), "CUDA"),
        (([[0.0] * 3] * 4, good), "tensor"),
    ]
    for args, msg in bad:
        with pytest.raises(ValueError, match=msg):
            chamfer_distance(*args)


def test_c_abi_argument_checks():
    lib = _lib.load()
    for name in ("distegnn_chamfer_distance", "distegnn_chamfer_distance_bwd",
                 "distegnn_chamfer_distance_bwd_workspace_bytes"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    p = 256                                                    # never dereferenced: the checks return first
    nb = C.c_int64(0)
    # forward: (N, B, pred, target, batch, out, nearest, ws, bytes, stream)
    assert lib.distegnn_chamfer_distance(-1, 1, p, p, None, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_chamfer_distance(4, 0, p, p, None, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_chamfer_distance(1 << 29, 1, p, p, None, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_chamfer_distance(4, 2, p, p, None, p, p, p, 1 << 20, None) == -1
    assert b"data_batch" in lib.distegnn_last_error()
    assert lib.distegnn_chamfer_distance(4, 1, p, p, None, None, p, p, 1 << 20, None) == -1      # out
    assert lib.distegnn_chamfer_distance(4, 1, p, p, None, p, None, p, 1 << 20, None) == -1      # nearest
    assert lib.distegnn_chamfer_distance(4, 1, None, p, None, p, p, p, 1 << 20, None) == -1      # pred
    assert lib.distegnn_chamfer_distance(4, 1, p, p, None, p, p, None, 1 << 20, None) == -1      # workspace
    assert lib.distegnn_chamfer_distance(4, 1, p, p, None, p, p, p + 8, 1 << 20, None) == -1     # alignment
    assert lib.distegnn_chamfer_distance(5000, 1, p, p, None, p, p, p, 8, None) != 0             # workspace too small
    # backward: (N, B, pred, target, batch, nearest, g, g_pred, g_target, ws, bytes, stream)
    assert lib.distegnn_chamfer_distance_bwd_workspace_bytes(-1, C.byref(nb)) == -1
    assert lib.distegnn_chamfer_distance_bwd_workspace_bytes(1 << 29, C.byref(nb)) == -1
    assert lib.distegnn_chamfer_distance_bwd_workspace_bytes(10, None) == -1
    assert lib.distegnn_chamfer_distance_bwd(-1, 1, p, p, None, p, p, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_chamfer_distance_bwd(4, 0, p, p, None, p, p, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_chamfer_distance_bwd(4, 2, p, p, None, p, p, p, p, p, 1 << 20, None) == -1
    assert b"data_batch" in lib.distegnn_last_error()
    assert lib.distegnn_chamfer_distance_bwd(4, 1, p, p, None, None, p, p, p, p, 1 << 20, None) == -1   # nearest
    assert lib.distegnn_chamfer_distance_bwd(4, 1, p, p, None, p, None, p, p, p, 1 << 20, None) == -1   # g
    assert lib.distegnn_chamfer_distance_bwd(4, 1, p, p, None, p, p, p, p, None, 1 << 20, None) == -1  # workspace
    assert lib.distegnn_chamfer_distance_bwd(4, 1, p, p, None, p, p, p, p, p + 4, 1 << 20, None) == -1  # alignment
    assert lib.distegnn_chamfer_distance_bwd(5000, 1, p, p, None, p, p, p, p, p, 8, None) != 0         # too small
    assert lib.distegnn_chamfer_distance_bwd(4, 1, p, p, None, p, p, None, None, p, 8, None) == 0      # nothing asked
    assert lib.distegnn_chamfer_distance_bwd(0, 1, None, None, None, None, None, p, p, None, 0, None) == 0


# ---- numpy references ---------------------------------------------------------------------------------------------------
def _nearest_ids(p, q):
    """(min, id) of d(p_i, ·) over q for every row of p (ids local to the graph) under the tie rule: the matched row i
    when it attains the minimum, else the smallest minimiser.  Brute force in row blocks; cKDTree candidates (and the
    matched row) re-scored with the same expression for large clouds."""
    n = len(p)
    mins, ids = np.zeros(n), np.zeros(n, np.int64)
    if n == 0:
        return mins, ids
    rows = np.arange(n)
    if n * n > 40_000_000:
        from scipy.spatial import cKDTree
        _, cand = cKDTree(q.astype(np.float64)).query(p.astype(np.float64), k=8, workers=-1)
        cand = np.concatenate([cand, rows[:, None]], 1)
        dd = (p[:, None, :] - q[cand]).astype(np.float64)
        d = (dd[..., 0] * dd[..., 0] + dd[..., 1] * dd[..., 1]) + dd[..., 2] * dd[..., 2]
        m = d.min(1)
        mins[:] = m
        big = np.where(d == m[:, None], cand, np.iinfo(np.int64).max).min(1)
        ids[:] = np.where(d[:, -1] == m, rows, big)
        return mins, ids
    step = max(1, 4_000_000 // n)
    for a in range(0, n, step):
        d = _d(p[a:a + step], q)
        m = d.min(1)
        r = rows[a:a + step]
        first = np.argmax(d == m[:, None], 1)                  # the smallest minimiser
        mins[a:a + step] = m
        ids[a:a + step] = np.where(d[np.arange(len(r)), r] == m, r, first)
    return mins, ids


def ref_nearest(pred, tg, batch, B):
    """int64 [2N] nearest ids (global) under the tie rule, −1 in a graph with a non-finite coordinate."""
    P, Q = pred.numpy().astype(F32), tg.numpy().astype(F32)
    N = len(P)
    b = np.zeros(N, np.int64) if batch is None else batch.numpy()
    out = np.full(2 * N, -1, np.int64)
    for g in range(B):
        i = np.nonzero(b == g)[0]
        if len(i) == 0 or not (np.isfinite(P[i]).all() and np.isfinite(Q[i]).all()):
            continue
        lo = i[0]
        out[i] = _nearest_ids(P[i], Q[i])[1] + lo
        out[N + i] = _nearest_ids(Q[i], P[i])[1] + lo
    return out


def ref_grad(pred, tg, batch, nearest, g):
    """The backward rule restated: row r's own term 2·g·fl32(x_r − y_{n(r)}), then the terms of the rows whose nearest it
    is, in ascending row, each product and sum in float64 round-to-nearest, rounded once to float32.  -> (g_pred, g_target)
    float32 [N,3]; NaN rows where the id is −1."""
    P, Q = pred.numpy().astype(F32), tg.numpy().astype(F32)
    N = len(P)
    b = np.zeros(N, np.int64) if batch is None else batch.numpy()
    n = np.asarray(nearest, np.int64)
    r = np.arange(2 * N)
    c = (r >= N).astype(np.int64)
    i = r - c * N
    X = np.concatenate([P, Q])                                 # the row's own point
    other = np.where(c[:, None] == 1, P[np.clip(n, 0, N - 1)], Q[np.clip(n, 0, N - 1)])
    g2 = 2.0 * np.asarray(g, np.float64)
    bb = b[i]
    g_own, g_in = g2[bb, c], g2[bb, 1 - c]
    valid = n >= 0
    acc = g_own[:, None] * (X - other).astype(np.float64)
    key = np.where(valid, np.where(r < N, N + n, n), 2 * N)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    rank = r - np.searchsorted(ks, ks, "left")
    for k in range(int(rank.max()) + 1 if N else 0):
        sel = (rank == k) & (ks < 2 * N)
        dst, src = ks[sel], order[sel]
        acc[dst] = acc[dst] + g_in[dst][:, None] * (X[dst] - X[src]).astype(np.float64)
    out = acc.astype(F32)
    out[~valid] = NAN
    return out[:N], out[N:]


# ---- GPU helpers ------------------------------------------------------------------------------------------------------
def _graphs(batch):
    return 1 if batch is None or len(batch) == 0 else int(batch.max()) + 1


def _fwd_raw(pred, tg, batch, B):
    """distegnn_chamfer_distance through the backend -> (out [B,2], nearest [2N]) on the CPU."""
    from distegnn_b200.backend import cuda_backend
    be = cuda_backend()
    N = pred.shape[0]
    out = torch.full((B, 2), -7.0, dtype=torch.float64, device=dev())
    nearest = torch.full((2 * N,), -9, dtype=torch.int32, device=dev())
    ws = be.rollout_chamfer_workspace(N, B, dev())
    ws.fill_(0x5A)                                             # needs no initialisation
    be.chamfer_distance(pred.to(dev()), tg.to(dev()), None if batch is None else batch.to(dev()), out, nearest, ws)
    torch.cuda.synchronize()
    return out.cpu(), nearest.cpu()


def _g(B, seed):
    """Per-graph, per-direction upstream values, some of them 0."""
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, 2, generator=gen, dtype=torch.float64)
    g[torch.rand(B, 2, generator=gen) < 0.25] = 0.0
    return g


def _autograd(pred, tg, batch, B, g, need=(True, True)):
    p = pred.to(dev()).clone().requires_grad_(need[0])
    t = tg.to(dev()).clone().requires_grad_(need[1])
    out = chamfer_distance(p, t, None if batch is None else batch.to(dev()), B)
    (out * g.to(dev())).sum().backward()
    return out.detach().cpu(), (None if p.grad is None else p.grad.cpu()), (None if t.grad is None else t.grad.cpu())


def _bits(x):
    return x.numpy().view(np.uint32) if isinstance(x, torch.Tensor) else x.view(np.uint32)


def _same_bits(got, want):
    got = got.numpy() if isinstance(got, torch.Tensor) else got
    want = want.numpy() if isinstance(want, torch.Tensor) else want
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    return np.array_equal(nan_g, nan_w) and np.array_equal(got[~nan_g].view(np.uint32), want[~nan_w].view(np.uint32))


def _lattice_ties():
    """Each record sits at the centre of 8 equidistant predictions, with the records' rows shuffled, so the matched node
    is not among them and the id is the smallest of 8; and each prediction has 8 equidistant records."""
    ijk = np.stack(np.meshgrid(*[np.arange(7)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(F32) * F32(0.5)
    P = ijk
    Q = (ijk + F32(0.25))[np.random.default_rng(11).permutation(len(ijk))]
    return torch.from_numpy(P), torch.from_numpy(Q), None


def _coincident_ties():
    """Duplicates in both clouds, coincident pairs and one point on top of many copies."""
    g = np.random.default_rng(12)
    base = g.random((40, 3), dtype=np.float32)
    P = np.concatenate([np.repeat(base, 5, 0), np.full((60, 3), 0.5, F32)])
    Q = np.concatenate([np.tile(base, (5, 1)), np.full((60, 3), 0.5, F32)])[g.permutation(260)]
    return torch.from_numpy(P), torch.from_numpy(Q), _batch([130, 130])


def _outlier_ties():
    """Far points whose nearest lie in a dense cluster, with 40 exact copies of the nearest one: the warp scan's lanes
    see tied minima."""
    g = np.random.default_rng(13)
    dense = g.random((3000, 3), dtype=np.float32) * F32(0.01)
    near_p = np.repeat(np.array([[0.02, 0.0, 0.0]], F32), 40, 0)
    near_q = np.repeat(np.array([[-0.02, 0.0, 0.0]], F32), 40, 0)
    far_p = np.array([[100.0, 0.0, 0.0], [90.0, 1.0, 0.0]], F32)
    far_q = np.array([[-100.0, 0.0, 0.0], [-95.0, 0.0, 1.0]], F32)
    P = np.concatenate([dense, near_p, far_p, far_q * F32(0.5)])
    Q = np.concatenate([dense[::-1] + F32(1e-4), near_q, far_q, far_p * F32(0.5)])
    return torch.from_numpy(P), torch.from_numpy(Q), None


CASES = dict(KERNEL_CASES)
CASES.update({
    "offset -1e3": lambda: _noisy([500, 400], seed=14, offset=-1e3),
    "offset 1e4": lambda: _noisy([600, 300], seed=15, offset=1e4, noise=5e-3),
    "lattice ties": _lattice_ties,
    "coincident ties": _coincident_ties,
    "outlier ties": _outlier_ties,
})


# ---- GPU: nearest ids, sums, gradients -----------------------------------------------------------------------------------
def _check_all(pred, tg, batch, seed=0):
    B = _graphs(batch)
    out, nearest = _fwd_raw(pred, tg, batch, B)
    want = ref_nearest(pred, tg, batch, B)
    assert np.array_equal(nearest.numpy().astype(np.int64), want), \
        f"{int((nearest.numpy() != want).sum())} nearest ids differ from the brute force"
    ev, _ = _chamfer_kernel(pred, tg, batch, B)                # the rollout's kernel at step 1 of 3
    assert _same_bits(out, ev[1]), "sums differ from distegnn_rollout_chamfer"
    g = _g(B, seed)
    for need in ((True, True), (True, False), (False, True)):
        val, gp, gt = _autograd(pred, tg, batch, B, g, need)
        assert _same_bits(val, out)
        wp, wt = ref_grad(pred, tg, batch, want, g.numpy())
        if need[0]:
            assert _same_bits(gp, wp), f"g_pred differs from the restated rule ({need})"
        else:
            assert gp is None
        if need[1]:
            assert _same_bits(gt, wt), f"g_target differs from the restated rule ({need})"
        else:
            assert gt is None


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_ids_sums_and_gradients(case):
    _check_all(*CASES[case](), seed=len(case))


@pytest.mark.gpu
def test_one_2m_node_graph():
    _check_all(*_noisy([2_000_000], seed=7, noise=2e-3), seed=3)


def _margin_case(seed):
    """Jittered lattice predictions and records drawn onto lattice sites with repetition: several records share a
    prediction, some predictions have none nearby."""
    g = np.random.default_rng(seed)
    sizes = [64, 125]
    P, Q = [], []
    for n in sizes:
        k = round(n ** (1 / 3))
        site = np.stack(np.meshgrid(*[np.arange(k)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
        P.append(site + g.uniform(-0.1, 0.1, site.shape))
        Q.append(site[g.integers(0, len(site), len(site))] + g.uniform(-0.1, 0.1, site.shape))
    return (torch.from_numpy(np.concatenate(P).astype(F32)), torch.from_numpy(np.concatenate(Q).astype(F32)),
            _batch(sizes))


def _margin(p, q):
    d = np.sort(_d(p, q), 1)
    return float(((d[:, 1] - d[:, 0]) / d[:, 1]).min())


@pytest.mark.gpu
def test_gradient_against_float64_autograd():
    """The formula itself: float64 torch autograd of Σ g·(brute-force min) on clouds whose minimisers are unique with a
    margin, within 1e-6 of each row's Σ|terms|."""
    pred, tg, batch = _margin_case(0)
    P, Q, b = pred.numpy(), tg.numpy(), batch.numpy()
    for gi in range(2):
        i = np.nonzero(b == gi)[0]
        assert _margin(P[i], Q[i]) > 1e-3 and _margin(Q[i], P[i]) > 1e-3
    g = _g(2, 5)
    _, gp, gt = _autograd(pred, tg, batch, 2, g)
    p64, t64 = pred.double().requires_grad_(True), tg.double().requires_grad_(True)
    loss, scale_p, scale_t = 0.0, torch.zeros(len(P), 3, dtype=torch.float64), torch.zeros(len(P), 3, dtype=torch.float64)
    for gi in range(2):
        i = torch.from_numpy(np.nonzero(b == gi)[0])
        d = ((p64[i][:, None] - t64[i][None]) ** 2).sum(-1)
        loss = loss + g[gi, 0] * d.min(1).values.sum() + g[gi, 1] * d.min(0).values.sum()
        with torch.no_grad():                                  # Σ|terms| per row: |own| + Σ |incoming|
            n0, n1 = d.argmin(1), d.argmin(0)
            dp0 = (p64[i] - t64[i][n0]).abs() * 2 * abs(g[gi, 0])
            dt1 = (t64[i] - p64[i][n1]).abs() * 2 * abs(g[gi, 1])
            scale_p[i] += dp0
            scale_t[i] += dt1
            scale_p[i] += torch.zeros_like(dp0).index_add_(0, n1, dt1)
            scale_t[i] += torch.zeros_like(dt1).index_add_(0, n0, dp0)
    wp, wt = torch.autograd.grad(loss, [p64, t64])
    for got, want, s, what in ((gp, wp, scale_p, "pred"), (gt, wt, scale_t, "target")):
        err = ((got.double() - want).abs() / s.clamp(min=1e-300)).max()
        assert float(err) <= 1e-6, (what, float(err))


@pytest.mark.gpu
def test_permutation_gives_zero_value_and_zero_gradient():
    pred, _, batch = _noisy([1000, 3000, 17], seed=8)
    perm = torch.cat([torch.randperm(n, generator=torch.Generator().manual_seed(n)) + o
                      for n, o in ((1000, 0), (3000, 1000), (17, 4000))])
    val, gp, gt = _autograd(pred, pred[perm], batch, 3, torch.ones(3, 2, dtype=torch.float64))
    assert (val == 0).all() and (gp == 0).all() and (gt == 0).all()


@pytest.mark.gpu
def test_non_finite_graph_gives_nan_rows_in_that_graph_only():
    pred, tg, batch = _noisy([300, 500, 400], seed=9)
    g = torch.ones(3, 2, dtype=torch.float64)
    ref = _autograd(pred, tg, batch, 3, g)
    rows = slice(300, 800)
    for cloud, bad in ((0, NAN), (1, float("inf")), (0, -float("inf"))):
        p2, t2 = pred.clone(), tg.clone()
        (p2 if cloud == 0 else t2)[550, 1] = bad
        val, gp, gt = _autograd(p2, t2, batch, 3, g)
        _, nearest = _fwd_raw(p2, t2, batch, 3)
        assert torch.isnan(val[1]).all() and torch.equal(val[[0, 2]], ref[0][[0, 2]])
        assert (nearest[300:800] == -1).all() and (nearest[1500:2000] == -1).all()
        assert torch.isnan(gp[rows]).all() and torch.isnan(gt[rows]).all()
        for got, want in ((gp, ref[1]), (gt, ref[2])):
            keep = torch.ones(1200, dtype=torch.bool)
            keep[rows] = False
            assert torch.equal(got[keep], want[keep])


@pytest.mark.gpu
def test_empty_cloud_and_empty_graphs():
    z = torch.zeros(0, 3, device=dev(), requires_grad=True)
    out = chamfer_distance(z, torch.zeros(0, 3, device=dev()), torch.zeros(0, dtype=torch.int64, device=dev()), 3)
    assert out.shape == (3, 2) and (out == 0).all()
    out.sum().backward()
    assert z.grad.shape == (0, 3)


# ---- GPU: reproducibility, capture, no synchronisation ---------------------------------------------------------------
def _raw_pair(be, p, t, batch, B, g, bufs):
    """One forward and one backward through the C ABI into preallocated buffers."""
    out, nearest, gp, gt, ws_f, ws_b = bufs
    be.chamfer_distance(p, t, batch, out, nearest, ws_f)
    be.chamfer_distance_bwd(p, t, batch, nearest, g, gp, gt, ws_b)


@pytest.mark.gpu
def test_bitwise_reproducible_across_calls_streams_and_graph_capture():
    from distegnn_b200.backend import cuda_backend
    be = cuda_backend()
    pred, tg, batch = _noisy([5000, 20_000, 3], seed=16, noise=0.05)
    p, t, b = pred.to(dev()), tg.to(dev()), batch.to(dev())
    B, N = 3, p.shape[0]
    g = _g(B, 17).to(dev())

    def bufs():
        return (torch.empty(B, 2, dtype=torch.float64, device=dev()), torch.empty(2 * N, dtype=torch.int32, device=dev()),
                torch.empty(N, 3, device=dev()), torch.empty(N, 3, device=dev()), be.rollout_chamfer_workspace(N, B, dev()),
                be.chamfer_distance_bwd_workspace(N, dev()))

    runs = {}
    for what in ("first", "second"):
        bb = bufs()
        _raw_pair(be, p, t, b, B, g, bb)
        runs[what] = bb
    side = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device=dev())
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        bb = bufs()
        _raw_pair(be, p, t, b, B, g, bb)
        runs["side stream"] = bb
    for _ in range(4):
        a = a @ a / 64.0                                       # work on the default stream meanwhile
    torch.cuda.synchronize()
    bb = bufs()
    _raw_pair(be, p, t, b, B, g, bb)                           # warm-up outside the capture
    for x in bb[:4]:
        x.fill_(-1)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _raw_pair(be, p, t, b, B, g, bb)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    runs["graphed"] = bb
    ref = runs.pop("first")
    for what, r in runs.items():
        for x, y in zip(ref[:4], r[:4]):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), what
    _, via_autograd_p, via_autograd_t = _autograd(pred, tg, batch, B, g.cpu())
    assert torch.equal(via_autograd_p, ref[2].cpu()) and torch.equal(via_autograd_t, ref[3].cpu())


@pytest.mark.gpu
def test_forward_and_backward_with_n_graphs_never_synchronise():
    pred, tg, batch = _noisy([700, 900], seed=18)
    p = pred.to(dev()).requires_grad_(True)
    t, b = tg.to(dev()), batch.to(dev())
    chamfer_distance(p, t, b, 2).sum().backward()              # warm-up: library load, allocator
    p.grad = None
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = chamfer_distance(p, t, b, 2)
        (out[:, 0] * 0.5 + out[:, 1]).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert p.grad is not None and torch.isfinite(p.grad).all()


# ---- GPU: through a differentiable rollout -------------------------------------------------------------------------------
@pytest.mark.gpu
def test_chamfer_loss_through_differentiable_rollout(tmp_path):
    """The INTEGRATION §1 Chamfer loss on differentiable_rollout(...).trajectory: the gradient reaching the trajectory is
    chamfer_distance's own on the detached trajectory, bit for bit; the parameter and input gradients match a second
    rollout driven by that gradient within §15's 1e-4 (the model's backward adds with atomics)."""
    from tests.test_rollout_grad import _param_errs, _rel
    K = 4
    ld, kw, ex = _fluid_batch(tmp_path, K, sizes=(170, 130), step=0.5)
    node, batch, B = _node(kw), kw["data_batch"], 2
    N = node["node_loc"].shape[0]
    m = _model().train()
    cap = 2 * rollout(m, **node, steps=K, radius=ld.radius, speed_col=2).capacity

    def leaves():
        return {k: (v.clone().requires_grad_(True) if k in ("node_loc", "node_vel") else v) for k, v in node.items()}

    seen = {}
    leaf = leaves()
    res = differentiable_rollout(m, **leaf, steps=K, radius=ld.radius, speed_col=2, capacity=cap)
    res.trajectory.register_hook(lambda g: seen.setdefault("g", g.clone()))
    loss = sum(chamfer_distance(res.trajectory[t], ex["targets"][t], batch, B).sum() for t in range(K)) / (3 * N * K)
    loss.backward()
    res.check()
    traj = res.trajectory.detach().clone().requires_grad_(True)
    direct = sum(chamfer_distance(traj[t], ex["targets"][t], batch, B).sum() for t in range(K)) / (3 * N * K)
    direct.backward()
    assert torch.equal(seen["g"], traj.grad)
    assert float(traj.grad.abs().max()) > 0
    got_p = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    got_in = {k: leaf[k].grad.clone() for k in ("node_loc", "node_vel")}
    m.zero_grad(set_to_none=True)
    leaf2 = leaves()
    res2 = differentiable_rollout(m, **leaf2, steps=K, radius=ld.radius, speed_col=2, capacity=cap)
    res2.trajectory.backward(traj.grad)
    res2.check()
    ref_p = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert set(ref_p) == set(got_p) and ref_p
    errs = _param_errs(got_p, ref_p)
    errs.update({k: _rel(got_in[k], leaf2[k].grad) for k in got_in})
    worst = max(errs, key=errs.get)
    assert errs[worst] <= 1e-4, (worst, errs[worst])
