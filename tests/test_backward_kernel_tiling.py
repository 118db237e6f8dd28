"""Tensor-core backward kernels (edge_layer_bwd_tc_kernel, virtual_layer_bwd_tc_kernel) on the shapes their tiling makes
fragile.  Edge stage: every edge-attribute count through both instantiations (weights only and with g_edge_attr), ragged
and tiny edge counts, a destination run that crosses warps and tiles next to degree-one rows, isolated nodes, self loops,
a device-side edge count far below the capacity, many tiles per CTA, extreme rows of P and upstream gradients over
2^-60 … 2^60, and rerun determinism.  Real↔virtual stage: channel counts that do and do not divide the 128-row tile,
thousands of tiny graphs (and graph ids without nodes), graphs spanning many strided tiles of one CTA, ragged node
counts, nodes sitting exactly on a virtual node, and upstream gradients over 2^-60 … 2^60.  Plus one whole-model
training step on a radius graph with self loops under normalize=True.

Each case runs the production kernel, its fp32-FMA twin (tests/twin_backend.py) and float64 autograd of the stage's
restatement (tests/shadow_autograd.py) on the same inputs.  Per-node and per-edge outputs are compared ROW-WISE
(max |got − ref| over a row over max |ref| of that row), so a hub row cannot hide a degree-one row and a large gradient
cannot hide a small one; rows that are structurally zero (isolated nodes, nodes never used as col, graphs without nodes)
must be exactly zero.  Parameter gradients are compared per field."""
import functools

import pytest
import torch

from distegnn_b200 import FastEGNN, _lib
from oracle import fastegnn_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 2e-5              # row-wise relative error against float64 autograd (the per-stage bound of the backward kernels)
# g_x rows have three entries, each a signed sum over the node's edges (or channels), and whole rows cancel.  Measured on
# an H100 80GB HBM3 (700 W): up to 4.6e-5 for the edge kernel (hub, FLAG_NORMALIZE) and 7.7e-5 for the virtual kernel
# (2^k upstream, FLAG_LAST); the fp32-FMA twins reach 4.6e-5 on the same inputs.
TOL_X = 1e-4
# Where a case needs more than TOL, the tensor-core kernel must still be within this factor of the twin's error (its
# operands are split into two fp16 terms with one power-of-two scale per row; the worst ratio measured is 9, on the
# rescued rows of test_edge_bwd_rescued_and_guarded_rows).
TWIN_FACTOR = 16
FLOOR = 1e-30           # denominator floor of the row-wise error (the smallest rows here are about 1e-20)
C_EDGE, NA = 3, 0       # virtual channels / node attributes of the layer whose edge stage is tested
EDGE_FIELDS = ("E_W1R", "E_W1E", "E_W2", "E_B2", "E_WC", "E_BC", "E_W3")
VIRT_FIELDS = ("V_W1R", "V_W2", "V_B2", "V_WXV", "V_BXV", "V_W3XV", "V_WX", "V_BX", "V_W3X")
FLAG_SETS = [0, _lib.FLAG_NORMALIZE, _lib.FLAG_LAST, _lib.FLAG_NORMALIZE | _lib.FLAG_LAST]


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def backend():
    from tests.twin_backend import twin_backend
    return twin_backend()


@functools.lru_cache(maxsize=None)
def layer_params(A, C, seed=2):
    sd = orc.init_state_dict(2, NA, A, 64, C, 1, seed=seed, coord_gain=1.0)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=2, node_attr_nf=NA, edge_attr_nf=A, virtual_channels=C,
                 n_layers=1)
    m.load_state_dict(sd)
    return m.to(dev()).eval()._packed_params(dev())["layers"][0]


def field_sizes(A):
    return {"E_W1R": 64, "E_W1E": A * 64, "E_W2": 4096, "E_B2": 64, "E_WC": 4096, "E_BC": 64, "E_W3": 64,
            "V_W1R": 64, "V_W2": 4096, "V_B2": 64, "V_WXV": 4096, "V_BXV": 64, "V_W3XV": 64, "V_WX": 4096,
            "V_BX": 64, "V_W3X": 64}


def rowwise(got, ref, zero_rows=None):
    """Largest row-wise relative error; rows flagged in `zero_rows` must be exactly zero in both."""
    got = got.detach().double().reshape(got.shape[0], -1)
    ref = ref.detach().double().reshape(ref.shape[0], -1)
    assert torch.isfinite(got).all(), "non-finite output"
    if zero_rows is not None and bool(zero_rows.any()):
        assert float(ref[zero_rows].abs().max()) == 0.0
        assert float(got[zero_rows].abs().max()) == 0.0, "structurally zero row is not exactly zero"
        got, ref = got[~zero_rows], ref[~zero_rows]
    if got.shape[0] == 0:
        return 0.0
    return float(((got - ref).abs().amax(1) / ref.abs().amax(1).clamp(min=FLOOR)).max())


def edge_attr_rowwise(got, ref, terms, row, N):
    """g_edge_attr[e,k] = Σ_n g_z1[e,n]·W_e[k,n] can cancel to any magnitude, and g_z1 of one edge carries the fp32
    rounding of its gφ = g_aggx[row]·Δ (a three-term dot product).  So each edge's error is taken relative to the largest
    sum of |terms| over the edges of its destination node: a node's edges are still judged on that node's own scale."""
    assert torch.isfinite(got).all(), "non-finite output"
    err = (got.double() - ref.double()).abs().amax(1)
    scale = torch.zeros(N, dtype=torch.float64, device=got.device).scatter_reduce(0, row, terms.amax(1), "amax")
    return float((err / scale[row].clamp(min=FLOOR)).max())


def check_bounds(errs, tols):
    """errs: {kernel: {field: error}}.  Every field within its bound; a field above TOL in the tensor-core kernel within
    TWIN_FACTOR of the twin's error."""
    for kind, e in errs.items():
        bad = {f: v for f, v in e.items() if v > tols.get(f, TOL)}
        assert not bad, (kind, bad)
    for f, v in errs["tc"].items():
        if v > TOL and f in errs["twin"]:
            assert v <= TWIN_FACTOR * max(errs["twin"][f], TOL), (f, v, errs["twin"][f])


def rel(got, ref):
    assert torch.isfinite(got).all(), "non-finite output"
    return float((got.double() - ref.double()).abs().max()) / max(FLOOR, float(ref.abs().max()))


def within_rerun_bound(a, b):
    """Two launches that differ only in the order of their float atomics (DESIGN §5)."""
    return float((a - b).abs().max()) <= 2e-6 * max(1.0, float(a.abs().max()))


def param_errors(glp, rlp, names, A, offs):
    sizes = field_sizes(A)
    return {k: rel(glp[offs[k]:offs[k] + sizes[k]], rlp[offs[k]:offs[k] + sizes[k]]) for k in names if sizes[k]}


def fmt(errs):
    return ", ".join(f"{k} {v:.1e}" for k, v in errs.items())


# ==== edge stage =======================================================================================================
def random_graph(N, E, seed, self_loops=False):
    g = torch.Generator().manual_seed(seed)
    row = torch.sort(torch.randint(0, N, (E,), generator=g))[0]
    col = torch.randint(0, N, (E,), generator=g)
    if not self_loops:
        col = torch.where(col == row, (col + 1) % N, col)
    return row, col


def edge_inputs(row, col, N, A, seed, E_cap=None):
    """row / col as CPU int64, row non-decreasing.  With E_cap the id arrays are padded with out-of-range ids and the
    edge attributes with NaN up to the capacity: the kernel must read neither."""
    g = torch.Generator().manual_seed(seed)
    E = row.numel()
    x4 = torch.zeros(N, 4)
    x4[:, :3] = torch.randn(N, 3, generator=g)
    gx = torch.zeros(N, 4)
    gx[:, :3] = torch.randn(N, 3, generator=g)
    ea = torch.randn(E, A, generator=g) * 0.5 if A else None
    if E_cap is not None:
        pad = torch.full((E_cap - E,), 2**30, dtype=torch.int64)
        row, col = torch.cat([row, pad]), torch.cat([col, pad])
        if A:
            ea = torch.cat([ea, torch.full((E_cap - E, A), float("nan"))])
    d = dev()
    t = lambda v: None if v is None else v.to(d)
    return dict(row=t(row.to(torch.int32)), col=t(col.to(torch.int32)), ea=t(ea), x4=t(x4),
                P=t(torch.randn(N, 64, generator=g)), Q=t(torch.randn(N, 64, generator=g)),
                g_m=t(torch.randn(N, 64, generator=g)), g_x=t(gx), n_valid=E)


def edge_reference(N, A, flags, inp, lp):
    """float64 autograd of the stage on the first n_valid edges -> (g_P, g_Q, g_x, g_lp, g_ea, |terms| of g_ea)."""
    from tests import shadow_autograd as sa
    n = inp["n_valid"]
    last = bool(flags & _lib.FLAG_LAST)
    leaves = [t.double().requires_grad_(True) for t in (inp["P"], inp["Q"], inp["x4"][:, :3], lp)]
    z1_shift = torch.zeros(n, 64, dtype=torch.float64, device=dev(), requires_grad=True)
    ead = inp["ea"][:n].double().requires_grad_(True) if A else None
    am, ax = sa.edge_stage((N, n, A, C_EDGE, NA), flags, inp["row"][:n], inp["col"][:n], ead, leaves[2], leaves[0],
                           leaves[1], leaves[3], z1_shift=z1_shift)
    loss = (ax * inp["g_x"][:, :3].double()).sum() + (0 if last else (am * inp["g_m"].double()).sum())
    grads = torch.autograd.grad(loss, leaves + [z1_shift] + ([ead] if A else []))
    terms = None
    if A:                                   # g_ea[e,k] = Σ_n g_z1[e,n]·W_e[k,n]: the sums of the terms' magnitudes
        offs, _ = _lib.param_layout(A, C_EDGE, NA)
        w1e = lp[offs["E_W1E"]:offs["E_W1E"] + A * 64].view(A, 64).double()
        terms = grads[4].abs() @ w1e.abs().t()
    return tuple(grads[:4]) + ((grads[5] if A else None), terms)


def edge_run(kind, N, A, flags, inp, lp):
    """kind: 'tc' (weights-only instantiation), 'tc_inputs' (with g_edge_attr) or 'twin' (fp32 FMA, first n_valid edges).
    -> (g_P, g_Q, g_x [N,3], g_lp, g_ea or None)"""
    be = backend()
    E, n = inp["row"].numel(), inp["n_valid"]
    last = bool(flags & _lib.FLAG_LAST)
    gP, gQ, gx4, glp = (torch.zeros_like(t) for t in (inp["P"], inp["Q"], inp["x4"], lp))
    g_ea = None
    if kind == "twin":
        ea = inp["ea"][:n] if A else None
        be.edge_layer_bwd_simt((N, n, A, C_EDGE, NA), flags, inp["row"][:n], inp["col"][:n], ea, inp["x4"], inp["P"],
                               inp["Q"], lp, None if last else inp["g_m"], inp["g_x"], gP, gQ, gx4, glp)
    else:
        if kind == "tc_inputs":
            g_ea = torch.full((E, A), float("nan"), device=dev())        # sentinel beyond the device-side count
            g_ea[:n] = 0
        n_dev = torch.tensor([n], dtype=torch.int32, device=dev()) if n < E else None
        be.edge_layer_bwd((N, E, A, C_EDGE, NA), flags, inp["row"], inp["col"], inp["ea"], inp["x4"], inp["P"],
                          inp["Q"], lp, None if last else inp["g_m"], inp["g_x"], gP, gQ, gx4, glp, n_dev, g_ea)
    torch.cuda.synchronize()
    if g_ea is not None:
        assert bool(torch.isnan(g_ea[n:]).all()), "g_edge_attr written beyond the device-side edge count"
        g_ea = g_ea[:n]
    return gP, gQ, gx4[:, :3], glp, g_ea


def edge_errors(got, ref, masks, row, A, offs):
    N = got[0].shape[0]
    errs = dict(P=rowwise(got[0], ref[0], masks[0]), Q=rowwise(got[1], ref[1], masks[1]),
                x=rowwise(got[2], ref[2], masks[2]))
    if got[4] is not None:
        errs["ea"] = edge_attr_rowwise(got[4], ref[4], ref[5], row, N)
    errs.update(param_errors(got[3], ref[3], EDGE_FIELDS, A, offs))
    return errs


def check_edge(N, A, flags, inp, what, tol=None, inputs_kernel=True, same_as_weights_only=False):
    """Weights-only kernel, the g_edge_attr instantiation (A > 0) and the twin against float64 autograd, row-wise.
    tol: per-field bounds that replace TOL / TOL_X where a case needs more.  same_as_weights_only: the g_edge_attr
    instantiation's other outputs must equal the weights-only kernel's up to atomic order."""
    lp = layer_params(A, C_EDGE)
    offs, _ = _lib.param_layout(A, C_EDGE, NA)
    n = inp["n_valid"]
    row, col = inp["row"][:n].long(), inp["col"][:n].long()
    has_row = torch.bincount(row, minlength=N) > 0
    has_col = torch.bincount(col, minlength=N) > 0
    masks = (~has_row, ~has_col, ~(has_row | has_col))
    ref = edge_reference(N, A, flags, inp, lp)
    kinds = ["tc", "twin"] + (["tc_inputs"] if (A and inputs_kernel) else [])
    got = {k: edge_run(k, N, A, flags, inp, lp) for k in kinds}
    errs = {k: edge_errors(got[k], ref, masks, row, A, offs) for k in kinds}
    for k in kinds:
        print(f"edge bwd {what} N={N} E={n} A={A} flags={flags} [{k}]: row-wise vs fp64 {fmt(errs[k])}")
    if same_as_weights_only and "tc_inputs" in got:     # same arithmetic as the weights-only kernel, up to atomic order
        for i, name in enumerate(("g_P", "g_Q", "g_x", "g_lp")):
            assert within_rerun_bound(got["tc_inputs"][i], got["tc"][i]), name
    check_bounds(errs, {"x": TOL_X, **(tol or {})})
    return errs


@pytest.mark.parametrize("flags", FLAG_SETS)
@pytest.mark.parametrize("A", [0, 1, 2, 3, 8])
def test_edge_bwd_attr_counts_and_flags(A, flags):
    """Every edge-attribute count through both instantiations, several 128-edge tiles per CTA."""
    N = 5_000
    row, col = random_graph(N, 100_003, seed=100 + A + 10 * flags)
    check_edge(N, A, flags, edge_inputs(row, col, N, A, seed=A + flags), "attr counts", same_as_weights_only=True)


@pytest.mark.parametrize("E", [1, 17, 127, 128, 129, 255, 1_000, 4_097])
def test_edge_bwd_small_and_ragged_edge_counts(E):
    """Fewer edges than one tile, ragged last tiles, fewer tiles than SMs."""
    N = 300
    row, col = random_graph(N, E, seed=E)
    check_edge(N, 2, 0, edge_inputs(row, col, N, 2, seed=E), "ragged")
    # Under FLAG_LAST every g_z1 row is gφ_e times nearly the same vector, so edges of opposite gφ cancel whole g_P / g_Q
    # rows: 2.1e-5 measured for both the tensor-core kernel and the twin (E = 1,000)
    check_edge(N, 2, _lib.FLAG_NORMALIZE | _lib.FLAG_LAST, edge_inputs(row, col, N, 2, seed=E + 1), "ragged",
               tol={"P": 5e-5, "Q": 5e-5})


@pytest.mark.parametrize("flags", [0, _lib.FLAG_NORMALIZE])
def test_edge_bwd_hub_next_to_degree_one_rows(flags):
    """One destination with 5,000 edges (its run crosses warps and tiles, one RED.v2 per run piece) among destinations of
    degree one; nodes 9,001.. are isolated (exact zero g_P, g_Q, g_x) and many nodes are never a source (exact zero g_Q)."""
    N = 20_000
    g = torch.Generator().manual_seed(5)
    row = torch.cat([torch.arange(0, 3_000), torch.full((5_000,), 3_000), torch.arange(3_001, 9_001)])
    col = torch.randint(0, 9_001, (row.numel(),), generator=g)
    col = torch.where(col == row, (col + 1) % 9_001, col)
    check_edge(N, 2, flags, edge_inputs(row, col, N, 2, seed=5), "hub")


@pytest.mark.parametrize("flags", [_lib.FLAG_NORMALIZE, 0])
def test_edge_bwd_self_loops(flags):
    """Every 7th edge is a self loop.  d f(x_i − x_i) / d x_i = 0: the kernel must not add +gΔ and −gΔ to the same
    node, which under FLAG_NORMALIZE (Δ = 0, 1/(‖Δ‖ + 1e-8) = 1e8) rounds the node's gradient to the ulp of 1e8·|g·φ|."""
    N = 5_000
    row, col = random_graph(N, 100_003, seed=7)
    col[::7] = row[::7]
    inp = edge_inputs(row, col, N, 2, seed=7)
    errs = check_edge(N, 2, flags, inp, "self loops")
    print(f"self loops flags={flags}: g_x row-wise tensor-core {errs['tc']['x']:.2e} twin {errs['twin']['x']:.2e}")


def test_edge_bwd_capacity_mode():
    """E is a capacity and the device-side count is far below it: padding ids are 2^30 and padding edge attributes NaN,
    so any read of them shows; g_edge_attr beyond the count keeps its NaN sentinel."""
    N, n, cap = 4_000, 30_011, 200_000
    row, col = random_graph(N, n, seed=8)
    check_edge(N, 2, 0, edge_inputs(row, col, N, 2, seed=8, E_cap=cap), "capacity")
    check_edge(N, 1, _lib.FLAG_LAST | _lib.FLAG_NORMALIZE, edge_inputs(row, col, N, 1, seed=9, E_cap=cap), "capacity")


def test_edge_bwd_many_tiles_per_cta():
    """About 60 tiles per CTA: the weight gradients accumulate in registers over all of them before the atomic flush."""
    N = 50_000
    row, col = random_graph(N, 1_000_003, seed=9)
    torch.cuda.reset_peak_memory_stats()
    check_edge(N, 2, _lib.FLAG_NORMALIZE, edge_inputs(row, col, N, 2, seed=9), "many tiles", inputs_kernel=False)
    print(f"many tiles: peak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


def test_edge_bwd_rescued_and_guarded_rows():
    """Every third row of P scaled by 10^3 … 10^7 and every fifth shifted to pre-activations of −20 … −45 in some
    columns: rescued, guarded and ordinary rows share one warp; every row is encoded with its own power-of-two scale."""
    N = 3_000
    row, col = random_graph(N, 60_000, seed=12)
    inp = edge_inputs(row, col, N, 2, seed=12)
    g = torch.Generator().manual_seed(13)
    ids = torch.arange(N)
    scale = torch.where(ids % 3 == 0, 10 ** (3 + 4 * torch.rand(N, generator=g)), torch.ones(N))
    cols = torch.rand(N, 64, generator=g) < 0.3
    shift = torch.where(ids % 5 == 0, -(20 + 25 * torch.rand(N, generator=g)), torch.zeros(N))
    inp["P"] = (inp["P"].cpu() * scale[:, None] + shift[:, None] * cols).to(dev())
    # z2 = a1·W2 recomputed from rows of 10^7 carries absolute errors of order one where it lands near zero, and
    # SiLU'(z2) there is not small: measured row-wise g_P 2.3e-4, g_Q 1.0e-4 (twin 2.6e-5, 4.1e-5), g_edge_attr 8.1e-5
    check_edge(N, 2, 0, inp, "rescue/guard", tol={"P": 5e-4, "Q": 5e-4, "ea": 5e-4})


@pytest.mark.parametrize("flags", [0, _lib.FLAG_NORMALIZE])
def test_edge_bwd_upstream_gradient_range(flags):
    """g_aggm and g_aggx scaled per node by 2^k, k in [−60, 60]: each row's power-of-two scale keeps it exact whatever its
    magnitude (the products stay in the fp32 normal range)."""
    N = 5_000
    row, col = random_graph(N, 100_003, seed=15)
    inp = edge_inputs(row, col, N, 2, seed=15)
    k = torch.randint(-60, 61, (N,), generator=torch.Generator().manual_seed(16)).double()
    s = torch.pow(2.0, k).float().to(dev())[:, None]
    inp["g_m"], inp["g_x"] = inp["g_m"] * s, inp["g_x"] * s
    check_edge(N, 2, flags, inp, "2^k upstream")


def test_edge_bwd_rerun_within_the_nondeterminism_bound():
    """Two launches on the same inputs differ only by the arrival order of the float atomics."""
    N = 50_000
    row, col = random_graph(N, 1_000_003, seed=14)
    inp = edge_inputs(row, col, N, 2, seed=14)
    lp = layer_params(2, C_EDGE)
    a = edge_run("tc", N, 2, _lib.FLAG_NORMALIZE, inp, lp)
    b = edge_run("tc", N, 2, _lib.FLAG_NORMALIZE, inp, lp)
    for x, y, name in zip(a[:4], b[:4], ("g_P", "g_Q", "g_x", "g_lp")):
        assert within_rerun_bound(x, y), name


# ==== real↔virtual stage ===============================================================================================
def virt_inputs(batch, B, C, last, seed, on_virtual=False):
    """batch: CPU int64, sorted.  on_virtual: every 5th node sits exactly on one of its graph's virtual nodes."""
    g = torch.Generator().manual_seed(seed)
    N = batch.numel()
    rnd = lambda *s: torch.randn(*s, generator=g)
    x4 = torch.zeros(N, 4)
    x4[:, :3] = rnd(N, 3)
    Xv = rnd(B, 3, C)
    if on_virtual:
        ids = torch.arange(0, N, 5)
        x4[ids, :3] = Xv[batch[ids], :, ids % C]
    K = 4 + 3 * C + 64 * C
    g_tv = torch.zeros(N, 4)
    g_tv[:, :3] = rnd(N, 3)
    g_vsum = rnd(B, K)
    if last:
        g_vsum[:, 4 + 3 * C:] = 0
    d = dev()
    return dict(batch=batch.to(torch.int32).to(d), x4=x4.to(d), Hn=rnd(N, 64).to(d), Xv=Xv.to(d), G=rnd(B, C, 64).to(d),
                g_aggv=rnd(N, 64).to(d), g_tv=g_tv.to(d), g_vsum=g_vsum.to(d), B=B, C=C)


def virt_reference(flags, inp, lp):
    from tests import shadow_autograd as sa
    N, B, C = inp["batch"].numel(), inp["B"], inp["C"]
    last = bool(flags & _lib.FLAG_LAST)
    xd, Hd, Xd, Gd, lpd = (t.double().requires_grad_(True) for t in (inp["x4"][:, :3], inp["Hn"], inp["Xv"], inp["G"], lp))
    av, tv, tail = sa.virtual_stage((N, B, 2, C, NA), flags, inp["batch"], xd, Hd, Xd, Gd, lpd)
    loss = (tv * inp["g_tv"][:, :3].double()).sum() + (tail * inp["g_vsum"][:, 4:].double()).sum()
    if not last:
        loss = loss + (av * inp["g_aggv"].double()).sum()
    rx, rH, rX, rG, rlp = torch.autograd.grad(loss, (xd, Hd, Xd, Gd, lpd))
    return rH, rx, rG, rX, rlp


def virt_run(kind, flags, inp, lp):
    """kind: 'tc' or 'twin' -> (g_Hn, g_xv [N,3], g_G, g_Xv, g_lp)"""
    be = backend()
    N, B, C = inp["batch"].numel(), inp["B"], inp["C"]
    last = bool(flags & _lib.FLAG_LAST)
    if kind == "tc":
        fn, w = be.virtual_layer_bwd, be.virtual_bwd_prepare(2, C, NA, lp)
    else:
        offs, _ = _lib.param_layout(2, C, NA)
        fn = be.virtual_layer_bwd_simt
        w = torch.stack([lp[offs[k]:offs[k] + 4096].view(64, 64).t().contiguous() for k in ("V_W2", "V_WXV", "V_WX")])
    gHn = torch.full((N, 64), float("nan"), device=dev())          # written, not accumulated
    gxv = torch.full((N, 4), float("nan"), device=dev())
    gG, gXv, glp = torch.zeros_like(inp["G"]), torch.zeros_like(inp["Xv"]), torch.zeros_like(lp)
    fn((N, B, 2, C, NA), flags, inp["batch"], inp["x4"], inp["Hn"], inp["Xv"], inp["G"], lp, w,
       None if last else inp["g_aggv"], inp["g_tv"], inp["g_vsum"], gHn, gxv, gG, gXv, glp)
    torch.cuda.synchronize()
    return gHn, gxv[:, :3], gG, gXv, glp


def check_virtual(batch, B, C, last, what, seed=0, on_virtual=False, inp=None):
    flags = _lib.FLAG_LAST if last else 0
    lp = layer_params(2, C)
    offs, _ = _lib.param_layout(2, C, NA)
    inp = inp or virt_inputs(batch, B, C, last, seed, on_virtual)
    empty = torch.bincount(batch, minlength=B) == 0
    ref = virt_reference(flags, inp, lp)
    errs = {}
    for kind in ("tc", "twin"):
        got = virt_run(kind, flags, inp, lp)
        e = dict(Hn=rowwise(got[0], ref[0]), x=rowwise(got[1], ref[1]),
                 G=rowwise(got[2].reshape(B * C, 64), ref[2].reshape(B * C, 64), empty.repeat_interleave(C).to(dev())),
                 Xv=rowwise(got[3], ref[3], empty.to(dev())))
        e.update(param_errors(got[4], ref[4], VIRT_FIELDS, 2, offs))
        print(f"virtual bwd {what} N={batch.numel()} B={B} C={C} last={last} [{kind}]: row-wise vs fp64 {fmt(e)}")
        errs[kind] = e
    check_bounds(errs, {"x": TOL_X})
    return errs


@pytest.mark.parametrize("last", [False, True])
@pytest.mark.parametrize("C", [1, 2, 3, 5, 7, 8, 9, 15, 16])
def test_virtual_bwd_channel_counts(C, last):
    """Divisors of 128 and channel counts that leave dead rows in every tile (C = 3: 42 nodes, 126 live rows)."""
    N, B = 5_003, 7
    g = torch.Generator().manual_seed(C)
    batch = torch.sort(torch.randint(0, B, (N,), generator=g)).values
    check_virtual(batch, B, C, last, "channels", seed=C)


@pytest.mark.parametrize("C", [3, 16])
def test_virtual_bwd_many_tiny_graphs_and_empty_graph_ids(C):
    """About 3,000 graphs of 1–4 nodes (almost every tile straddles graph boundaries: the atomic path); every 10th graph
    id has no nodes and must get exact zero g_G and g_Xv rows."""
    g = torch.Generator().manual_seed(20 + C)
    B = 3_000
    sizes = torch.randint(1, 5, (B,), generator=g)
    sizes[::10] = 0
    batch = torch.repeat_interleave(torch.arange(B), sizes)
    check_virtual(batch, B, C, False, "tiny graphs", seed=21)


@pytest.mark.parametrize("layout", ["three_large", "large_then_singletons"])
def test_virtual_bwd_graphs_spanning_many_tiles_of_one_cta(layout):
    """C = 16 (8 nodes per tile): graphs of tens of thousands of nodes span dozens of strided tiles of each CTA, driving
    the accumulate-and-flush path; then a large graph followed by 2,000 one-node graphs."""
    if layout == "three_large":
        sizes = torch.tensor([30_000, 29_993, 30_011])
    else:
        sizes = torch.cat([torch.tensor([60_000]), torch.ones(2_000, dtype=torch.int64)])
    B = sizes.numel()
    batch = torch.repeat_interleave(torch.arange(B), sizes)
    check_virtual(batch, B, 16, False, layout, seed=22)


RAGGED_N = {"1": lambda tn, sm: 1, "TN-1": lambda tn, sm: tn - 1, "TN": lambda tn, sm: tn,
            "TN+1": lambda tn, sm: tn + 1, "TN*SM+1": lambda tn, sm: tn * sm + 1,
            "TN*SM+TN-1": lambda tn, sm: tn * sm + tn - 1}


@pytest.mark.parametrize("n_spec", list(RAGGED_N))
@pytest.mark.parametrize("C", [3, 16])
def test_virtual_bwd_ragged_node_counts(C, n_spec):
    """Node counts around one tile (TN = 128 / C nodes) and just above one tile per SM."""
    N = RAGGED_N[n_spec](128 // C, torch.cuda.get_device_properties(dev()).multi_processor_count)
    B = 1 if N < 4 else 3
    g = torch.Generator().manual_seed(N)
    batch = torch.sort(torch.randint(0, B, (N,), generator=g)).values
    check_virtual(batch, B, C, False, f"ragged {n_spec}", seed=N)


def test_virtual_bwd_node_on_a_virtual_node():
    """‖ΔX‖ = 0 for every 5th node in one channel: the radial gradient there is zero (autograd through the norm gives 0,
    the kernel takes g_r/‖ΔX‖ as 0)."""
    N, B, C = 4_001, 4, 5
    batch = torch.sort(torch.randint(0, B, (N,), generator=torch.Generator().manual_seed(30))).values
    check_virtual(batch, B, C, False, "on virtual node", seed=31, on_virtual=True)


@pytest.mark.parametrize("last", [False, True])
def test_virtual_bwd_upstream_gradient_range(last):
    """g_trans_v and g_aggv scaled per node, g_vsum per graph, by independent 2^k, k in [−60, 60]."""
    N, B, C = 5_003, 40, 5
    g = torch.Generator().manual_seed(40)
    batch = torch.sort(torch.randint(0, B, (N,), generator=g)).values
    inp = virt_inputs(batch, B, C, last, seed=41)
    p2 = lambda n: torch.pow(2.0, torch.randint(-60, 61, (n,), generator=g).double()).float().to(dev())[:, None]
    inp["g_tv"], inp["g_aggv"], inp["g_vsum"] = inp["g_tv"] * p2(N), inp["g_aggv"] * p2(N), inp["g_vsum"] * p2(B)
    check_virtual(batch, B, C, last, "2^k upstream", inp=inp)


# ==== the whole model ==================================================================================================
def test_model_gradients_on_a_radius_graph_with_self_loops():
    """One training step of FastEGNN on a radius graph built with loop=True, normalize=True: parameter gradients and the
    node_loc gradient against float64 autograd through the oracle (the self loops' geometry gradient is exactly zero)."""
    from distegnn_b200 import radius_graph, synth
    w = synth.WORKLOADS["water3d_10k"]
    host = synth.make_partitions(w, n_nodes=2_000, seed=33)[0]
    n = host["node_loc"].shape[0]
    ei, ea = radius_graph(host["node_loc"].to(dev()), w.radius, loop=True)
    assert int((ei[0] == ei[1]).sum()) == n
    host = {**host, "edge_index": ei.cpu(), "edge_attr": ea.cpu()}
    F, Na, A, C = w.node_feat_nf, w.node_attr_nf, 2, w.virtual_channels
    sd = orc.init_state_dict(F, Na, A, 64, C, 3, seed=34, coord_gain=0.05)
    g = torch.Generator().manual_seed(35)
    cot_out, cot_X = torch.randn(n, 3, generator=g), torch.randn(1, 3, C, generator=g)
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    inp64 = {k: (v.double() if (v is not None and v.is_floating_point()) else v) for k, v in host.items()}
    inp64["node_loc"].requires_grad_(True)
    o64, X64 = orc.forward(sd64, **inp64, normalize=True)
    keys = list(sd64)
    grads = torch.autograd.grad((o64 * cot_out.double()).sum() + (X64 * cot_X.double()).sum(),
                                [inp64["node_loc"]] + [sd64[k] for k in keys], allow_unused=True)
    ref_loc, ref = grads[0], dict(zip(keys, grads[1:]))
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=C,
                 n_layers=3, normalize=True)
    m.load_state_dict(sd)
    m.input_grads = True
    m = m.to(dev()).train()
    d = {k: (v.to(dev()) if v is not None else None) for k, v in host.items()}
    d["node_loc"] = d["node_loc"].clone().requires_grad_(True)
    out, X = m(**d)
    ((out * cot_out.to(dev())).sum() + (X * cot_X.to(dev())).sum()).backward()
    errs = {"node_loc": rel(d["node_loc"].grad.cpu(), ref_loc)}
    for k, p in m.named_parameters():
        r = ref[k]
        if r is None or float(r.abs().max()) == 0.0:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        errs[k] = rel(p.grad.cpu(), r)
    worst = max(errs, key=errs.get)
    print(f"radius graph with self loops n={n} E={ei.shape[1]}: node_loc {errs['node_loc']:.2e}, worst {worst} "
          f"{errs[worst]:.2e}")
    assert errs[worst] <= 5e-4                           # as test_training_path_gradients_batched_nbody
