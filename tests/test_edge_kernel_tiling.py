"""Edge kernel (distegnn_edge_layer_fwd) on the graph shapes its tiling makes fragile: every edge-attribute
instantiation, edge counts that do not fill a 64-edge warpgroup tile, destination runs that cross warps, tiles and
warpgroups, self loops and isolated nodes, a device-side edge count far below the capacity, grids with fewer tiles than
warpgroups, and range-rescued / SiLU-guarded rows sharing a quad and a warp with ordinary ones.

Each case is compared with the fp32-FMA twin (1e-5 relative over the tensor, as the other edge-kernel tests) and with
the float64 restatement (tests/shadow_autograd.py edge_terms) ROW BY ROW: a row of agg_m against its own largest entry,
a row of agg_x (a short signed sum that cancels) against the largest summed magnitude of its terms, Σ_e |Δx|·Σ_k
|w3_k·s_k| (φ = Σ_k w3_k·s_k is a 64-term dot product that cancels too), both within helpers.TOL; rows without edges
must be exactly zero.  Where a field needs more than TOL, the kernel must stay within helpers.TWIN_FACTOR of the twin's
error on the same metric.  `check` and `rescued_and_guarded` take the kernel under test as an argument:
tests/test_forward_det_tiling.py runs the deterministic kernel and its combine through them."""
import pytest
import torch

from distegnn_b200 import FastEGNN, _lib
from oracle import fastegnn_oracle as orc
from tests.helpers import check_bounds, rowwise, terms_rowwise
from tests.shadow_autograd import edge_terms

pytestmark = pytest.mark.gpu

REL_TOL = 1e-5          # the tensor-core kernel against its fp32-FMA twin, over the whole tensor


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def layer_params(A, seed=2):
    sd = orc.init_state_dict(3, 0, A, 64, 3, 1, seed=seed, coord_gain=1.0)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=3, node_attr_nf=0, edge_attr_nf=A, virtual_channels=3,
                 n_layers=1)
    m.load_state_dict(sd)
    return m.to(dev()).eval()._packed_params(dev())["layers"][0]


def make_inputs(row, col, N, A, seed):
    """row / col as CPU int64 with row non-decreasing; returns device tensors of the kernel's inputs."""
    g = torch.Generator().manual_seed(seed)
    E = row.numel()
    d = dev()
    x4 = torch.zeros(N, 4)
    x4[:, :3] = torch.randn(N, 3, generator=g)
    P, Q = torch.randn(N, 64, generator=g), torch.randn(N, 64, generator=g)
    ea = torch.randn(E, A, generator=g) if A else None
    t = lambda v: None if v is None else v.to(d)
    return dict(row=t(row.to(torch.int32)), col=t(col.to(torch.int32)), ea=t(ea), x4=t(x4), P=t(P), Q=t(Q))


def run(be, fn_name, N, E, A, flags, inp, lp, n_edges_dev=None, det_ws=None):
    d = dev()
    agg_m = None if flags & _lib.FLAG_LAST else torch.zeros(N, 64, device=d)
    agg_x = torch.zeros(N, 4, device=d)
    args = ((N, E, A, 3, 0), flags, inp["row"], inp["col"], inp["ea"], inp["x4"], inp["P"], inp["Q"], lp, agg_m, agg_x)
    kw = {k: v for k, v in (("n_edges_dev", n_edges_dev), ("det_ws", det_ws)) if v is not None}
    getattr(be, fn_name)(*args, **kw)
    torch.cuda.synchronize()
    assert not agg_x[:, 3].any(), "agg_x column 3 written"
    return agg_m, agg_x[:, :3]


def production(be, N, E, A, flags, inp, lp, n_edges_dev=None):
    """The kernel under test by default: distegnn_edge_layer_fwd -> (agg_m or None, agg_x[:, :3])."""
    return run(be, "edge_layer", N, E, A, flags, inp, lp, n_edges_dev)


def shadow(N, E, A, flags, inp, lp):
    """float64 restatement -> (agg_m or None, agg_x, the summed magnitudes of the terms of agg_x)."""
    dbl = lambda v: None if v is None else v.double()
    m, x, terms = edge_terms((N, E, A, 3, 0), flags, inp["row"], inp["col"], dbl(inp["ea"]), inp["x4"][:, :3].double(),
                             inp["P"].double(), inp["Q"].double(), lp.double())
    return (None if flags & _lib.FLAG_LAST else m), x, terms


def rel(o, r):
    return float((o.double() - r.double()).abs().max()) / max(1e-9, float(r.abs().max()))


def errors(got, ref, isolated):
    """agg_m row-wise, agg_x against its terms; rows without edges (`isolated`) exactly zero."""
    e = {}
    if got[0] is not None:
        e["agg_m"] = rowwise(got[0], ref[0], zero_rows=isolated)
    assert not got[1][isolated].any(), "agg_x row without edges is not exactly zero"
    e["agg_x"] = terms_rowwise(got[1][~isolated], ref[1][~isolated], ref[2][~isolated])
    return e


def fmt(errs):
    return ", ".join(f"{k} {v:.1e}" for k, v in errs.items())


def check(N, row, col, A, flags, seed=0, n_valid=None, tols=None, kernel=production, inp=None):
    """The kernel under test vs float64 row by row (and, for the production kernel, vs the twin over the tensor).
    n_valid: the device-side edge count (capacity mode: row / col hold n_valid real edges followed by padding, which the
    kernel must not read).  kernel(be, N, E, A, flags, inp, lp, n_edges_dev) -> (agg_m or None, agg_x)."""
    from tests.twin_backend import twin_backend
    be = twin_backend()
    E = row.numel()
    lp = layer_params(A)
    inp = inp or make_inputs(row, col, N, A, seed)
    if n_valid is None:
        got = kernel(be, N, E, A, flags, inp, lp)
        ref_inp, E_ref = inp, E
    else:
        got = kernel(be, N, E, A, flags, inp, lp, torch.tensor([n_valid], dtype=torch.int32, device=dev()))
        ref_inp = {k: (None if v is None else (v[:n_valid] if k in ("row", "col", "ea") else v)) for k, v in inp.items()}
        E_ref = n_valid
    twin = run(be, "edge_layer_simt", N, E_ref, A, flags, ref_inp, lp)
    ref = shadow(N, E_ref, A, flags, ref_inp, lp)
    isolated = torch.bincount(ref_inp["row"].long(), minlength=N) == 0
    if kernel is production:
        for k, name in ((1, "agg_x"), (0, "agg_m")):
            if got[k] is not None:
                assert rel(got[k], twin[k]) <= REL_TOL, (name, rel(got[k], twin[k]))
    errs = {"tc": errors(got, ref, isolated), "twin": errors(twin, ref, isolated)}
    print(f"{kernel.__name__} N={N} E={E} A={A} flags={flags}: row-wise vs fp64 {fmt(errs['tc'])} "
          f"(twin {fmt(errs['twin'])})")
    check_bounds(errs, tols or {})
    return got


def random_graph(N, E, seed, self_loops=True):
    g = torch.Generator().manual_seed(seed)
    row = torch.sort(torch.randint(0, N, (E,), generator=g))[0]
    col = torch.randint(0, N, (E,), generator=g)
    if not self_loops:
        col = torch.where(col == row, (col + 1) % N, col)
    return row, col


FLAG_SETS = [0, _lib.FLAG_NORMALIZE, _lib.FLAG_LAST, _lib.FLAG_NORMALIZE | _lib.FLAG_LAST]
ATTR_COUNTS = [0, 1, 2, 3, 8]
RAGGED_E = [1, 17, 63, 64, 65, 130, 1_000, 4_097]


def attr_case(A, flags, kernel=production):
    N = 5_000
    row, col = random_graph(N, 100_003, seed=A + 10 * flags)
    check(N, row, col, A, flags, seed=A, kernel=kernel)


def ragged_case(E, kernel=production):
    N = 300
    row, col = random_graph(N, E, seed=E)
    check(N, row, col, 2, 0, seed=E, kernel=kernel)
    check(N, row, col, 2, _lib.FLAG_LAST | _lib.FLAG_NORMALIZE, seed=E, kernel=kernel)


def hub_case(kernel=production):
    N = 20_000
    g = torch.Generator().manual_seed(5)
    lo = torch.arange(0, 3_000)                                  # degree 1
    hub = torch.full((5_000,), 3_000)                            # degree 5,000
    hi = torch.arange(3_001, 9_001)                              # degree 1; nodes 9,001.. are isolated
    row = torch.cat([lo, hub, hi])
    col = torch.randint(0, N, (row.numel(),), generator=g)
    col[::7] = row[::7]                                          # self loops
    for flags in (0, _lib.FLAG_NORMALIZE):
        agg_m, agg_x = check(N, row, col, 2, flags, seed=5, kernel=kernel)
        assert float(agg_m[9_001:].abs().max()) == 0.0 and float(agg_x[9_001:].abs().max()) == 0.0


def capacity_case(kernel=production):
    N = 4_000
    row, col = random_graph(N, 30_011, seed=8)
    cap = 200_000
    pad = torch.full((cap - row.numel(),), 2**30, dtype=torch.int64)
    check(N, torch.cat([row, pad]), torch.cat([col, pad]), 2, 0, seed=8, n_valid=row.numel(), kernel=kernel)
    check(N, torch.cat([row, pad]), torch.cat([col, pad]), 1, _lib.FLAG_LAST, seed=8, n_valid=row.numel(),
          kernel=kernel)


def many_tiles_case(kernel=production):
    N = 200_000
    row, col = random_graph(N, 4_000_037, seed=9)
    check(N, row, col, 2, 0, seed=9, kernel=kernel)


@pytest.mark.parametrize("A", ATTR_COUNTS)
@pytest.mark.parametrize("flags", FLAG_SETS)
def test_edge_attr_instantiations(A, flags):
    """A = 0, 1, 2, the generic count (3) and the widest (8), with and without FLAG_LAST / FLAG_NORMALIZE, on a graph
    that spans several tiles per warpgroup."""
    attr_case(A, flags)


@pytest.mark.parametrize("E", RAGGED_E)
def test_small_and_ragged_edge_counts(E):
    """Fewer edges than one tile, ragged tails, and fewer tiles than warpgroups in the grid."""
    ragged_case(E)


def test_hub_destination_next_to_degree_one_rows():
    """One destination with 5,000 edges (its run crosses warps, tiles and warpgroups) between many destinations of
    degree one; plus self loops and isolated nodes."""
    hub_case()


def test_capacity_mode_device_count_below_bound():
    """E is a capacity; the device count is far below it.  Padding entries hold out-of-range ids, so any read of them
    would fault or corrupt the sums."""
    capacity_case()


def test_many_tiles_per_warpgroup():
    many_tiles_case()


def rescued_and_guarded(kernel=production):
    """Every third destination row is scaled far beyond the fp16 range and every fifth is shifted to pre-activations
    of −20 … −45 (the SiLU batch guard), in some columns only: rescued, guarded and ordinary rows sit in one quad and
    one warp.  Row-wise error against fp64, as in the range-rescue test."""
    from tests.twin_backend import twin_backend
    be = twin_backend()
    N = 3_000
    row, col = random_graph(N, 60_000, seed=12)
    lp = layer_params(2)
    inp = make_inputs(row, col, N, 2, seed=12)
    g = torch.Generator().manual_seed(13)
    ids = torch.arange(N)
    scale = torch.where(ids % 3 == 0, 10 ** (3 + 4 * torch.rand(N, generator=g)), torch.ones(N))
    cols = torch.rand(N, 64, generator=g) < 0.3
    shift = torch.where(ids % 5 == 0, -(18 + 30 * torch.rand(N, generator=g)), torch.zeros(N))
    inp["P"] = (inp["P"].cpu() * scale[:, None] + shift[:, None] * cols).to(dev())
    E = row.numel()
    got = kernel(be, N, E, 2, 0, inp, lp)
    twin = run(be, "edge_layer_simt", N, E, 2, 0, inp, lp)
    ref = shadow(N, E, 2, 0, inp, lp)
    assert float(ref[0].abs().max()) > 1e5
    e_m, e_x = rowwise(got[0], ref[0]), rowwise(got[1], ref[1])
    e_twin_x = rowwise(twin[1], ref[1])
    print(f"{kernel.__name__} mixed rescue/guard rows: row-wise rel err agg_m {e_m:.2e} agg_x {e_x:.2e} "
          f"(twin agg_x {e_twin_x:.2e})")
    assert e_m <= 2e-5
    # Δx·φ cancels heavily on rows that are both scaled and shifted (about 6e-4 row-wise for the 22-bit operand split
    # here, against 4e-5 for fp32 FMA): the bound is the range-rescue test's absolute cap
    assert e_x <= 1e-3


def test_rescued_and_guarded_rows_share_quads_and_warps():
    rescued_and_guarded()


def test_rerun_within_the_nondeterminism_bound():
    """Two launches on the same inputs differ only by the arrival order of the RED.ADD partial sums (DESIGN §5)."""
    from tests.twin_backend import twin_backend
    be = twin_backend()
    N = 50_000
    row, col = random_graph(N, 1_000_003, seed=14)
    lp = layer_params(2)
    inp = make_inputs(row, col, N, 2, seed=14)
    a = run(be, "edge_layer", N, row.numel(), 2, 0, inp, lp)
    b = run(be, "edge_layer", N, row.numel(), 2, 0, inp, lp)
    for x, y in zip(a, b):
        assert float((x - y).abs().max()) <= 2e-6 * max(1.0, float(x.abs().max()))
