"""Real<->virtual kernel (distegnn_virtual_layer_fwd) on the shapes its tiling makes fragile: every channel count 1..16
(full and ragged 64-row tiles, nodes that straddle warps), node counts below one tile and grids with fewer tiles than
warpgroups, graph boundaries inside a warp / on a warp boundary / on a tile boundary, tiles spanning many graphs, empty
graph ids, one graph per node, a warpgroup whose consecutive tiles sit in different graphs, one graph over many tiles,
and range-rescued / SiLU-guarded rows sharing a quad and a warp with ordinary ones.  vsum is pre-filled, so the
accumulate semantics (columns 0..3 and the rows of graphs without nodes left alone) are checked too.  Every case runs
with and without FLAG_LAST.

Each case is compared with the fp32-FMA twin (2e-5 relative over the tensor, as the other virtual-kernel tests) and with
the float64 restatement (tests/shadow_autograd.py virtual_terms) ROW BY ROW and GRAPH BY GRAPH, within helpers.TOL: a
row of agg_v against its own largest entry; a row of trans_v (a short signed sum that cancels) against the largest
summed magnitude of its terms, mean_c |ΔX|·Σ_k |w3xv_k·s_k| (the head φ_xv = Σ_k w3xv_k·s_k cancels too); per graph,
the Σ mv block of vsum (64·C entries) against its own largest entry and the Σ ΔX·φ_X block (3·C entries) against the
largest Σ |ΔX|·Σ_k |w3x_k·s_k| of its entries (plus the pre-filled value it is added to).  Where a field needs more
than TOL, the kernel must stay within helpers.TWIN_FACTOR of the twin's error on the same metric.  `check` and
`rescued_and_guarded` take the kernel under test as an argument: tests/test_forward_det_tiling.py runs the deterministic
kernel and its combine through them (from vsum = 0, as the model does)."""
import pytest
import torch

from distegnn_b200 import FastEGNN, _lib
from oracle import fastegnn_oracle as orc
from tests.helpers import check_bounds, rowwise, terms_rowwise
from tests.shadow_autograd import virtual_terms

pytestmark = pytest.mark.gpu

REL_TOL = 2e-5          # the tensor-core kernel against its fp32-FMA twin, over the whole tensor
FLAGS = [0, _lib.FLAG_LAST]


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def layer_params(C, seed=3):
    sd = orc.init_state_dict(3, 0, 2, 64, C, 1, seed=seed, coord_gain=1.0)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=3, node_attr_nf=0, edge_attr_nf=2, virtual_channels=C,
                 n_layers=1)
    m.load_state_dict(sd)
    return m.to(dev()).eval()._packed_params(dev())["layers"][0]


def make_inputs(batch, B, C, seed):
    """batch: CPU int64, non-decreasing, values < B.  Returns device tensors of the kernel's inputs."""
    g = torch.Generator().manual_seed(seed)
    N = batch.numel()
    x4 = torch.zeros(N, 4)
    x4[:, :3] = torch.randn(N, 3, generator=g)
    inp = dict(batch=batch.to(torch.int32), x4=x4, Hn=torch.randn(N, 64, generator=g),
               Xv=torch.randn(B, 3, C, generator=g), G=torch.randn(B, C, 64, generator=g),
               vsum0=torch.randn(B, 4 + 3 * C + 64 * C, generator=g))
    return {k: v.to(dev()) for k, v in inp.items()}


def run(fn, B, C, flags, inp, lp, vsum0):
    N = inp["batch"].numel()
    d = dev()
    agg_v = torch.zeros(N, 64, device=d)
    trans_v = torch.zeros(N, 4, device=d)
    vsum = vsum0.clone()
    fn((N, B, 2, C, 0), flags, inp["batch"], inp["x4"], inp["Hn"], inp["Xv"], inp["G"], lp,
       None if flags & _lib.FLAG_LAST else agg_v, trans_v, vsum)
    torch.cuda.synchronize()
    assert not trans_v[:, 3].any(), "trans_v column 3 written"
    return (None if flags & _lib.FLAG_LAST else agg_v), trans_v[:, :3], vsum


def production(be, B, C, flags, inp, lp, vsum0):
    """The kernel under test by default: distegnn_virtual_layer_fwd -> (agg_v or None, trans_v[:, :3], vsum)."""
    return run(be.virtual_layer, B, C, flags, inp, lp, vsum0)


def shadow(B, C, flags, inp, lp, vsum0):
    """float64 restatement -> virtual_terms' dict, plus vsum = vsum0 + the sums (no Σ mv under FLAG_LAST) and
    vsum_x_terms = |vsum0| + the terms of the Σ ΔX·φ_X entries."""
    N = inp["batch"].numel()
    r = virtual_terms((N, B, 2, C, 0), inp["batch"], inp["x4"][:, :3].double(), inp["Hn"].double(), inp["Xv"].double(),
                      inp["G"].double(), lp.double())
    v0 = vsum0.double()
    r["vsum"] = v0.clone()
    r["vsum"][:, 4:4 + 3 * C] += r["tail_x"]
    if not flags & _lib.FLAG_LAST:
        r["vsum"][:, 4 + 3 * C:] += r["tail_m"]
    r["vsum_x_terms"] = v0[:, 4:4 + 3 * C].abs() + r["tail_x_terms"]
    return r


def rel(o, r):
    return float((o.double() - r.double()).abs().max()) / max(1e-9, float(r.abs().max()))


def errors(got, ref, C, empty):
    """agg_v row-wise, trans_v against its terms; per graph with nodes, Σ mv row-wise and Σ ΔX·φ_X against its
    terms."""
    agg_v, trans_v, vsum = got
    e = {}
    if agg_v is not None:
        e["agg_v"] = rowwise(agg_v, ref["agg_v"])
    e["trans_v"] = terms_rowwise(trans_v, ref["trans_v"], ref["trans_terms"])
    v, r = vsum[~empty], ref["vsum"][~empty]
    e["vsum_x"] = terms_rowwise(v[:, 4:4 + 3 * C], r[:, 4:4 + 3 * C], ref["vsum_x_terms"][~empty])
    if agg_v is not None:
        e["vsum_m"] = rowwise(v[:, 4 + 3 * C:], r[:, 4 + 3 * C:])
    return e


def fmt(errs):
    return ", ".join(f"{k} {v:.1e}" for k, v in errs.items())


def check(batch, B, C, flags, seed=0, tols=None, kernel=production):
    """The kernel under test vs float64 row by row and graph by graph (and, for the production kernel, vs the twin over
    the tensor).  kernel(be, B, C, flags, inp, lp, vsum0) -> (agg_v or None, trans_v[:, :3], vsum); the production
    kernel accumulates into a pre-filled vsum, any other kernel starts from vsum = 0."""
    from tests.twin_backend import twin_backend
    be = twin_backend()
    lp = layer_params(C)
    inp = make_inputs(batch, B, C, seed)
    vsum0 = inp["vsum0"] if kernel is production else torch.zeros_like(inp["vsum0"])
    got = kernel(be, B, C, flags, inp, lp, vsum0)
    twin = run(be.virtual_layer_simt, B, C, flags, inp, lp, vsum0)
    ref = shadow(B, C, flags, inp, lp, vsum0)
    N = batch.numel()
    empty = torch.bincount(batch, minlength=B).to(dev()) == 0
    last = bool(flags & _lib.FLAG_LAST)
    vs = got[2]
    # the rows of graphs without nodes are not the kernel's; under FLAG_LAST neither is the Σ mv block
    assert torch.equal(vs[empty], vsum0[empty])
    if last:
        assert torch.equal(vs[:, 4 + 3 * C:], vsum0[:, 4 + 3 * C:])
    if kernel is production:
        assert torch.equal(vs[:, :4], vsum0[:, :4])             # columns 0..3 are the node kernel's
        for k, name in ((0, "agg_v"), (1, "trans_v"), (2, "vsum")):
            if got[k] is not None:
                assert rel(got[k], twin[k]) <= REL_TOL, (name, rel(got[k], twin[k]))
    errs = {"tc": errors(got, ref, C, empty), "twin": errors(twin, ref, C, empty)}
    print(f"{kernel.__name__} N={N} B={B} C={C} flags={flags}: row-wise / per graph vs fp64 {fmt(errs['tc'])} "
          f"(twin {fmt(errs['twin'])})")
    check_bounds(errs, tols or {})
    return got


def sorted_batch(N, B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.sort(torch.randint(0, B, (N,), generator=g))[0]


def batch_of_sizes(sizes):
    """Graph i gets sizes[i] nodes (0 = a graph id with no nodes)."""
    return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))


SMALL_N = [1, 2, 3, 7, 13, 100, 257, 1_001]
SMALL_N_C = [1, 3, 8, 11, 16]
# C = 8: 2 nodes per warp, 8 per tile; C = 3: 21 nodes per tile, warps split nodes; C = 5: 12 nodes per tile
BOUNDARY_SIZES = {
    "inside_a_warp": [1, 2, 1, 3, 5, 1, 1, 7, 9, 2, 4, 1, 30, 1],
    "on_warp_boundaries": [2, 2, 4, 6, 2, 8, 16, 2, 10, 2, 2, 24],
    "on_tile_boundaries": [8, 16, 8, 24, 21, 42, 12, 36, 64, 8, 40],
    "tiles_over_three_or_more_graphs_and_empty_ids": [1, 0, 1, 1, 0, 0, 2, 1, 1, 1, 3, 0, 1, 1, 1, 1, 5, 1, 0, 2, 1],
}
BOUNDARY_C = [1, 3, 5, 8, 16]


def every_channel_case(C, flags, kernel=production):
    check(sorted_batch(5_003, 3, seed=C), 3, C, flags, seed=C, kernel=kernel)


def small_n_case(N, C, flags, kernel=production):
    check(sorted_batch(N, 2, seed=N), 2, C, flags, seed=N + C, kernel=kernel)


def boundary_case(layout, C, flags, kernel=production):
    sizes = BOUNDARY_SIZES[layout] * 5
    check(batch_of_sizes(sizes), len(sizes), C, flags, seed=len(sizes) + C, kernel=kernel)


def one_graph_per_node_case(C, flags, kernel=production):
    N = 3_001
    check(torch.arange(N), N, C, flags, seed=C, kernel=kernel)


def graph_change_case(C, flags, kernel=production):
    sizes = [997 + 13 * (i % 7) for i in range(200)]
    check(batch_of_sizes(sizes), len(sizes), C, flags, seed=C, kernel=kernel)


def many_tiles_case(C, flags, kernel=production):
    check(torch.zeros(400_003, dtype=torch.int64), 1, C, flags, seed=C, kernel=kernel)


@pytest.mark.parametrize("C", list(range(1, 17)))
@pytest.mark.parametrize("flags", FLAGS)
def test_every_channel_count(C, flags):
    """Full tiles (C divides 64), ragged tiles and nodes that straddle warps (C does not divide 16), a few graphs."""
    every_channel_case(C, flags)


@pytest.mark.parametrize("N", SMALL_N)
@pytest.mark.parametrize("C", SMALL_N_C)
@pytest.mark.parametrize("flags", FLAGS)
def test_small_node_counts(N, C, flags):
    """N = 1, N below one tile's node count, N not a multiple of it, and grids with fewer tiles than warpgroups."""
    small_n_case(N, C, flags)


@pytest.mark.parametrize("layout", list(BOUNDARY_SIZES))
@pytest.mark.parametrize("C", BOUNDARY_C)
@pytest.mark.parametrize("flags", FLAGS)
def test_graph_boundaries(layout, C, flags):
    boundary_case(layout, C, flags)


@pytest.mark.parametrize("C", [2, 7, 8])
@pytest.mark.parametrize("flags", FLAGS)
def test_one_graph_per_node(C, flags):
    """B = N: every tile straddles graphs, every row goes to vsum directly."""
    one_graph_per_node_case(C, flags)


@pytest.mark.parametrize("C", [4, 8, 13])
@pytest.mark.parametrize("flags", FLAGS)
def test_graph_changes_between_a_groups_tiles(C, flags):
    """Graphs of about a thousand nodes: a warpgroup's consecutive tiles (one grid stride apart) sit in different graphs,
    so the G cache is reloaded and the per-graph sums flushed while the kernel runs."""
    graph_change_case(C, flags)


@pytest.mark.parametrize("C", [3, 8, 16])
@pytest.mark.parametrize("flags", FLAGS)
def test_one_graph_over_many_tiles(C, flags):
    many_tiles_case(C, flags)


def rescued_and_guarded(C, flags, kernel=production):
    """Every third node has Hn (or, for one graph, G) scaled far beyond the fp16 range — stage 1 and, through D, stage 2
    are range-rescued — and every fifth is shifted to pre-activations of −20 … −50 in some columns (the SiLU batch
    guard): rescued, guarded and ordinary rows sit in one quad and one warp.  Row-wise error against fp64, vsum per
    graph."""
    from tests.twin_backend import twin_backend
    be = twin_backend()
    N, B = 4_000, 3
    batch = sorted_batch(N, B, seed=21)
    lp = layer_params(C)
    inp = make_inputs(batch, B, C, seed=21)
    g = torch.Generator().manual_seed(22)
    ids = torch.arange(N)
    scale = torch.where(ids % 3 == 0, 10 ** (3 + 4 * torch.rand(N, generator=g)), torch.ones(N))
    cols = torch.rand(N, 64, generator=g) < 0.3
    shift = torch.where(ids % 5 == 0, -(20 + 30 * torch.rand(N, generator=g)), torch.zeros(N))
    inp["Hn"] = (inp["Hn"].cpu() * scale[:, None] + shift[:, None] * cols).to(dev())
    G = inp["G"].cpu()
    G[1] *= 3e4
    inp["G"] = G.to(dev())
    vsum0 = inp["vsum0"] if kernel is production else torch.zeros_like(inp["vsum0"])
    got = kernel(be, B, C, flags, inp, lp, vsum0)
    twin = run(be.virtual_layer_simt, B, C, flags, inp, lp, vsum0)
    ref = shadow(B, C, flags, inp, lp, vsum0)

    for x in got:
        assert x is None or torch.isfinite(x).all()
    e_t = rowwise(got[1], ref["trans_v"])
    e_s, e_s_twin = rowwise(got[2][:, 4:], ref["vsum"][:, 4:]), rowwise(twin[2][:, 4:], ref["vsum"][:, 4:])
    print(f"{kernel.__name__} C={C} flags={flags} mixed rescue/guard rows: row-wise rel err trans_v {e_t:.2e} "
          f"(twin {rowwise(twin[1], ref['trans_v']):.2e}), vsum per graph {e_s:.2e} (twin {e_s_twin:.2e})")
    if got[0] is not None:
        e_a = rowwise(got[0], ref["agg_v"])
        print(f"  agg_v row-wise {e_a:.2e} (twin {rowwise(twin[0], ref['agg_v']):.2e})")
        assert e_a <= 2e-5
    # ΔX·φ cancels on rows that are both scaled and shifted: the bound is the edge kernel's range-rescue cap
    assert e_t <= 1e-3 and e_s <= 1e-4


@pytest.mark.parametrize("C", [3, 8])
@pytest.mark.parametrize("flags", FLAGS)
def test_rescued_and_guarded_rows_share_quads_and_warps(C, flags):
    rescued_and_guarded(C, flags)
