"""Real<->virtual kernel (distegnn_virtual_layer_fwd) on the shapes its tiling makes fragile: every channel count 1..16
(full and ragged 64-row tiles, nodes that straddle warps), node counts below one tile and grids with fewer tiles than
warpgroups, graph boundaries inside a warp / on a warp boundary / on a tile boundary, tiles spanning many graphs, empty
graph ids, one graph per node, a warpgroup whose consecutive tiles sit in different graphs, one graph over many tiles,
and range-rescued / SiLU-guarded rows sharing a quad and a warp with ordinary ones.  vsum is pre-filled, so the
accumulate semantics (and columns 0..3 left alone) are checked too.  Every case runs with and without FLAG_LAST and is
compared with the fp32-FMA twin (2e-5 relative, as the other virtual-kernel tests) and with the float64 restatement."""
import pytest
import torch

from distegnn_b200 import FastEGNN, _lib
from oracle import fastegnn_oracle as orc
from tests.shadow_backend import ShadowBackend

pytestmark = pytest.mark.gpu

REL_TOL = 2e-5
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


def run(fn, B, C, flags, inp, lp, dtype=torch.float32):
    N = inp["batch"].numel()
    d = dev()
    cast = (lambda v: v.double()) if dtype == torch.float64 else (lambda v: v)
    agg_v = torch.zeros(N, 64, device=d, dtype=dtype)
    trans_v = torch.zeros(N, 4, device=d, dtype=dtype)
    vsum = inp["vsum0"].to(dtype).clone()
    fn((N, B, 2, C, 0), flags, inp["batch"], cast(inp["x4"]), cast(inp["Hn"]), cast(inp["Xv"]), cast(inp["G"]),
       cast(lp), None if flags & _lib.FLAG_LAST else agg_v, trans_v, vsum)
    torch.cuda.synchronize()
    return (None if flags & _lib.FLAG_LAST else agg_v), trans_v, vsum


def rel(o, r):
    return float((o.double() - r.double()).abs().max()) / max(1e-9, float(r.abs().max()))


def check(batch, B, C, flags, seed=0, tol_shadow=REL_TOL):
    from tests.twin_backend import twin_backend
    be = twin_backend()
    lp = layer_params(C)
    inp = make_inputs(batch, B, C, seed)
    got = run(be.virtual_layer, B, C, flags, inp, lp)
    twin = run(be.virtual_layer_simt, B, C, flags, inp, lp)
    ref = run(ShadowBackend().virtual_layer, B, C, flags, inp, lp, dtype=torch.float64)
    N = batch.numel()
    # columns 0..3 of vsum are not the kernel's, nor is column 3 of trans_v
    assert torch.equal(got[2][:, :4], inp["vsum0"][:, :4])
    assert float(got[1][:, 3].abs().max()) == 0.0
    for k, name in ((0, "agg_v"), (1, "trans_v"), (2, "vsum")):
        if got[k] is None:
            continue
        o, t, r = (x[:, :3] if k == 1 else x for x in (got[k], twin[k], ref[k]))
        assert torch.isfinite(o).all(), name
        e_twin, e_ref = rel(o, t), rel(o, r)
        print(f"N={N} B={B} C={C} flags={flags} {name}: rel err vs twin {e_twin:.2e} vs fp64 {e_ref:.2e}")
        assert e_twin <= REL_TOL and e_ref <= tol_shadow, (name, e_twin, e_ref)
    return got


def sorted_batch(N, B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.sort(torch.randint(0, B, (N,), generator=g))[0]


def batch_of_sizes(sizes):
    """Graph i gets sizes[i] nodes (0 = a graph id with no nodes)."""
    return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))


@pytest.mark.parametrize("C", list(range(1, 17)))
@pytest.mark.parametrize("flags", FLAGS)
def test_every_channel_count(C, flags):
    """Full tiles (C divides 64), ragged tiles and nodes that straddle warps (C does not divide 16), a few graphs."""
    check(sorted_batch(5_003, 3, seed=C), 3, C, flags, seed=C)


@pytest.mark.parametrize("N", [1, 2, 3, 7, 13, 100, 257, 1_001])
@pytest.mark.parametrize("C", [1, 3, 8, 11, 16])
@pytest.mark.parametrize("flags", FLAGS)
def test_small_node_counts(N, C, flags):
    """N = 1, N below one tile's node count, N not a multiple of it, and grids with fewer tiles than warpgroups."""
    check(sorted_batch(N, 2, seed=N), 2, C, flags, seed=N + C)


# C = 8: 2 nodes per warp, 8 per tile; C = 3: 21 nodes per tile, warps split nodes; C = 5: 12 nodes per tile
BOUNDARY_SIZES = {
    "inside_a_warp": [1, 2, 1, 3, 5, 1, 1, 7, 9, 2, 4, 1, 30, 1],
    "on_warp_boundaries": [2, 2, 4, 6, 2, 8, 16, 2, 10, 2, 2, 24],
    "on_tile_boundaries": [8, 16, 8, 24, 21, 42, 12, 36, 64, 8, 40],
    "tiles_over_three_or_more_graphs_and_empty_ids": [1, 0, 1, 1, 0, 0, 2, 1, 1, 1, 3, 0, 1, 1, 1, 1, 5, 1, 0, 2, 1],
}


@pytest.mark.parametrize("layout", list(BOUNDARY_SIZES))
@pytest.mark.parametrize("C", [1, 3, 5, 8, 16])
@pytest.mark.parametrize("flags", FLAGS)
def test_graph_boundaries(layout, C, flags):
    sizes = BOUNDARY_SIZES[layout] * 5
    check(batch_of_sizes(sizes), len(sizes), C, flags, seed=len(sizes) + C)


@pytest.mark.parametrize("C", [2, 7, 8])
@pytest.mark.parametrize("flags", FLAGS)
def test_one_graph_per_node(C, flags):
    """B = N: every tile straddles graphs, every row goes to vsum directly."""
    N = 3_001
    check(torch.arange(N), N, C, flags, seed=C)


@pytest.mark.parametrize("C", [4, 8, 13])
@pytest.mark.parametrize("flags", FLAGS)
def test_graph_changes_between_a_groups_tiles(C, flags):
    """Graphs of about a thousand nodes: a warpgroup's consecutive tiles (one grid stride apart) sit in different graphs,
    so the G cache is reloaded and the per-graph sums flushed while the kernel runs."""
    sizes = [997 + 13 * (i % 7) for i in range(200)]
    check(batch_of_sizes(sizes), len(sizes), C, flags, seed=C)


@pytest.mark.parametrize("C", [3, 8, 16])
@pytest.mark.parametrize("flags", FLAGS)
def test_one_graph_over_many_tiles(C, flags):
    check(torch.zeros(400_003, dtype=torch.int64), 1, C, flags, seed=C)


@pytest.mark.parametrize("C", [3, 8])
@pytest.mark.parametrize("flags", FLAGS)
def test_rescued_and_guarded_rows_share_quads_and_warps(C, flags):
    """Every third node has Hn (or, for one graph, G) scaled far beyond the fp16 range — stage 1 and, through D, stage 2
    are range-rescued — and every fifth is shifted to pre-activations of −20 … −50 in some columns (the SiLU batch
    guard): rescued, guarded and ordinary rows sit in one quad and one warp.  Row-wise error against fp64."""
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
    got = run(be.virtual_layer, B, C, flags, inp, lp)
    twin = run(be.virtual_layer_simt, B, C, flags, inp, lp)
    ref = run(ShadowBackend().virtual_layer, B, C, flags, inp, lp, dtype=torch.float64)

    def rowwise(o, r):
        return float(((o.double() - r).abs().amax(dim=1) / r.abs().amax(dim=1).clamp(min=1e-9)).max())

    for x in got:
        assert x is None or torch.isfinite(x).all()
    e_t = rowwise(got[1][:, :3], ref[1][:, :3])
    e_s = rel(got[2], ref[2])
    print(f"C={C} flags={flags} mixed rescue/guard rows: row-wise rel err trans_v {e_t:.2e} "
          f"(twin {rowwise(twin[1][:, :3], ref[1][:, :3]):.2e}), vsum {e_s:.2e} (twin {rel(twin[2], ref[2]):.2e})")
    if got[0] is not None:
        e_a = rowwise(got[0], ref[0])
        print(f"  agg_v row-wise {e_a:.2e} (twin {rowwise(twin[0], ref[0]):.2e})")
        assert e_a <= 2e-5
    # ΔX·φ cancels on rows that are both scaled and shifted: the bound is the edge kernel's range-rescue cap
    assert e_t <= 1e-3 and e_s <= 1e-4
