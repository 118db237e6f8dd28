"""The node-stage forward kernels (node_layer_tc_kernel, embed_tc_kernel) on the shapes their register-fragment tiling
makes fragile.  A CTA runs four independent warpgroup pipelines over 64-node tiles; thread (g, q) of warp w holds rows
16w + g and 16w + g + 8 of its warpgroup's tile, and the four threads of a quad share those rows (per-row maxima and φ_v
come from quad shuffles, the coordinate update is split over the quad's lanes).

Cases: graph boundaries between the two rows of a thread, on 16-row warp blocks and on 64-row tiles; a graph of exactly
one tile; consecutive tiles of a warpgroup in different graphs, and one graph over many tiles; N = 64k − 1, 64k, 64k + 1
around one tile and at eight tiles per warpgroup; rows outside the fp16 range confined to one quad of one warp per tile,
and one such row per warp, at every encode site (h, agg_m/deg, agg_v, t1 and h' through attr, h0 through node_feat).
Node cases run for Na = 0 and 8 and C = 1 and 16, each with and without FLAG_LAST; every case goes through check_node /
check_embed of test_node_kernel_tiling.py (buffer contract, in place against out of place, reruns, the fp32-FMA twin and
the float64 restatement)."""
import pytest
import torch

from tests.test_node_kernel_tiling import (RESCUE_CAP, check_embed, check_node, embed_inputs, node_inputs, random_deg,
                                           sm_count)

pytestmark = pytest.mark.gpu

TILE, WG = 64, 4                        # rows per warpgroup tile, warpgroups per CTA
NA_C = [(0, 1), (0, 16), (8, 1), (8, 16)]


def many_tiles_k():
    """Tiles that give every warpgroup of a full grid at least eight."""
    return 8 * WG * sm_count() + 3


def layout_sizes(name):
    """Nodes per graph."""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    if name == "between_thread_rows":      # boundaries at every offset inside the 16-row blocks, rows g | g + 8 split
        return torch.tensor([3, 8, 5, 13, 9, 7, 19, 2, 11, 4] * 60)
    if name == "on_warp_rows":
        return 16 * torch.randint(1, 4, (200,), generator=g)
    if name == "on_tiles":                  # each tile one graph; a warpgroup's consecutive tiles in different graphs
        return TILE * torch.randint(1, 3, (3 * WG * sm_count(),), generator=g)
    if name == "one_tile_graph":            # graph 2 is exactly tile 2
        return torch.tensor([100, 28, TILE, 300, 7])
    if name == "one_graph_many_tiles":      # graph 1 spans at least eight tiles of every warpgroup
        return torch.tensor([40, TILE * many_tiles_k(), 50])
    raise ValueError(name)


LAYOUTS = ["between_thread_rows", "on_warp_rows", "on_tiles", "one_tile_graph", "one_graph_many_tiles"]


def layout_batch(name):
    sizes = layout_sizes(name)
    return torch.repeat_interleave(torch.arange(sizes.numel()), sizes), sizes.numel()


def node_count(spec):
    k = 1 if spec.startswith("one_tile") else many_tiles_k()
    return TILE * k + {"minus_1": -1, "exact": 0, "plus_1": 1}[spec.split(":")[1]]


NODE_COUNTS = [f"{k}:{d}" for k in ("one_tile", "8_tiles_per_warpgroup") for d in ("minus_1", "exact", "plus_1")]


def batch_of(N, B, seed):
    return torch.sort(torch.randint(0, B, (N,), generator=torch.Generator().manual_seed(seed))).values


@pytest.mark.parametrize("Na,C", NA_C)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_node_regfrag_graph_layouts(layout, Na, C):
    batch, B = layout_batch(layout)
    N = batch.numel()
    check_node(node_inputs(batch, random_deg(N, 11), Na, seed=12), B, Na, C, layout, seed=13)


@pytest.mark.parametrize("Na,C", NA_C)
@pytest.mark.parametrize("n_spec", NODE_COUNTS)
def test_node_regfrag_node_counts(n_spec, Na, C):
    N = node_count(n_spec)
    B = 3
    check_node(node_inputs(batch_of(N, B, N), random_deg(N, N), Na, seed=N), B, Na, C, f"N {n_spec}", seed=N)


def extreme_rows(N, pattern):
    """Rows put outside the fp16 range: the two rows of one quad of one warp in every tile (the warp and quad vary from
    tile to tile), or one row in every 16-row warp block."""
    r = torch.arange(N)
    tile, off = r // TILE, r % TILE
    if pattern == "one_quad":
        w, g = tile % WG, tile % 8
        return (off == 16 * w + g) | (off == 16 * w + g + 8)
    if pattern == "one_row_per_warp":
        blk = r // 16
        return r % 16 == (5 * blk) % 16
    raise ValueError(pattern)


NODE_SITES = ["h", "agg_m", "agg_v", "attr_t1_h_prime"]


@pytest.mark.parametrize("Na,C", NA_C)
@pytest.mark.parametrize("pattern", ["one_quad", "one_row_per_warp"])
@pytest.mark.parametrize("site", NODE_SITES)
def test_node_regfrag_fp16_range_rescue(site, pattern, Na, C):
    """h (φ_v and layer 1 start scaled), agg_m/deg and agg_v (D brought to the new row scale), and attr ×1e5 … 1e7 with
    h ordinary (t1 and h' leave the range; h' is re-encoded from h_out, which in place is h; needs Na > 0)."""
    if site == "attr_t1_h_prime" and Na == 0:
        pytest.skip("t1 and h' are driven out of range through node_attr")
    N, B = 64 * 90 + 17, 4
    g = torch.Generator().manual_seed(120 + NODE_SITES.index(site))
    inp = node_inputs(batch_of(N, B, 121), random_deg(N, 122), Na, seed=123)
    ext = extreme_rows(N, pattern)
    scale = torch.where(ext, 10 ** (5 + 2 * torch.rand(N, generator=g)), torch.ones(N)).to(inp["h"].device)[:, None]
    key = {"h": "h", "agg_m": "agg_m", "agg_v": "agg_v", "attr_t1_h_prime": "attr"}[site]
    inp[key] = inp[key] * scale
    check_node(inp, B, Na, C, f"rescue {site} {pattern}", seed=124,
               tols=dict.fromkeys(("h", "x", "P", "Q", "Hn", "loc", "vsum"), RESCUE_CAP))


@pytest.mark.parametrize("F", [1, 16])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_embed_regfrag_graph_layouts(layout, F):
    batch, B = layout_batch(layout)
    check_embed(embed_inputs(batch, F, seed=14), B, F, layout, seed=15)


@pytest.mark.parametrize("n_spec", NODE_COUNTS)
def test_embed_regfrag_node_counts(n_spec):
    N = node_count(n_spec)
    check_embed(embed_inputs(batch_of(N, 3, N), 5, seed=N), 3, 5, f"N {n_spec}", seed=N)


@pytest.mark.parametrize("pattern", ["one_quad", "one_row_per_warp"])
def test_embed_regfrag_h0_out_of_fp16_range(pattern):
    N, B, F = 64 * 90 + 17, 3, 4
    inp = embed_inputs(batch_of(N, B, 130), F, seed=131)
    g = torch.Generator().manual_seed(132)
    s = torch.where(extreme_rows(N, pattern), 10 ** (4 + 2 * torch.rand(N, generator=g)), torch.ones(N))
    inp["feat"] = inp["feat"] * s.to(inp["feat"].device)[:, None]
    check_embed(inp, B, F, f"h0 out of range {pattern}", seed=133,
                tols=dict.fromkeys(("h", "P", "Q", "Hn", "vsum"), RESCUE_CAP))
