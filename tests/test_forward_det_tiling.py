"""Deterministic forward kernels (DESIGN §17) against float64, row by row and graph by graph, on the shapes their tiling
makes fragile.

GPU: distegnn_edge_layer_fwd_det + distegnn_edge_combine_det run through every case of
tests/test_edge_kernel_tiling.py and distegnn_virtual_layer_fwd_det + distegnn_vsum_combine_det through every case of
tests/test_virtual_kernel_tiling.py, with the same float64 restatement and the same bounds (helpers.TOL per row and
per graph; where a field needs more, the default kernel's fp32-FMA twin error on the same case times
helpers.TWIN_FACTOR).  Every case runs at the full grid and under the testing library's grid caps 1 and 7, and the
three must be bitwise equal.  On top of those shapes, layouts
aimed at what the deterministic instantiations do differently: 16-edge slices (warp w of tile t owns edges
16(4t + w) .. +15) whose runs are stored to the row or to the slice's slot, rows crossing slices, tiles and grid
strides, the device edge count ending mid-slice, a capacity tail that must not reach the valid rows; vsum chunks of
(64 // C) << s nodes with graphs starting and ending on chunk boundaries, empty graph ids there, and chunk shifts 4, 5
and 6.  After the vsum combine, Σx per graph (judged against Σ|x|), the exact count, and all-zero rows of graphs without
nodes.  Both rollout centroids against float64 per graph.

CPU: the float64 restatement with term magnitudes equals the torch stand-in, and the row-wise metrics reject a 1e-4
error on a small row next to a large one, which the old whole-tensor metric accepted."""
import pytest
import torch

from distegnn_b200 import _lib
from tests import test_edge_kernel_tiling as ek
from tests import test_virtual_kernel_tiling as vk
from tests.helpers import TOL, rel, rowwise, terms_rowwise
from tests.shadow_autograd import edge_terms, virtual_terms
from tests.shadow_backend import ShadowBackend
from tests.test_deterministic import _CappedLib, _chunk_nodes, _vsum_part

H = 64
LAST, NORM = _lib.FLAG_LAST, _lib.FLAG_NORMALIZE
CAPS = (None, 1, 7)     # the product at the full grid, then the testing library's capped twins


# ==== CPU =============================================================================================================
def _cpu_params(A, C, seed):
    _, total = _lib.param_layout(A, C, 0)
    return torch.randn(total, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * 0.2


@pytest.mark.parametrize("A", [0, 2])
@pytest.mark.parametrize("flags", [0, NORM, LAST, NORM | LAST])
def test_edge_terms_restate_the_stand_in(A, flags):
    g = torch.Generator().manual_seed(A + flags)
    N, E = 300, 2_000
    row = torch.sort(torch.randint(0, N - 20, (E,), generator=g))[0]        # nodes N−20.. have no edges
    col = torch.randint(0, N, (E,), generator=g)
    col[::9] = row[::9]
    x4 = torch.zeros(N, 4, dtype=torch.float64)
    x4[:, :3] = torch.randn(N, 3, generator=g, dtype=torch.float64)
    P, Q = (torch.randn(N, H, generator=g, dtype=torch.float64) for _ in range(2))
    ea = torch.randn(E, A, generator=g, dtype=torch.float64) if A else None
    lp = _cpu_params(A, 3, seed=A)
    want_m, want_x = torch.zeros(N, H, dtype=torch.float64), torch.zeros(N, 4, dtype=torch.float64)
    ShadowBackend().edge_layer((N, E, A, 3, 0), flags, row, col, ea, x4, P, Q, lp, want_m, want_x)
    m, x, terms = edge_terms((N, E, A, 3, 0), flags, row, col, ea, x4[:, :3], P, Q, lp)
    assert float((x - want_x[:, :3]).abs().max()) <= 1e-12 * float(want_x.abs().max())
    if not flags & LAST:
        assert float((m - want_m).abs().max()) <= 1e-12 * float(want_m.abs().max())
    assert bool((terms >= x.abs() * (1 - 1e-12)).all())
    assert torch.equal(terms.amax(1) > 0, torch.bincount(row[col != row], minlength=N) > 0)


@pytest.mark.parametrize("C", [1, 3, 16])
@pytest.mark.parametrize("flags", [0, LAST])
def test_virtual_terms_restate_the_stand_in(C, flags):
    g = torch.Generator().manual_seed(C + flags)
    sizes = [5, 0, 40, 1, 300, 0]
    B = len(sizes)
    batch = vk.batch_of_sizes(sizes)
    N = batch.numel()
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    x4 = torch.zeros(N, 4, dtype=torch.float64)
    x4[:, :3] = r(N, 3)
    Hn, Xv, G, vsum0 = r(N, H), r(B, 3, C), r(B, C, H), r(B, 4 + 3 * C + H * C)
    lp = _cpu_params(2, C, seed=C)
    agg_v, trans_v, vsum = torch.zeros(N, H, dtype=torch.float64), torch.zeros(N, 4, dtype=torch.float64), vsum0.clone()
    ShadowBackend().virtual_layer((N, B, 2, C, 0), flags, batch.int(), x4, Hn, Xv, G, lp, agg_v, trans_v, vsum)
    t = virtual_terms((N, B, 2, C, 0), batch.int(), x4[:, :3], Hn, Xv, G, lp)
    close = lambda a, b: float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max()))
    assert close(t["trans_v"], trans_v[:, :3])
    assert close(t["tail_x"], vsum[:, 4:4 + 3 * C] - vsum0[:, 4:4 + 3 * C])
    if not flags & LAST:
        assert close(t["agg_v"], agg_v)
        assert close(t["tail_m"], vsum[:, 4 + 3 * C:] - vsum0[:, 4 + 3 * C:])
    assert bool((t["trans_terms"] >= t["trans_v"].abs() * (1 - 1e-12)).all())
    assert bool((t["tail_x_terms"] >= t["tail_x"].abs() * (1 - 1e-12)).all())
    empty = torch.tensor(sizes) == 0
    assert not t["tail_x_terms"][empty].any() and not t["tail_m"][empty].any()


def _inject(got, scale, i, j):
    """A copy of `got` with entry (i, j) off by 1e-4 of `scale` (row i's own scale)."""
    got = got.clone()
    got[i, j] += 1e-4 * scale
    return got


def test_rowwise_metrics_reject_a_small_row_error_the_global_metric_accepted():
    """A 1e-4 relative error in one degree-one row next to a 6,000-edge hub (agg_m, agg_x) and in one 1-node graph's
    vsum row next to a 300k-node graph (Σ mv, Σ ΔX·φ_X): the whole-tensor metric of the old tiling tests accepts every
    one of them, the row-wise and per-graph metrics reject every one."""
    g = torch.Generator().manual_seed(3)
    # edge stage: rows 0..99 and 101..199 of degree one, row 100 a hub
    row = torch.cat([torch.arange(100), torch.full((6_000,), 100), torch.arange(101, 200)])
    N, E = 400, row.numel()
    col = torch.randint(0, N, (E,), generator=g)
    x3 = torch.randn(N, 3, generator=g, dtype=torch.float64)
    P, Q = (torch.randn(N, H, generator=g, dtype=torch.float64) for _ in range(2))
    m, x, terms = edge_terms((N, E, 0, 3, 0), 0, row, col, None, x3, P, Q, _cpu_params(0, 3, seed=4))
    r = 50
    bad_m = _inject(m, float(m[r].abs().max()), r, 7)
    bad_x = _inject(x, float(terms[r].max()), r, 1)
    assert rel(bad_m, m) <= ek.REL_TOL and rel(bad_x, x) <= ek.REL_TOL
    assert rowwise(bad_m, m) > TOL and terms_rowwise(bad_x, x, terms) > TOL
    # real<->virtual stage: graph 1 has one node, graph 0 300,000
    C, sizes = 2, [300_000, 1, 40]
    batch = vk.batch_of_sizes(sizes).int()
    B, N = len(sizes), batch.numel()
    t = virtual_terms((N, B, 2, C, 0), batch, torch.randn(N, 3, generator=g, dtype=torch.float64),
                      torch.randn(N, H, generator=g, dtype=torch.float64),
                      torch.randn(B, 3, C, generator=g, dtype=torch.float64),
                      torch.randn(B, C, H, generator=g, dtype=torch.float64), _cpu_params(2, C, seed=5))
    vsum = torch.cat([torch.zeros(B, 4, dtype=torch.float64), t["tail_x"], t["tail_m"]], 1)
    bad_vm = _inject(t["tail_m"], float(t["tail_m"][1].abs().max()), 1, 5)
    bad_vx = _inject(t["tail_x"], float(t["tail_x_terms"][1].max()), 1, 2)
    for bad in (torch.cat([vsum[:, :4 + 3 * C], bad_vm], 1), torch.cat([vsum[:, :4], bad_vx, vsum[:, 4 + 3 * C:]], 1)):
        assert rel(bad, vsum) <= vk.REL_TOL
    assert rowwise(bad_vm, t["tail_m"]) > TOL
    assert terms_rowwise(bad_vx, t["tail_x"], t["tail_x_terms"]) > TOL


# ==== GPU: the kernels under test =====================================================================================
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def _backend(cap):
    from distegnn_b200.backend import CudaBackend
    be = CudaBackend()
    if cap is not None:
        be.lib = _CappedLib(cap)
    return be


def _same_bits(outs, what):
    for cap, o in zip(CAPS[1:], outs[1:]):
        for a, b in zip(outs[0], o):
            assert a is None or torch.equal(a, b), f"{what}: grid cap {cap} is not bit-identical to the full grid"


def det_edge(be, N, E, A, flags, inp, lp, n_edges_dev=None):
    """distegnn_edge_layer_fwd_det + distegnn_edge_combine_det at the full grid and at grid caps 1 and 7 (bitwise equal)
    -> the full grid's (agg_m or None, agg_x).  The workspace starts as NaN: a slot read before it is written shows."""
    ws = torch.empty(_lib.deterministic_workspace_bytes(N, E, 3), dtype=torch.uint8, device=dev())
    outs = []
    for cap in CAPS:
        ws.fill_(255)
        outs.append(ek.run(_backend(cap), "edge_layer", N, E, A, flags, inp, lp, n_edges_dev, det_ws=ws))
    _same_bits(outs, "edge")
    return outs[0]


def det_virtual(be, B, C, flags, inp, lp, vsum0):
    """distegnn_virtual_layer_fwd_det + distegnn_vsum_combine_det from vsum = 0, at the full grid and at grid caps 1 and
    7 (bitwise equal) -> the full grid's (agg_v or None, trans_v, vsum).  Also checks the combine's Σ(x, 1) per
    graph."""
    N = inp["batch"].numel()
    assert not vsum0.any()
    ws = torch.empty(_vsum_part(N, C)[2], dtype=torch.uint8, device=dev())
    outs = []
    for cap in CAPS:
        b = _backend(cap)

        def layer(dims, fl, batch, x4, Hn, Xv, G, lp_, agg_v, trans_v, vsum):
            b.virtual_layer(dims, fl, batch, x4, Hn, Xv, G, lp_, agg_v, trans_v, vsum, det_ws=ws)
            b._vsum_combine(N, B, C, fl & LAST, batch, x4, vsum, ws)
        ws.fill_(255)
        outs.append(vk.run(layer, B, C, flags, inp, lp, vsum0))
    _same_bits(outs, "vsum")
    vsum = outs[0][2]
    bl, x = inp["batch"].long(), inp["x4"][:, :3].double()
    cnt = torch.bincount(bl, minlength=B)
    assert torch.equal(vsum[:, 3], cnt.float()), "node count per graph"
    sx = torch.zeros(B, 3, dtype=torch.float64, device=x.device).index_add(0, bl, x)
    sx_terms = torch.zeros(B, 3, dtype=torch.float64, device=x.device).index_add(0, bl, x.abs())
    e = terms_rowwise(vsum[cnt > 0, :3], sx[cnt > 0], sx_terms[cnt > 0])
    assert not vsum[cnt == 0].any(), "vsum row of a graph without nodes is not exactly zero"
    print(f"det_virtual N={N} B={B} C={C}: Σx per graph vs fp64 {e:.1e}")
    assert e <= TOL, e
    return outs[0]


# ==== GPU: edge kernel, the shapes of test_edge_kernel_tiling.py ======================================================
@pytest.mark.gpu
@pytest.mark.parametrize("A", ek.ATTR_COUNTS)
@pytest.mark.parametrize("flags", ek.FLAG_SETS)
def test_det_edge_attr_instantiations(A, flags):
    ek.attr_case(A, flags, kernel=det_edge)


@pytest.mark.gpu
@pytest.mark.parametrize("E", ek.RAGGED_E)
def test_det_edge_small_and_ragged_edge_counts(E):
    ek.ragged_case(E, kernel=det_edge)


@pytest.mark.gpu
def test_det_edge_hub_destination_next_to_degree_one_rows():
    ek.hub_case(kernel=det_edge)


@pytest.mark.gpu
def test_det_edge_capacity_mode_device_count_below_bound():
    ek.capacity_case(kernel=det_edge)


@pytest.mark.gpu
def test_det_edge_many_tiles_per_warpgroup():
    ek.many_tiles_case(kernel=det_edge)


@pytest.mark.gpu
def test_det_edge_rescued_and_guarded_rows_share_quads_and_warps():
    ek.rescued_and_guarded(kernel=det_edge)


# ==== GPU: edge kernel, slice layouts =================================================================================
def _rows(deg):
    return torch.repeat_interleave(torch.arange(len(deg)), torch.tensor(deg))


def _cols(row, N, seed):
    return torch.randint(0, N, (row.numel(),), generator=torch.Generator().manual_seed(seed))


def slice_offsets_layout():
    """Rows of degree 15, 16, 17, 31, 32, 33 whose first edge sits at offset 0, 1 and 15 of a 16-edge slice (offset 15:
    the row's first edge is the slice's last), each after two isolated node ids and degree-one rows; -> (degrees,
    first edge of every such row)."""
    deg, e, starts = [], 0, []
    for d in (15, 16, 17, 31, 32, 33):
        for o in (0, 1, 15):
            fill = (o - e) % 16
            deg += [0, 0] + [1] * fill
            e += fill
            starts.append((e, d))
            deg.append(d)
            e += d
    deg += [0, 0, 1, 1]
    return deg, starts


def boundary_layout(seed):
    """Rows that cross a tile boundary (64 edges), the grid strides of caps 1 and 7 and of the full grid (4 warpgroups
    per CTA: 4·64 edges per CTA), a row over many slices, and runs that end exactly on a slice boundary with isolated
    node ids on both sides; between them rows of degree 0 … 5.  -> (degrees, [(first edge, degree)])."""
    stride = 4 * 64 * torch.cuda.get_device_properties(dev()).multi_processor_count
    targets = [(60, 10), (250, 12), (4 * 64 * 7 - 3, 5), (5_000, 300), (6_000, 16), (6_016, 16), (6_032, 1),
               (stride - 9, 20), (stride + 100, 16)]
    g = torch.Generator().manual_seed(seed)
    deg, e = [], 0
    for start, d in targets + [(stride + 3_000, 0)]:
        while e < start:
            k = min(int(torch.randint(0, 6, (1,), generator=g)), start - e)
            deg.append(k)
            e += k
        if start in (6_000, 6_016, 6_032):
            deg += [0, 0, 0]
        if d:
            deg.append(d)
            e += d
    return deg, targets


@pytest.mark.gpu
@pytest.mark.parametrize("A,flags", [(0, 0), (2, NORM), (3, 0), (1, LAST)])
def test_det_edge_rows_across_slices_at_every_offset(A, flags):
    deg, starts = slice_offsets_layout()
    row = _rows(deg)
    for s, d in starts:
        assert bool((row[s:s + d] == row[s]).all()) and (s == 0 or row[s - 1] != row[s])
    N = len(deg)
    ek.check(N, row, _cols(row, N, 30), A, flags, seed=30, kernel=det_edge)


@pytest.mark.gpu
@pytest.mark.parametrize("A,flags", [(2, 0), (8, NORM | LAST)])
def test_det_edge_rows_across_tiles_and_grid_strides(A, flags):
    deg, targets = boundary_layout(seed=31)
    row = _rows(deg)
    for s, d in targets:
        assert bool((row[s:s + d] == row[s]).all()) and row[s - 1] != row[s]
    N = len(deg)
    ek.check(N, row, _cols(row, N, 31), A, flags, seed=31, kernel=det_edge)


@pytest.mark.gpu
@pytest.mark.parametrize("tail", ["past_the_count", "continues_the_last_row"])
def test_det_edge_device_count_ends_mid_slice(tail):
    """n_valid = 16k + 7 with the last valid row over the last two slices; the capacity's padding holds out-of-range ids
    or continues the last valid row (so that a combine reading past the count would add a slot to it)."""
    deg, _ = slice_offsets_layout()
    deg[-1] = 17 + (7 - sum(deg[:-1]) - 17) % 16
    row = _rows(deg)
    n_valid = row.numel()
    assert n_valid % 16 == 7
    N = len(deg) + 10
    col = _cols(row, N, 32)
    pad = 4_000
    if tail == "past_the_count":
        row_t = torch.full((pad,), 2**30)
        col_t = row_t
    else:
        row_t = torch.full((pad,), int(row[-1]))
        col_t = _cols(row_t, N, 33)
    ek.check(N, torch.cat([row, row_t]), torch.cat([col, col_t]), 2, 0, seed=32, n_valid=n_valid, kernel=det_edge)


@pytest.mark.gpu
@pytest.mark.parametrize("A,flags", [(2, 0), (3, LAST)])
def test_det_edge_capacity_tail_cannot_reach_the_valid_rows(A, flags):
    """The padding past the device count holds valid ids of isolated nodes (no valid edge references them) whose P and Q
    rows, and the padding's edge attributes, are ±1e30 and NaN.  The result equals, bit for bit, the same call with
    out-of-range padding ids, and the isolated rows stay exactly zero."""
    N, n_iso = 4_000, 1_000
    row, col = ek.random_graph(N - n_iso, 30_011, seed=34)
    pad = 200_000 - row.numel()
    g = torch.Generator().manual_seed(35)
    iso_row = torch.sort(torch.randint(N - n_iso, N, (pad,), generator=g))[0]
    iso_col = torch.randint(N - n_iso, N, (pad,), generator=g)
    far = torch.full((pad,), 2**30)
    inp = ek.make_inputs(torch.cat([row, iso_row]), torch.cat([col, iso_col]), N, A, seed=34)
    junk = torch.tensor([1e30, -1e30, float("nan")], device=dev())
    for k in ("P", "Q"):
        inp[k][N - n_iso:] = junk[torch.arange(n_iso * H, device=dev()) % 3].view(n_iso, H)
    inp["ea"][row.numel():] = junk[torch.arange(pad * A, device=dev()) % 3].view(pad, A)
    got = ek.check(N, torch.cat([row, iso_row]), torch.cat([col, iso_col]), A, flags, n_valid=row.numel(),
                   kernel=det_edge, inp=inp)
    inp_far = dict(inp, row=torch.cat([row, far]).int().to(dev()), col=torch.cat([col, far]).int().to(dev()))
    plain = ek.check(N, torch.cat([row, far]), torch.cat([col, far]), A, flags, n_valid=row.numel(),
                     kernel=det_edge, inp=inp_far)
    for a, b in zip(got, plain):
        assert a is None or torch.equal(a, b)


# ==== GPU: real<->virtual kernel, the shapes of test_virtual_kernel_tiling.py =========================================
@pytest.mark.gpu
@pytest.mark.parametrize("C", list(range(1, 17)))
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_every_channel_count(C, flags):
    vk.every_channel_case(C, flags, kernel=det_virtual)


@pytest.mark.gpu
@pytest.mark.parametrize("N", vk.SMALL_N)
@pytest.mark.parametrize("C", vk.SMALL_N_C)
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_small_node_counts(N, C, flags):
    vk.small_n_case(N, C, flags, kernel=det_virtual)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(vk.BOUNDARY_SIZES))
@pytest.mark.parametrize("C", vk.BOUNDARY_C)
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_graph_boundaries(layout, C, flags):
    vk.boundary_case(layout, C, flags, kernel=det_virtual)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 7, 8])
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_one_graph_per_node(C, flags):
    vk.one_graph_per_node_case(C, flags, kernel=det_virtual)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [4, 8, 13])
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_graph_changes_between_a_groups_tiles(C, flags):
    vk.graph_change_case(C, flags, kernel=det_virtual)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 8, 16])
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_one_graph_over_many_tiles(C, flags):
    vk.many_tiles_case(C, flags, kernel=det_virtual)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 8])
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_rescued_and_guarded_rows_share_quads_and_warps(C, flags):
    vk.rescued_and_guarded(C, flags, kernel=det_virtual)


# ==== GPU: real<->virtual kernel, chunk layouts =======================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 5, 16])
@pytest.mark.parametrize("flags", vk.FLAGS)
def test_det_virtual_graphs_on_chunk_boundaries(C, flags):
    per = (64 // C) << 4
    g = torch.Generator().manual_seed(C)
    sizes = [per, 0,                                # exactly chunk 0; an empty id on the boundary
             5, 7, per - 13, 1, 0, 0,               # chunk 1: graphs inside it, the last one its last node; empty ids
             per - 1,                               # chunk 2 but its last node
             per + 1,                               # from chunk 2's last node over all of chunk 3, to its last node
             per - 3, 3,                            # chunk 4: the second graph ends on its last node
             2 * per + 5]                           # chunks 5, 6 and into 7
    sizes += torch.randint(0, 9, (60,), generator=g).tolist()
    N = sum(sizes)
    assert _chunk_nodes(N, C) == per
    starts = set(torch.cumsum(torch.tensor([0] + sizes[:-1]), 0).tolist())
    assert {per, 2 * per - 1, 2 * per, 3 * per - 1, 4 * per, 5 * per - 3, 5 * per} <= starts
    vk.check(vk.batch_of_sizes(sizes), len(sizes), C, flags, seed=40 + C, kernel=det_virtual)


@pytest.mark.gpu
@pytest.mark.parametrize("N,shift", [(200_003, 4), (300_003, 5), (600_003, 6)])
def test_det_virtual_chunk_shifts(N, shift):
    """C = 16: 4 << s nodes per chunk, s = 4 up to N = 262,144, 5 up to 524,288.  Tiny graphs and empty ids next to one
    large graph, graph boundaries on chunk boundaries."""
    C = 16
    per = _chunk_nodes(N, C)
    assert per == 4 << shift
    sizes = [1, 2, 0, per - 3, 3 * per, 1, per - 1, 0]
    sizes += [N - sum(sizes) - 7, 0, 1, 2, 3, 1]
    assert sum(sizes) == N
    for flags in (0, LAST) if shift < 6 else (0,):
        vk.check(vk.batch_of_sizes(sizes), len(sizes), C, flags, seed=50 + shift, kernel=det_virtual)


@pytest.mark.gpu
def test_det_virtual_tiny_graphs_next_to_a_300k_node_graph():
    C = 16
    sizes = [1, 0, 2, 300_000, 1, 0, 3, 1]
    for flags in vk.FLAGS:
        vk.check(vk.batch_of_sizes(sizes), len(sizes), C, flags, seed=60, kernel=det_virtual)


# ==== GPU: rollout centroids ==========================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("deterministic", [False, True])
def test_rollout_centroid_per_graph(deterministic):
    """Σx per graph in fp64 against float64 (judged against Σ|x|, far below fp32 rounding) and the exact count; graphs
    of 0, 1, 31 and 33 nodes so that warps straddle graphs, one of 2M nodes; and one graph without data_batch."""
    from distegnn_b200.backend import CudaBackend
    be = CudaBackend()
    g = torch.Generator().manual_seed(70)
    sizes = [0, 1, 31, 33, 0, 1, 1, 2_000_000, 33, 31, 0, 1, 64, 17]
    B = len(sizes)
    batch = vk.batch_of_sizes(sizes)
    N = batch.numel()
    pos = torch.randn(N, 3, generator=g) * 2 + 100 * torch.randn(B, 3, generator=g)[batch]
    want = torch.zeros(B, 3, dtype=torch.float64).index_add(0, batch, pos.double())
    terms = torch.zeros(B, 3, dtype=torch.float64).index_add(0, batch, pos.double().abs())
    cnt = torch.bincount(batch, minlength=B)
    runs = []
    for b, nb in ((batch, B), (None, 1)):
        p = pos if b is not None else pos[:sizes[2]]
        sums = torch.zeros(nb, 4, dtype=torch.float64, device=dev())
        be.rollout_centroid(p.to(dev()), None if b is None else b.to(dev()), sums, deterministic=deterministic)
        torch.cuda.synchronize()
        runs.append(sums.cpu())
    s = runs[0]
    assert torch.equal(s[:, 3], cnt.double())
    assert not s[cnt == 0].any()
    e = terms_rowwise(s[cnt > 0, :3], want[cnt > 0], terms[cnt > 0])
    one = runs[1]
    assert float(one[0, 3]) == sizes[2]
    e1 = float(((one[0, :3] - pos[:sizes[2]].double().sum(0)).abs() / pos[:sizes[2]].double().abs().sum(0)).max())
    print(f"rollout centroid deterministic={deterministic}: Σx per graph vs fp64 {e:.1e}, one graph {e1:.1e}")
    assert e <= 1e-12 and e1 <= 1e-12
    if deterministic:
        again = torch.zeros(B, 4, dtype=torch.float64, device=dev())
        be.rollout_centroid(pos.to(dev()), batch.to(dev()), again, deterministic=True)
        assert torch.equal(again.cpu(), s)
