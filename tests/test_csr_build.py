"""The CSR builds of csrc/csr.cu against an exact host reference, bit for bit.

`distegnn_build_csr` (rows in id order) and `distegnn_build_csr_cells` (rows in (graph, cell, id) order, DESIGN §3) turn
an int64 `edge_index` into the int32 `rowptr`, `row`, `col` and `perm` every kernel reads, and count the edges whose ids
lie outside [0, N).  Neither has a float reduction whose order matters, nor an expression nvcc could contract into an
FMA, so the reference below restates them in numpy and every output is compared for equality, not within a tolerance.

CPU: the id-order reference against `CSRGraph.from_edge_index`, the cell-order reference against the invariants of
DESIGN §3, and the comparator against planted faults (an unstable edge sort, a node sort on too few key bits, the cell
index computed in float64 or with a fused multiply-add).
GPU: both builds against the reference at the edges of the two radix sorts' key widths, on edge patterns, empty and
out-of-range inputs, adversarial positions and graph batches (`n_graphs` = 2^30 + 3 among them); repeatability and the
workspace size; `gather_rows` / `scatter_rows` against torch indexing, past 2^31 elements too; and one training step at
scale through the cell order against float64 autograd of the oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

F32 = np.float32
FIELDS = ("rowptr", "row", "col", "perm", "n_invalid")
NODES_PER_CELL = 4                         # kCsrNodesPerCell of csrc/csr.cu


# ======================================================================================================================
# The host reference
# ======================================================================================================================
def key_bits(n):
    """Bits of the radix sort of keys in [0, n): the least b >= 1 with 2^b >= n, at most 31."""
    b = 1
    while b < 31 and (1 << b) < n:
        b += 1
    return b


def cell_budget(n_nodes, n_graphs):
    """Cells per graph of the row order: about four nodes per cell, at most 2^30 / n_graphs and at least one, so every
    (graph, cell) key lies below max(2^30, n_graphs)."""
    return max(min(n_nodes // (n_graphs * NODES_PER_CELL) + 1, (1 << 30) // n_graphs), 1)


def stable_order(keys):
    """The stable argsort of int keys in [0, 2^31), as cub's radix sort orders them: one sort of the unique composite
    key·2^32 + index."""
    k = np.asarray(keys, np.int64)
    return np.sort((k << 32) | np.arange(k.size, dtype=np.int64)) & 0xFFFFFFFF


def chamfer_grid_size(ext, budget):
    """distegnn_chamfer_grid_size of the testing library -> (cell, dims, ncell)."""
    from tests import twin_backend
    fn = twin_backend.load_testing().distegnn_chamfer_grid_size
    fn.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    fn.restype = C.c_int
    cell, dims, ncell = C.c_float(0), (C.c_int32 * 3)(), C.c_int64(0)
    e = (C.c_float * 3)(*[float(x) for x in ext])
    twin_backend.check(fn(C.addressof(e), int(budget), C.addressof(cell), C.addressof(dims), C.addressof(ncell)),
                       "chamfer_grid_size")
    return F32(cell.value), [int(d) for d in dims], int(ncell.value)


def q_f32(x, o, inv):
    """The cell coordinate as axis_cell computes it: fl(fl(x − o) · inv), two fp32 roundings."""
    return (x - o) * inv


def axis_cell(x, o, inv, n, q=q_f32):
    """axis_cell of cell_grid.cuh: q > 0 ? (q < n ? ⌊q⌋ : n − 1) : 0, so NaN -> 0 and +inf -> n − 1."""
    with np.errstate(invalid="ignore", over="ignore"):
        v = q(x, o, inv)
        inside = (v > 0) & (v < n)
        return np.where(inside, np.where(inside, v, 0).astype(np.int64), np.where(v > 0, n - 1, 0))


def cell_grid(pos, n_nodes, n_graphs, budget=cell_budget):
    """One grid for all graphs over the finite coordinates of `pos` (per axis; an axis without one gets origin 0 and
    extent 0), sized by distegnn_chamfer_grid_size for the cell budget of the build."""
    o, ext = np.zeros(3, F32), np.zeros(3, F32)
    for k in range(3):
        v = pos[:, k][np.isfinite(pos[:, k])]
        if v.size:
            with np.errstate(over="ignore"):
                o[k], ext[k] = v.min(), v.max() - v.min()      # hi − lo in fp32: +inf past FLT_MAX
    b = budget(n_nodes, n_graphs)
    cell, dims, ncell = chamfer_grid_size(ext, b) if b >= 1 else (F32(np.finfo(F32).max), [1, 1, 1], 1)
    return dict(o=o, ext=ext, budget=b, cell=cell, inv=F32(1) / cell, dims=dims, ncell=ncell)


def node_keys(pos, batch, n_graphs, g, q=q_f32):
    """(graph, cell, id) keys without the id: clamp(batch)·ncell + (ix·ny + iy)·nz + iz."""
    nx, ny, nz = g["dims"]
    ix, iy, iz = (axis_cell(pos[:, k], g["o"][k], g["inv"], g["dims"][k], q) for k in range(3))
    gid = np.zeros(pos.shape[0], np.int64) if batch is None else np.clip(np.asarray(batch, np.int64), 0, n_graphs - 1)
    return gid * g["ncell"] + (ix * ny + iy) * nz + iz


def ref_csr(edge_index, n_nodes, rank=None):
    """distegnn_build_csr restated (rank = None), or the edge half of distegnn_build_csr_cells: ids clamped into [0, N)
    and counted when either is outside, rowptr from the in-degrees in id order, the edges stably sorted by the rank of
    their clamped destination."""
    ei = np.asarray(edge_index, np.int64)
    E, N = ei.shape[1], n_nodes
    if E == 0:
        e = np.zeros(0, np.int32)
        return dict(rowptr=np.zeros(N + 1, np.int32), row=e, col=e.copy(), perm=e.copy(), n_invalid=0)
    r, c = ei
    n_invalid = int(((r < 0) | (r >= N) | (c < 0) | (c >= N)).sum())
    r, c = np.clip(r, 0, N - 1), np.clip(c, 0, N - 1)
    rowptr = np.zeros(N + 1, np.int64)
    rowptr[1:] = np.cumsum(np.bincount(r, minlength=N))
    perm = stable_order(r if rank is None else rank[r])
    return dict(rowptr=rowptr.astype(np.int32), row=r[perm].astype(np.int32), col=c[perm].astype(np.int32),
                perm=perm.astype(np.int32), n_invalid=n_invalid)


def ref_csr_cells(edge_index, n_nodes, pos, batch, n_graphs, q=q_f32, budget=cell_budget, bits=None):
    """distegnn_build_csr_cells restated: the nodes stably sorted by their (graph, cell) key, the edges by the rank of
    their destination.  `q`, `budget` and `bits` (sort only the bits(n_graphs · budget) low bits of the key, as a radix
    sort does) exist for the planted faults; the reference sorts by the whole key.  The grid goes to result["grid"]."""
    if np.asarray(edge_index).shape[1] == 0:
        return ref_csr(edge_index, n_nodes)
    pos = np.asarray(pos, F32)
    g = cell_grid(pos, n_nodes, n_graphs, budget)
    keys = node_keys(pos, batch, n_graphs, g, q)
    if bits is not None:
        keys = keys & ((1 << bits(n_graphs * g["budget"])) - 1)
    order = stable_order(keys)
    rank = np.empty(n_nodes, np.int64)
    rank[order] = np.arange(n_nodes)
    out = ref_csr(edge_index, n_nodes, rank)
    out["grid"] = g
    return out


def assert_same(got, want, what=""):
    """Bitwise equality of the five build outputs; the message names the first differing entry."""
    for k in FIELDS:
        a, b = got[k], want[k]
        if k == "n_invalid":
            assert a == b, f"{what}: n_invalid {a} != {b}"
            continue
        assert a.dtype == np.int32 and a.shape == b.shape, f"{what}: {k} {a.dtype}{a.shape} vs {b.dtype}{b.shape}"
        bad = np.flatnonzero(a != b)
        assert bad.size == 0, f"{what}: {k} differs at {bad.size} entries, first [{bad[0]}]: {a[bad[0]]} != {b[bad[0]]}"


# ---- faults planted into the reference -------------------------------------------------------------------------------
def q_f64(x, o, inv):
    return (x.astype(np.float64) - np.float64(o)) * np.float64(inv)


def q_fma(x, o, inv):
    """fma(x, inv, −fl(o·inv)), the contraction of x·inv − o·inv, emulated in float64 (x·inv is exact there)."""
    return (x.astype(np.float64) * np.float64(inv) - np.float64(F32(o * inv))).astype(F32)


def budget_without_floor(n_nodes, n_graphs):
    """cell_budget without its floor of one cell: 0 for n_graphs > 2^30."""
    return min(n_nodes // (n_graphs * NODES_PER_CELL) + 1, (1 << 30) // n_graphs)


def swap_two_edges_of_a_row(res):
    out = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in res.items()}
    starts = np.flatnonzero(out["row"][1:] == out["row"][:-1])
    i = int(starts[0])
    for k in ("col", "perm"):
        out[k][[i, i + 1]] = out[k][[i + 1, i]]
    return out


def boundary_points(n=4096, seed=0):
    """One graph of n nodes in the box [lo, lo + 100] x [0, 0.05]^2, lo = −37.3 (a grid of 820 x 1 x 1 cells), whose x
    coordinates lie within 16 ulps of the cell planes, chosen where the cell index axis_cell computes differs from the
    one computed in float64 (up to a quarter of the nodes) or with a fused multiply-add (another quarter).  Every other
    node is uniform in the box; two corners pin the bounds.  Returns (pos [n,3] float32, {variant: its node count})."""
    lo, w = F32(-37.3), F32(0.05)
    hi = F32(lo + F32(100))
    g = cell_grid(np.array([[lo, 0, 0], [hi, w, w]], F32), n, 1)
    nx = g["dims"][0]
    planes = (np.float64(lo) + np.arange(1, nx) * np.float64(g["cell"])).astype(F32)
    cand = np.unique((planes.view(np.int32)[:, None] + np.arange(-16, 17)).astype(np.int32).view(F32))
    cand = cand[(cand > lo) & (cand < hi)]
    base = axis_cell(cand, lo, g["inv"], nx)
    picked, counts = [], {}
    for name, q in (("fp64", q_f64), ("fma", q_fma)):
        moved = cand[axis_cell(cand, lo, g["inv"], nx, q) != base][: n // 4]
        counts[name] = moved.size
        picked.append(moved)
    rng = np.random.default_rng(seed)
    pos = np.minimum(rng.random((n, 3)) * np.array([hi - lo, w, w]) + np.array([lo, 0, 0]), [hi, w, w]).astype(F32)
    xs = np.concatenate(picked)
    pos[rng.permutation(np.arange(2, n))[: xs.size], 0] = xs
    pos[0], pos[1] = (lo, 0, 0), (hi, w, w)
    return pos, counts


def every_node_a_row(rng, n, extra):
    """Edges that give every node at least one in-edge (so the row array shows the whole node order), shuffled."""
    row = np.concatenate([np.arange(n), rng.integers(0, n, extra)])
    ei = np.stack([row, rng.integers(0, n, row.size)])
    return ei[:, rng.permutation(row.size)]


# ======================================================================================================================
# CPU
# ======================================================================================================================
def test_id_order_reference_matches_csrgraph_from_edge_index():
    from distegnn_b200.shards import CSRGraph
    rng = np.random.default_rng(1)
    for N, E in ((1, 5), (7, 40), (1_000, 6_000), (5_000, 1)):
        ei = rng.integers(0, N, (2, E))
        ei[1, ::5] = ei[0, ::5]                                     # self loops
        ei = np.concatenate([ei, ei[:, ::3]], 1)                    # duplicates
        want = ref_csr(ei, N)
        ids = torch.arange(ei.shape[1], dtype=torch.float64)[:, None]
        g, pe = CSRGraph.from_edge_index(torch.from_numpy(ei), N, ids)
        assert want["n_invalid"] == 0
        assert np.array_equal(want["rowptr"], g.rowptr.numpy()) and np.array_equal(want["col"], g.col.numpy())
        assert np.array_equal(want["row"], g.rows().numpy()) and np.array_equal(want["perm"], pe[:, 0].long().numpy())


def check_design_invariants(res, ei, N, batch):
    """DESIGN §3: perm a permutation, each row one run in the caller's relative order, graphs contiguous and in order,
    rowptr the id-order rowptr."""
    row, col, perm = (res[k].astype(np.int64) for k in ("row", "col", "perm"))
    assert np.array_equal(np.sort(perm), np.arange(perm.size)), "perm is not a permutation"
    assert np.array_equal(ei[0][perm], row) and np.array_equal(ei[1][perm], col)
    starts = np.ones(row.size, bool)
    starts[1:] = row[1:] != row[:-1]
    assert np.unique(row[starts]).size == starts.sum(), "a row's edges are split into several runs"
    run = np.cumsum(starts)
    assert np.all((perm[1:] > perm[:-1]) | (run[1:] != run[:-1])), "a row's edges left the caller's relative order"
    gid = np.zeros(row.size, np.int64) if batch is None else np.asarray(batch)[row]
    assert np.all(gid[1:] >= gid[:-1]), "graphs are not contiguous and in order"
    assert np.array_equal(res["rowptr"], ref_csr(ei, N)["rowptr"])


def three_clouds():
    from tests.test_edge_row_order import batch_of_clouds
    _, inp = batch_of_clouds()
    return inp["edge_index"].numpy(), inp["node_loc"].shape[0], inp["node_loc"].numpy(), inp["data_batch"].numpy(), 3


def test_cell_order_reference_keeps_the_design_invariants():
    ei, N, pos, batch, B = three_clouds()
    res = ref_csr_cells(ei, N, pos, batch, B)
    check_design_invariants(res, ei, N, batch)
    assert not np.all(res["row"][1:] >= res["row"][:-1]), "the rows came out in id order"
    rng = np.random.default_rng(2)
    sizes = rng.integers(1, 6, 3_000)
    batch = np.repeat(np.arange(sizes.size), sizes)
    ei = graph_local_edges(rng, batch, 3 * batch.size)
    check_design_invariants(ref_csr_cells(ei, batch.size, rng.normal(size=(batch.size, 3)).astype(F32), batch,
                                          sizes.size), ei, batch.size, batch)


def test_comparator_rejects_an_unstable_edge_sort():
    ei, N, pos, batch, B = three_clouds()
    for res in (ref_csr(ei, N), ref_csr_cells(ei, N, pos, batch, B)):
        with pytest.raises(AssertionError, match="(col|perm) differs"):
            assert_same(swap_two_edges_of_a_row(res), res, "swapped")


def huge_graph_count_case():
    """8 nodes whose graph ids lie around 2^30, n_graphs = 2^30 + 3: the cap 2^30 / n_graphs on the cell budget is 0."""
    B = (1 << 30) + 3
    batch = np.array([-2, 0, 1 << 30, (1 << 30) - 1, (1 << 30) + 1, (1 << 30) + 1, (1 << 30) + 2, 1 << 40]) \
        .clip(0, B - 1)
    batch = np.sort(batch)
    rng = np.random.default_rng(3)
    return every_node_a_row(rng, 8, 16), 8, rng.normal(size=(8, 3)).astype(F32), batch, B


def test_comparator_rejects_a_node_sort_on_too_few_key_bits():
    # n_graphs = 2^30 + 3 with the budget of 0 cells: a 1-bit sort leaves the graphs out of order
    ei, N, pos, batch, B = huge_graph_count_case()
    want = ref_csr_cells(ei, N, pos, batch, B)
    assert want["grid"]["budget"] == 1 and want["grid"]["ncell"] == 1
    check_design_invariants(want, ei, N, batch)
    assert budget_without_floor(N, B) == 0 and key_bits(B * budget_without_floor(N, B)) == 1
    with pytest.raises(AssertionError, match="row differs"):
        assert_same(ref_csr_cells(ei, N, pos, batch, B, budget=budget_without_floor, bits=key_bits), want,
                    "budget 0")
    # n_graphs · budget = 2^11 and keys filling [0, 2^11): a sort on one bit fewer reorders the nodes
    ei, N, pos, batch, B = pow2_case(1024)
    want = ref_csr_cells(ei, N, pos, batch, B)
    assert B * want["grid"]["budget"] == B * want["grid"]["ncell"] == 2048
    with pytest.raises(AssertionError, match="row differs"):
        assert_same(ref_csr_cells(ei, N, pos, batch, B, bits=lambda n: key_bits(n) - 1), want, "10-bit node sort")


@pytest.mark.parametrize("variant", ["fp64", "fma"])
def test_comparator_rejects_a_cell_index_rounded_otherwise(variant):
    pos, counts = boundary_points()
    assert counts[variant] > 100, counts
    ei = every_node_a_row(np.random.default_rng(4), pos.shape[0], 3 * pos.shape[0])
    want = ref_csr_cells(ei, pos.shape[0], pos, None, 1)
    with pytest.raises(AssertionError, match="row differs"):
        assert_same(ref_csr_cells(ei, pos.shape[0], pos, None, 1, q={"fp64": q_f64, "fma": q_fma}[variant]), want,
                    variant)


# ======================================================================================================================
# GPU: inputs
# ======================================================================================================================
def graph_local_edges(rng, batch, E):
    """E edges whose two ends lie in the same graph of the sorted `batch`."""
    batch = np.asarray(batch)
    N = batch.size
    start = np.searchsorted(batch, batch, "left")
    size = np.searchsorted(batch, batch, "right") - start
    r = rng.integers(0, N, E)
    return np.stack([r, start[r] + (rng.random(E) * size[r]).astype(np.int64)])


def uniform(rng, n, scale=1.0):
    return (rng.random((n, 3)) * scale).astype(F32)


def pow2_case(B):
    """B graphs, 6,000 nodes on a line: a cell budget of 2 per graph, and a grid of exactly 2 cells, so the node keys
    fill [0, 2B) and the node sort needs key_bits(2B) bits (11 for B = 1024, 12 for 1025)."""
    rng = np.random.default_rng(B)
    N = 6_000
    batch = np.sort(np.concatenate([np.arange(B), rng.integers(0, B, N - B)]))
    pos = np.zeros((N, 3), F32)
    pos[:, 0] = rng.random(N)
    return graph_local_edges(rng, batch, 4 * N), N, pos, batch, B


# ======================================================================================================================
# GPU: the production builds against the reference
# ======================================================================================================================
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def _np(res):
    out = dict(zip(FIELDS[:4], (t.cpu().numpy() for t in res[:4])))
    out["n_invalid"] = 0 if res[4] is None else int(res[4].item())
    return out


def device_builds(ei, N, pos=None, batch=None, B=1):
    """Both builds through CudaBackend, with the out-of-range counter handed back instead of raised."""
    from distegnn_b200.backend import CudaBackend
    be, d = CudaBackend(), dev()
    eid = torch.from_numpy(np.ascontiguousarray(ei, np.int64)).to(d)
    got = {"id": _np(be.build_csr(eid, N, validate="defer"))}
    if pos is not None:
        p = torch.from_numpy(np.ascontiguousarray(pos, F32)).to(d)
        b = None if batch is None else torch.from_numpy(np.ascontiguousarray(batch, np.int64)).to(d)
        got["cells"] = _np(be.build_csr_cells(eid, N, p, b, B, validate="defer"))
    return got


def check_builds(ei, N, pos, batch=None, B=1, what=""):
    """Both builds bitwise against the reference; returns the cell-order reference (its grid included)."""
    got = device_builds(ei, N, pos, batch, B)
    assert_same(got["id"], ref_csr(ei, N), f"{what} id order")
    want = ref_csr_cells(ei, N, pos, batch, B)
    assert_same(got["cells"], want, f"{what} cell order")
    return want


def raw_build(ei, N, pos=None, batch=None, B=1, short=0):
    """The C ABI directly, with a workspace of distegnn_csr_workspace_bytes − `short` bytes -> return code."""
    from distegnn_b200 import _lib
    from distegnn_b200._lib import ptr
    lib, d = _lib.load(), dev()
    E = ei.shape[1]
    eid = torch.from_numpy(np.ascontiguousarray(ei, np.int64)).to(d)
    rowptr = torch.empty(N + 1, dtype=torch.int32, device=d)
    row, col, perm = (torch.empty(E, dtype=torch.int32, device=d) for _ in range(3))
    need = C.c_int64(0)
    assert lib.distegnn_csr_workspace_bytes(N, E, C.byref(need)) == 0
    ws = torch.empty(max(need.value, 1), dtype=torch.uint8, device=d)
    s = torch.cuda.current_stream(d).cuda_stream
    if pos is None:
        rc = lib.distegnn_build_csr(ptr(eid), N, E, ptr(rowptr), ptr(row), ptr(col), ptr(perm), ptr(ws),
                                    need.value - short, None, s)
    else:
        p = torch.from_numpy(np.ascontiguousarray(pos, F32)).to(d)
        b = None if batch is None else torch.from_numpy(np.ascontiguousarray(batch, np.int64)).to(d)
        rc = lib.distegnn_build_csr_cells(ptr(eid), N, E, ptr(p), ptr(b), B, ptr(rowptr), ptr(row), ptr(col), ptr(perm),
                                          ptr(ws), need.value - short, None, s)
    torch.cuda.synchronize()
    return rc


# ---- the key widths of the two sorts ---------------------------------------------------------------------------------
SORT_WIDTHS = [(1, 0), (1, 1), (1, 4), (2, 8), (3, 1), (3, 12), (5, 20), (1 << 16, 3), (1 << 16, 1 << 18),
               ((1 << 16) + 1, 1 << 15), ((1 << 16) + 1, (1 << 18) + 4), ((1 << 20) + 1, (1 << 22) + 4),
               ((1 << 24) + 1, (1 << 25) + 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,E", SORT_WIDTHS)
def test_sort_widths(N, E):
    """key_bits(N) bits for the edge sort and key_bits(budget) for the node sort, at and one past powers of two."""
    rng = np.random.default_rng(N + E)
    ei = rng.integers(0, N, (2, E))
    check_builds(ei, N, uniform(rng, N), what=f"N={N} E={E}")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1024, 1025])
def test_node_sort_width_at_a_power_of_two(B):
    """n_graphs · budget = 2048 (keys fill all 11 bits) and 2050 (12 bits)."""
    ei, N, pos, batch, B = pow2_case(B)
    want = check_builds(ei, N, pos, batch, B, f"B={B}")
    assert want["grid"]["budget"] == want["grid"]["ncell"] == 2
    assert key_bits(B * 2) == (11 if B == 1024 else 12)


# ---- edge patterns ---------------------------------------------------------------------------------------------------
def edge_pattern(kind, N, rng):
    if kind == "unsorted":
        return rng.integers(0, N, (2, 4 * N))
    if kind == "reverse_sorted":
        ei = rng.integers(0, N, (2, 4 * N))
        return ei[:, np.argsort(-ei[0], kind="stable")]
    if kind == "duplicates_and_self_loops":
        ei = rng.integers(0, N, (2, N))
        ei[1, ::3] = ei[0, ::3]
        ei = np.repeat(ei, rng.integers(1, 4, N), axis=1)
        return ei[:, rng.permutation(ei.shape[1])]
    if kind == "hub":                                    # 2^20 edges into one row among degree-one rows
        row = np.concatenate([np.full(1 << 20, 777), np.delete(np.arange(N), 777)])
        ei = np.stack([row, rng.integers(0, N, row.size)])
        return ei[:, rng.permutation(row.size)]
    if kind == "isolated":                               # edges only into every third node of the first half
        return np.stack([rng.integers(0, N // 6, 2 * N) * 3, rng.integers(0, N, 2 * N)])
    if kind == "one_destination":
        return np.stack([np.full(3 * N, N - 1), rng.integers(0, N, 3 * N)])
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["unsorted", "reverse_sorted", "duplicates_and_self_loops", "hub", "isolated",
                                  "one_destination"])
def test_edge_patterns(kind):
    N = 50_000
    rng = np.random.default_rng(len(kind))
    check_builds(edge_pattern(kind, N, rng), N, uniform(rng, N), what=kind)


# ---- empty and invalid input -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_empty_inputs():
    e = np.zeros((2, 0), np.int64)
    for N in (0, 1, 1_000):
        got = device_builds(e, N, np.zeros((N, 3), F32))
        for order in ("id", "cells"):
            assert_same(got[order], ref_csr(e, N), f"N={N} E=0 {order} order")
            assert not got[order]["rowptr"].any()
    ei = np.zeros((2, 3), np.int64)
    assert raw_build(ei, 0) == -1                                    # DISTEGNN_EINVAL: edges on an empty node set
    assert raw_build(ei, 0, np.zeros((0, 3), F32)) == -1


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["row", "col", "both"])
def test_out_of_range_ids_are_counted_and_clamped(where):
    """500 edges with ids −1, −7, N, N + 5 or 2^40 are counted into n_invalid once per edge and clamped into [0, N):
    row / col in id order, and in cell order through the rank of the clamped destination."""
    N, E = 3_000, 12_000
    rng = np.random.default_rng(7)
    ei = rng.integers(0, N, (2, E))
    bad_ids = np.array([-1, -7, N, N + 5, 1 << 40])
    sel = rng.choice(E, 500, replace=False)
    for k in ((0,) if where == "row" else (1,) if where == "col" else (0, 1)):
        ei[k, sel] = bad_ids[rng.integers(0, bad_ids.size, sel.size)]
    want = check_builds(ei, N, uniform(rng, N), what=where)
    assert want["n_invalid"] == 500                                  # an edge with both ends out of range counts once


# ---- positions -------------------------------------------------------------------------------------------------------
def position_case(kind, N, rng):
    u = uniform(rng, N)
    if kind == "uniform":
        return u
    if kind == "cluster_and_outlier":
        p = (u * 1e-3).astype(F32)
        p[N // 2] = (3e7, -3e7, 3e7)
        return p
    if kind == "coincident":
        return np.full((N, 3), 0.3, F32)
    if kind == "collinear":
        return np.stack([u[:, 0], np.full(N, 2.0, F32), np.zeros(N, F32)], 1)
    if kind == "flat":
        return np.stack([u[:, 0], u[:, 1], np.full(N, -5.0, F32)], 1)
    if kind == "offset_plus_1e4":
        return (u + F32(1e4)).astype(F32)
    if kind == "offset_minus_1e4":
        return (u - F32(1e4)).astype(F32)
    if kind == "extent_past_flt_max":                 # hi − lo overflows to +inf on x: one slab there
        u[0, 0], u[1, 0] = -3e38, 3e38
        return u
    if kind == "non_finite_rows":
        u[::97, 0], u[5::89, 1], u[7::83, 2] = np.nan, np.inf, -np.inf
        u[11::101] = np.nan
        return u
    if kind == "all_non_finite":
        return np.array([np.nan, np.inf, -np.inf], F32)[rng.integers(0, 3, (N, 3))]
    if kind == "signed_zeros":
        p = np.where(rng.random((N, 3)) < 0.5, F32(-0.0), F32(0.0)).astype(F32)
        p[::3] = u[::3]
        return p
    raise ValueError(kind)


POSITIONS = ["uniform", "cluster_and_outlier", "coincident", "collinear", "flat", "offset_plus_1e4", "offset_minus_1e4",
             "extent_past_flt_max", "non_finite_rows", "all_non_finite", "signed_zeros"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", POSITIONS)
def test_positions(kind):
    N = 6_000
    rng = np.random.default_rng(POSITIONS.index(kind))
    pos = position_case(kind, N, rng)
    want = check_builds(every_node_a_row(rng, N, 3 * N), N, pos, what=kind)
    if kind == "extent_past_flt_max":
        assert np.isinf(want["grid"]["ext"][0]) and want["grid"]["dims"][0] == 1
    if kind in ("coincident", "all_non_finite"):
        assert want["grid"]["ncell"] == 1


@pytest.mark.gpu
def test_positions_on_cell_boundaries():
    """Nodes on which an index computed in float64 or with an FMA would differ get the cell of the fp32 expression."""
    pos, counts = boundary_points()
    N = pos.shape[0]
    check_builds(every_node_a_row(np.random.default_rng(4), N, 3 * N), N, pos, what=f"cell boundaries {counts}")


# ---- graphs ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_graph_with_and_without_batch():
    N = 5_000
    rng = np.random.default_rng(8)
    ei, pos = every_node_a_row(rng, N, 4 * N), uniform(rng, N)
    a = device_builds(ei, N, pos, None, 1)["cells"]
    b = device_builds(ei, N, pos, np.zeros(N, np.int64), 1)["cells"]
    assert_same(a, ref_csr_cells(ei, N, pos, None, 1), "batch=None")
    assert_same(b, a, "all-zero batch")


def graph_case(kind, rng):
    if kind == "three_clouds":
        return three_clouds()
    if kind == "20000_tiny_graphs":
        sizes = rng.integers(1, 6, 20_000)
        batch = np.repeat(np.arange(sizes.size), sizes)
        pos = (uniform(rng, batch.size) + 3 * rng.random((sizes.size, 3))[batch]).astype(F32)
        return graph_local_edges(rng, batch, 3 * batch.size), batch.size, pos, batch, sizes.size
    if kind == "graphs_without_nodes":
        batch = np.repeat([0, 3, 4, 17, 49], [900, 1, 2_000, 300, 1_000])
        return graph_local_edges(rng, batch, 4 * batch.size), batch.size, uniform(rng, batch.size), batch, 60
    if kind == "more_graphs_than_nodes":
        batch = np.sort(rng.integers(0, 5_000, 300))
        return graph_local_edges(rng, batch, 900), 300, uniform(rng, 300), batch, 5_000
    if kind == "batch_out_of_range":
        batch = np.concatenate([[-5, -1], np.sort(rng.integers(0, 7, 2_000)), [7, 12, 1 << 40]])
        N = batch.size
        return every_node_a_row(rng, N, 3 * N), N, uniform(rng, N), batch, 7
    if kind == "2^30+3_graphs":
        return huge_graph_count_case()
    raise ValueError(kind)


GRAPHS = ["three_clouds", "20000_tiny_graphs", "graphs_without_nodes", "more_graphs_than_nodes", "batch_out_of_range",
          "2^30+3_graphs"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", GRAPHS)
def test_graph_batches(kind):
    ei, N, pos, batch, B = graph_case(kind, np.random.default_rng(GRAPHS.index(kind)))
    want = check_builds(ei, N, pos, batch, B, kind)
    check_design_invariants(want, ei, N, np.clip(batch, 0, B - 1))


# ---- repeatability and workspace -------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_repeatable_on_a_side_stream_and_workspace_size():
    """The same bits from a second build on a side stream after unrelated work; distegnn_csr_workspace_bytes suffices
    (every build here runs with exactly that many bytes), one byte less is DISTEGNN_EWORKSPACE."""
    N = (1 << 20) + 1
    rng = np.random.default_rng(9)
    ei, pos = rng.integers(0, N, (2, 4 * N)), uniform(rng, N)
    first = device_builds(ei, N, pos)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        x = torch.randn(4096, 4096, device=dev())
        for _ in range(8):
            x = torch.tanh(x @ x)
        second = device_builds(ei, N, pos)
    torch.cuda.synchronize()
    for order in ("id", "cells"):
        assert_same(second[order], first[order], f"side stream, {order} order")
    assert_same(first["cells"], ref_csr_cells(ei, N, pos, None, 1), "cell order")
    for p in (None, pos):
        assert raw_build(ei, N, p) == 0
        assert raw_build(ei, N, p, short=1) == -3                   # DISTEGNN_EWORKSPACE


# ---- gather_rows / scatter_rows --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("width", [1, 2, 3, 4, 5, 6, 7, 8, 64])
def test_gather_scatter_rows(width):
    from distegnn_b200.backend import CudaBackend
    be, d = CudaBackend(), dev()
    g = torch.Generator(device=d).manual_seed(width)
    for n in (0, 1, 2, 300_007):
        src = torch.randn(n, width, device=d, generator=g)
        perm = torch.randperm(n, device=d, generator=g).to(torch.int32)
        got = be.gather_rows(src, perm)
        assert torch.equal(got, src[perm.long()]), (n, width)
        assert torch.equal(be.gather_rows(got, perm, inverse=True), src), (n, width)       # scatter ∘ gather = identity
        want = torch.empty_like(src)
        want[perm.long()] = src
        assert torch.equal(be.gather_rows(src, perm, inverse=True), want), (n, width)
    from distegnn_b200 import _lib
    lib = _lib.load()
    assert lib.distegnn_gather_rows(None, None, 0, width, None, None) == 0     # nothing to move: no pointer is read
    assert lib.distegnn_scatter_rows(None, None, 0, width, None, None) == 0


@pytest.mark.gpu
def test_gather_scatter_rows_past_2_31_elements():
    """n_rows · width = 2^31 + 192 elements (8.6 GB a tensor, 26 GB in all): the element index needs 64 bits."""
    from distegnn_b200.backend import CudaBackend
    be, d = CudaBackend(), dev()
    n, w = (1 << 25) + 3, 64
    g = torch.Generator(device=d).manual_seed(10)
    src = torch.randn(n, w, device=d, generator=g)
    perm = torch.randperm(n, device=d, generator=g).to(torch.int32)
    dst = be.gather_rows(src, perm)
    step = 1 << 22
    for a in range(0, n, step):
        assert torch.equal(dst[a:a + step], src[perm[a:a + step].long()]), a
    back = be.gather_rows(dst, perm, inverse=True)
    del dst
    for a in range(0, n, step):
        assert torch.equal(back[a:a + step], src[a:a + step]), a


# ======================================================================================================================
# GPU: one training step through the cell order, at scale
# ======================================================================================================================
def many_graphs_batch(seed=12):
    """2,000 graphs of 1..60 nodes and, in the middle, one of 20,000 (fluid113k density); edge_index shuffled."""
    from distegnn_b200 import synth
    w = synth.WORKLOADS["fluid113k"]
    rng = np.random.default_rng(seed)
    big = synth.make_partitions(w, n_nodes=20_000, seed=seed)[0]
    parts, off = [], 0
    sizes = list(rng.integers(1, 61, 2_000))
    sizes.insert(1_000, big["node_loc"].shape[0])
    for b, n in enumerate(sizes):
        if b == 1_000:
            pos, ei = big["node_loc"].numpy(), big["edge_index"].numpy()
        else:
            pos = (rng.random((n, 3)) * synth.box_side(n, w.radius, 8.0) + rng.random(3) * 4).astype(F32)
            ei = synth.radius_graph_np(pos, w.radius) if n > 1 else np.zeros((2, 0), np.int64)
        parts.append((pos, ei + off))
        off += n
    pos = np.concatenate([p for p, _ in parts])
    ei = np.concatenate([e for _, e in parts], 1)
    ei = ei[:, rng.permutation(ei.shape[1])]
    N, B = pos.shape[0], len(sizes)
    batch = np.repeat(np.arange(B), sizes)
    d = np.sqrt(((pos[ei[0]] - pos[ei[1]]) ** 2).sum(-1, dtype=np.float32))
    loc_mean = np.add.reduceat(pos.astype(np.float64), np.cumsum([0] + sizes[:-1])) / np.array(sizes)[:, None]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    inp = dict(node_feat=t(rng.normal(size=(N, w.node_feat_nf)).astype(F32)), node_loc=t(pos),
               node_vel=t((rng.normal(size=(N, 3)) * 0.01).astype(F32)), loc_mean=t(loc_mean.astype(F32)),
               edge_index=t(ei), data_batch=t(batch), edge_attr=t(np.repeat(d[:, None], w.edge_attr_nf, 1)),
               node_attr=t(rng.normal(size=(N, w.node_attr_nf)).astype(F32)))
    return w, inp


@pytest.mark.gpu
def test_training_step_through_the_cell_order_at_scale():
    """Parameter and input gradients (model.input_grads) of a training step whose graph the model caches in cell order,
    against float64 autograd of the oracle, with the gates of the training-path and input-gradient tests.  g_edge_attr
    comes back in the caller's shuffled edge order through scatter_rows; the same step on the graph passed as an
    id-order CSRGraph is printed next to it."""
    from distegnn_b200 import FastEGNN
    from distegnn_b200.shards import CSRGraph
    from oracle import fastegnn_oracle as orc
    from tests.test_gpu_parity import _param_grad_errors
    from tests.test_input_grads import INPUTS, _rel, leaves
    w, host = many_graphs_batch()
    d = dev()
    N, B, E = host["node_loc"].shape[0], host["loc_mean"].shape[0], host["edge_index"].shape[1]
    F, Na, A, Cv = w.node_feat_nf, w.node_attr_nf, w.edge_attr_nf, w.virtual_channels
    sd = orc.init_state_dict(F, Na, A, 64, Cv, 3, seed=12, coord_gain=0.05)
    g = torch.Generator().manual_seed(13)
    cot, cotX = torch.randn(N, 3, generator=g).to(d), torch.randn(B, 3, Cv, generator=g).to(d)
    # float64 autograd through the oracle (on the device: the same ops, in float64)
    sd64 = {k: v.to(d, torch.float64).requires_grad_(True) for k, v in sd.items()}
    in64 = leaves(host, dtype=torch.float64, device=d)
    o64, X64 = orc.forward(sd64, **in64)
    keys = list(sd64)
    leaves64 = [sd64[k] for k in keys] + [in64[k] for k in INPUTS]
    gr = torch.autograd.grad((o64 * cot.double()).sum() + (X64 * cotX.double()).sum(), leaves64, allow_unused=True)
    ref_p = {k: (v if v is not None else torch.zeros_like(sd64[k])).cpu() for k, v in zip(keys, gr)}
    ref_in = dict(zip(INPUTS, gr[len(keys):]))
    del o64, X64, gr, in64, leaves64

    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=Cv,
                 n_layers=3)
    m.load_state_dict(sd)
    m.input_grads = True
    m = m.to(d).train()

    def step(inp):
        m.zero_grad()
        inp = leaves(inp)
        out, X = m(**inp)
        ((out * cot).sum() + (X * cotX).sum()).backward()
        gp = {k: (torch.zeros_like(p) if p.grad is None else p.grad.clone()) for k, p in m.named_parameters()}
        return gp, {k: inp[k].grad for k in INPUTS}

    dh = {k: v.to(d) for k, v in host.items()}
    gp, gi = step(dh)
    rows = [e[3][1] for k, e in m._graphs.entries.items() if k[1] and e[0] is dh["edge_index"]]
    assert len(rows) == 1 and not bool((rows[0][1:] >= rows[0][:-1]).all()), "the cached graph is not in cell order"
    errs, dead = _param_grad_errors(m, ref_p)
    worst = max(errs, key=errs.get)
    ierr = {k: _rel(gi[k], ref_in[k]) for k in INPUTS if float(ref_in[k].abs().max()) > 0}
    iworst = max(ierr, key=ierr.get)
    print(f"N={N} B={B} E={E}: parameter gradients vs oracle fp64: worst {worst} {errs[worst]:.2e} (gate 5e-4), "
          f"{dead} dead; input gradients: " + ", ".join(f"{k} {v:.1e}" for k, v in ierr.items()) + " (gate 5e-4)")
    assert errs[worst] <= 5e-4 and ierr[iworst] <= 5e-4
    # the same graph as an id-order CSRGraph: g_edge_attr in its CSR order
    csr, ea = CSRGraph.from_edge_index(dh["edge_index"], N, dh["edge_attr"].detach())
    cp, ci = step(dict(dh, edge_index=csr, edge_attr=ea))
    order = torch.argsort(dh["edge_index"][0], stable=True)
    ci["edge_attr"] = torch.empty_like(ci["edge_attr"]).index_copy_(0, order, ci["edge_attr"])
    dp = max(_rel(cp[k], gp[k]) for k in gp if float(gp[k].abs().max()) > 0)
    di = {k: _rel(ci[k], gi[k]) for k in ierr}
    print("cell order vs id-order CSRGraph: parameters " + f"{dp:.1e}, inputs "
          + ", ".join(f"{k} {v:.1e}" for k, v in di.items()))
