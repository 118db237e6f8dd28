"""The radius-graph builder (DESIGN §10) against a float64 brute force, through both of its outputs:
`partition.radius_graph_csr` (csrc/radius_csr.cu, a CSRGraph) and `partition.radius_graph` (the int64 edge_index over it).

The reference classifies every same-graph pair of the fp32 positions in float64 against r2 = fp32(r·r): required if
d² < r2·(1 − 2^-20), forbidden if d² ≥ r2·(1 + 2^-20), either way in between; a node with a non-finite coordinate has
no edges.  Every build is checked for no duplicates, exact mirror symmetry, ascending rows under a monotone rowptr that
ends at the count, edge_attr columns equal to each other and to the float64 length within 3e-7 relative, and
`CSRGraph.validate()`.

CPU: the grid sizing through the testing library (every key inside the cell table for normal, huge, infinite and NaN
extents) and the fp32 emulation of the cell index that constructs pairs closer than r two cells apart when the cell is
exactly r.  GPU: far from the grid origin, lattices at the boundary, degenerate boxes, grid growth, capacity mode,
determinism, non-finite and extreme positions, the edge cutoff and a rollout step on top."""
import ctypes as C

import numpy as np
import pytest
import torch

F32 = np.float32
MARGIN = F32(1.0) + F32(2.0 ** -10)        # the first cell edge is fp32(r) * MARGIN (csrc/radius_grid.cuh)
DEFAULT_TABLE = 1 << 22


def dev():
    return torch.device("cuda")


# ---- fp32 emulation of the builders' cell index -------------------------------------------------------------------------
def _f2ord(x):
    i = np.asarray(x, dtype=np.float32).view(np.int32).astype(np.int64)
    return np.where(i >= 0, i, i ^ 0x7FFFFFFF)


def _ord2f(o):
    o = np.asarray(o, dtype=np.int64)
    return np.where(o >= 0, o, o ^ 0x7FFFFFFF).astype(np.int32).view(np.float32)


def cell_index(x, lo, cell):
    """⌊fl(fl(x − lo) · fl(1/cell))⌋, the kernels' fp32 expression (unclamped)."""
    q = (np.asarray(x, dtype=np.float32) - F32(lo)) * (F32(1.0) / F32(cell))
    return np.floor(q).astype(np.int64)


def straddling_pairs(lo, r, n_cells, cell):
    """Axis-aligned pairs (x1, x2) with fp32 (x2 − x1)² < fp32(r·r), float64-required (d² < r2·(1 − 2^-20)), whose cell
    indices under `cell` differ by two: x1 = the last fp32 value of cell k − 1, x2 = the first of cell k + 1."""
    k = np.arange(1, n_cells, dtype=np.int64)
    a = np.full(k.shape, _f2ord(F32(lo)))
    b = np.full(k.shape, _f2ord(F32(float(lo) + (n_cells + 2) * float(cell))))
    while (b - a > 1).any():                      # bisection on the fp32 order: b = first value with index >= k
        m = (a + b) // 2
        ok = cell_index(_ord2f(m), lo, cell) >= k
        b, a = np.where(ok, m, b), np.where(ok, a, m)
    first = _ord2f(b)
    x1, x2 = _ord2f(_f2ord(first[:-1]) - 1), first[1:]
    r2 = F32(r) * F32(r)
    dd = x2 - x1
    sel = (dd * dd < r2) & (cell_index(x2, lo, cell) - cell_index(x1, lo, cell) >= 2)
    x1, x2 = x1[sel], x2[sel]
    req = (x2.astype(np.float64) - x1.astype(np.float64)) ** 2 < float(r2) * (1 - 2.0 ** -20)
    return x1[req], x2[req]


def far_corner_cloud(r, axis, n=3000, seed=0):
    """A slab 1000 cells long on `axis` (2 cells across the others) whose lower corner lies 970 cells below the coordinate
    origin, a random cloud in it, and the pairs the fp32 cell index of a cell of exactly r puts two cells apart
    (they exist where a node is nearer the coordinate origin than the grid corner)."""
    rng = np.random.default_rng(seed)
    r32 = F32(r)
    lo = F32(-970.0 * float(r32))
    length = F32(1000.0 * float(r32))
    x1, x2 = straddling_pairs(lo, r, 1001, r32)
    width = 2.0 * float(r32)
    pts = rng.uniform(0.0, width, size=(n, 3))
    pts[:, axis] = rng.uniform(float(lo), float(lo) + float(length), size=n)
    pairs = rng.uniform(0.0, width, size=(2 * len(x1), 3))
    pairs[1::2] = pairs[0::2]                      # same off-axis coordinates: axis-aligned pairs
    pairs[0::2, axis], pairs[1::2, axis] = x1, x2
    corners = np.zeros((2, 3))
    corners[:, axis] = [float(lo), float(lo) + float(length)]
    corners[1, [a for a in range(3) if a != axis]] = width
    pos = np.concatenate([corners, pairs, pts]).astype(np.float32)      # pair k = nodes 2 + 2k and 3 + 2k
    assert pos[:, axis].min() == lo
    return pos, len(x1)


# ---- float64 brute force ------------------------------------------------------------------------------------------------
def reference(pos, batch, r, loop):
    """(required, possible) edge keys i·N + j, sorted int64: required = d² < r2·(1 − 2^-20), possible = required or in
    the band below r2·(1 + 2^-20).  `batch` sorted (or None); pairs of one graph only; non-finite nodes get nothing."""
    pos = np.asarray(pos, dtype=np.float32)
    N = pos.shape[0]
    batch = np.zeros(N, dtype=np.int64) if batch is None else np.asarray(batch, dtype=np.int64)
    assert (np.diff(batch) >= 0).all()
    p = pos.astype(np.float64)
    finite = np.isfinite(p).all(axis=1)
    r2 = float(F32(r) * F32(r))
    lo_t, hi_t = r2 * (1 - 2.0 ** -20), r2 * (1 + 2.0 ** -20)
    max_size = int(np.bincount(batch).max())
    req, pos_ = [], []
    ids = np.arange(N, dtype=np.int64)
    for k in range(1, max_size):                   # i and i + k of one graph (sorted batch)
        i, j = ids[:-k], ids[k:]
        m = (batch[i] == batch[j]) & finite[i] & finite[j]
        i, j = i[m], j[m]
        d2 = ((p[i] - p[j]) ** 2).sum(axis=1)
        for sel, out in ((d2 < lo_t, req), (d2 < hi_t, pos_)):
            out += [i[sel] * N + j[sel], j[sel] * N + i[sel]]
    if loop:
        self_keys = ids[finite] * N + ids[finite]
        req.append(self_keys)
        pos_.append(self_keys)
    cat = lambda xs: np.sort(np.concatenate(xs)) if xs else np.zeros(0, dtype=np.int64)
    return cat(req), cat(pos_)


def check_graph(g, ea, pos, batch, r, loop):
    """The invariants of the module docstring; returns the edge keys (i·N + j, CSR order)."""
    pos = np.asarray(pos, dtype=np.float32)
    N = pos.shape[0]
    E = int(g.n_edges_dev.item()) if g.n_edges_dev is not None else g.num_edges
    rowptr = g.rowptr.cpu().numpy().astype(np.int64)
    assert rowptr.shape == (N + 1,) and rowptr[0] == 0 and rowptr[-1] == E, (rowptr[0], rowptr[-1], E)
    assert (np.diff(rowptr) >= 0).all(), "rowptr not monotone"
    row = g.rows()[:E].cpu().numpy().astype(np.int64)
    col = g.col[:E].cpu().numpy().astype(np.int64)
    assert np.array_equal(row, np.repeat(np.arange(N), np.diff(rowptr))), "rows not ascending / not as rowptr says"
    assert ((col >= 0) & (col < N)).all()
    keys = row * N + col
    skeys = np.sort(keys)
    assert (np.diff(skeys) > 0).all(), "duplicate edges"
    assert np.array_equal(skeys, np.sort(col * N + row)), "not mirror-symmetric"
    req, possible = reference(pos, batch, r, loop)
    missing = np.setdiff1d(req, skeys, assume_unique=True)
    extra = np.setdiff1d(skeys, possible, assume_unique=True)
    assert missing.size == 0, f"{missing.size} required edges missing, e.g. {[divmod(int(k), N) for k in missing[:4]]}"
    assert extra.size == 0, f"{extra.size} forbidden edges, e.g. {[divmod(int(k), N) for k in extra[:4]]}"
    if ea is not None and E:
        a = ea[:E].cpu().numpy()
        assert (a == a[:, :1]).all(), "edge_attr columns differ"
        d = np.sqrt(((pos[row].astype(np.float64) - pos[col].astype(np.float64)) ** 2).sum(axis=1))
        assert (np.abs(a[:, 0].astype(np.float64) - d) <= 3e-7 * d).all(), "edge_attr is not the edge length"
    g.validate(g.rowptr.device)
    return keys


# ---- the two outputs -----------------------------------------------------------------------------------------------------
def build_csr(pos, batch, r, loop=False, n_graphs=None, **kw):
    from distegnn_b200.partition import radius_graph_csr
    pd = torch.from_numpy(np.ascontiguousarray(pos, dtype=np.float32)).to(dev())
    bd = None if batch is None else torch.from_numpy(np.asarray(batch, dtype=np.int64)).to(dev())
    return radius_graph_csr(pd, r, bd, loop=loop, n_graphs=n_graphs, **kw)


def build_coo(pos, batch, r, loop=False):
    from distegnn_b200 import radius_graph
    from distegnn_b200.shards import CSRGraph
    pd = torch.from_numpy(np.ascontiguousarray(pos, dtype=np.float32)).to(dev())
    bd = None if batch is None else torch.from_numpy(np.asarray(batch, dtype=np.int64)).to(dev())
    ei, ea = radius_graph(pd, r, bd, loop=loop, max_num_neighbors=pd.shape[0])
    N = pd.shape[0]
    rowptr = torch.zeros(N + 1, dtype=torch.int32, device=dev())
    rowptr[1:] = torch.cumsum(torch.bincount(ei[0], minlength=N), 0).to(torch.int32)
    return CSRGraph(rowptr, ei[1].to(torch.int32).contiguous(), ei[0].to(torch.int32).contiguous()), ea


BUILDERS = {"csr": build_csr, "coo": build_coo}


def check_both(pos, batch, r, loop=False, builders=("csr", "coo")):
    for name in builders:
        g, ea = BUILDERS[name](pos, batch, r, loop)
        check_graph(g, ea, pos, batch, r, loop)


# ---- CPU: grid sizing through the testing library -----------------------------------------------------------------------
def _grid_size(ext, r, B, table):
    """distegnn_radius_grid_size (include/distegnn_b200_testing_grid.h) -> (cell, dims, ncell)."""
    from tests import twin_backend
    fn = twin_backend.load_testing().distegnn_radius_grid_size
    fn.argtypes = [C.c_void_p, C.c_float, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    fn.restype = C.c_int
    cell, dims, ncell = C.c_float(0), (C.c_int32 * 3)(), C.c_int64(0)
    e = (C.c_float * 3)(*ext)
    twin_backend.check(fn(C.addressof(e), float(r), int(B), int(table), C.addressof(cell), C.addressof(dims),
                          C.addressof(ncell)), "radius_grid_size")
    return cell.value, list(dims), ncell.value


INF, NAN, FLT_MAX = float("inf"), float("nan"), float(np.finfo(np.float32).max)
EXTENTS = [(1.0, 1.0, 1.0), (0.0, 0.0, 0.0), (30.0, 0.1, 0.1), (1e3, 1e3, 1e3), (1e4, 0.0, 2.0), (3e38, 3e38, 3e38),
           (3e38, 0.0, 0.0), (INF, 1.0, 1.0), (INF, INF, INF), (-INF, -INF, -INF), (NAN, 1.0, 2.0), (NAN, NAN, NAN),
           (1.0, -INF, NAN), (3.4028235e38, 1e-30, 7.0)]


@pytest.mark.parametrize("ext", EXTENTS)
def test_grid_size_keeps_every_key_inside_the_table(ext):
    """For any extent, radius, graph count and table: dims in [1, 1024], n_graphs·Πdims + 1 <= table_cells, and the cell
    at least r·(1 + 2^-10) (the margin) unless one cell per graph covers everything."""
    for r in (1e-38, 1e-6, 0.035, 0.075, 1.0, 1e30):
        for B, table in ((1, 27), (5, 27), (26, 27), (3, 64), (1, DEFAULT_TABLE), (20_000, DEFAULT_TABLE),
                         (DEFAULT_TABLE - 1, DEFAULT_TABLE), (7, (1 << 30) - 1)):
            cell, dims, ncell = _grid_size(ext, r, B, table)
            assert all(1 <= d <= 1024 for d in dims), (ext, r, B, table, dims)
            assert ncell == dims[0] * dims[1] * dims[2] and B * ncell + 1 <= table, (ext, r, B, table, dims)
            assert np.isfinite(cell) and cell > 0
            if ncell > 1:
                assert F32(cell) >= F32(r) * MARGIN, (ext, r, cell)
            for e, d in zip(ext, dims):                 # the grid covers the extent: nothing relies on clamping
                if np.isfinite(e) and e >= 0 and d > 1:
                    assert e / cell < d + 1e-3


def test_grid_size_first_cell_carries_the_margin_and_grows_by_half():
    r = 0.075
    cell, dims, _ = _grid_size((1.0, 1.0, 1.0), r, 1, DEFAULT_TABLE)
    assert F32(cell) == F32(r) * MARGIN and dims == [14, 14, 14]
    cell, dims, _ = _grid_size((100.0, 100.0, 100.0), r, 1, DEFAULT_TABLE)      # 1334 cells per axis: grows
    assert cell > 1.4 * r and all(d <= 1024 for d in dims)
    # r tiny against 3e38: the old 200 steps of growth ended at ~1e29 with 10^9 cells; now the growth goes on
    cell, dims, _ = _grid_size((3e38, 1.0, 1.0), 1e-6, 5, DEFAULT_TABLE)
    assert dims[1:] == [1, 1] and 600 < dims[0] <= 1024 and 3e38 / 1024 <= cell <= FLT_MAX
    # FLT_MAX on every axis and too many graphs for 2 cells per axis: the growth overflows fp32 -> one cell per graph
    assert _grid_size((FLT_MAX,) * 3, 1.0, 600_000, DEFAULT_TABLE)[1:] == ([1, 1, 1], 1)


def test_grid_size_rejects_what_no_grid_can_hold():
    for ext, r, B, table in (((1.0, 1.0, 1.0), 0.1, 27, 27), ((1.0, 1.0, 1.0), 0.0, 1, 27),
                             ((1.0, 1.0, 1.0), NAN, 1, 27), ((1.0, 1.0, 1.0), 0.1, 1, 26)):
        with pytest.raises(ValueError):
            _grid_size(ext, r, B, table)


# ---- CPU: the emulation behind the far-from-origin cases ----------------------------------------------------------------
@pytest.mark.parametrize("r", [0.035, 0.075, 0.1, 0.3])
def test_emulated_cell_of_exactly_r_splits_pairs_and_the_margin_does_not(r):
    """With a cell of exactly r the fp32 index puts pairs closer than r two cells apart (the builders missed them); with
    the cell r·(1 + 2^-10) no pair is split, neither the constructed ones nor any the same search finds."""
    for axis in range(3):
        pos, n_pairs = far_corner_cloud(r, axis, n=10)
        assert n_pairs > 0
        lo = pos[:, axis].min()
        x1, x2 = pos[2:2 + 2 * n_pairs:2, axis], pos[3:3 + 2 * n_pairs:2, axis]
        assert (cell_index(x2, lo, F32(r)) - cell_index(x1, lo, F32(r)) == 2).all()
        fixed = F32(r) * MARGIN
        assert (cell_index(x2, lo, fixed) - cell_index(x1, lo, fixed) <= 1).all()
        assert len(straddling_pairs(lo, r, 1001, fixed)[0]) == 0


# ---- GPU: 1. far from the grid origin -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("builder", ["csr", "coo"])
@pytest.mark.parametrize("r", [0.035, 0.075, 0.1, 0.3])
def test_no_missed_edges_far_from_the_grid_origin(builder, r):
    """Pairs closer than r that a cell of exactly r splits over two cells are found, on every axis."""
    for axis in range(3):
        pos, n_pairs = far_corner_cloud(r, axis, seed=axis)
        assert n_pairs > 0
        g, ea = BUILDERS[builder](pos, None, r)
        keys = check_graph(g, ea, pos, None, r, False)
        N = pos.shape[0]
        i = np.arange(2, 2 + 2 * n_pairs, 2)
        assert np.isin(i * N + i + 1, keys).all()


@pytest.mark.gpu
@pytest.mark.parametrize("builder", ["csr", "coo"])
@pytest.mark.parametrize("offset", [1e3, -1e3, 1e4, -1e4])
def test_clouds_at_large_offsets(builder, offset):
    """Random clouds 1000 cells long at coordinates ±1e3 and ±1e4, where the fp32 spacing of the coordinates (up to 1e-3)
    is a sizeable part of r: every pair near r is classified as in float64."""
    rng = np.random.default_rng(int(abs(offset)) + (offset < 0))
    for r in (0.035, 0.075, 0.1, 0.3):
        pos = (rng.uniform(0.0, 1.0, size=(4000, 3)) * np.array([1000 * r, 3 * r, 3 * r]) + offset).astype(np.float32)
        g, ea = BUILDERS[builder](pos, None, r)
        check_graph(g, ea, pos, None, r, False)


# ---- GPU: 2. lattices at the boundary -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("builder", ["csr", "coo"])
@pytest.mark.parametrize("s,offset", [(0.125, 0.0), (0.1015625, 1e3), (0.03515625, -1e4), (0.375, 1e4)])
def test_lattice_at_spacing_r_and_just_below(builder, s, offset):
    """A 10³ lattice of exact fp32 spacing s at an offset: with r = s the neighbours at d = r are absent (strict), with
    r = nextafter(s, inf) (so that d = nextafter(r, 0)) every node has exactly its axis neighbours."""
    idx = np.stack(np.meshgrid(*[np.arange(10)] * 3, indexing="ij"), -1).reshape(-1, 3)
    pos = (offset + idx * s).astype(np.float32)
    assert np.array_equal(pos.astype(np.float64), offset + idx * s), "lattice not exact in fp32"
    g, ea = BUILDERS[builder](pos, None, float(F32(s)))
    assert check_graph(g, ea, pos, None, float(F32(s)), False).size == 0
    r_up = float(np.nextafter(F32(s), F32(np.inf)))
    g, ea = BUILDERS[builder](pos, None, r_up)
    keys = check_graph(g, ea, pos, None, r_up, False)
    deg = np.diff(g.rowptr.cpu().numpy())
    want = ((idx > 0).astype(int) + (idx < 9).astype(int)).sum(axis=1)
    assert keys.size == want.sum() and np.array_equal(deg, want)


# ---- GPU: 3. degenerate boxes -------------------------------------------------------------------------------------------
def _degenerate(kind, rng):
    if kind == "coincident":
        return np.full((1500, 3), [0.3, -2.0, 7.5], dtype=np.float32)
    if kind == "collinear":
        t = rng.uniform(0, 3, size=(3000, 1))
        return (np.array([1.0, -2.0, 0.5]) + t * np.array([0.48, 0.6, 0.64])).astype(np.float32)
    if kind == "coplanar":
        uv = rng.uniform(0, 2, size=(3000, 2))
        return (uv[:, :1] * np.array([0.6, 0.8, 0.0]) + uv[:, 1:] * np.array([0.0, 0.6, 0.8]) + 5.0).astype(np.float32)
    if kind == "flat_z":
        p = rng.uniform(0, 2, size=(3000, 3))
        p[:, 2] = -1.25
        return p.astype(np.float32)
    if kind == "line_x":
        p = np.zeros((3000, 3))
        p[:, 0] = rng.uniform(-4, 4, size=3000)
        p[:, 1:] = [0.5, 100.0]
        return p.astype(np.float32)
    if kind == "duplicates":
        p = rng.uniform(0, 1, size=(1500, 3))
        return np.repeat(p, 2, axis=0).astype(np.float32)
    raise KeyError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("loop", [False, True])
@pytest.mark.parametrize("kind", ["coincident", "collinear", "coplanar", "flat_z", "line_x", "duplicates"])
def test_degenerate_boxes(kind, loop):
    rng = np.random.default_rng(11)
    pos = _degenerate(kind, rng)
    check_both(pos, None, 0.1, loop)
    batch = np.sort(rng.integers(0, 3, size=pos.shape[0]))
    check_both(pos, batch, 0.1, loop)


# ---- GPU: 4. grid growth ------------------------------------------------------------------------------------------------
def _close_pairs(rng, n, box, d):
    p = rng.uniform(0, box, size=(n, 3))
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return np.concatenate([p, p + d * u]).astype(np.float32)


@pytest.mark.gpu
def test_radius_tiny_against_the_extent():
    """More than 1024 cells per axis at cell = r: the cell grows, pairs well below r and right at it are still found."""
    rng = np.random.default_rng(1)
    r = 1e-3
    pos = np.concatenate([rng.uniform(0, 10, size=(3000, 3)).astype(np.float32),
                          _close_pairs(rng, 500, 10.0, 0.7 * r), _close_pairs(rng, 500, 10.0, r * (1 - 1e-6))])
    check_both(pos, None, r)


@pytest.mark.gpu
@pytest.mark.parametrize("table,B", [(27, 5), (27, 26), (64, 3), (64, 21)])
def test_small_tables_with_several_graphs(table, B):
    rng = np.random.default_rng(table + B)
    pos = rng.uniform(0, 2, size=(3000, 3)).astype(np.float32)
    batch = np.sort(rng.integers(0, B, size=3000))
    batch[0], batch[-1] = 0, B - 1
    g, ea = build_csr(pos, batch, 0.2, n_graphs=B, table_cells=table)
    check_graph(g, ea, pos, batch, 0.2, False)
    gc, eac = build_csr(pos, batch, 0.2, n_graphs=B, table_cells=table, capacity=g.num_edges + 1)
    assert int(gc.info[2].item()) + 1 <= table                         # cells used
    assert torch.equal(gc.rowptr, g.rowptr) and torch.equal(gc.col[:g.num_edges], g.col)


@pytest.mark.gpu
def test_twenty_thousand_tiny_graphs():
    """20k graphs of 1-3 nodes sharing one box: edges only inside a graph, on the default table."""
    rng = np.random.default_rng(2)
    sizes = rng.integers(1, 4, size=20_000)
    batch = np.repeat(np.arange(20_000), sizes)
    pos = rng.uniform(0, 1, size=(batch.size, 3)).astype(np.float32)
    for loop in (False, True):
        g, ea = build_csr(pos, batch, 0.6, loop, n_graphs=20_000)
        check_graph(g, ea, pos, batch, 0.6, loop)
    check_both(pos, batch, 0.6, False, builders=("coo",))


@pytest.mark.gpu
def test_graph_ids_without_nodes():
    """Empty graph ids in the middle and at the end (n_graphs > max id + 1)."""
    rng = np.random.default_rng(3)
    batch = np.sort(rng.choice([0, 1, 3, 4], size=2000))
    pos = rng.uniform(0, 1, size=(2000, 3)).astype(np.float32)
    for n_graphs in (5, 9, 64):
        g, ea = build_csr(pos, batch, 0.15, n_graphs=n_graphs)
        check_graph(g, ea, pos, batch, 0.15, False)
    check_both(pos, batch, 0.15, False, builders=("coo",))


@pytest.mark.gpu
@pytest.mark.parametrize("outlier", [1e3, -1e6, 3e7])
def test_one_far_outlier(outlier):
    rng = np.random.default_rng(4)
    pos = rng.uniform(0, 1, size=(3000, 3)).astype(np.float32)
    pos[1234] = [outlier, 0.5, -outlier]
    pos[1235] = pos[1234] + [0.05, 0.0, 0.0]                           # the outlier has a neighbour out there
    check_both(pos, None, 0.08)


# ---- GPU: 5. capacity mode ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_capacity_below_at_and_count_only():
    rng = np.random.default_rng(5)
    B = 3
    pos = rng.uniform(0, 1.5, size=(4000, 3)).astype(np.float32)
    batch = np.sort(rng.integers(0, B, size=4000))
    g, ea = build_csr(pos, batch, 0.1, n_graphs=B)
    check_graph(g, ea, pos, batch, 0.1, False)
    E = g.num_edges
    assert E > 1000
    small, ea_s = build_csr(pos, batch, 0.1, n_graphs=B, capacity=E // 3)
    info = small.info.tolist()
    assert info[0] == E and info[1] == 1 and small.overflowed()
    assert torch.equal(small.rowptr, g.rowptr)
    cap = E // 3
    assert torch.equal(small.col, g.col[:cap]) and torch.equal(small.row, g.rows()[:cap])
    assert torch.equal(ea_s, ea[:cap])
    exact, ea_e = build_csr(pos, batch, 0.1, n_graphs=B, capacity=E)
    assert exact.info.tolist()[:2] == [E, 0] and not exact.overflowed()
    assert torch.equal(exact.rowptr, g.rowptr) and torch.equal(exact.col, g.col) and torch.equal(ea_e, ea)
    count, ea_c = build_csr(pos, batch, 0.1, n_graphs=B, capacity=0)   # count-only: rowptr and the count, no edges
    assert count.num_edges == 0 and int(count.info[0].item()) == E and torch.equal(count.rowptr, g.rowptr)


# ---- GPU: 6. determinism ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_builds_are_bitwise_equal_even_after_other_work():
    """`differentiable_rollout` rebuilds each step's graph in the backward and relies on getting the same one."""
    from distegnn_b200.partition import RadiusGraphBuffers, radius_graph_csr
    rng = np.random.default_rng(6)
    pos = torch.from_numpy(rng.uniform(-3, 3, size=(12_000, 3)).astype(np.float32)).to(dev())
    batch = torch.from_numpy(np.sort(rng.integers(0, 4, size=12_000))).to(dev())
    g0, _ = radius_graph_csr(pos, 0.2, batch, n_graphs=4)
    cap = g0.num_edges + 64
    outs = []
    side = torch.cuda.Stream()
    for k in range(2):
        if k:
            with torch.cuda.stream(side):                              # unrelated work on another stream
                a = torch.randn(2048, 2048, device=dev())
                for _ in range(8):
                    a = torch.tanh(a @ a * 1e-3)
        buf = RadiusGraphBuffers(12_000, cap, 2, dev())
        radius_graph_csr(pos, 0.2, batch, n_graphs=4, out=buf)
        outs.append(buf)
    torch.cuda.synchronize()
    a, b = outs
    E = int(a.info[0])
    assert 0 < E <= cap and not a.graph.overflowed()
    for name in ("rowptr", "info", "col", "row", "edge_attr"):          # the edge buffers past the count are unused
        x, y = getattr(a, name), getattr(b, name)
        if name not in ("rowptr", "info"):
            x, y = x[:E], y[:E]
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), name
    check_graph(a.graph, a.edge_attr, pos.cpu().numpy(), batch.cpu().numpy(), 0.2, False)


# ---- GPU: 7. non-finite and extreme positions ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_non_finite_nodes_get_no_edges_and_the_rest_are_exact():
    rng = np.random.default_rng(7)
    B, N = 6, 3000
    pos = rng.uniform(0, 1, size=(N, 3)).astype(np.float32)
    batch = np.sort(rng.integers(0, B, size=N))
    bad = rng.choice(N, size=60, replace=False)
    for k, v in enumerate((np.inf, -np.inf, np.nan)):
        pos[bad[k::3], k] = v
    pos[bad[:5]] = np.nan                                              # all three coordinates
    for loop in (False, True):
        g, ea = build_csr(pos, batch, 0.12, loop, n_graphs=B)
        check_graph(g, ea, pos, batch, 0.12, loop)
        deg = np.diff(g.rowptr.cpu().numpy())
        assert (deg[bad] == 0).all()
        gc, _ = build_csr(pos, batch, 0.12, loop, n_graphs=B, capacity=g.num_edges)
        assert int(gc.info[2].item()) <= DEFAULT_TABLE and not gc.overflowed()


@pytest.mark.gpu
def test_all_positions_non_finite():
    for v in (np.nan, np.inf):
        pos = np.full((500, 3), v, dtype=np.float32)
        batch = np.sort(np.random.default_rng(8).integers(0, 5, size=500))
        g, ea = build_csr(pos, batch, 0.1, True, n_graphs=5, capacity=64)
        assert g.info.tolist()[:2] == [0, 0] and int(g.info[2].item()) <= DEFAULT_TABLE
        assert int(g.rowptr[-1]) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("r,scale", [(1e-6, 2e-5), (0.05, 1.0)])
def test_extent_near_float_max(r, scale):
    """Two nodes at ±3e38 stretch the box beyond FLT_MAX (the fp32 extent overflows); with r = 1e-6 the cell's growth
    would overflow fp32 before the table fits.  The other nodes' edges are still exact."""
    rng = np.random.default_rng(9)
    B, N = 5, 2000
    pos = rng.uniform(0, scale, size=(N, 3)).astype(np.float32)
    pos[0] = [3e38, -3e38, 3e38]
    pos[1] = [-3e38, 3e38, 1.0]
    batch = np.sort(rng.integers(0, B, size=N))
    g, ea = build_csr(pos, batch, r, n_graphs=B)
    check_graph(g, ea, pos, batch, r, False)
    assert g.num_edges > 0
    gc, _ = build_csr(pos, batch, r, n_graphs=B, capacity=g.num_edges)
    assert int(gc.info[2].item()) <= DEFAULT_TABLE
    check_both(pos, batch, r, builders=("coo",))


@pytest.mark.gpu
def test_coo_builder_rejects_non_finite_positions():
    pos = np.random.default_rng(10).uniform(0, 1, size=(100, 3)).astype(np.float32)
    for v in (np.inf, -np.inf, np.nan):
        p = pos.copy()
        p[17, 1] = v
        with pytest.raises(ValueError, match="finite"):
            build_coo(p, None, 0.1)


# ---- GPU: 8. on top of the builders -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("r", [0.035, 0.3])
def test_cutoff_keeps_half_of_the_complete_candidate_set(r):
    pos, _ = far_corner_cloud(r, 0, seed=12)
    N = pos.shape[0]
    batch = (np.arange(N) >= N // 2).astype(np.int64)
    g, ea = build_csr(pos, batch, r, n_graphs=2)
    keys = check_graph(g, ea, pos, batch, r, False)
    E_b = np.bincount(batch[keys // N], minlength=2)
    cut, ea_c = build_csr(pos, batch, r, n_graphs=2, cutoff_rate=0.5)
    rows = cut.rows().cpu().numpy().astype(np.int64)
    kept = rows * N + cut.col.cpu().numpy().astype(np.int64)
    assert np.array_equal(np.bincount(batch[rows], minlength=2), (E_b * 0.5).astype(np.int64))
    assert np.isin(kept, keys).all()


@pytest.mark.gpu
def test_rollout_step_at_offset_coordinates_builds_the_reference_graph():
    from distegnn_b200 import FastEGNN, rollout, synth
    from oracle import fastegnn_oracle as orc
    w = synth.WORKLOADS["fluid113k"]
    inp = synth.make_partitions(w, n_nodes=4000, seed=3)[0]
    sd = orc.init_state_dict(3, 2, 2, 64, 5, 4, seed=1, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, normalize=w.normalize, node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2,
                 virtual_channels=5, n_layers=4)
    m.load_state_dict(sd)
    m = m.to(dev()).eval()
    node = {k: (v.to(dev()) if v is not None else None) for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
    shift = torch.tensor([-1e3, 250.0, 1e3], device=dev())
    node["node_loc"] = node["node_loc"] + shift
    node["loc_mean"] = node["loc_mean"] + shift
    res = rollout(m, **node, steps=1, radius=w.radius)
    pos = node["node_loc"].cpu().numpy()
    batch = node["data_batch"].cpu().numpy()
    check_graph(res.graph, res.edge_attr, pos, batch, w.radius, False)
    g, _ = build_csr(pos, batch, w.radius, n_graphs=int(batch.max()) + 1)
    E = int(res.graph.n_edges_dev.item())
    assert torch.equal(res.graph.rowptr, g.rowptr) and torch.equal(res.graph.col[:E], g.col)
