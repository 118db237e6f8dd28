"""The edge kernels need one thing from the edge order: the edges of a destination row are contiguous.  Rows need not come
in id order, and the cached graph of FastEGNN stores them in a spatial order (distegnn_build_csr_cells, DESIGN §3).

Here the forward kernel, the deterministic forward kernel with its combine pass and the backward kernel run on graphs
whose rows are shuffled as whole blocks (hubs next to degree-one rows, isolated rows, self loops), checked row by row
against float64 with the metrics of tests/helpers.py.  The cell-order CSR build is checked against the id-order build
(same rowptr, same edges per row in the same relative order, graphs contiguous), the edge kernel's outputs on the two
orders against each other, and whole forwards through the cached cell-order graph against a pre-sorted id-order
CSRGraph.  In the deterministic mode the cached graph is in id order, and its bits do not depend on the positions of
earlier calls."""
import pytest
import torch

from distegnn_b200 import FastEGNN, _lib, synth
from distegnn_b200.shards import CSRGraph
from oracle import fastegnn_oracle as orc
from tests import test_backward_kernel_tiling as bk
from tests import test_edge_kernel_tiling as ek
from tests import test_forward_det_tiling as dk
from tests.helpers import TOL, rel_disp_err, rowwise, within_rerun_bound

pytestmark = pytest.mark.gpu


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def shuffle_row_blocks(row, col, N, seed):
    """The edges of every row kept together and in their order, the rows in a random order."""
    g = torch.Generator().manual_seed(seed)
    rank = torch.randperm(N, generator=g)
    order = torch.sort(rank[row], stable=True).indices
    return row[order], col[order]


def hub_graph(N, seed):
    """Degree-one rows around a 5,000-edge hub, random rows, self loops, and isolated rows."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.arange(0, 3_000)
    hub = torch.full((5_000,), 3_000)
    mid = torch.sort(torch.randint(3_001, N // 2, (20_000,), generator=g))[0]     # nodes N/2.. are isolated
    row = torch.cat([lo, hub, mid])
    col = torch.randint(0, N, (row.numel(),), generator=g)
    col[::7] = row[::7]
    return row, col


def assert_row_runs(row):
    """Every row's edges form one contiguous run."""
    r = row.long().cpu()
    starts = torch.ones_like(r, dtype=torch.bool)
    starts[1:] = r[1:] != r[:-1]
    assert torch.unique(r[starts]).numel() == int(starts.sum()), "a row's edges are split into several runs"


KERNELS = {"default": ek.production, "deterministic": dk.det_edge}


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("flags", [0, _lib.FLAG_NORMALIZE | _lib.FLAG_LAST])
def test_edge_fwd_rows_in_shuffled_blocks(kernel, flags):
    N = 20_000
    row, col = shuffle_row_blocks(*hub_graph(N, seed=3), N, seed=4)
    assert_row_runs(row)
    agg_m, agg_x = ek.check(N, row, col, 2, flags, seed=3, kernel=KERNELS[kernel])
    assert float(agg_x[N // 2:].abs().max()) == 0.0
    if agg_m is not None:
        assert float(agg_m[N // 2:].abs().max()) == 0.0


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_edge_fwd_many_tiles_rows_in_shuffled_blocks(kernel):
    N = 200_000
    row, col = shuffle_row_blocks(*ek.random_graph(N, 2_000_003, seed=9), N, seed=10)
    ek.check(N, row, col, 2, 0, seed=9, kernel=KERNELS[kernel])


@pytest.mark.parametrize("flags", [0, _lib.FLAG_NORMALIZE])
def test_edge_bwd_hub_rows_in_shuffled_blocks(flags):
    """The graph of test_backward_kernel_tiling's hub case (a 5,000-edge hub among degree-one rows, isolated rows), its
    rows shuffled as whole blocks."""
    N = 20_000
    g = torch.Generator().manual_seed(5)
    row = torch.cat([torch.arange(0, 3_000), torch.full((5_000,), 3_000), torch.arange(3_001, 9_001)])
    col = torch.randint(0, 9_001, (row.numel(),), generator=g)
    col = torch.where(col == row, (col + 1) % 9_001, col)
    row, col = shuffle_row_blocks(row, col, N, seed=6)
    bk.check_edge(N, 2, flags, bk.edge_inputs(row, col, N, 2, seed=5), "hub, rows in shuffled blocks")


@pytest.mark.parametrize("flags", [0, _lib.FLAG_NORMALIZE | _lib.FLAG_LAST])
def test_edge_bwd_rows_in_shuffled_blocks(flags):
    """Several 128-edge tiles per CTA, as test_backward_kernel_tiling's attribute-count case, rows shuffled."""
    N = 5_000
    row, col = shuffle_row_blocks(*bk.random_graph(N, 100_003, seed=102 + 10 * flags), N, seed=7)
    bk.check_edge(N, 2, flags, bk.edge_inputs(row, col, N, 2, seed=2 + flags), "rows in shuffled blocks",
                  same_as_weights_only=True)


def batch_of_clouds(seed=0):
    """Three fluid-like clouds of different sizes as one batch (sorted data_batch)."""
    w = synth.WORKLOADS["fluid113k"]
    parts = [synth.make_partitions(w, n_nodes=n, seed=seed + i)[0] for i, n in enumerate((3_000, 1_200, 5_000))]
    cat = lambda k: torch.cat([p[k] for p in parts])
    off, eis = 0, []
    for p in parts:
        eis.append(p["edge_index"] + off)
        off += p["node_loc"].shape[0]
    inp = dict(node_feat=cat("node_feat"), node_loc=cat("node_loc"), node_vel=cat("node_vel"),
               node_attr=cat("node_attr"), edge_attr=cat("edge_attr"), edge_index=torch.cat(eis, 1),
               loc_mean=torch.cat([p["loc_mean"] for p in parts]),
               data_batch=torch.cat([torch.full((p["node_loc"].shape[0],), i, dtype=torch.long)
                                     for i, p in enumerate(parts)]))
    return w, inp


def test_build_csr_cells_against_id_order():
    from distegnn_b200.backend import CudaBackend
    be = CudaBackend()
    _, inp = batch_of_clouds()
    d = dev()
    N, B = inp["node_loc"].shape[0], 3
    ei = inp["edge_index"].to(d)
    ref = be.build_csr(ei, N)
    got = be.build_csr_cells(ei, N, inp["node_loc"].to(d), inp["data_batch"].to(d), B)
    assert torch.equal(got[0], ref[0]), "rowptr differs from the id-order build"
    row, col, perm = (t.long().cpu() for t in got[1:])
    assert_row_runs(row)
    gid = inp["data_batch"][row]
    assert bool((gid[1:] >= gid[:-1]).all()), "graphs are not contiguous and in order"
    assert not bool((row[1:] >= row[:-1]).all()), "the rows came out in id order"
    assert torch.equal(perm.sort().values, torch.arange(row.numel())), "perm is not a permutation"
    assert torch.equal(ei[0].cpu()[perm], row) and torch.equal(ei[1].cpu()[perm], col)
    s = torch.sort(row, stable=True).indices                     # each row's edges in the id build's relative order
    for a, b in ((row[s], ref[1]), (col[s], ref[2]), (perm[s], ref[3])):
        assert torch.equal(a, b.long().cpu())


def test_edge_kernel_cell_order_matches_id_order():
    """distegnn_edge_layer_fwd on the cell-order and the id-order build of one graph: agg_m row by row, agg_x within the
    bound of two launches that differ only in the order of their atomics."""
    from tests.twin_backend import twin_backend
    be = twin_backend()
    _, inp = batch_of_clouds(seed=7)
    d = dev()
    N, E = inp["node_loc"].shape[0], inp["edge_index"].shape[1]
    ei = inp["edge_index"].to(d)
    x4 = torch.zeros(N, 4, device=d)
    x4[:, :3] = inp["node_loc"].to(d)
    g = torch.Generator().manual_seed(7)
    P, Q = torch.randn(N, 64, generator=g).to(d), torch.randn(N, 64, generator=g).to(d)
    ea = inp["edge_attr"].to(d)
    lp = ek.layer_params(2)
    outs = []
    for csr in (be.build_csr(ei, N), be.build_csr_cells(ei, N, inp["node_loc"].to(d), inp["data_batch"].to(d), 3)):
        row, col, perm = csr[1:]
        agg_m, agg_x = torch.zeros(N, 64, device=d), torch.zeros(N, 4, device=d)
        be.edge_layer((N, E, 2, 3, 0), 0, row, col, be.gather_rows(ea, perm), x4, P, Q, lp, agg_m, agg_x)
        outs.append((agg_m, agg_x))
    torch.cuda.synchronize()
    e_m = rowwise(outs[1][0], outs[0][0], zero_rows=~outs[0][0].any(1))
    print(f"cell vs id order: agg_m row-wise {e_m:.1e}")
    assert e_m <= TOL
    assert within_rerun_bound(outs[1][1], outs[0][1])


def model_and_inputs():
    w, inp = batch_of_clouds(seed=11)
    sd = orc.init_state_dict(w.node_feat_nf, w.node_attr_nf, w.edge_attr_nf, 64, w.virtual_channels, 4, seed=0,
                             coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=w.node_feat_nf, node_attr_nf=w.node_attr_nf,
                 edge_attr_nf=w.edge_attr_nf, virtual_channels=w.virtual_channels, n_layers=4)
    m.load_state_dict(sd)
    d = dev()
    return m.to(d).eval(), {k: v.to(d) for k, v in inp.items()}


def id_order_inputs(inp):
    N = inp["node_loc"].shape[0]
    g, ea = CSRGraph.from_edge_index(inp["edge_index"], N, inp["edge_attr"])
    return dict(inp, edge_index=g, edge_attr=ea)


def cached_rows(m, edge_index):
    """The `row` array of the model's cached graph of `edge_index` (there must be exactly one)."""
    rows = [e[3][1] for e in m._graphs.entries.values() if e[0] is edge_index]
    assert len(rows) == 1
    return rows[0].long().cpu()


def test_forward_cached_cell_order_matches_id_order():
    """A forward through the cached graph (rows in cell order) against the same graph passed in id order; the cached
    order is the one of the first call's positions, and later calls with other positions reuse it."""
    m, inp = model_and_inputs()
    ref = id_order_inputs(inp)
    with torch.no_grad():
        out, X = m(**inp)
        row = cached_rows(m, inp["edge_index"])
        assert_row_runs(row)
        assert not bool((row[1:] >= row[:-1]).all()), "the cached graph is in id order, not in cell order"
        out_r, X_r = m(**ref)
        e = rel_disp_err(out, out_r, inp["node_loc"])
        print(f"cell vs id order, displacement {e:.1e}")
        assert e <= 1e-5 and within_rerun_bound(X, X_r)
        moved = dict(inp, node_loc=inp["node_loc"] + 0.01 * inp["node_vel"])
        builds = m._graphs.builds
        out_m, _ = m(**moved)
        assert m._graphs.builds == builds, "the cached graph was rebuilt for new positions"
        assert torch.equal(cached_rows(m, inp["edge_index"]), row)
        out_mr, _ = m(**dict(ref, node_loc=moved["node_loc"]))
        assert rel_disp_err(out_m, out_mr, moved["node_loc"]) <= 1e-5


def test_deterministic_bits_do_not_depend_on_the_cache_history():
    """In the deterministic mode the cached graph is in id order, which depends on edge_index alone: after forwards at
    other positions, in either mode, a forward at positions b has the bits of a fresh model's forward at b, and of the
    same graph passed as an id-order CSRGraph."""
    m, inp = model_and_inputs()
    fresh, _ = model_and_inputs()
    fresh.deterministic = True
    moved = dict(inp, node_loc=inp["node_loc"] + 0.01 * inp["node_vel"])
    with torch.no_grad():
        m(**inp)                                               # default mode first: a cell-order entry for edge_index
        m.deterministic = True
        m(**inp)
        ids = [e[3][1].long().cpu() for e in m._graphs.entries.values()
               if e[0] is inp["edge_index"] and bool((e[3][1][1:] >= e[3][1][:-1]).all())]
        assert len(ids) == 1, "the deterministic mode has no id-order entry of its own"
        out, X = m(**moved)
        out_f, X_f = fresh(**moved)
        assert torch.equal(out, out_f) and torch.equal(X, X_f), "the bits depend on the positions of an earlier call"
        out_r, X_r = m(**dict(id_order_inputs(inp), node_loc=moved["node_loc"]))
        assert torch.equal(out, out_r) and torch.equal(X, X_r), "the cached graph is not in id order"
        out2, X2 = m(**moved)
        assert torch.equal(out, out2) and torch.equal(X, X2), "not bitwise reproducible"
