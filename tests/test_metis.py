"""split_mode="metis": the reference's METIS partitioner (distribute_graphs.py:54-87, 151-185) — the host call into the
toolkit's METIS with its validation, the device sort that turns the radius build's CSR into METIS's input, the labels
against the host restatement `synth.metis_partition`, and the split through split_large_graph and FrameLoader."""
import threading

import numpy as np
import pytest
import torch

from distegnn_b200 import _lib, synth
from distegnn_b200.partition import metis_recursive


def dev():
    return torch.device("cuda:0")


def grid_csr(rows, cols):
    """The rows x cols 4-neighbour grid, node r*cols + c, neighbours ascending."""
    adj = [[] for _ in range(rows * cols)]
    for r in range(rows):
        for c in range(cols):
            for rr, cc in ((r - 1, c), (r, c - 1), (r, c + 1), (r + 1, c)):
                if 0 <= rr < rows and 0 <= cc < cols:
                    adj[r * cols + c].append(rr * cols + cc)
    xadj = np.zeros(rows * cols + 1, dtype=np.int64)
    np.cumsum([len(a) for a in adj], out=xadj[1:])
    return xadj, np.array(sum(adj, []), dtype=np.int64)


def kdtree_csr(pos, r):
    """The reference's METIS input written out again: cKDTree pairs both ways, sorted by (row, col), index2ptr."""
    from scipy.spatial import cKDTree
    n = pos.shape[0]
    pairs = cKDTree(pos).query_pairs(r, output_type="ndarray").astype(np.int64).reshape(-1, 2)
    row = np.concatenate([pairs[:, 0], pairs[:, 1]])
    col = np.concatenate([pairs[:, 1], pairs[:, 0]])
    order = np.lexsort((col, row))
    return np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n))]).astype(np.int64), col[order]


def assert_clean(pos, r):
    """No pair's float64 squared distance lies within 2^-20 (relative) of r²: there the device's fp32 strict `<` and the
    cKDTree's float64 `<=` could disagree, and this file compares graphs built both ways."""
    from scipy.spatial import cKDTree
    if pos.shape[0] < 2:
        return
    p = pos.astype(np.float64)
    pairs = cKDTree(p).query_pairs(r * (1 + 2.0 ** -19), output_type="ndarray").reshape(-1, 2)
    d2 = ((p[pairs[:, 0]] - p[pairs[:, 1]]) ** 2).sum(1)
    assert not (np.abs(d2 - r * r) <= 2.0 ** -20 * r * r).any(), "a pair lies at r within the fp32 tolerance"


def cut_edges(xadj, adjncy, labels):
    row = np.repeat(np.arange(xadj.shape[0] - 1), np.diff(xadj))
    return int((labels[row] != labels[adjncy]).sum()) // 2


# ---- host side (no GPU) ----------------------------------------------------------------------------------------------
def test_metis_symbols_are_not_exported():
    lib = _lib.load()
    assert hasattr(lib, "distegnn_metis_recursive")
    for name in ("METIS_PartGraphRecursive", "METIS_SetDefaultOptions", "gk_sigtrap", "libmetis__Match_RM"):
        assert not hasattr(lib, name), name


def test_grid_bisects_into_its_two_halves():
    xadj, adjncy = grid_csr(2, 4)
    labels, cut = metis_recursive(xadj, adjncy, 2)
    assert cut == 2
    assert labels.dtype == np.int64
    halves = {frozenset(np.nonzero(labels == p)[0].tolist()) for p in (0, 1)}
    assert halves == {frozenset({0, 1, 4, 5}), frozenset({2, 3, 6, 7})}
    assert cut_edges(xadj, adjncy, labels) == 2


def test_inputs_are_left_unchanged_and_calls_repeat():
    xadj, adjncy = kdtree_csr(np.random.default_rng(0).random((3000, 3)).astype(np.float32), 0.08)
    x0, a0 = xadj.copy(), adjncy.copy()
    first, cut = metis_recursive(xadj, adjncy, 5)
    assert np.array_equal(xadj, x0) and np.array_equal(adjncy, a0)
    again, cut2 = metis_recursive(xadj, adjncy, 5)
    assert np.array_equal(first, again) and cut == cut2 == cut_edges(xadj, adjncy, first)
    assert set(np.unique(first)) == set(range(5))


def test_one_part_is_zeros_without_metis():
    """METIS itself labels everything 1 at nparts = 1; the reference's metis() returns zeros without calling it."""
    xadj, adjncy = grid_csr(3, 3)
    labels, cut = metis_recursive(xadj, adjncy, 1)
    assert labels.dtype == np.int64 and np.array_equal(labels, np.zeros(9, dtype=np.int64)) and cut == 0


@pytest.mark.parametrize("case,match", [
    ("xadj0", "xadj\\[0\\]"), ("decreasing", "decreases"), ("negative", "outside"), ("past_n", "outside"),
    ("self_loop", "self loop"), ("parts0", "n_parts=0"), ("parts_past_n", "n_parts=10"), ("short_adjncy", "past adjncy"),
])
def test_malformed_input_is_rejected_before_metis(case, match):
    xadj, adjncy = grid_csr(3, 3)
    parts = 2
    if case == "xadj0":
        xadj[0] = 1
    elif case == "decreasing":
        xadj[4], xadj[5] = xadj[5], xadj[4]
    elif case == "negative":
        adjncy[3] = -1
    elif case == "past_n":
        adjncy[7] = 9
    elif case == "self_loop":
        adjncy[xadj[4]] = 4
    elif case == "parts0":
        parts = 0
    elif case == "parts_past_n":
        parts = 10
    elif case == "short_adjncy":
        adjncy = adjncy[:-1]
    with pytest.raises(ValueError, match=match):
        metis_recursive(xadj, adjncy, parts)


def test_malformed_input_sets_the_last_error_through_the_c_abi():
    lib = _lib.load()
    xadj, adjncy = grid_csr(2, 2)
    part = np.empty(4, dtype=np.int64)
    rc = lib.distegnn_metis_recursive(4, xadj.ctypes.data, adjncy.ctypes.data, 5, part.ctypes.data, None)
    assert rc == -1 and b"n_parts=5" in lib.distegnn_last_error()
    rc = lib.distegnn_metis_recursive(0, xadj.ctypes.data, adjncy.ctypes.data, 1, part.ctypes.data, None)
    assert rc == -1


@pytest.mark.parametrize("n,parts", [(1, 1), (7, 7), (16, 16), (40, 3), (100, 8)])
def test_edgeless_graph_gives_balanced_parts(n, parts):
    labels, cut = metis_recursive(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int64), parts)
    assert cut == 0 and labels.min() >= 0 and labels.max() < parts
    sizes = np.bincount(labels, minlength=parts)
    assert sizes.max() - sizes.min() <= 1, sizes


def test_concurrent_calls_give_the_serial_labels():
    rng = np.random.default_rng(1)
    graphs = [kdtree_csr(rng.random((4000, 3)).astype(np.float32), 0.07) for _ in range(4)]
    serial = [metis_recursive(x, a, 2 + k)[0] for k, (x, a) in enumerate(graphs)]
    got = [None] * 4

    def work(k):
        x, a = graphs[k]
        for _ in range(3):
            lab = metis_recursive(x, a, 2 + k)[0]
            assert got[k] is None or np.array_equal(got[k], lab)
            got[k] = lab
    threads = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for k in range(4):
        assert np.array_equal(got[k], serial[k]), k


@pytest.mark.parametrize("n,P,r", [(500, 2, 0.15), (3000, 4, 0.08), (2500, 7, 0.1)])
def test_synth_metis_partition_is_the_c_call_on_the_kdtree_csr(n, P, r):
    pos = np.random.default_rng(n).random((n, 3)).astype(np.float32)
    xadj, adjncy = kdtree_csr(pos, r)
    sx, sa = synth.metis_csr_np(pos, r)
    assert np.array_equal(sx, xadj) and np.array_equal(sa, adjncy)
    labels, _ = metis_recursive(xadj, adjncy, P)
    chunks = synth.metis_partition(pos, P, r)
    assert len(chunks) == P
    for i in range(P):
        assert np.array_equal(chunks[i], np.nonzero(labels == i)[0])


def test_frame_loader_metis_needs_outer_radius(tmp_path):
    from distegnn_b200.frames import FrameLoader, load_scenes, sample_list
    rng = np.random.default_rng(0)
    p = str(tmp_path / "water_0.npz")
    np.savez(p, position=rng.random((4, 40, 3)).astype(np.float32), particle_type=rng.integers(1, 9, 40))
    traj = load_scenes([p], "water3d")
    samples = sample_list(traj, seed=0, max_samples=1, delta_t=1, max_frame=2)
    with pytest.raises(ValueError, match="outer_radius"):
        FrameLoader(traj, samples, radius=0.2, world_size=2, rank=0, split_mode="metis")
    FrameLoader(traj, samples, radius=0.2, world_size=2, rank=0, split_mode="metis", outer_radius=0.3)   # accepted
    FrameLoader(traj, samples, radius=0.2, world_size=1, rank=0, split_mode="metis")                     # one rank


# ---- the sort kernel -------------------------------------------------------------------------------------------------
def ragged_cloud(seed):
    """Clusters dense enough for rows past 32 and past 1024 entries, a sparse field and isolated far nodes."""
    rng = np.random.default_rng(seed)
    return np.concatenate([
        rng.uniform(0, 0.05, (1300, 3)),                 # degree ~1299 at r = 0.1
        rng.uniform(0, 0.2, (400, 3)) + [1, 0, 0],       # degree ~tens to hundreds
        rng.uniform(0, 3, (2000, 3)) + [0, 2, 0],        # sparse
        rng.uniform(0, 1, (9, 3)) * 100 + 50,            # isolated
    ]).astype(np.float32)[rng.permutation(3709)]


def device_graph(pos, r, capacity=None):
    from distegnn_b200 import radius_graph_csr
    return radius_graph_csr(torch.from_numpy(pos).to(dev()), r, edge_attr_nf=0, capacity=capacity)[0]


def host_lexsort(g):
    """index2ptr(sort_edge_index(.)) of the device graph's own edges, on the host."""
    E = int(g.n_edges_dev.item()) if g.n_edges_dev is not None else g.num_edges
    rowptr = g.rowptr.cpu().numpy().astype(np.int64)
    col = g.col[:E].cpu().numpy().astype(np.int64)
    row = np.repeat(np.arange(rowptr.shape[0] - 1), np.diff(rowptr))
    return rowptr, col[np.lexsort((col, row))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ragged0", "ragged1", "complete2000", "n1", "edgeless", "capacity"])
def test_sorted_csr_is_the_host_lexsort(case):
    from distegnn_b200.partition import csr_sorted_i64
    rng = np.random.default_rng(3)
    cap = None
    if case.startswith("ragged"):
        pos, r = ragged_cloud(int(case[-1])), 0.1
    elif case == "complete2000":
        pos, r = rng.random((2000, 3)).astype(np.float32), 10.0
    elif case == "n1":
        pos, r = np.zeros((1, 3), np.float32), 1.0
    elif case == "edgeless":
        pos, r = rng.random((300, 3)).astype(np.float32), 1e-4
    else:
        pos, r, cap = ragged_cloud(2), 0.1, 3_000_000
    g = device_graph(pos, r, cap)
    xadj, adjncy = csr_sorted_i64(g)
    want_x, want_a = host_lexsort(g)
    E = want_a.shape[0]
    assert xadj.dtype == adjncy.dtype == torch.int64
    assert np.array_equal(xadj.cpu().numpy(), want_x)
    assert np.array_equal(adjncy[:E].cpu().numpy(), want_a)
    deg = np.diff(want_x)
    print(f"{case}: N={pos.shape[0]} E={E} max degree {deg.max()} rows past 32: {(deg > 32).sum()}, "
          f"past 1024: {(deg > 1024).sum()}")
    if case == "complete2000":
        assert E == 2000 * 1999 and deg.min() == 1999
    if case.startswith("ragged"):
        assert (deg > 1024).any() and ((deg > 32) & (deg <= 1024)).any() and (deg == 0).any()
    if case in ("n1", "edgeless"):
        assert E == 0 and np.array_equal(xadj.cpu().numpy(), np.zeros(pos.shape[0] + 1))


@pytest.mark.gpu
@pytest.mark.parametrize("seed,n,r", [(0, 5000, 0.1), (1, 20000, 0.05), (3, 3709, 0.1)])
def test_sorted_csr_is_the_kdtree_csr(seed, n, r):
    from distegnn_b200.partition import csr_sorted_i64
    pos = ragged_cloud(seed) if n == 3709 else np.random.default_rng(seed).random((n, 3)).astype(np.float32)
    assert_clean(pos, r)
    xadj, adjncy = csr_sorted_i64(device_graph(pos, r))
    want_x, want_a = kdtree_csr(pos, r)
    assert np.array_equal(xadj.cpu().numpy(), want_x) and np.array_equal(adjncy.cpu().numpy(), want_a)


# ---- the labels ------------------------------------------------------------------------------------------------------
def label_case(name, P, n, seed):
    """(positions, outer radius) of one metis_labels case."""
    rng = np.random.default_rng(seed)
    if name == "fluid":
        w = synth.WORKLOADS["fluid113k"]
        return synth.make_points(w, seed=seed, n_nodes=n)["pos"], w.radius
    if name == "blobs":                                  # two far-apart blobs: a disconnected graph
        return np.concatenate([rng.normal(0, 0.1, (n // 2, 3)),
                               rng.normal(0, 0.1, (n - n // 2, 3)) + 5]).astype(np.float32), 0.05
    if name == "coincident":                             # every point three times over
        base = rng.random(((n + 2) // 3, 3)).astype(np.float32)
        return np.repeat(base, 3, axis=0)[:n], 0.12
    if name == "edgeless":                               # r below the spacing
        return (np.stack(np.meshgrid(*[np.arange(12)] * 3), -1).reshape(-1, 3)[:n] * 0.1).astype(np.float32), 0.05
    raise KeyError(name)


# seeds of the larger fluid clouds picked so that assert_clean holds (about one pair in 10^6 lies that close to r)
LABEL_CASES = [("fluid", 2, 2, 2), ("fluid", 3, 40, 3), ("fluid", 4, 1000, 4), ("fluid", 5, 7777, 5),
               ("fluid", 8, 10000, 8), ("fluid", 16, 30000, 17), ("fluid", 2, 113140, 37), ("fluid", 8, 113140, 37),
               ("blobs", 2, 3000, 0), ("blobs", 5, 3000, 1), ("coincident", 4, 3000, 2), ("coincident", 16, 3000, 3),
               ("edgeless", 3, 1000, 0), ("edgeless", 16, 1728, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,P,n,seed", LABEL_CASES)
def test_labels_equal_the_host_restatement(name, P, n, seed):
    from distegnn_b200 import metis_labels
    pos, r = label_case(name, P, n, seed)
    assert_clean(pos, r)
    got = metis_labels(torch.from_numpy(pos).to(dev()), P, r)
    assert got.dtype == torch.int64 and got.device == dev() and got.shape == (n,)
    got = got.cpu().numpy()
    want = synth.metis_partition(pos, P, r)
    sizes = np.bincount(got, minlength=P)
    print(f"{name} N={n} P={P} r={r}: sizes {sizes.min()}..{sizes.max()}")
    for i in range(P):
        assert np.array_equal(np.nonzero(got == i)[0], want[i]), i
    if name == "edgeless":
        assert sizes.max() - sizes.min() <= 1


@pytest.mark.gpu
def test_labels_reject_bad_input():
    from distegnn_b200 import metis_labels
    pos = torch.rand(100, 3, device=dev())
    bad = pos.clone()
    bad[7, 1] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        metis_labels(bad, 2, 0.2)
    bad[7, 1] = float("inf")
    with pytest.raises(ValueError, match="finite"):
        metis_labels(bad, 2, 0.2)
    for r in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="outer_radius"):
            metis_labels(pos, 2, r)
    for P in (0, 101):
        with pytest.raises(ValueError, match="n_parts"):
            metis_labels(pos, P, 0.2)
    assert torch.equal(metis_labels(pos, 1, 0.2), torch.zeros(100, dtype=torch.int64, device=dev()))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 8])
def test_metis_cuts_fewer_edges_than_kmeans_with_balanced_parts(P):
    from distegnn_b200 import kmeans_labels, metis_labels
    w = synth.WORKLOADS["fluid113k"]
    pos = synth.make_points(w, seed=0)["pos"]
    xadj, adjncy = kdtree_csr(pos, w.radius)
    p = torch.from_numpy(pos).to(dev())
    met = metis_labels(p, P, w.radius).cpu().numpy()
    km = kmeans_labels(p, P).cpu().numpy()
    cm, ck = cut_edges(xadj, adjncy, met), cut_edges(xadj, adjncy, km)
    sizes = np.bincount(met, minlength=P)
    print(f"P={P}: METIS cuts {cm} of {adjncy.shape[0] // 2} edges, k-means {ck}; METIS sizes {sizes.tolist()}")
    assert cm < ck
    # recursive bisection's default tolerance, 1.001 per level (ufactor 1)
    levels = int(np.ceil(np.log2(P)))
    assert sizes.max() <= np.ceil(pos.shape[0] / P * 1.001 ** levels) and sizes.min() > 0


# ---- the split -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_split_large_graph_metis_equals_the_host_restatement_and_runs_in_the_model():
    from distegnn_b200 import FastEGNN, split_large_graph
    w = synth.WORKLOADS["fluid113k"]
    n, P, outer = 6000, 4, 0.09
    pts = synth.make_points(w, seed=8, n_nodes=n)
    pos_np = pts["pos"]
    assert_clean(pos_np, outer)
    d = dev()
    pos, vel = torch.from_numpy(pos_np).to(d), torch.from_numpy(pts["vel"]).to(d)
    feat, attr = torch.from_numpy(pts["feat"]).to(d), torch.from_numpy(pts["attr"]).to(d)
    target = pos + 0.01 * vel
    mine = split_large_graph(pos, feat, target, vel, attr, w.radius, P, split_mode="metis", outer_radius=outer)
    # split_large_graph_metis restated: labels from the outer graph, pos[cluster == i], an inner graph per part
    labels = np.empty(n, dtype=np.int64)
    for i, idx in enumerate(synth.metis_partition(pos_np, P, outer)):
        labels[idx] = i
    loc_mean = pos.mean(dim=0, keepdim=True)
    for i in range(P):
        m_ = labels == i
        part = mine[i]
        assert torch.equal(part["pos"].cpu(), torch.from_numpy(pos_np[m_]))
        for key, src in (("x", feat), ("vel", vel), ("attr", attr), ("target", target)):
            assert torch.equal(part[key].cpu(), src.cpu()[torch.from_numpy(m_)]), key
        assert torch.equal(part["loc_mean"], loc_mean)
        assert_clean(pos_np[m_], w.radius)
        ei = synth.radius_graph_np(pos_np[m_], w.radius)
        got = part["edge_index"].edge_index().cpu().numpy()
        assert {tuple(e) for e in ei.T.tolist()} == {tuple(e) for e in got.T.tolist()}
        assert part["special_nodes"].all()
    m = FastEGNN(node_feat_nf=w.node_feat_nf, node_attr_nf=w.node_attr_nf, edge_attr_nf=w.edge_attr_nf, hidden_nf=64,
                 virtual_channels=w.virtual_channels, world_size=1, n_layers=2).to(d).eval()
    part = mine[0]
    with torch.no_grad():
        out, X = m(part["x"], part["pos"], part["vel"], part["loc_mean"], part["edge_index"],
                   torch.zeros(part["pos"].shape[0], dtype=torch.long, device=d), part["edge_attr"], part["attr"])
    assert torch.isfinite(out).all() and torch.isfinite(X).all()


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 4])
def test_frame_loaders_cover_each_node_once_and_call_metis_once_per_sample(tmp_path, monkeypatch, P):
    from distegnn_b200 import partition
    from distegnn_b200.frames import FrameLoader, load_scenes, sample_list
    rng = np.random.default_rng(4)
    paths = []
    for k, n in enumerate((900, 700)):
        p = str(tmp_path / f"water_{k}.npz")
        steps = rng.normal(0.0, 0.01, (6, n, 3))
        steps[0] = rng.random((n, 3))
        np.savez(p, position=np.cumsum(steps, 0).astype(np.float32), particle_type=rng.integers(1, 9, n))
        paths.append(p)
    traj = load_scenes(paths, "water3d")
    samples = sample_list(traj, seed=1, max_samples=4, delta_t=1, max_frame=3)
    calls = []
    real = partition.metis_recursive

    def counting(xadj, adjncy, n_parts):
        calls.append(int(n_parts))
        return real(xadj, adjncy, n_parts)
    monkeypatch.setattr(partition, "metis_recursive", counting)
    loaders = [FrameLoader(traj, samples, radius=0.1, batch_size=2, shuffle=True, device=dev(), world_size=P, rank=r,
                           split_mode="metis", outer_radius=0.15, prefetch=0) for r in range(P)]
    for _ in range(2):
        for ld in loaders:
            assert sum(1 for _ in ld) == len(ld)
    assert len(calls) == P * len(samples) and set(calls) == {P}
    for i, (s, f) in enumerate(samples):
        n = traj.scenes[s].n_nodes
        parts = [ld.partition(i) for ld in loaders]
        nodes = torch.cat([idx.to(torch.int64) for idx, _ in parts])
        assert torch.equal(torch.sort(nodes).values, torch.arange(n)), i
        assert all(c == parts[0][1] for _, c in parts)
        pos = np.array(traj.scenes[s].position[f], dtype=np.float32)
        want = synth.metis_partition(pos, P, 0.15)
        for r in range(P):
            assert np.array_equal(parts[r][0].numpy().astype(np.int64), want[r])
    assert len(calls) == P * len(samples) + len(samples)         # the host restatement above, nothing more
