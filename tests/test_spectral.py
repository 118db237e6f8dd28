"""split_mode="spectral": the reference's spectral-clustering partitioner (distribute_graphs.py:90-115, 201-223) on the
device — the matrix-free RBF product against float64 dense S·X, the embedding against float64 eigh, the labels against
sklearn's SpectralClustering run by the reference's recipe, and the split through split_large_graph and FrameLoader."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from distegnn_b200 import _lib, synth
from distegnn_b200.spectral import RESIDUAL_TOL, SpectralOperator, rbf_gamma, spectral_embedding, spectral_labels


def dev():
    return torch.device("cuda:0")


def ref_gamma(X):
    """The reference's σ recipe (distribute_graphs.py:205-213), written out again."""
    X = X.astype(np.float32)
    N = X.shape[0]
    m = min(N, 2000)
    idx = np.random.RandomState(0).choice(N, size=m, replace=False)
    D = np.linalg.norm(X[idx, None, :] - X[None, idx, :], axis=2)
    sigma = np.median(D[D > 0]) + 1e-12
    return 1.0 / (2.0 * (sigma ** 2))


def ref_labels(X, P):
    """The reference's spectral_clustering through sklearn."""
    from sklearn.cluster import SpectralClustering
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sc = SpectralClustering(n_clusters=P, affinity="rbf", gamma=ref_gamma(X), assign_labels="kmeans",
                                random_state=0, eigen_solver="arpack")
        return sc.fit_predict(X.astype(np.float32))


def clouds(n=1500, seed=0):
    rng = np.random.default_rng(seed)
    return {
        "box": (rng.uniform(0, 1, (n, 3)) * [1, 1.5, 2.3]).astype(np.float32),
        "cube": rng.uniform(0, 1, (n, 3)).astype(np.float32),
        "blob_sheet": np.concatenate([rng.normal(0, .2, (n * 8 // 15, 3)),
                                      rng.uniform(0, 1, (n - n * 8 // 15, 3)) * [3, 3, .1] + [1, 0, 0]]).astype(np.float32),
    }


def dense_S(X, gamma, scaled=True):
    """float64 A_off and (scaled) D^-1/2 A_off D^-1/2 from float32 positions."""
    X = X.astype(np.float64)
    A = np.exp(-gamma * ((X[:, None] - X[None]) ** 2).sum(-1))
    np.fill_diagonal(A, 0.0)
    d = A.sum(1)
    dd = np.where(d > 0, np.sqrt(d), 1.0)
    return (A / dd[:, None] / dd[None]) if scaled else A, d, dd


# ---- host side (no GPU) ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [7, 1999, 2000, 2500])
def test_rbf_gamma_is_the_reference_recipe_bit_for_bit(n):
    rng = np.random.default_rng(n)
    X = (rng.normal(0, 3, (n, 3)) + 500).astype(np.float32)
    X[1] = X[0]                                                   # a coincident pair: zero distances are skipped
    assert rbf_gamma(X) == ref_gamma(X)
    assert rbf_gamma(X.astype(np.float64)) == ref_gamma(X)        # positions are taken as float32 as the reference does


def test_rbf_gamma_rejects_a_cloud_of_one_point():
    with pytest.raises(ValueError, match="coincide"):
        rbf_gamma(np.ones((5, 3), np.float32))


def test_spectral_labels_argument_checks():
    pos = torch.rand(20, 3)
    for bad in (0, 17, 2.0, True):
        with pytest.raises(ValueError, match="n_clusters"):
            spectral_labels(pos, bad)
    with pytest.raises(ValueError, match="cannot form"):
        spectral_labels(pos[:3], 4)
    with pytest.raises(ValueError, match=r"\[N, 3\]"):
        spectral_labels(torch.rand(20, 2), 2)
    nan = pos.clone()
    nan[3, 1] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        spectral_labels(nan, 2)
    with pytest.raises(_lib.DistEGNNError, match="CUDA"):
        spectral_labels(pos, 2)


def test_spectral_c_abi_validates_its_arguments():
    lib = _lib.load()
    nb = C.c_int64(0)
    assert lib.distegnn_spectral_workspace_bytes(1000, 16, 40, C.byref(nb)) == 0 and nb.value > 0
    assert lib.distegnn_spectral_workspace_bytes(1000, 17, 1, C.byref(nb)) == -1
    assert lib.distegnn_spectral_workspace_bytes(0, 1, 1, C.byref(nb)) == -1
    p = 256                                                        # a non-null stand-in: validation fails before use
    assert lib.distegnn_spectral_apply(100, 0, p, 1.0, None, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_spectral_apply(100, 17, p, 1.0, None, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_spectral_apply(100, 2, p, 1.0, None, None, p, p, 1 << 20, None) == -1    # x = NULL needs k = 1
    assert b"k == 1" in lib.distegnn_last_error()
    assert lib.distegnn_spectral_apply(100, 1, p, -1.0, None, None, p, p, 1 << 20, None) == -1
    assert lib.distegnn_spectral_apply(100, 1, p, float("nan"), None, None, p, p, 1 << 20, None) == -1
    assert lib.distegnn_spectral_apply(100, 1, p, 1.0, None, None, p, p, 8, None) == -1             # workspace
    assert b"workspace" in lib.distegnn_last_error()
    assert lib.distegnn_spectral_apply(100, 1, None, 1.0, None, None, p, p, 1 << 20, None) == -1
    assert lib.distegnn_spectral_gram(100, 3, 17, p, p, p, p, 1 << 20, None) == -1
    assert lib.distegnn_spectral_combine(100, 3, 0, p, p, p, 0, None) == -1
    assert lib.distegnn_spectral_combine(100, 3, 2, p, p, p, 2, None) == -1
    assert lib.distegnn_kmeans_lloyd_d(100, 4, 17, p, p, p, p, p, 0.0, 1, None, None) == -1
    assert lib.distegnn_kmeans_lloyd_d(100, 65, 3, p, p, p, p, p, 0.0, 1, None, None) == -1


def test_make_partitions_spectral_is_sklearn_spectral_clustering():
    w = synth.WORKLOADS["fluid113k"]
    n, P = 600, 3
    parts = synth.make_partitions(w, world_size=P, split_mode="spectral", seed=3, n_nodes=n)
    pos = synth.make_points(w, seed=3, n_nodes=n)["pos"]
    want = ref_labels(pos, P)
    for r in range(P):
        assert np.array_equal(parts[r]["node_loc"].numpy(), pos[want == r])
    assert sum(p["node_loc"].shape[0] for p in parts) == n


def test_frame_loader_spectral_split_limits(tmp_path):
    from distegnn_b200.frames import FrameLoader, load_scenes, sample_list
    rng = np.random.default_rng(0)
    p = str(tmp_path / "water_0.npz")
    np.savez(p, position=rng.random((4, 40, 3)).astype(np.float32), particle_type=rng.integers(1, 9, 40))
    traj = load_scenes([p], "water3d")
    samples = sample_list(traj, seed=0, max_samples=1, delta_t=1, max_frame=2)
    with pytest.raises(ValueError, match="at most 16"):
        FrameLoader(traj, samples, radius=0.2, world_size=17, rank=0, split_mode="spectral")
    FrameLoader(traj, samples, radius=0.2, world_size=4, rank=0, split_mode="spectral")      # accepted


# ---- the block product on the device ---------------------------------------------------------------------------------
def _kernel_cases():
    rng = np.random.default_rng(7)
    dup = rng.uniform(0, 1, (300, 3)).astype(np.float32)
    dup[100:150] = dup[:50]                                        # duplicates
    dup[200:220] = dup[199]                                        # a coincident clump
    far = rng.uniform(0, 1, (500, 3)).astype(np.float32)
    far[17] = [1e4, -1e4, 1e4]                                     # every affinity of node 17 underflows to 0
    return {
        "n1000": rng.uniform(0, 1, (1000, 3)).astype(np.float32),  # not a multiple of the 128-row tile
        "n77": rng.uniform(0, 1, (77, 3)).astype(np.float32),      # below one tile
        "dup": dup,
        "plus1e3": (rng.normal(0, 1, (700, 3)) + 1e3).astype(np.float32),
        "minus1e3": (rng.normal(0, 1, (700, 3)) - 1e3).astype(np.float32),
        "far": far,
        "n5000": rng.uniform(0, 2, (5000, 3)).astype(np.float32),  # several column splits
    }


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(_kernel_cases()))
@pytest.mark.parametrize("k", [1, 2, 8, 16])
def test_block_product_matches_float64_dense(case, k):
    X = _kernel_cases()[case]
    N = X.shape[0]
    gamma = rbf_gamma(X)
    S, d, dd = dense_S(X, gamma)
    op = SpectralOperator(torch.from_numpy(X).to(dev()), gamma)
    g = torch.Generator().manual_seed(k)
    x = torch.randn(N, k, generator=g, dtype=torch.float64)
    scale = torch.from_numpy(1.0 / dd)
    y = op.apply(x.to(dev()), scale.to(dev())).cpu().numpy()
    want = S @ x.numpy()
    err = np.abs(y - want).max(0) / np.abs(want).max(0)
    print(f"{case} N={N} k={k}: worst column error relative to its largest value {err.max():.2e}")
    assert np.isfinite(y).all()
    assert err.max() <= 2e-5
    if case == "far":
        assert np.all(y[17] == 0.0)
    # degree mode: x = 1, no scaling
    deg = op.apply(None)[:, 0].cpu().numpy()
    assert np.abs(deg - d).max() <= 2e-5 * d.max()
    if case == "far":
        assert deg[17] == 0.0


@pytest.mark.gpu
def test_block_product_is_bitwise_reproducible_across_calls_and_streams():
    X = _kernel_cases()["n5000"]
    gamma = rbf_gamma(X)
    op = SpectralOperator(torch.from_numpy(X).to(dev()), gamma)
    x = torch.randn(X.shape[0], 16, generator=torch.Generator().manual_seed(0), dtype=torch.float64).to(dev())
    s = torch.rand(X.shape[0], generator=torch.Generator().manual_seed(1), dtype=torch.float64).to(dev()) + 0.5
    a = op.apply(x, s)
    b = op.apply(x, s)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c = op.apply(x, s)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(a, b) and torch.equal(a, c)
    q = torch.randn(40, X.shape[0], generator=torch.Generator().manual_seed(2), dtype=torch.float64).to(dev())
    assert np.array_equal(op.gram(q, q[:16]), op.gram(q, q[:16]))
    want = q.cpu().numpy() @ q[:16].cpu().numpy().T
    assert np.abs(op.gram(q, q[:16]) - want).max() <= 1e-12 * np.abs(want).max()
    cm = np.random.default_rng(3).standard_normal((40, 16))
    assert torch.equal(op.combine(q, cm), op.combine(q, cm))
    assert np.abs(op.combine(q, cm).cpu().numpy() - cm.T @ q.cpu().numpy()).max() <= 1e-12 * 40


# ---- the embedding -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,n,P", [("box", 1500, 4), ("blob_sheet", 1500, 4), ("cube", 2000, 2), ("box", 3000, 8)])
def test_embedding_matches_float64_eigh(name, n, P):
    """Each sign-flipped column within 5·tol/gap of float64 eigh (relative to the column's largest value), where tol is
    the eigensolver's residual bound and gap the distance of the eigenvalue to the rest of the spectrum (Davis–Kahan
    bounds the angle by residual/gap; the fp32 affinity adds a perturbation of the same order)."""
    from sklearn.utils.extmath import _deterministic_vector_sign_flip
    X = clouds(n)[name]
    gamma = rbf_gamma(X)
    S, d, dd = dense_S(X, gamma)
    w, V = np.linalg.eigh(S)
    w, V = w[::-1], V[:, ::-1]
    gaps = np.array([min(abs(w[i] - w[i - 1]) if i else np.inf, abs(w[i] - w[i + 1])) for i in range(P)])
    assert (gaps / np.abs(w[:P]) >= 1e-3).all(), "the cloud does not have the eigen-gaps this test is for"
    want = _deterministic_vector_sign_flip((V[:, :P] / dd[:, None]).T).T
    got, info = spectral_embedding(torch.from_numpy(X).to(dev()), P)
    err = np.abs(got - want).max(0) / np.abs(want).max(0)
    bound = 5 * RESIDUAL_TOL / gaps
    print(f"{name} N={n} P={P}: {info['products']} products, column errors {np.array2string(err, precision=2)}, "
          f"bounds {np.array2string(bound, precision=2)}, eigenvalue error {np.abs(info['eigenvalues'] - w[:P]).max():.1e}")
    assert (err <= bound).all()
    assert np.abs(info["eigenvalues"] - w[:P]).max() <= 1e-5


# ---- the labels --------------------------------------------------------------------------------------------------------
LABEL_CASES = [(name, P) for name in ("box", "cube", "blob_sheet") for P in (2, 4, 8)] + [("fluid", 2), ("fluid", 4),
                                                                                         ("fluid", 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,P", LABEL_CASES)
def test_labels_match_the_reference_recipe(name, P):
    """The three clouds at N = 1500, where the recipe reproduces sklearn exactly, must agree exactly; the synth fluid
    cloud (N = 4000) at >= 0.999, as for k-means."""
    if name == "fluid":
        X = synth.make_points(synth.WORKLOADS["fluid113k"], seed=5, n_nodes=4000)["pos"].astype(np.float32)
    else:
        X = clouds(1500)[name]
    want = ref_labels(X, P)
    got = spectral_labels(torch.from_numpy(X).to(dev()), P)
    assert got.dtype == torch.int64 and got.device.type == "cuda"
    got = got.cpu().numpy()
    agree = float((got == want).mean())
    print(f"{name} N={X.shape[0]} P={P}: label agreement {agree:.6f}, sizes {np.bincount(got, minlength=P).tolist()}")
    assert agree == 1.0 if name != "fluid" else agree >= 0.999
    again = spectral_labels(torch.from_numpy(X).to(dev()), P).cpu().numpy()
    assert np.array_equal(got, again)


# ---- the split -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_split_large_graph_spectral_equals_the_host_restatement_and_runs_in_the_model():
    from distegnn_b200 import FastEGNN, split_large_graph
    w = synth.WORKLOADS["fluid113k"]
    n, P = 3000, 4
    pts = synth.make_points(w, seed=6, n_nodes=n)
    d = dev()
    pos, vel = torch.from_numpy(pts["pos"]).to(d), torch.from_numpy(pts["vel"]).to(d)
    feat, attr = torch.from_numpy(pts["feat"]).to(d), torch.from_numpy(pts["attr"]).to(d)
    host = synth.make_partitions(w, world_size=P, split_mode="spectral", seed=6, n_nodes=n)
    mine = split_large_graph(pos, feat, pos + 0.01 * vel, vel, attr, w.radius, P, split_mode="spectral")
    m = FastEGNN(node_feat_nf=w.node_feat_nf, node_attr_nf=w.node_attr_nf, edge_attr_nf=w.edge_attr_nf, hidden_nf=64,
                 virtual_channels=w.virtual_channels, world_size=1, n_layers=2).to(d).eval()
    for r in range(P):
        assert torch.equal(mine[r]["pos"].cpu(), host[r]["node_loc"]), r
        part = mine[r]
        with torch.no_grad():
            out, X = m(part["x"], part["pos"], part["vel"], part["loc_mean"], part["edge_index"],
                       torch.zeros(part["pos"].shape[0], dtype=torch.long, device=d), part["edge_attr"], part["attr"])
        assert torch.isfinite(out).all() and torch.isfinite(X).all()


@pytest.mark.gpu
def test_frame_loaders_of_every_rank_cover_each_node_once(tmp_path):
    from distegnn_b200.frames import FrameLoader, load_scenes, sample_list
    from distegnn_b200.partition import node_chunks
    rng = np.random.default_rng(4)
    paths = []
    for k, n in enumerate((600, 450)):
        p = str(tmp_path / f"water_{k}.npz")
        steps = rng.normal(0.0, 0.01, (6, n, 3))
        steps[0] = rng.random((n, 3))
        np.savez(p, position=np.cumsum(steps, 0).astype(np.float32), particle_type=rng.integers(1, 9, n))
        paths.append(p)
    traj = load_scenes(paths, "water3d")
    samples = sample_list(traj, seed=1, max_samples=3, delta_t=1, max_frame=3)
    P = 3
    loaders = [FrameLoader(traj, samples, radius=0.2, device=dev(), world_size=P, rank=r, split_mode="spectral",
                           prefetch=0) for r in range(P)]
    for i, (s, f) in enumerate(samples):
        n = traj.scenes[s].n_nodes
        parts = [ld.partition(i) for ld in loaders]
        nodes = torch.cat([idx.to(torch.int64) for idx, _ in parts])
        assert torch.equal(torch.sort(nodes).values, torch.arange(n)), i
        assert all(c == parts[0][1] for _, c in parts)
        pos = torch.from_numpy(np.array(traj.scenes[s].position[f], dtype=np.float32)).to(dev())
        ref = node_chunks(n, P, "spectral", pos=pos)
        for r in range(P):
            assert torch.equal(parts[r][0].to(torch.int64), ref[r].cpu())


@pytest.mark.gpu
def test_eigensolver_accepts_an_exhausted_krylov_space():
    """Three distinct positions, 20 nodes each, and a two-vector start block: the Krylov space is invariant after six
    vectors, fewer than the wanted pairs plus the guard pairs; the wanted pairs are exact there and must be returned."""
    from distegnn_b200.spectral import top_eigenvectors
    rng = np.random.default_rng(1)
    X = np.repeat(rng.uniform(0, 1, (3, 3)), 20, axis=0).astype(np.float32)
    gamma = rbf_gamma(X)
    S, d, dd = dense_S(X, gamma)
    op = SpectralOperator(torch.from_numpy(X).to(dev()), gamma)
    start = np.stack([np.sqrt(d) / np.linalg.norm(np.sqrt(d)), rng.standard_normal(60) / np.sqrt(60)])
    U, theta, products = top_eigenvectors(op, torch.from_numpy(1.0 / dd).to(dev()), torch.from_numpy(start).to(dev()), 3)
    w = np.linalg.eigvalsh(S)[::-1]
    assert np.abs(theta - w[:3]).max() <= 1e-5
    U = U.cpu().numpy()
    assert np.abs(U @ U.T - np.eye(3)).max() <= 1e-10
    assert np.linalg.norm(S @ U.T - U.T * theta, axis=0).max() <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("max_iter", [1, 2, 300])
def test_kmeans_runs_match_sklearn_with_and_without_convergence(max_iter):
    """kmeans_best_of = sklearn's k_means(X, P, random_state=rs, n_init=10, max_iter=...) on 5-dimensional points,
    also when the runs stop at the iteration cap: every run ends with sklearn's closing assignment and its own inertia."""
    from sklearn.cluster import k_means
    from distegnn_b200.spectral import kmeans_best_of
    rng = np.random.default_rng(max_iter)
    X = np.concatenate([rng.normal(c, 0.6, (400, 5)) for c in range(6)]).astype(np.float32)
    _, want, want_inertia = k_means(X, 6, random_state=np.random.RandomState(3), n_init=10, max_iter=max_iter)
    got, inertia = kmeans_best_of(X, 6, np.random.RandomState(3), dev(), max_iter=max_iter)
    agree = float((got == want).mean())
    print(f"max_iter={max_iter}: agreement {agree:.6f}, inertia {inertia:.6g} vs sklearn {want_inertia:.6g}")
    assert np.isfinite(inertia) and inertia > 0
    assert agree >= 0.999
    assert abs(inertia - want_inertia) <= 1e-4 * want_inertia
