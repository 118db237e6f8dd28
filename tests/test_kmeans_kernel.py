"""The Lloyd kernels of the k-means partitioner (csrc/kmeans.cu: `distegnn_kmeans_lloyd`, `distegnn_kmeans_lloyd_d`) and
the Gram / combine products of the spectral eigensolver (csrc/spectral.cu), against plain references.

The host part restates one sklearn Lloyd run from given centres (`_k_means_lloyd.pyx`, `_k_means_common.pyx` and
`_kmeans_single_lloyd`): first-minimum argmin, relocation of empty clusters, averaging as fp32(sum)·fp32(1/count),
strict convergence or the `tol` stop and the iteration cap, each followed by the closing assignment.  It is checked
against `KMeans(K, init=C0, n_init=1, algorithm="lloyd")` on exact data: small integer or quarter-integer coordinates in
a point set symmetric about 0, so that sklearn's centring is a no-op and every sum is exact in fp32 and fp64.  Later
iterations have centres that are not on the grid; there the restatement refuses (`Ambiguous`) any point whose nearest
centre is not ahead of the next one by more than the rounding of an fp32 distance, any relocation whose farthest points
are that close, and any centre shift that close to `tol`, so a comparison bit for bit never depends on rounding.

The GPU part runs the kernels against the restatement bit for bit on such data (labels, centres and state after every
call), walks the device state machine, checks general float clouds against float64, and checks the Gram and combine
products against float64 across their 8192-row chunks."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from distegnn_b200 import _lib
from distegnn_b200.spectral import _same_clustering

U32 = 2.0 ** -24                      # unit roundoff of fp32


class Ambiguous(AssertionError):
    """The data puts a decision of the run within rounding of its threshold: no exact comparison is possible."""


# ---- the restatement ---------------------------------------------------------------------------------------------------
def _on_grid(v):
    """Every value a multiple of 1/4 and below 64 in magnitude: its fp32 distances are exact in either form."""
    v = np.asarray(v, dtype=np.float64)
    return bool(np.all(v * 4 == np.round(v * 4)) and np.all(np.abs(v) < 64))


def _distances(X, Cc, rows=65536):
    """float64 ‖x − c‖² [N,K] in blocks of rows (fp32 inputs: each difference and square is exact)."""
    X64, C64 = X.astype(np.float64), Cc.astype(np.float64)
    for s in range(0, X.shape[0], rows):
        yield s, ((X64[s:s + rows, None, :] - C64[None]) ** 2).sum(-1)


def assign(X, Cc, strict):
    """First-minimum argmin of every point over the centres, with the ambiguity guard: a runner-up within the rounding
    of an fp32 distance (the kernel's direct form, or with `strict` also sklearn's ‖c‖² − 2x·c) must be an exact tie
    between identical centres or between grid centres of a grid point."""
    N, D = X.shape
    labels = np.empty(N, dtype=np.int32)
    cn = (Cc.astype(np.float64) ** 2).sum(1)
    for s, d in _distances(X, Cc):
        k0 = np.argmin(d, axis=1)
        d0 = d[np.arange(d.shape[0]), k0]
        labels[s:s + d.shape[0]] = k0
        if Cc.shape[0] == 1:
            continue
        xn = (X[s:s + d.shape[0]].astype(np.float64) ** 2).sum(1)
        if strict:
            scale = (np.sqrt(xn)[:, None] + np.sqrt(cn)[None]) ** 2
            scale = scale + scale[np.arange(d.shape[0]), k0][:, None]
        else:
            scale = d0[:, None] + d
        near = d <= d0[:, None] + (D + 3) * U32 * scale
        near[np.arange(d.shape[0]), k0] = False
        for r, k in zip(*np.nonzero(near)):
            i, a = s + r, k0[r]
            if d[r, k] == d0[r] and (np.array_equal(Cc[k], Cc[a]) or _on_grid(np.concatenate([X[i], Cc[k], Cc[a]]))):
                continue
            raise Ambiguous(f"point {i}: centres {a} and {k} at {d0[r]!r} and {d[r, k]!r}")
    return labels


def m_step(X, C_old, labels, K, strict):
    """sklearn's M-step: sums and counts, relocation of the empty clusters (the e-th empty cluster, ascending, takes the
    e-th point in the order distance to its centre descending, index ascending; sklearn's order among the relocated points
    is unspecified, so with several empty clusters a comparison with sklearn goes up to a permutation), then the
    averaging.  Returns (centres fp32, squared shift, number of relocated clusters)."""
    N, D = X.shape
    X64 = X.astype(np.float64)
    counts = np.bincount(labels, minlength=K).astype(np.float64)
    sums = np.stack([np.bincount(labels, weights=X64[:, c], minlength=K) for c in range(D)], 1)
    empty = np.nonzero(counts == 0)[0]
    moved = 0
    if empty.size:
        d = ((X64 - C_old.astype(np.float64)[labels]) ** 2).sum(1)
        if d.max() > 0:
            order = np.lexsort((np.arange(N), -d))[:empty.size + 1]
            dd = d[order]
            for j in range(min(empty.size, N - 1)):
                i1, i2 = order[j], order[j + 1]
                if dd[j] - dd[j + 1] > 2 * (D + 3) * U32 * dd[j]:
                    continue
                same = np.array_equal(X[i1], X[i2]) and labels[i1] == labels[i2]
                if not (dd[j] == dd[j + 1] and (same or (not strict and _on_grid(np.concatenate(
                        [X[i1], X[i2], C_old[labels[i1]], C_old[labels[i2]]]))))):
                    raise Ambiguous(f"relocation: points {i1} and {i2} at {dd[j]!r} and {dd[j + 1]!r}")
            for e, i in zip(empty, order):
                old = labels[i]
                sums[old] -= X64[i]
                counts[old] -= 1
                sums[e] = X64[i]
                counts[e] = 1
                moved += 1
    m = int(np.argmax(counts))
    new = np.empty_like(C_old)
    for k in range(K):
        src = k if counts[k] > 0 else m
        if counts[k] > 0 or m < k:
            new[k] = (sums[src] * np.float64(np.float32(1.0 / counts[src]))).astype(np.float32)
        else:
            new[k] = sums[src].astype(np.float32)
    shift = float(((new.astype(np.float64) - C_old.astype(np.float64)) ** 2).sum())
    return new, shift, moved


class RefLloyd:
    """The device state machine of csrc/kmeans.cu restated on the host: `call(iters)` is one `distegnn_kmeans_lloyd*`
    call, `close()` the header's closing call (state[0] = 1, iters = 1)."""

    def __init__(self, X, C0, tol, strict=False):
        self.X, self.centers, self.tol, self.strict = X, C0.astype(np.float32).copy(), float(tol), strict
        self.labels = np.full(X.shape[0], -1, dtype=np.int32)
        self.state = [0, 0, 0, 0]
        self.relocated = []                                  # (iteration, clusters relocated)

    def iterate(self):
        st = self.state[0]
        if st == 2:
            return
        lab = assign(self.X, self.centers, self.strict)
        self.state[2] += int((lab != self.labels).sum())
        self.labels = lab
        if st == 1:
            self.state[0] = 2
            return
        self.centers, shift, moved = m_step(self.X, self.centers, lab, self.centers.shape[0], self.strict)
        self.state[1] += 1
        if moved:
            self.relocated.append((self.state[1], moved))
        if self.state[2] == 0:
            self.state[0] = 2
        else:
            if shift != 0 and (abs(shift - self.tol) <= 1e-3 * self.tol or shift < 1e-30):
                raise Ambiguous(f"centre shift {shift!r} against tol {self.tol!r}")
            if shift <= self.tol:
                self.state[0] = 1
        self.state[2] = 0

    def call(self, iters):
        for _ in range(iters):
            self.iterate()

    def close(self):
        self.state[0] = 1
        self.iterate()

    def run(self, max_iter):
        self.call(max_iter)
        if self.state[0] != 2:
            self.close()
        return self


def sklearn_fit(X, C0, tol, max_iter):
    from sklearn.cluster import KMeans
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return KMeans(C0.shape[0], init=C0, n_init=1, algorithm="lloyd", tol=tol, max_iter=max_iter).fit(X)


def tol_abs(X, tol):
    """sklearn's `_tolerance`."""
    return float(np.mean(np.var(X, axis=0)) * tol)


def exact_cloud(rng, n, D, hi=7, step=1.0):
    """n points with coordinates k·step, |k| <= hi, symmetric about 0 (its fp32 mean is exactly 0), rows shuffled."""
    half = rng.integers(-hi, hi + 1, (n // 2, D)) * step
    pts = np.concatenate([half, -half] + ([np.zeros((1, D))] if n % 2 else []))
    return np.ascontiguousarray(pts[rng.permutation(n)], dtype=np.float32)


def blobs():
    """The two-blob case: unit Gaussian blobs at −3 and +3 (one the mirror of the other) on a 1/4 grid, 300 points each,
    and a third initial centre far from both, which empties in the first pass."""
    a = np.round(np.random.default_rng(0).normal(-3.0, 1.0, (300, 3)) * 4) / 4
    X = np.concatenate([a, -a]).astype(np.float32)
    return X, np.array([[-3, -3, -3], [3, 3, 3.25], [57, 57, 57]], np.float32)


def several_empty():
    rng = np.random.default_rng(1)
    X = exact_cloud(rng, 400, 3)
    C0 = np.concatenate([X[:5], [[40, 40, 40], [-50, 30, 20], [30, -60, 45]]]).astype(np.float32)
    return X, C0


def coincident():
    """Every point on one of the initial centres, and two centres with no point: relocation does nothing (every distance
    is 0), and sklearn's averaging puts the empty clusters on the first largest cluster (its plain sum before it)."""
    P = np.array([[1, 0, 0]] * 3 + [[-1, 0, 0]] * 3 + [[0, 2, 0]] * 2 + [[0, -2, 0]] * 2, np.float32)
    C0 = np.array([[9, 9, 9], [1, 0, 0], [-1, 0, 0], [0, 2, 0], [0, -2, 0], [5, 5, 5]], np.float32)
    return P, C0


def later_empty():
    """A cluster that holds points after the first pass and loses them all in the second (1-D; found by a seeded
    search)."""
    rng = np.random.default_rng(4127)
    X = exact_cloud(rng, 40, 1, hi=8)
    return X, np.ascontiguousarray(np.round(rng.uniform(-8, 8, (5, 1)) * 2) / 2, dtype=np.float32)


HOST_CASES = {"blobs": blobs, "several_empty": several_empty, "coincident": coincident, "later_empty": later_empty}


def _check_against_sklearn(X, C0, tol, max_iter, permute=False):
    ref = RefLloyd(X, C0, tol_abs(X, tol), strict=True).run(max_iter)
    km = sklearn_fit(X, C0, tol, max_iter)
    assert ref.state[0] == 2 and ref.state[1] == km.n_iter_
    if permute:
        assert _same_clustering(ref.labels, km.labels_, C0.shape[0])
        assert _same_clustering(km.labels_, ref.labels, C0.shape[0])
        perm = np.full(C0.shape[0], -1)
        perm[ref.labels] = km.labels_
        assert np.array_equal(np.sort(ref.centers, axis=0), np.sort(km.cluster_centers_, axis=0))
        occupied = np.unique(ref.labels)
        assert np.array_equal(ref.centers[occupied], km.cluster_centers_[perm[occupied]])
    else:
        assert np.array_equal(ref.labels, km.labels_)
        assert np.array_equal(ref.centers, km.cluster_centers_)
    return ref, km


@pytest.mark.parametrize("case", list(HOST_CASES))
def test_restatement_matches_sklearn_on_exact_data(case):
    X, C0 = HOST_CASES[case]()
    assert X.astype(np.float64).sum(0).tolist() == [0.0] * X.shape[1]
    ref, km = _check_against_sklearn(X, C0, 1e-12, 300, permute=case == "several_empty")
    sizes = np.bincount(ref.labels, minlength=C0.shape[0]).tolist()
    print(f"{case}: {ref.state[1]} iterations, sizes {sizes}, relocations {ref.relocated}")
    if case == "blobs":
        assert ref.relocated[0] == (1, 1) and min(sizes) > 0
    elif case == "several_empty":
        assert ref.relocated[0] == (1, 3)
    elif case == "coincident":
        assert ref.relocated == [] and ref.state[1] == 2
        assert ref.centers[0].tolist() == [3, 0, 0] and ref.centers[5].tolist() == [1, 0, 0]
    else:
        assert ref.relocated == [(2, 1)]


@pytest.mark.parametrize("tol,max_iter", [(0.0, 300), (1e-12, 300), (0.05, 300), (1e-12, 1), (1e-12, 2), (1e-12, 3)])
def test_restatement_stops_as_sklearn(tol, max_iter):
    """The tol stop with its closing pass, tol = 0, and the cap followed by the closing assignment."""
    rng = np.random.default_rng(7)
    X = exact_cloud(rng, 512, 3, hi=12)
    C0 = X[rng.choice(512, 6, replace=False)].copy()
    ref, km = _check_against_sklearn(X, C0, tol, max_iter)
    print(f"tol={tol} max_iter={max_iter}: {ref.state[1]} iterations, state {ref.state}")


def test_restatement_refuses_ambiguous_data():
    X = np.array([[-1.0], [0.0], [1.0]], np.float32)
    with pytest.raises(Ambiguous):                           # 0 is equidistant from two centres off the grid
        RefLloyd(X, np.array([[-1 / 3], [1 / 3]], np.float32), 0.0).run(5)
    RefLloyd(X, np.array([[-0.5], [0.5]], np.float32), 0.0).run(5)   # an exact grid tie: the lower index wins


# ---- the kernels -------------------------------------------------------------------------------------------------------
def dev():
    return torch.device("cuda:0")


class Lloyd:
    """Device buffers of one run and the entry point (`entry` "d": distegnn_kmeans_lloyd_d, "3": distegnn_kmeans_lloyd)."""

    def __init__(self, X, C0, tol, entry="d", stream=None):
        self.lib = _lib.load()
        self.N, self.D = X.shape
        self.K = C0.shape[0]
        self.tol, self.entry, self.stream = float(tol), entry, stream
        self.x = torch.from_numpy(np.ascontiguousarray(X)).to(dev())
        self.centers = torch.from_numpy(np.ascontiguousarray(C0, dtype=np.float32)).to(dev())
        self.labels = torch.full((self.N,), -1, dtype=torch.int32, device=dev())
        self.sums = torch.zeros(self.K, self.D + 1, dtype=torch.float64, device=dev())
        self.state = torch.zeros(4, dtype=torch.int32, device=dev())
        self.inertia = torch.full((1,), float("nan"), dtype=torch.float64, device=dev())

    def call(self, iters):
        s = _lib.stream_ptr(dev()) if self.stream is None else C.c_void_p(self.stream.cuda_stream)
        p = _lib.ptr
        if self.entry == "3":
            rc = self.lib.distegnn_kmeans_lloyd(self.N, self.K, p(self.x), p(self.centers), p(self.labels), p(self.sums),
                                                p(self.state), self.tol, iters, s)
        else:
            rc = self.lib.distegnn_kmeans_lloyd_d(self.N, self.K, self.D, p(self.x), p(self.centers), p(self.labels),
                                                  p(self.sums), p(self.state), self.tol, iters, p(self.inertia), s)
        _lib.check(rc, "kmeans_lloyd")

    def close(self):
        self.state[0] = 1
        self.call(1)

    def snapshot(self):
        torch.cuda.synchronize()
        return self.labels.cpu().numpy(), self.centers.cpu().numpy(), self.state.cpu().tolist()


def _agree(run, ref, where):
    lab, cen, st = run.snapshot()
    assert st == ref.state, f"{where}: state {st} != {ref.state}"
    assert np.array_equal(lab, ref.labels), f"{where}: {(lab != ref.labels).sum()} labels differ"
    assert np.array_equal(cen, ref.centers), f"{where}: centres differ by {np.abs(cen - ref.centers).max()}"


def _run_both(X, C0, tol, max_iter, chunk, entry="d"):
    run, ref = Lloyd(X, C0, tol, entry), RefLloyd(X, C0, tol)
    done = 0
    while done < max_iter and ref.state[0] != 2:
        n = min(chunk, max_iter - done)
        run.call(n)
        ref.call(n)
        done += n
        _agree(run, ref, f"after {done} iterations")
    if ref.state[0] != 2:
        run.close()
        ref.close()
        _agree(run, ref, "after the closing call")
    return run, ref


def unambiguous(make, seed, tol, max_iter, tries=64):
    """The first data set make(seed), make(seed + 1), ... on which the whole run can be compared exactly."""
    for s in range(seed, seed + tries):
        X, C0 = make(s)
        try:
            RefLloyd(X, C0, tol(X)).run(max_iter)
            return X, C0
        except Ambiguous:
            pass
    raise AssertionError(f"no unambiguous data among seeds {seed}..{seed + tries - 1}")


def _grid_case(K, D, N, seed):
    def make(s):
        rng = np.random.default_rng(s)
        X = exact_cloud(rng, N, D, hi=7)
        return X, (np.round(rng.uniform(-7, 7, (K, D)) * 2) / 2).astype(np.float32)
    return unambiguous(make, seed, lambda X: tol_abs(X, 1e-4), 60)


GRID = ([(K, D, N) for K in (1, 2, 7, 63, 64) for D in (1, 3, 16) for N in sorted({1, max(K - 1, 1), K, 255, 1025})]
        + [(7, 2, N) for N in (256, 1023, 1024, 4097)] + [(64, 16, 4097), (63, 5, 1024), (2, 5, 256)])


@pytest.mark.gpu
@pytest.mark.parametrize("K,D,N", GRID)
def test_kernel_matches_the_restatement_bitwise(K, D, N):
    X, C0 = _grid_case(K, D, N, seed=K * 1000 + D * 100 + N % 97)
    run, ref = _run_both(X, C0, tol_abs(X, 1e-4), 60, 7)
    if D == 3:
        run3, _ = _run_both(X, C0, tol_abs(X, 1e-4), 60, 7, entry="3")
        assert np.array_equal(run3.snapshot()[1], run.snapshot()[1])
    print(f"K={K} D={D} N={N}: {ref.state[1]} iterations, relocations {ref.relocated}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(HOST_CASES))
def test_kernel_matches_sklearn_on_the_empty_cluster_cases(case):
    X, C0 = HOST_CASES[case]()
    tol = tol_abs(X, 1e-12)
    for entry in ("d", "3") if X.shape[1] == 3 else ("d",):
        run, ref = _run_both(X, C0, tol, 300, 16, entry)
    km = sklearn_fit(X, C0, 1e-12, 300)
    lab, cen, st = run.snapshot()
    assert st[1] == km.n_iter_
    if case == "several_empty":
        assert _same_clustering(lab, km.labels_, C0.shape[0]) and _same_clustering(km.labels_, lab, C0.shape[0])
    else:
        assert np.array_equal(lab, km.labels_) and np.array_equal(cen, km.cluster_centers_)
    print(f"{case}: sizes {np.bincount(lab, minlength=C0.shape[0]).tolist()} after {st[1]} iterations")


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["d", "3"])
def test_kernel_over_more_than_one_grid_stride_pass(entry):
    """≈1.2 M points: more than 8 CTAs per SM × 1024 points, so every thread takes several points."""
    rng = np.random.default_rng(11)
    X = exact_cloud(rng, 1_200_017, 3, hi=7)
    C0 = np.concatenate([np.round(rng.uniform(-6, 6, (6, 3)) * 2) / 2, [[40, 40, 40]]]).astype(np.float32)
    run, ref = _run_both(X, C0, tol_abs(X, 1e-4), 12, 5, entry)
    assert ref.relocated and ref.relocated[0][0] == 1


@pytest.mark.gpu
def test_ties_duplicates_and_fewer_distinct_points_than_clusters():
    rng = np.random.default_rng(5)
    # exact ties between identical centres and between grid centres: the lower index wins
    X = exact_cloud(rng, 2000, 3, hi=4)
    C0 = np.array([[1, 1, 1], [1, 1, 1], [-1, -1, -1], [0, 0, 2], [0, 0, -2], [-1, -1, -1]], np.float32)
    _run_both(X, C0, 0.0, 100, 3)
    # four distinct points, many copies each, and 9 clusters
    P = np.array([[2, 0, 0], [-2, 0, 0], [0, 3, 0], [0, -3, 0]], np.float32)
    X = np.ascontiguousarray(P[rng.integers(0, 4, 999)])
    X = np.concatenate([X, -X, P])
    C0 = (np.round(rng.uniform(-3, 3, (9, 3)) * 2) / 2).astype(np.float32)
    run, ref = _run_both(X, C0, 0.0, 100, 4)
    assert len(np.unique(ref.labels)) <= 4


@pytest.mark.gpu
def test_state_machine_chunking_and_inertia():
    """The same run as 1 × 300, 16 × 19 and 300 × 1 calls gives the same bits; iterations after state 2 do nothing; the
    cap ends with the closing call; no inertia is written before state 2."""
    def make(s):
        rng = np.random.default_rng(s)
        X = exact_cloud(rng, 3000, 5, hi=9)
        return X, X[rng.choice(3000, 12, replace=False)].copy()
    X, C0 = unambiguous(make, 3, lambda X: 0.0, 300)
    tol = tol_abs(X, 0.01)
    RefLloyd(X, C0, tol).run(300)                             # the tol stop below is unambiguous too
    ref = RefLloyd(X, C0, 0.0).run(300)
    assert ref.state[:2] == [2, ref.state[1]] and ref.state[1] < 250
    outs = []
    for calls, iters in ((1, 300), (16, 19), (300, 1)):
        run = Lloyd(X, C0, 0.0)
        for _ in range(calls):
            run.call(iters)
            if run.state[0].item() != 2:
                assert torch.isnan(run.inertia).all()
        outs.append(run.snapshot() + (run.inertia.item(),))
    for o in outs[1:]:
        assert np.array_equal(o[0], outs[0][0]) and np.array_equal(o[1], outs[0][1]) and o[2] == outs[0][2]
        assert o[3] == outs[0][3]
    assert outs[0][2] == ref.state and np.array_equal(outs[0][0], ref.labels) and np.array_equal(outs[0][1], ref.centers)
    # the cap: after max_iter passes without convergence the closing call assigns to the final centres
    for cap in (1, 2, 5):
        run, want = _run_both(X, C0, 0.0, cap, 2)
        assert want.state[1] == cap and not np.isnan(run.inertia.item())
    # a tol stop: one more assignment pass inside the same call
    run, want = _run_both(X, C0, tol, 300, 300)
    assert want.state[1] < ref.state[1]


@pytest.mark.gpu
@pytest.mark.parametrize("name,K,D", [("offset1e3", 8, 3), ("heavy", 16, 3), ("offset100_d16", 12, 16), ("mixed", 64, 7)])
def test_general_float_clouds_against_float64(name, K, D):
    rng = np.random.default_rng(K + D)
    N = 50_000
    if name == "offset1e3":
        X = rng.uniform(0, 10, (N, D)) + 1e3
    elif name == "heavy":
        X = rng.standard_cauchy((N, D)).clip(-1e4, 1e4)
    elif name == "offset100_d16":
        X = rng.normal(0, 1, (N, D)) * rng.uniform(0.1, 5, D) + 100
    else:
        X = np.concatenate([rng.normal(c, 0.3, (N // 8, D)) for c in rng.uniform(-20, 20, 8)]) * 1.7 - 4
    X = np.ascontiguousarray(X, dtype=np.float32)
    N = X.shape[0]
    C0 = X[rng.choice(N, K, replace=False)].copy()
    run = Lloyd(X, C0, 0.0)
    run.call(300)
    if run.state[0].item() != 2:
        run.close()
    lab, cen, st = run.snapshot()
    X64, c64 = X.astype(np.float64), cen.astype(np.float64)
    # every label an argmin of the final centres, within the fp32 rounding of the distance
    best = np.full(N, np.inf)
    for s, d in _distances(X, cen):
        best[s:s + d.shape[0]] = d.min(1)
    mine = ((X64 - c64[lab]) ** 2).sum(1)
    assert (mine <= best + 2 * (D + 2) * U32 * (mine + best)).all()
    # every centre within one fp32 step of fp32(float64 mean of its points), when the labels are the last M-step's
    if st[2] == 0:
        for k in np.unique(lab):
            m = X64[lab == k].mean(0).astype(np.float32)
            ok = (cen[k] == m) | (cen[k] == np.nextafter(m, np.inf)) | (cen[k] == np.nextafter(m, -np.inf))
            assert ok.all(), (k, cen[k], m)
    # the inertia: fp32 terms, fp64 sum — within the terms' rounding of float64, the same bits when recomputed
    ine = run.inertia.item()
    want = mine.sum()
    print(f"{name}: {st[1]} iterations, state {st}, inertia {ine:.9g} vs float64 {want:.9g}")
    assert abs(ine - want) <= (D + 2) * U32 * want
    for stream in (None, torch.cuda.Stream()):
        run.inertia.fill_(float("nan"))
        run.stream = stream
        if stream is not None:
            stream.wait_stream(torch.cuda.current_stream())
        run.call(1)                                            # state 2: only the inertia runs again
        torch.cuda.synchronize()
        assert run.inertia.item() == ine
        assert np.array_equal(run.snapshot()[1], cen)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0.0, 100.0, 1000.0])
def test_kmeans_labels_on_an_offset_uniform_cloud(offset):
    """kmeans_labels against the reference call on 20,000 uniform points at an offset: the iterations run on the centred
    positions, so the offset costs no digits."""
    from sklearn.cluster import KMeans
    from distegnn_b200.partition import kmeans_labels
    X = (np.random.default_rng(0).uniform(0, 1, (20_000, 3)) + offset).astype(np.float32)
    want = KMeans(n_clusters=8, random_state=0, n_init="auto").fit_predict(X)
    got = kmeans_labels(torch.from_numpy(X).to(dev()), 8).cpu().numpy()
    agree = float((got == want).mean())
    print(f"offset {offset}: agreement {agree:.6f}")
    assert agree >= 0.9999


# ---- the spectral eigensolver's Gram and combine products --------------------------------------------------------------
def _gamma(n):
    u = 2.0 ** -53
    return n * u / (1 - n * u)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 8191, 8192, 8193, 3 * 8192 + 1, 113_140])
@pytest.mark.parametrize("a,b", [(1, 1), (17, 7), (300, 16), (17, 16), (300, 1)])
def test_gram_and_combine_against_float64(N, a, b):
    lib = _lib.load()
    p = _lib.ptr
    g = torch.Generator().manual_seed(N + a * b)
    u = (torch.randn(a, N, generator=g, dtype=torch.float64) * torch.logspace(-3, 3, a, dtype=torch.float64)[:, None])
    v = torch.randn(b, N, generator=g, dtype=torch.float64)
    c = torch.randn(a, b, generator=g, dtype=torch.float64)
    ud, vd, cd = u.to(dev()), v.to(dev()), c.to(dev())
    nb = C.c_int64(0)
    _lib.check(lib.distegnn_spectral_workspace_bytes(N, b, a, C.byref(nb)), "workspace")
    ws = torch.empty(int(nb.value), dtype=torch.uint8, device=dev())
    s = _lib.stream_ptr(dev())

    def gram():
        out = torch.full((a, b), float("nan"), dtype=torch.float64, device=dev())
        _lib.check(lib.distegnn_spectral_gram(N, a, b, p(ud), p(vd), p(out), p(ws), ws.numel(), s), "gram")
        return out.cpu().numpy()

    def combine(out, subtract):
        _lib.check(lib.distegnn_spectral_combine(N, a, b, p(ud), p(cd), p(out), subtract, s), "combine")
        return out

    un, vn, cn = u.numpy(), v.numpy(), c.numpy()
    got = gram()
    want = un @ vn.T
    bound = 2 * _gamma(N) * (np.abs(un) @ np.abs(vn).T)
    assert np.isfinite(got).all() and (np.abs(got - want) <= bound).all()
    assert np.array_equal(got, gram())
    y = combine(torch.full((b, N), float("nan"), dtype=torch.float64, device=dev()), 0).cpu().numpy()
    want = cn.T @ un
    assert np.isfinite(y).all() and (np.abs(y - want) <= 2 * _gamma(a) * (np.abs(cn).T @ np.abs(un))).all()
    assert np.array_equal(y, combine(torch.empty(b, N, dtype=torch.float64, device=dev()), 0).cpu().numpy())
    y0 = torch.randn(b, N, generator=g, dtype=torch.float64)
    z = combine(y0.to(dev()), 1).cpu().numpy()
    want = y0.numpy() - cn.T @ un
    assert (np.abs(z - want) <= 2 * _gamma(a + 1) * (np.abs(y0.numpy()) + np.abs(cn).T @ np.abs(un))).all()
    assert np.array_equal(z, combine(y0.to(dev()), 1).cpu().numpy())
