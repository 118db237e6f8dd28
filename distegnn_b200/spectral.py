"""Spectral node partitioner on the device — the reference's `split_mode="spectral"` (datasets/distribute_graphs.py:90-115,
201-223: `sklearn.cluster.SpectralClustering(affinity="rbf", gamma=1/(2σ²), assign_labels="kmeans", random_state=0,
eigen_solver="arpack")` with σ the median pairwise distance of 2000 sampled nodes).

    labels = spectral_labels(pos, n_clusters)        # int64 [N] on pos.device, the reference's cluster of every node

The recipe, restated (DESIGN §10):
  1. σ on the host, exactly as the reference: `rbf_gamma`.
  2. The P eigenvectors of S = D^−½ (A − I) D^−½, A_ij = exp(−γ‖x_i − x_j‖²), with the largest eigenvalues (the trivial
     one, √d/‖√d‖, included), each divided by √d and sign-flipped as sklearn does.  A is never formed: every product
     S·X recomputes it from the positions (`distegnn_spectral_apply`, csrc/spectral.cu, O(N) memory), and a block Krylov
     eigensolver with full reorthogonalisation and Rayleigh–Ritz in fp64 runs over that product (`top_eigenvectors`).
  3. k-means on the float32 embedding as sklearn's `k_means(maps, P, random_state=rs, n_init=10)`: ten k-means++
     seedings on the host from the one RandomState (after ARPACK's N `v0` draws), Lloyd on the device
     (`distegnn_kmeans_lloyd_d`), the lowest inertia kept by sklearn's rule.

The operator, the eigensolver and the embedding are bitwise deterministic (fixed summation orders on the device, fp64
eigenproblems on the host).  The Lloyd cluster sums use fp64 atomics, so ranks computing the labels from the same
positions agree with high probability, not with certainty (DESIGN §10).  CUDA only; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr

Tensor = torch.Tensor
MAX_CLUSTERS = 16           # = DISTEGNN_SPECTRAL_MAX_K = DISTEGNN_KMEANS_MAX_DIM
BLOCK = 16                  # vectors per block product
RESIDUAL_TOL = 1e-6         # ‖S·u − θu‖₂ of every wanted Ritz pair (u unit-norm, ‖S‖₂ <= 1) at convergence
MAX_ITER = 60               # block products after the first
GUARD = 8                   # Ritz pairs past the wanted ones that must converge too: a small residual alone does not
                            # say that no eigenvalue above the P-th is still missing from the basis
N_INIT = 10                 # k-means runs, as spectral_clustering's default
LOG2E = 1.4426950408889634


class EigensolverNotConverged(RuntimeError):
    """The eigensolver hit its iteration cap; `residuals` holds the last residual norm of every wanted Ritz pair."""

    def __init__(self, msg: str, residuals: np.ndarray):
        super().__init__(msg)
        self.residuals = residuals


def rbf_gamma(pos: np.ndarray) -> float:
    """γ = 1/(2σ²) of the reference's spectral partitioner (distribute_graphs.py:205-213), on the host, bit for bit:
    σ = the median of the nonzero float32 pairwise distances among min(N, 2000) nodes drawn by RandomState(0) without
    replacement, plus 1e-12 (float32 arithmetic throughout, as numpy does it there)."""
    X = np.asarray(pos, dtype=np.float32)
    N = X.shape[0]
    m = min(N, 2000)
    idx = np.random.RandomState(0).choice(N, size=m, replace=False)
    D = np.linalg.norm(X[idx, None, :] - X[None, idx, :], axis=2)
    nz = D[D > 0]
    if nz.size == 0:
        raise ValueError("spectral partitioning: the sampled positions all coincide, the RBF width σ is undefined")
    sigma = np.median(nz) + 1e-12
    return float(1.0 / (2.0 * (sigma ** 2)))


class SpectralOperator:
    """S·X = s ⊙ (A_off · (s ⊙ X)) for a fixed cloud, plus the deterministic tall-skinny products of the eigensolver.
    `pos` [N,3] on a CUDA device, centred here (fp64 mean on the host, then fp32: the kernel's distances are fp32, and a
    cloud far from the origin would lose its digits to the offset), `gamma` the RBF parameter, `max_vectors` the largest
    number of stored vectors a Gram product will see."""

    def __init__(self, pos: Tensor, gamma: float, max_vectors: int = BLOCK):
        self.lib = _lib.load()
        x = pos.detach().to(torch.float64).cpu().numpy()
        self.pos = torch.from_numpy((x - x.mean(axis=0)).astype(np.float32)).to(pos.device).contiguous()
        self.n = int(self.pos.shape[0])
        self.dev = pos.device
        self.g2 = float(np.float32(gamma * LOG2E))
        nbytes = C.c_int64(0)
        check(self.lib.distegnn_spectral_workspace_bytes(self.n, BLOCK, max(1, int(max_vectors)), C.byref(nbytes)),
              "spectral_workspace_bytes")
        self.ws = torch.empty(int(nbytes.value), dtype=torch.uint8, device=self.dev)

    def apply(self, x: Optional[Tensor], scale: Optional[Tensor] = None) -> Tensor:
        """y [N,k] = scale ⊙ (A_off · (scale ⊙ x)) for x fp64 [N,k] (k <= 16; None: all ones, k = 1)."""
        k = 1 if x is None else int(x.shape[1])
        y = torch.empty(self.n, k, dtype=torch.float64, device=self.dev)
        with torch.cuda.device(self.dev):
            check(self.lib.distegnn_spectral_apply(self.n, k, ptr(self.pos), self.g2, ptr(scale), ptr(x), ptr(y),
                                                   ptr(self.ws), self.ws.numel(), _lib.stream_ptr(self.dev)),
                  "spectral_apply")
        return y

    def gram(self, u: Tensor, v: Tensor) -> np.ndarray:
        """u·vᵀ on the host (fp64 [a,b]) for u [a,N], v [b,N] (b <= 16)."""
        g = torch.empty(u.shape[0], v.shape[0], dtype=torch.float64, device=self.dev)
        with torch.cuda.device(self.dev):
            check(self.lib.distegnn_spectral_gram(self.n, int(u.shape[0]), int(v.shape[0]), ptr(u), ptr(v), ptr(g),
                                                  ptr(self.ws), self.ws.numel(), _lib.stream_ptr(self.dev)),
                  "spectral_gram")
        return g.cpu().numpy()

    def combine(self, u: Tensor, c: np.ndarray, out: Optional[Tensor] = None, subtract: bool = False) -> Tensor:
        """cᵀ-combination of the rows of u [a,N]: [b,N] (subtract: out −= it in place)."""
        c = np.ascontiguousarray(c, dtype=np.float64)
        ct = torch.from_numpy(c).to(self.dev)
        if out is None:
            out = torch.empty(c.shape[1], self.n, dtype=torch.float64, device=self.dev)
        with torch.cuda.device(self.dev):
            check(self.lib.distegnn_spectral_combine(self.n, int(u.shape[0]), int(c.shape[1]), ptr(u), ptr(ct),
                                                     ptr(out), int(subtract), _lib.stream_ptr(self.dev)),
                  "spectral_combine")
        return out


def _orthonormalise(op: SpectralOperator, w: Tensor, q: Tensor) -> Tensor:
    """w [b,N] (rows of norm <= 1) made orthonormal and orthogonal to the orthonormal rows of q [m,N]: two classical
    Gram–Schmidt passes, then the block whitened by the eigen-decomposition of its Gram matrix (host fp64); all of it
    twice.  Directions whose norm fell below 1e-6 after the projection (the Krylov space is exhausted there: what is left
    is rounding, not orthogonal to q) are dropped, so the result may have fewer rows."""
    for _ in range(2):
        for _ in range(2):
            if q.shape[0]:
                op.combine(q, op.gram(q, w), out=w, subtract=True)
        g = op.gram(w, w)
        lam, vec = np.linalg.eigh((g + g.T) / 2)
        keep = lam > 1e-12
        if not keep.any():
            return w[:0]
        w = op.combine(w, vec[:, keep] / np.sqrt(lam[keep]))
    return w


def _residuals(op: SpectralOperator, q: Tensor, sq: Tensor, y: np.ndarray, theta: np.ndarray) -> np.ndarray:
    """‖S·(q y_i) − θ_i (q y_i)‖₂ of Ritz pairs, with S·q = sq."""
    y = np.ascontiguousarray(y)
    r = op.combine(sq, y)
    op.combine(op.combine(q, y), np.diag(theta), out=r, subtract=True)
    return np.sqrt(np.maximum(np.diag(op.gram(r, r)), 0.0))


def top_eigenvectors(op: SpectralOperator, scale: Tensor, start: Tensor, n_vectors: int, tol: float = RESIDUAL_TOL,
                     max_iter: int = MAX_ITER) -> Tuple[Tensor, np.ndarray, int]:
    """The `n_vectors` eigenpairs of S (the operator with `scale`) with the largest eigenvalues, by a block Krylov method
    (block Lanczos with full reorthogonalisation): the basis grows by S·(last block), every block orthonormalised twice
    against the whole basis, and the Rayleigh–Ritz problem H = Qᵀ S Q solved on the host in fp64 after every product.
    `start` [b,N] is the first block (its first row the known top vector).  Stops once the wanted Ritz pairs and `GUARD`
    more all have ‖S u − θ u‖₂ <= tol, or once the Krylov space is exhausted (span Q invariant: fewer guard pairs exist,
    the wanted ones still need the residual bound); raises `EigensolverNotConverged` with the residuals after `max_iter`
    products.  The basis Q and S·Q (2·m·N fp64 for m basis vectors) grow with the products actually made, doubling their
    storage when full.  Returns (vectors fp64 [n_vectors, N] in descending eigenvalue order, eigenvalues, products)."""
    n, b = op.n, int(start.shape[0])
    cap = min(n, b * (max_iter + 1))
    Q = torch.empty(0, n, dtype=torch.float64, device=op.dev)
    SQ = torch.empty_like(Q)
    H = np.zeros((cap, cap))
    m, w, res, products = 0, start.clone(), np.full(n_vectors, np.inf), 0
    while True:
        w = _orthonormalise(op, w, Q[:m])
        bw = min(int(w.shape[0]), cap - m)
        exhausted = bw == 0 or m + bw == n
        if bw:
            if m + bw > Q.shape[0]:                                  # grow the stored basis on demand
                rows = min(cap, max(m + bw, 2 * Q.shape[0]))
                Q2 = torch.empty(rows, n, dtype=torch.float64, device=op.dev)
                SQ2 = torch.empty_like(Q2)
                Q2[:m], SQ2[:m] = Q[:m], SQ[:m]
                Q, SQ = Q2, SQ2
            Q[m:m + bw] = w[:bw]
            SQ[m:m + bw] = op.apply(Q[m:m + bw].t().contiguous(), scale).t()
            products += 1
            H[:m + bw, m:m + bw] = op.gram(Q[:m + bw], SQ[m:m + bw])
            H[m:m + bw, :m] = H[:m, m:m + bw].T
            m += bw
        Hs = (H[:m, :m] + H[:m, :m].T) / 2
        theta, Y = np.linalg.eigh(Hs)
        sel = np.argsort(-theta, kind="stable")[:min(n_vectors + GUARD, m)]
        theta, Y = theta[sel], Y[:, sel]
        res = np.concatenate([_residuals(op, Q[:m], SQ[:m], Y[:, c:c + BLOCK], theta[c:c + BLOCK])
                              for c in range(0, len(sel), BLOCK)])
        if (len(sel) == n_vectors + GUARD or exhausted) and len(sel) >= n_vectors and res.max() <= tol:
            return op.combine(Q[:m], np.ascontiguousarray(Y[:, :n_vectors])), theta[:n_vectors], products
        if exhausted or m == cap or products > max_iter:
            break
        w = SQ[m - bw:m].clone()
    raise EigensolverNotConverged(
        f"spectral eigensolver: {m} basis vectors after {products} block products"
        f"{' (Krylov space exhausted)' if exhausted else ''}, residuals ‖S·u − θu‖ of the {len(res)} leading pairs "
        f"{np.array2string(res, precision=3)} not all below {tol:g} (or fewer than the {n_vectors} wanted)", res)


def _same_clustering(l1: np.ndarray, l2: np.ndarray, k: int) -> bool:
    """sklearn's `_is_same_clustering`: every label of l1 maps to one label of l2."""
    mapping = np.full(k, -1, dtype=np.int64)
    first = np.unique(l1, return_index=True)[1]
    mapping[l1[first]] = l2[first]
    return bool(np.array_equal(mapping[l1], l2))


def kmeans_best_of(X: np.ndarray, n_clusters: int, rs: np.random.RandomState, device, n_init: int = N_INIT,
                   max_iter: int = 300, tol: float = 1e-4, chunk: int = 16) -> Tuple[np.ndarray, float]:
    """`sklearn.cluster.k_means(X, n_clusters, random_state=rs, n_init=n_init)` for float32 X [N,D] (D <= 16): each run
    draws its k-means++ seeding from `rs` on the host (on the centred X, as KMeans.fit does) and runs Lloyd on the device
    with sklearn's stopping rules; a run replaces the best so far when its inertia is lower and its clustering differs
    (sklearn's rule).  Returns (labels int32 [N], inertia)."""
    from sklearn.cluster import kmeans_plusplus
    lib = _lib.load()
    X = np.ascontiguousarray(X, dtype=np.float32)
    N, D = X.shape
    tol_abs = float(np.mean(np.var(X, axis=0)) * tol)           # sklearn's _tolerance
    Xc = X - X.mean(axis=0)
    xd = torch.from_numpy(Xc).to(device)
    best_l, best_i = None, None
    with torch.cuda.device(device):
        for _ in range(n_init):
            c0, _ = kmeans_plusplus(Xc, n_clusters, random_state=rs)
            centers = torch.from_numpy(np.ascontiguousarray(c0, dtype=np.float32)).to(device)
            labels = torch.full((N,), -1, dtype=torch.int32, device=device)
            sums = torch.zeros(n_clusters, D + 1, dtype=torch.float64, device=device)
            state = torch.zeros(4, dtype=torch.int32, device=device)
            inertia = torch.full((1,), float("nan"), dtype=torch.float64, device=device)

            def lloyd(k):
                check(lib.distegnn_kmeans_lloyd_d(N, n_clusters, D, ptr(xd), ptr(centers), ptr(labels), ptr(sums),
                                                  ptr(state), tol_abs, k, ptr(inertia), _lib.stream_ptr(device)),
                      "kmeans_lloyd_d")
            done = 0
            while done < max_iter and int(state[0].item()) != 2:
                k = min(chunk, max_iter - done)
                lloyd(k)
                done += k
            if int(state[0].item()) != 2:
                # max_iter passes without strict convergence: sklearn's closing E-step, labels to the final centres
                state[0] = 1
                lloyd(1)
            lab, ine = labels.cpu().numpy(), float(inertia.item())
            if not np.isfinite(ine):
                raise _lib.DistEGNNError(f"k-means run ended without an inertia (state {state.tolist()})")
            if best_l is None or (ine < best_i and not _same_clustering(lab, best_l, n_clusters)):
                best_l, best_i = lab, ine
    return best_l, best_i


def spectral_embedding(pos: Tensor, n_components: int, gamma: Optional[float] = None, tol: float = RESIDUAL_TOL,
                       max_iter: int = MAX_ITER) -> Tuple[np.ndarray, dict]:
    """The reference's spectral embedding on the device: fp64 [N, n_components] on the host, columns = the eigenvectors
    of S with the largest eigenvalues divided by √d (1 for a zero degree), sign-flipped by sklearn's
    `_deterministic_vector_sign_flip`.  `gamma` None: `rbf_gamma(pos)`.  Also returns a dict with the eigenvalues, the
    products used and γ."""
    from sklearn.utils.extmath import _deterministic_vector_sign_flip
    X = pos.detach().to(torch.float32).cpu().numpy()
    N = X.shape[0]
    if gamma is None:
        gamma = rbf_gamma(X)
    b = min(BLOCK, N)
    op = SpectralOperator(pos, gamma, max_vectors=min(N, b * (max_iter + 1)))
    d = op.apply(None)[:, 0]
    dd = torch.where(d > 0, d.sqrt(), torch.ones_like(d))
    scale = (1.0 / dd).contiguous()
    start = np.empty((b, N))
    sd = d.sqrt().cpu().numpy()
    nrm = np.linalg.norm(sd)
    start[0] = sd / nrm if nrm > 0 else 1.0 / np.sqrt(N)
    if b > 1:
        start[1:] = np.random.default_rng(0).standard_normal((b - 1, N)) / np.sqrt(N)
    U, theta, its = top_eigenvectors(op, scale, torch.from_numpy(start).to(pos.device), n_components, tol, max_iter)
    emb = (U / dd[None, :]).cpu().numpy()
    emb = _deterministic_vector_sign_flip(emb)
    return np.ascontiguousarray(emb.T), dict(eigenvalues=theta, products=its, gamma=gamma)


def _check_pos(pos: Tensor, n_clusters) -> int:
    if pos.dim() != 2 or pos.shape[1] != 3:
        raise ValueError(f"positions must be [N, 3] (got {tuple(pos.shape)})")
    if isinstance(n_clusters, bool) or not isinstance(n_clusters, (int, np.integer)) or not 1 <= n_clusters <= MAX_CLUSTERS:
        raise ValueError(f"n_clusters must be an int in [1, {MAX_CLUSTERS}] (got {n_clusters!r})")
    N = int(pos.shape[0])
    if N < n_clusters:
        raise ValueError(f"{N} nodes cannot form {n_clusters} clusters")
    if not bool(torch.isfinite(pos).all()):
        raise ValueError("spectral_labels: positions must be finite")
    if pos.device.type != "cuda":
        raise _lib.DistEGNNError("distegnn_b200.spectral_labels runs only on CUDA tensors (no CPU path)")
    return N


def spectral_labels(pos: Tensor, n_clusters: int, random_state: int = 0) -> Tensor:
    """The reference's `spectral_clustering(pos, n_clusters, random_state)` (distribute_graphs.py:201-223) with the
    affinity products, the eigensolver's products and the Lloyd iterations on the device: int64 labels [N] on
    `pos.device`.  n_clusters in [1, 16], N >= n_clusters, finite positions (ValueError otherwise)."""
    N = _check_pos(pos, n_clusters)
    if n_clusters == 1:
        return torch.zeros(N, dtype=torch.int64, device=pos.device)
    emb, _ = spectral_embedding(pos, n_clusters)
    rs = np.random.RandomState(random_state)
    rs.uniform(-1, 1, N)                                         # ARPACK's v0, drawn from the same RandomState first
    labels, _ = kmeans_best_of(emb.astype(np.float32), n_clusters, rs, pos.device)
    return torch.from_numpy(labels.astype(np.int64)).to(pos.device)
