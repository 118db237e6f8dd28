"""Golden vectors for the edge cutoff (FastEGNN's cutoff_edges mode), from the UNMODIFIED reference.

    python oracle/make_golden_cutoff.py       # build container only (/root/reference)

Calls `cutoff_edge` of datasets/process_dataset.py:300-305 as it lies, once per sample as `process_key` does.  The module
is imported unmodified; the packages it imports but `cutoff_edge` does not use (h5py, msgpack(_numpy), zstandard,
MDAnalysis(Data), joblib, torch_geometric.data / .nn.pool, and the sibling module datasets.distribute_graphs) are
`sys.modules` stubs.  Writes tests/golden/cutoff_*.npz with: pos [N,3] fp32, batch [N], the candidate edge list
`candidates` int64 [2,E] in the order given to the reference (per graph: destination ascending, then source ascending),
`rate`, `radius` (−1: fully connected), and the reference's kept edge list `kept` (samples concatenated, node ids global).  Test infrastructure.

Cases: (a) dyadic lattices — every squared distance is exact in fp32, so torch's lengths equal the kernel's bit for bit
and there are ties far beyond the mirror pairs — at rates 0.5 and 0.3; (b) a 2k-node fluid-like radius graph at 0.5;
(c) three fully connected 100-node N-body graphs at 0.5; (d) graphs with odd k_b, so one mirror pair is split.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")


def import_cutoff_edge():
    class _Stub(types.ModuleType):
        def __getattr__(self, name):
            if name.startswith("__"):
                raise AttributeError(name)
            return lambda *a, **k: None

    for name in ("h5py", "msgpack", "msgpack_numpy", "zstandard", "MDAnalysis", "MDAnalysis.transformations",
                 "MDAnalysis.analysis", "MDAnalysis.analysis.distances", "MDAnalysisData", "joblib",
                 "torch_geometric", "torch_geometric.data", "torch_geometric.nn", "torch_geometric.nn.pool",
                 "datasets.distribute_graphs"):
        sys.modules[name] = _Stub(name)
    import importlib.util
    # the reference's own `datasets` / `utils` packages (an installed package of the same name must not shadow them)
    for pkg in ("datasets", "utils"):
        mod = types.ModuleType(pkg)
        mod.__path__ = [os.path.join(REF, pkg)]
        sys.modules[pkg] = mod
    spec = importlib.util.spec_from_file_location("datasets.process_dataset",
                                                  os.path.join(REF, "datasets", "process_dataset.py"))
    P = importlib.util.module_from_spec(spec)     # the unmodified reference module
    spec.loader.exec_module(P)
    return P.cutoff_edge


def _pairs(pos, r=None):
    """Ordered pairs of one graph (i != j, and |x_i − x_j| < r unless r is None), destination ascending then source."""
    n = pos.shape[0]
    d = np.linalg.norm(pos[:, None, :].astype(np.float64) - pos[None, :, :], axis=2)
    ok = ~np.eye(n, dtype=bool) if r is None else (d < r) & ~np.eye(n, dtype=bool)
    i, j = np.nonzero(ok)
    return np.stack([i, j]).astype(np.int64)


def _case(cutoff_edge, name, samples, rate, radius):
    """samples: list of (pos fp32 [n,3], candidates [2,E] local ids)."""
    pos, batch, cand, kept, off = [], [], [], [], 0
    for b, (p, ei) in enumerate(samples):
        out = cutoff_edge(torch.from_numpy(ei), torch.from_numpy(p), rate)
        pos.append(p)
        batch.append(np.full(p.shape[0], b, dtype=np.int64))
        cand.append(ei + off)
        kept.append(out.numpy() + off)
        off += p.shape[0]
    path = os.path.join(OUT, f"cutoff_{name}.npz")
    np.savez_compressed(path, pos=np.concatenate(pos), batch=np.concatenate(batch), candidates=np.concatenate(cand, 1),
                        rate=np.float64(rate), radius=np.float64(radius), kept=np.concatenate(kept, 1))
    print(path, "candidates", sum(c.shape[1] for c in cand), "kept", sum(k.shape[1] for k in kept))


def main():
    cutoff_edge = import_cutoff_edge()
    rng = np.random.default_rng(0)
    # (a) dyadic lattices: coordinates k/4, radius graph of r = 0.8 (neighbours up to (2,1,0)/4 ...), two graphs
    lat = []
    for shape in ((5, 4, 3), (3, 3, 3)):
        g = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"), -1).reshape(-1, 3)
        p = (0.25 * g + 0.25 * rng.integers(0, 4, size=3)).astype(np.float32)
        p = p[rng.permutation(p.shape[0])]
        lat.append((p, _pairs(p, 0.8)))
    _case(cutoff_edge, "lattice_r05", lat, 0.5, 0.8)
    _case(cutoff_edge, "lattice_r03", lat, 0.3, 0.8)
    # (b) fluid-like radius graph, 2k nodes in a unit box, ~20 neighbours each
    p = rng.random((2000, 3)).astype(np.float32)
    _case(cutoff_edge, "fluid2k_r05", [(p, _pairs(p, 0.135))], 0.5, 0.135)
    # (c) three fully connected 100-node N-body graphs
    nb = [(rng.standard_normal((100, 3)).astype(np.float32), None) for _ in range(3)]
    _case(cutoff_edge, "nbody3x100_r05", [(p, _pairs(p)) for p, _ in nb], 0.5, -1)
    # (d) odd k_b: fully connected 5-node graphs (E = 20) at 0.25 -> k = 15, and 4-node (E = 12) -> k = 9
    odd = [(rng.standard_normal((5, 3)).astype(np.float32), None), (rng.standard_normal((4, 3)).astype(np.float32), None)]
    _case(cutoff_edge, "odd_k", [(p, _pairs(p)) for p, _ in odd], 0.25, -1)


if __name__ == "__main__":
    main()
