"""Restatement of the edge cutoff (FastEGNN's cutoff_edges mode) in numpy, for the tests.

The reference (datasets/process_dataset.py:300-305, once per sample) sorts a graph's edges by length and keeps the first
int(E * (1 - cutoff_rate)).  The rule restated here is the one csrc/cutoff_csr.cu implements (DESIGN §16):
  - candidates: the edges of a CSR graph; graph b's are those whose destination row is one of its nodes
  - k_b = int(E_b * (1 - rate)), Python float arithmetic (fp64)
  - kept: the k_b smallest by (length, position in the candidate CSR): a stable sort, NaN last
  - output: the kept edges in candidate order, rowptr_out[i] = kept edges before rowptr_in[i]
Lengths are fp64 ‖pos_i − pos_j‖ by default, or given (e.g. the kernel's fp32 lengths, for a bit-exact comparison).
"""
from __future__ import annotations

from typing import Optional

import numpy as np


def k_of(E: int, rate: float) -> int:
    return int(E * (1 - rate))


def lengths64(pos, row, col) -> np.ndarray:
    p = np.asarray(pos, dtype=np.float64)
    return np.linalg.norm(p[np.asarray(row)] - p[np.asarray(col)], axis=1)


def keep_mask(row, col, pos, rate: float, batch=None, n_graphs: Optional[int] = None,
              lengths: Optional[np.ndarray] = None) -> np.ndarray:
    """bool [E]: which candidates (in the given order, grouped by graph) are kept."""
    row, col = np.asarray(row, dtype=np.int64), np.asarray(col, dtype=np.int64)
    E = row.shape[0]
    length = lengths64(pos, row, col) if lengths is None else np.asarray(lengths)
    g = np.zeros(E, dtype=np.int64) if batch is None else np.asarray(batch, dtype=np.int64)[row]
    B = (int(g.max()) + 1 if E else 1) if n_graphs is None else int(n_graphs)
    counts = np.bincount(g, minlength=B)
    k = np.array([k_of(int(c), rate) for c in counts], dtype=np.int64)
    order = np.lexsort((np.arange(E), length, g))           # by graph, then length (NaN last), then position
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    gs = g[order]
    rank = np.arange(E) - start[gs]
    mask = np.zeros(E, dtype=bool)
    mask[order[rank < k[gs]]] = True
    return mask


def cutoff_csr(rowptr, row, col, pos, rate: float, batch=None, n_graphs: Optional[int] = None,
               lengths: Optional[np.ndarray] = None):
    """The kept sub-graph: (rowptr_out [N+1], row_out, col_out, length_out, mask) in candidate CSR order."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    row, col = np.asarray(row, dtype=np.int64), np.asarray(col, dtype=np.int64)
    length = lengths64(pos, row, col) if lengths is None else np.asarray(lengths)
    mask = keep_mask(row, col, pos, rate, batch, n_graphs, length)
    before = np.concatenate([[0], np.cumsum(mask)])
    return before[rowptr], row[mask], col[mask], length[mask], mask


def cutoff_edge_index(edge_index, pos, rate: float, batch=None, n_graphs: Optional[int] = None,
                      lengths: Optional[np.ndarray] = None) -> np.ndarray:
    """The same rule on an int64 [2,E] edge list whose graphs are contiguous: the kept columns, in the given order."""
    ei = np.asarray(edge_index)
    return ei[:, keep_mask(ei[0], ei[1], pos, rate, batch, n_graphs, lengths)]
