"""Shared helpers for the test-suite (fixtures loader, error metrics)."""
from __future__ import annotations

import ast
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SINGLE_CASES = ["nbody24_norm", "fluid160_c5", "batch3_c8_multigraph"]
DIST_CASE = "dist2_fluid300_c5"
INPUT_KEYS = ["node_feat", "node_loc", "node_vel", "loc_mean", "edge_index", "data_batch", "edge_attr",
              "node_attr"]


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    kw = ast.literal_eval(str(z["meta.kw"]))
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd.")}
    return z, kw, sd


def golden_inputs(z, prefix="in."):
    d = {k: (torch.from_numpy(z[prefix + k]) if prefix + k in z.files else None) for k in INPUT_KEYS}
    return d


def golden_trace(z, key, prefix="trace."):
    out, i = [], 0
    while f"{prefix}{key}.{i}" in z.files:
        out.append(torch.from_numpy(z[f"{prefix}{key}.{i}"]))
        i += 1
    return out


def max_abs(a, b):
    return float((a.double() - b.double()).abs().max()) if a.numel() else 0.0


TOL = 2e-5              # row-wise relative error against float64 (the per-stage bound of the kernels)
# Where a case needs more than TOL, the tensor-core kernel must still be within this factor of the twin's error (its
# operands are split into two fp16 terms with one power-of-two scale per row; the worst ratio measured is 9, on the
# rescued rows of test_edge_bwd_rescued_and_guarded_rows).
TWIN_FACTOR = 16
FLOOR = 1e-30           # denominator floor of the row-wise error (the smallest rows here are about 1e-20)


def rowwise(got, ref, zero_rows=None):
    """Largest row-wise relative error; rows flagged in `zero_rows` must be exactly zero in both."""
    got = got.detach().double().reshape(got.shape[0], -1)
    ref = ref.detach().double().reshape(ref.shape[0], -1)
    assert torch.isfinite(got).all(), "non-finite output"
    if zero_rows is not None and bool(zero_rows.any()):
        assert float(ref[zero_rows].abs().max()) == 0.0
        assert float(got[zero_rows].abs().max()) == 0.0, "structurally zero row is not exactly zero"
        got, ref = got[~zero_rows], ref[~zero_rows]
    if got.shape[0] == 0:
        return 0.0
    return float(((got - ref).abs().amax(1) / ref.abs().amax(1).clamp(min=FLOOR)).max())


def terms_rowwise(got, ref, terms):
    """Row-wise error of a short signed sum, relative to the largest magnitude of the terms summed into the row."""
    assert torch.isfinite(got).all(), "non-finite output"
    if got.shape[0] == 0:
        return 0.0
    err = (got.double() - ref.double()).abs().amax(1)
    return float((err / terms.amax(1).clamp(min=FLOOR)).max())


def rel(got, ref):
    assert torch.isfinite(got).all(), "non-finite output"
    return float((got.double() - ref.double()).abs().max()) / max(FLOOR, float(ref.abs().max()))


def check_bounds(errs, tols):
    """errs: {kernel: {field: error}}.  Every field within its bound; a field above TOL in the tensor-core kernel within
    TWIN_FACTOR of the twin's error (kernels without a twin: no 'twin' entry, every field within its bound)."""
    for kind, e in errs.items():
        bad = {f: v for f, v in e.items() if v > tols.get(f, TOL)}
        assert not bad, (kind, bad)
    twin = errs.get("twin", {})
    for f, v in errs["tc"].items():
        if v > TOL and f in twin:
            assert v <= TWIN_FACTOR * max(twin[f], TOL), (f, v, twin[f])


def within_rerun_bound(a, b):
    """Two launches that differ only in the order of their float atomics (DESIGN §5)."""
    return float((a - b).abs().max()) <= 2e-6 * max(1.0, float(a.abs().max()))


def rel_disp_err(out, ref, pos):
    """‖(out−pos)−(ref−pos)‖∞ / ‖ref−pos‖∞ — parity on the *displacement*, which is what the model
    actually computes (SURVEY §7 'parity is deceptively easy at init')."""
    den = float((ref.double() - pos.double()).abs().max())
    return max_abs(out, ref) / max(den, 1e-30)
