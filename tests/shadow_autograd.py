"""Differentiable (functional) torch restatements of the C-ABI stages — TEST INFRASTRUCTURE for the backward kernels.

Same decomposition as tests/shadow_backend.py (per-node P/Q/Hn split, SUMS instead of means, packed vsum), but
out-of-place so that torch.autograd can differentiate them; the gradient tests run them in float64 and compare the
CUDA backward kernels with torch.autograd.grad.  Never imported by the package.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from distegnn_b200 import _lib
from .shadow_backend import _fields

H = 64


def edge_stage(dims, flags, row, col, ea, x3, P, Q, lp, z1_shift=None):
    """-> (agg_m [N,64] sums, agg_x [N,3] sums).  z1_shift: optional [E,64] added to the first pre-activation (zeros
    whose gradient is the per-edge g_z1)."""
    N, E, A, C, Na = dims
    f = _fields(lp, A, C, Na)
    r, c = row.long(), col.long()
    dx = x3[r] - x3[c]
    radial = (dx ** 2).sum(1, keepdim=True)
    if flags & _lib.FLAG_NORMALIZE:
        dx = dx / (radial.sqrt().detach() + 1e-8)
    pre = P[r] + Q[c] + radial * f["E_W1R"]
    if A:
        pre = pre + ea @ f["E_W1E"]
    if z1_shift is not None:
        pre = pre + z1_shift
    m = F.silu(F.silu(pre) @ f["E_W2"] + f["E_B2"])
    phi = F.silu(m @ f["E_WC"] + f["E_BC"]) @ f["E_W3"]
    agg_m = torch.zeros(N, H, dtype=P.dtype, device=P.device).index_add(0, r, m)
    agg_x = torch.zeros(N, 3, dtype=P.dtype, device=P.device).index_add(0, r, dx * phi.unsqueeze(1))
    return agg_m, agg_x


def virtual_stage(dims, flags, batch32, x3, Hn, Xv, G, lp):
    """-> (agg_v [N,64] means over channels, trans_v [N,3], vsum_tail [B, 3C + 64C] sums)"""
    N, B, A, C, Na = dims
    f = _fields(lp, A, C, Na)
    b = batch32.long()
    dX = Xv[b] - x3.unsqueeze(-1)                                  # [N,3,C]
    vr = dX.norm(dim=1)                                            # [N,C]
    pre = Hn.unsqueeze(1) + G[b] + vr.unsqueeze(-1) * f["V_W1R"]   # [N,C,64]
    mv = F.silu(F.silu(pre) @ f["V_W2"] + f["V_B2"])
    phi_xv = F.silu(mv @ f["V_WXV"] + f["V_BXV"]) @ f["V_W3XV"]    # [N,C]
    phi_x = F.silu(mv @ f["V_WX"] + f["V_BX"]) @ f["V_W3X"]
    trans_v = (-dX * phi_xv.unsqueeze(1)).mean(-1)
    tail_x = torch.zeros(B, 3 * C, dtype=Hn.dtype, device=Hn.device).index_add(0, b, (dX * phi_x.unsqueeze(1)).reshape(N, 3 * C))
    tail_m = torch.zeros(B, C * H, dtype=Hn.dtype, device=Hn.device).index_add(0, b, mv.reshape(N, C * H))
    return mv.mean(1), trans_v, torch.cat([tail_x, tail_m], 1)
