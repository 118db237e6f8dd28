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


def edge_messages(dims, flags, row, col, ea, x3, P, Q, lp, z1_shift=None):
    """Per edge: -> (destination row, m [E,64], Δx [E,3] (normalized under FLAG_NORMALIZE), φ [E], Σ_k |w3_k·s_k| [E],
    the magnitudes of the 64 products φ = Σ_k w3_k·s_k sums)."""
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
    s = F.silu(m @ f["E_WC"] + f["E_BC"])
    return r, m, dx, s @ f["E_W3"], s.abs() @ f["E_W3"].abs()


def edge_stage(dims, flags, row, col, ea, x3, P, Q, lp, z1_shift=None):
    """-> (agg_m [N,64] sums, agg_x [N,3] sums).  z1_shift: optional [E,64] added to the first pre-activation (zeros
    whose gradient is the per-edge g_z1)."""
    N = dims[0]
    r, m, dx, phi, _ = edge_messages(dims, flags, row, col, ea, x3, P, Q, lp, z1_shift)
    agg_m = torch.zeros(N, H, dtype=P.dtype, device=P.device).index_add(0, r, m)
    agg_x = torch.zeros(N, 3, dtype=P.dtype, device=P.device).index_add(0, r, dx * phi.unsqueeze(1))
    return agg_m, agg_x


def virtual_messages(dims, batch32, x3, Hn, Xv, G, lp):
    """Per node: -> (graph, ΔX [N,3,C], mv [N,C,64], φ_xv [N,C], φ_X [N,C], and the magnitudes of the products the two
    heads sum, Σ_k |w3_k·s_k| [N,C] each)."""
    N, B, A, C, Na = dims
    f = _fields(lp, A, C, Na)
    b = batch32.long()
    dX = Xv[b] - x3.unsqueeze(-1)                                  # [N,3,C]
    vr = dX.norm(dim=1)                                            # [N,C]
    pre = Hn.unsqueeze(1) + G[b] + vr.unsqueeze(-1) * f["V_W1R"]   # [N,C,64]
    mv = F.silu(F.silu(pre) @ f["V_W2"] + f["V_B2"])
    s_xv = F.silu(mv @ f["V_WXV"] + f["V_BXV"])
    s_x = F.silu(mv @ f["V_WX"] + f["V_BX"])
    return (b, dX, mv, s_xv @ f["V_W3XV"], s_x @ f["V_W3X"], s_xv.abs() @ f["V_W3XV"].abs(),
            s_x.abs() @ f["V_W3X"].abs())


def virtual_stage(dims, flags, batch32, x3, Hn, Xv, G, lp):
    """-> (agg_v [N,64] means over channels, trans_v [N,3], vsum_tail [B, 3C + 64C] sums)"""
    N, B, A, C, Na = dims
    b, dX, mv, phi_xv, phi_x, _, _ = virtual_messages(dims, batch32, x3, Hn, Xv, G, lp)
    trans_v = (-dX * phi_xv.unsqueeze(1)).mean(-1)
    tail_x = torch.zeros(B, 3 * C, dtype=Hn.dtype, device=Hn.device).index_add(0, b, (dX * phi_x.unsqueeze(1)).reshape(N, 3 * C))
    tail_m = torch.zeros(B, C * H, dtype=Hn.dtype, device=Hn.device).index_add(0, b, mv.reshape(N, C * H))
    return mv.mean(1), trans_v, torch.cat([tail_x, tail_m], 1)


# ---- the forward stages with the magnitudes of their signed sums, the scale a sum that cancels is judged against.  A
# coordinate sum Σ Δx·φ is fully expanded a sum of the products Δx·w3_k·s_k: φ = Σ_k w3_k·s_k is itself a 64-term dot
# product that cancels, and a kernel's error on it scales with Σ_k |w3_k·s_k|, not with |φ|
def edge_terms(dims, flags, row, col, ea, x3, P, Q, lp):
    """-> (agg_m [N,64], agg_x [N,3], x_terms [N,3] = Σ_e |Δx|·Σ_k |w3_k·s_k| per row and component)."""
    N = dims[0]
    r, m, dx, phi, phi_mag = edge_messages(dims, flags, row, col, ea, x3, P, Q, lp)
    z = lambda w: torch.zeros(N, w, dtype=P.dtype, device=P.device)
    return (z(H).index_add(0, r, m), z(3).index_add(0, r, dx * phi.unsqueeze(1)),
            z(3).index_add(0, r, dx.abs() * phi_mag.unsqueeze(1)))


def virtual_terms(dims, batch32, x3, Hn, Xv, G, lp):
    """-> dict: agg_v [N,64], trans_v [N,3], trans_terms [N,3] = mean_c |ΔX|·Σ_k |w3xv_k·s_k|, tail_x [B,3C] = Σ ΔX·φ_X
    and tail_x_terms = Σ |ΔX|·Σ_k |w3x_k·s_k| per graph ([3][C] order, as vsum[:, 4:4+3C]), tail_m [B,64C] = Σ mv per
    graph."""
    N, B, A, C, Na = dims
    b, dX, mv, phi_xv, phi_x, mag_xv, mag_x = virtual_messages(dims, batch32, x3, Hn, Xv, G, lp)
    z = lambda w: torch.zeros(B, w, dtype=Hn.dtype, device=Hn.device)
    return dict(agg_v=mv.mean(1), trans_v=(-dX * phi_xv.unsqueeze(1)).mean(-1),
                trans_terms=(dX.abs() * mag_xv.unsqueeze(1)).mean(-1),
                tail_x=z(3 * C).index_add(0, b, (dX * phi_x.unsqueeze(1)).reshape(N, 3 * C)),
                tail_x_terms=z(3 * C).index_add(0, b, (dX.abs() * mag_x.unsqueeze(1)).reshape(N, 3 * C)),
                tail_m=z(C * H).index_add(0, b, mv.reshape(N, C * H)))
