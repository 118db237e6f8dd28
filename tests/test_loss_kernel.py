"""Fused training loss (distegnn_b200.train_loss, csrc/loss.cu) against a float64 restatement, at the shapes where its
structure breaks: more than one node block of LOSS_NODES_PER_CTA = 2048 nodes (graphs straddling a block edge, 1M
nodes), every channel count 1..16 at S·C below, at and far above the 256 threads of an MMD block, sample rows padded
with −1, graph ids without nodes, thousands of MMD blocks, coincident points (the `dist > 0` guards), underflowing and
saturated kernel terms, accumulation steps, the upstream gradient, world sizes 3 and 4 with an empty rank, and a NaN
prediction.

Every output is checked element by element, not by one max over the tensor (a wrong row whose values are small next to
the largest row passes that):
  g_pred   each element against its own float64 value; an element with pred == target must be exactly 0
  g_Xv     each entry (b, k, c) against cV·Σ|term| over the C + S pair terms summed into it (the sum cancels)
  loss, logged   against the float64 value (the MSE part is a sum of positive terms)
  mmd      against |l_vv|/(B·C²) + 2|l_rv|/(B·S·C) (the difference cancels)
Each bound is γ_n = n·u/(1 − n·u), u = 2⁻²⁴, with n counted from the kernels' summation structure (see `bounds`), and
every case prints its observed errors next to them."""
import math

import pytest
import torch

from distegnn_b200.loss import graph_offsets
from oracle import train_loss_oracle as tlo
from tests.helpers import FLOOR
from tests.test_loss import CASES, _pad, load

U = 2.0 ** -24                      # unit roundoff of float32
NODES_PER_CTA, THREADS = 2048, 256  # loss.cu: LOSS_NODES_PER_CTA, LOSS_THREADS
CHAIN = -(-3 * NODES_PER_CTA // THREADS)   # fmaf terms per thread of a node block: ⌈6144/256⌉ = 24
TREE = 5 + 3                        # block_sum: 5 shuffle levels in a warp, 3 over the 8 warps


def gamma(n):
    return n * U / (1 - n * U)


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatement
# ---------------------------------------------------------------------------------------------------------------------

def _dist(diff):
    """‖diff‖ over the last axis with cdist's zero gradient at coincident points."""
    d2 = (diff * diff).sum(-1)
    pos = d2 > 0
    return torch.where(pos, torch.sqrt(torch.where(pos, d2, torch.ones_like(d2))), torch.zeros_like(d2))


def reference(pred, target, Xv, batch, samples, node_counts, rank, sigma, weight, accumulation_steps=1):
    """Vectorised float64 restatement of oracle/train_loss_oracle.py on the padded samples [B,S] (−1 = none).

    l_rv is divided by the full S, the kernel is exp(−‖x−y‖/(2σ²)) (distance not squared), and the gradient at
    coincident points is zero.  Returns loss, this rank's term of the logged loss n_r/Σn·MSE_r, mmd, g_pred, g_Xv and
    the magnitudes the bounds need: mse, mmd_scale = l_vv/(B·C²) + 2·l_rv/(B·S·C), g_terms [B,3,C] = |cV|·Σ|term|, and
    max_arg, the largest ‖x−y‖/(2σ²) of a term whose float32 value is normal."""
    world = len(node_counts)
    n_r, n_tot = float(node_counts[rank]), float(sum(node_counts))
    B, _, C = Xv.shape
    S = samples.shape[1]
    p = pred.detach().double().requires_grad_(True)
    V = Xv.detach().double().requires_grad_(True)
    t = target.detach().double()
    sse = ((p - t) ** 2).sum()
    mse = sse / (3 * n_r) if n_r > 0 else sse * math.nan        # the reference's mean over an empty tensor: NaN
    inv2s2 = 1.0 / (2 * sigma * sigma)
    Vt = V.transpose(1, 2)                                        # [B,C,3]
    dvv = Vt[:, :, None, :] - Vt[:, None, :, :]                   # [B,C,C,3] every ordered pair (c, c')
    rvv = _dist(dvv)
    kvv = torch.exp(-rvv * inv2s2)
    smp = samples.long()
    b_i, s_i = (smp >= 0).nonzero(as_tuple=True)                  # the slots that hold a node
    off = graph_offsets(batch, B)
    drv = t[off[b_i] + smp[b_i, s_i]][:, None, :] - Vt[b_i]      # [M,C,3]
    rrv = _dist(drv)
    krv = torch.exp(-rrv * inv2s2)
    l_vv, l_rv = kvv.sum(), krv.sum()
    mmd = l_vv / (B * C * C) - 2 * l_rv / (B * S * C)
    coef = world * n_r / n_tot / accumulation_steps
    loss = coef * (mse + weight * mmd)
    g_pred, g_Xv = torch.autograd.grad(loss, [p, V], allow_unused=True)
    with torch.no_grad():
        fvv = torch.where(rvv > 0, 2.0 / (B * C * C) * kvv * inv2s2 / rvv.clamp(min=FLOOR), torch.zeros_like(rvv))
        frv = torch.where(rrv > 0, 2.0 / (B * S * C) * krv * inv2s2 / rrv.clamp(min=FLOOR), torch.zeros_like(rrv))
        terms = (fvv[..., None] * dvv.abs()).sum(2)               # [B,C,3]
        terms.index_add_(0, b_i, frv[..., None] * drv.abs())
        args = torch.cat([rvv.flatten(), rrv.flatten()]) * inv2s2
        args = args[args <= 87.0]                                 # exp(−87) > 2⁻¹²⁶: k normal in float32
    return dict(loss=float(loss.detach()), logged=float(n_r / n_tot * mse.detach()), mmd=float(mmd.detach()),
                g_pred=g_pred if g_pred is not None else torch.zeros_like(t), g_Xv=g_Xv,
                mse=float(mse.detach()), mmd_scale=float(l_vv.detach() / (B * C * C) + 2 * l_rv.detach() / (B * S * C)),
                g_terms=abs(coef * weight) * terms.transpose(1, 2), max_arg=float(args.max()), coef=coef)


# ---------------------------------------------------------------------------------------------------------------------
# bounds and metrics
# ---------------------------------------------------------------------------------------------------------------------

def bounds(ref, n_nodes, C, S, B, weight, world=1, upstream=False):
    """Relative error bounds of the kernels' float32 outputs, n counted from loss.cu (n_nodes: nodes of every rank)."""
    nb = max(max(1, -(-n // NODES_PER_CTA)) for n in n_nodes)
    # SSE of a rank: d = pred − target and d·d (2 per term), a chain of CHAIN fmaf per thread, TREE levels, ×(1/3)
    # (the rounded constant and the product: 2), then one atomicAdd per node block
    e_sse = gamma(2 + CHAIN + TREE + 2 + nb)
    # k = expf(−dist·inv2s2): the argument carries 7 roundings (dx, the squares and two adds, sqrtf, σ·σ, the
    # reciprocal, the product), which exp turns into 7·arg·u relative; expf itself is within 2 ulp (4 u)
    e_k = 7 * ref["max_arg"] * U
    # l_vv, l_rv (positive): k (4 u + e_k), ⌈S·C/256⌉ terms per thread (C·C ≤ 256 needs one pass), TREE levels, one
    # atomicAdd per graph; then the divisions by B·C·C and B·S·C (the products and the quotient: 3), the subtraction (1)
    passes = -(-S * C // THREADS)
    e_mmd = gamma(4 + passes + TREE + B + 4) + e_k
    # finalize: coef = world·(n_r/n_tot)·(1/accum) (4), mse = acc/n_r (1), float(weight) and weight·mmd (2), the sum
    # (1), coef·(…) (1)
    chain = gamma(9)
    coef, w = ref["coef"], abs(weight)
    loss_abs = coef * ref["mse"] * (e_sse + chain) + coef * w * (e_mmd * ref["mmd_scale"] + chain * abs(ref["mmd"]))
    return dict(
        loss=loss_abs / abs(ref["loss"]) if ref["loss"] else 0.0,
        # the packed vectors of the ranks are added by world − 1 float32 sums, then packed[1]/n_tot (1)
        logged=gamma(2 + CHAIN + TREE + 2 + nb + world),
        mmd=e_mmd,
        # cp = coef·2/(3·n_r): coef (4), 3·n_r and the quotient (2); d = pred − target (1); cp·d (1); g_loss·g (1)
        g_pred=gamma(8 + upstream),
        # a term w·k·inv2s2/dist·dx: w = 1/(B·C·C) or 2/(B·S·C) (3), three products and the quotient (4), inv2s2
        # (2), dist (4), dx (1), k (4 + e_k); C + S terms added by shared-memory atomics (C + S − 1); cV = coef·weight
        # (6) and cV·(…) (1); g_loss·g (1)
        g_Xv=gamma(18 + C + S - 1 + 7 + upstream) + e_k,
    )


def elem_err(got, ref):
    """Largest |got − ref|/|ref| element by element; elements whose reference is 0 must be exactly 0."""
    got, ref = got.detach().double(), ref.detach().double()
    assert torch.isfinite(got).all(), "non-finite output"
    zero = ref == 0
    assert bool((got[zero] == 0).all()), "an element with pred == target is not exactly 0"
    if bool(zero.all()):
        return 0.0
    return float(((got - ref).abs()[~zero] / ref.abs()[~zero]).max())


def terms_err(got, ref, terms):
    """Largest |got − ref| of an entry over the magnitudes summed into it."""
    got, ref = got.detach().double(), ref.detach().double()
    assert torch.isfinite(got).all(), "non-finite output"
    return float(((got - ref).abs() / terms.clamp(min=FLOOR)).max())


def scalar_err(got, ref, scale=None):
    assert math.isfinite(got), "non-finite output"
    return abs(got - ref) / max(FLOOR, abs(ref) if scale is None else scale)


def global_gate(got, ref):
    """The one-max-over-the-tensor gate of tests/test_loss.py."""
    return float((got.double() - ref).abs().max() / ref.abs().max())


def check(name, got, ref, bd, skip=()):
    """got: loss, logged, mmd (floats), g_pred [N,3], g_Xv [B,3,C] from the kernels."""
    errs = {}
    if "loss" not in skip:
        errs["loss"] = scalar_err(got["loss"], ref["loss"])
    if "logged" not in skip:
        errs["logged"] = scalar_err(got["logged"], ref["logged"])
    if "mmd" not in skip:
        errs["mmd"] = scalar_err(got["mmd"], ref["mmd"], ref["mmd_scale"])
    if "g_pred" not in skip:
        errs["g_pred"] = elem_err(got["g_pred"], ref["g_pred"])
    if "g_Xv" not in skip:
        errs["g_Xv"] = terms_err(got["g_Xv"], ref["g_Xv"], ref["g_terms"])
    print(f"{name}: " + "  ".join(f"{k} {v:.2e} (bound {bd[k]:.2e})" for k, v in errs.items()))
    bad = {k: (v, bd[k]) for k, v in errs.items() if not v <= bd[k]}
    assert not bad, (name, bad)
    return errs


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------

def make_case(sizes, C, mmd_samples, *, seed, sigma=3.0, weight=0.01, spread=2.0):
    """Graphs of `sizes` nodes (0 allowed), target ~ spread·N(0,1), pred = target + 0.2·N(0,1) except every 97th row,
    where pred == target (g_pred exactly 0), samples drawn like the reference (randperm per graph, −1 padded)."""
    g = torch.Generator().manual_seed(seed)
    B, N, S = len(sizes), sum(sizes), mmd_samples * C
    batch = torch.repeat_interleave(torch.arange(B), torch.tensor(sizes, dtype=torch.long))
    target = spread * torch.randn(N, 3, generator=g)
    pred = target + 0.2 * torch.randn(N, 3, generator=g)
    pred[::97] = target[::97]
    Xv = spread * torch.randn(B, 3, C, generator=g)
    samples = _pad([torch.randperm(n, generator=g)[:S] for n in sizes], S)
    return dict(pred=pred, target=target, Xv=Xv, batch=batch, samples=samples, C=C, S=S, mmd_samples=mmd_samples,
                sigma=sigma, weight=weight)


def ref_of(case, node_counts=None, rank=0, accum=1):
    n = case["pred"].shape[0]
    return reference(case["pred"], case["target"], case["Xv"], case["batch"], case["samples"],
                     node_counts or [n], rank, case["sigma"], case["weight"], accum)


def bounds_of(case, ref, node_counts=None, **kw):
    return bounds(ref, node_counts or [case["pred"].shape[0]], case["C"], case["S"], case["Xv"].shape[0],
                  case["weight"], world=len(node_counts or [0]), **kw)


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def fused(case, accum=1, loc_mean=None):
    """One rank through train_loss with explicit samples; loss.backward() with the upstream gradient 1."""
    from distegnn_b200 import train_loss
    d = dev()
    p = case["pred"].to(d).requires_grad_(True)
    V = case["Xv"].to(d).requires_grad_(True)
    loss, info = train_loss(p, case["target"].to(d), V, case["batch"].to(d), world_size=1,
                            mmd_samples=case["mmd_samples"], mmd_sigma=case["sigma"], mmd_weight=case["weight"],
                            accumulation_steps=accum, loc_mean=None if loc_mean is None else loc_mean.to(d),
                            samples=case["samples"].to(d))
    loss.backward()
    torch.cuda.synchronize()
    return dict(loss=float(loss.detach()), logged=float(info["logged"]), mmd=float(info["mmd"]),
                dev=float(info["loc_mean_dev"]), g_pred=p.grad.cpu(), g_Xv=V.grad.cpu())


def run_case(name, case, accum=1):
    ref = ref_of(case, accum=accum)
    return check(name, fused(case, accum), ref, bounds_of(case, ref))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement against the oracle, and the metrics against the global gate
# ---------------------------------------------------------------------------------------------------------------------

def _oracle(case, node_counts, rank, accum, weight=None):
    """oracle/train_loss_oracle.py on the same inputs: loss, logged, g_pred, g_Xv."""
    p = case["pred"].double().requires_grad_(True)
    V = case["Xv"].double().requires_grad_(True)
    smp = [row[row >= 0].long() for row in case["samples"]]
    loss, logged = tlo.train_loss(p, case["target"].double(), V, case["batch"], smp, node_counts=node_counts, rank=rank,
                                  sigma=case["sigma"], weight=case["weight"] if weight is None else weight,
                                  samples_per_channel=case["mmd_samples"], accumulation_steps=accum)
    gp, gV = torch.autograd.grad(loss, [p, V])
    return float(loss.detach()), float(logged), gp, gV


def _golden_case(name):
    z, meta, smp = load(name)
    S = meta["samples"] * meta["C"]
    return dict(pred=torch.from_numpy(z["pred"]), target=torch.from_numpy(z["target"]), Xv=torch.from_numpy(z["V"]),
                batch=torch.from_numpy(z["batch"]), samples=_pad(smp, S), C=meta["C"], S=S,
                mmd_samples=meta["samples"], sigma=meta["sigma"], weight=meta["weight"])


def _random_padded_case():
    c = make_case([0, 3, 19, 20, 21, 40, 0], 4, 5, seed=11, sigma=1.5, weight=0.05)   # S = 20
    return c, [int(c["pred"].shape[0]), 17, 123], 0, 3


@pytest.mark.parametrize("which", CASES + ["random_padded_world3"])
def test_restatement_matches_the_oracle(which):
    """The vectorised restatement agrees with the oracle within 1e-12 (the oracle is pinned to the reference's own train
    step by the loss_* fixtures, tests/test_loss.py)."""
    if which in CASES:
        case = _golden_case(which)
        counts, rank, accum = [int(case["pred"].shape[0])], 0, 1
    else:
        case, counts, rank, accum = _random_padded_case()
    ref = ref_of(case, counts, rank, accum)
    loss, logged, gp, gV = _oracle(case, counts, rank, accum)
    # the oracle has no MMD output: the weight-linear part of its loss is coef·weight·mmd
    mmd = (loss - _oracle(case, counts, rank, accum, weight=0.0)[0]) / (ref["coef"] * case["weight"])
    assert scalar_err(ref["loss"], loss) <= 1e-12
    assert scalar_err(ref["logged"], logged) <= 1e-12
    assert scalar_err(ref["mmd"], mmd, ref["mmd_scale"]) <= 1e-12
    assert elem_err(ref["g_pred"], gp) <= 1e-12
    assert terms_err(ref["g_Xv"], gV, ref["g_terms"]) <= 1e-12


def test_restatement_keeps_the_reference_rules():
    """l_rv over the full S, distance not squared, zero gradient at coincident points — on a hand-sized case."""
    sigma = 2.0
    V = torch.tensor([[[0.0, 0.0], [0.0, 0.0], [0.0, 3.0]]])            # B=1, C=2: V_0 = 0, V_1 = (0,0,3)
    target = torch.tensor([[0.0, 0.0, 0.0], [4.0, 0.0, 0.0]])
    samples = torch.tensor([[0, -1, -1, -1]], dtype=torch.int32)         # S = 4, one slot filled, on top of V_0
    ref = reference(target.clone(), target, V, torch.zeros(2, dtype=torch.long), samples, [2], 0, sigma, 1.0)
    k = math.exp(-3.0 / (2 * sigma * sigma))
    l_vv, l_rv = 2 + 2 * k, 1 + k
    assert abs(ref["mmd"] - (l_vv / 4 - 2 * l_rv / (4 * 2))) <= 1e-15
    # g at V_0: only the vv pair with V_1 (the sample sits on V_0: zero gradient); at V_1: vv pair + rv pair
    dk = k / (2 * sigma * sigma)                                         # −∂k/∂dist
    assert torch.allclose(ref["g_Xv"][0, :, 0], torch.tensor([0.0, 0.0, 2 * dk / 4], dtype=torch.float64), atol=1e-15)
    assert torch.allclose(ref["g_Xv"][0, :, 1],
                          torch.tensor([0.0, 0.0, -2 * dk / 4 + 2 * dk / 8], dtype=torch.float64), atol=1e-15)


def test_metrics_catch_what_the_global_gate_misses():
    """A 1e-4 relative error in one g_pred row of 10⁶, and one in a graph whose g_Xv is 10³ times smaller than the rest
    of the tensor: the element-wise metrics reject both, the one-max-over-the-tensor gates (2e-6 and 2e-5 in
    tests/test_loss.py) accept both."""
    case = make_case([10 ** 6], 2, 1, seed=5)
    ref = ref_of(case)
    bd = bounds_of(case, ref)
    exact = ref["g_pred"].float()
    assert elem_err(exact, ref["g_pred"]) <= bd["g_pred"]              # rounding the reference to float32 passes
    amax = ref["g_pred"].abs().amax(1)
    row = int(amax.masked_fill(amax == 0, math.inf).argmin())          # the smallest row that is not exactly 0
    bad = exact.clone()
    bad[row] *= 1 + 1e-4
    assert elem_err(bad, ref["g_pred"]) > bd["g_pred"]
    assert global_gate(bad, ref["g_pred"]) <= 2e-6

    C = 4
    case = make_case([30, 30, 30, 30], C, 2, seed=6)
    far = torch.tensor([200.0, 0.0, 0.0])                               # graph 1: every pair ≥ 200 apart, σ = 3
    jitter = 0.1 * torch.randn(3, C, generator=torch.Generator().manual_seed(1))
    case["Xv"][1] = far[:, None] * torch.arange(C) + jitter
    lo, hi = int(case["batch"].eq(1).nonzero().min()), int(case["batch"].eq(1).nonzero().max()) + 1
    case["target"][lo:hi] -= 2 * far
    case["pred"][lo:hi] -= 2 * far
    ref = ref_of(case)
    bd = bounds_of(case, ref)
    others = torch.cat([ref["g_Xv"][:1], ref["g_Xv"][2:]])
    assert float(others.abs().max()) >= 1e3 * float(ref["g_terms"][1].max())
    exact = ref["g_Xv"].float()
    assert terms_err(exact, ref["g_Xv"], ref["g_terms"]) <= bd["g_Xv"]
    bad = exact.double()
    bad[1] += 1e-4 * ref["g_terms"][1]
    assert terms_err(bad.float(), ref["g_Xv"], ref["g_terms"]) > bd["g_Xv"]
    assert global_gate(bad.float(), ref["g_Xv"]) <= 2e-5


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the production kernels against the restatement
# ---------------------------------------------------------------------------------------------------------------------

def _block_sizes(N, several):
    """One graph, or graphs that end at 2047, 2048, 2049 (a graph straddles the first node-block edge) and at the
    later block edges."""
    if not several:
        return [N]
    cuts = sorted({c for c in (N // 2, 2047, 2048, 2049, 4096, 6144, 50_000) if 0 < c < N})
    return [b - a for a, b in zip([0] + cuts, cuts + [N])]


@pytest.mark.gpu
@pytest.mark.parametrize("several", [False, True], ids=["one_graph", "several_graphs"])
@pytest.mark.parametrize("N", [2047, 2048, 2049, 4095, 4097, 6145, 100_003])
def test_node_blocks(N, several):
    """More than one node block of the partials and the finalize kernel: g_pred checked on every row."""
    run_case(f"N={N} B={len(_block_sizes(N, several))}", make_case(_block_sizes(N, several), 4, 3, seed=N))


@pytest.mark.gpu
def test_config5_shape():
    """1M nodes in one graph, C = 8, mmd_samples = 50 (S = 400): 489 node blocks added by atomicAdd."""
    run_case("N=1_000_000 B=1 C=8 S=400", make_case([1_000_000], 8, 50, seed=7))


@pytest.mark.gpu
@pytest.mark.parametrize("mmd_samples", [1, 7, 50])
@pytest.mark.parametrize("C", range(1, 17))
def test_every_channel_count(C, mmd_samples):
    """S·C below, at and far above the 256 threads of an MMD block (C·C = 256 at C = 16); one graph with fewer nodes
    than S."""
    S = mmd_samples * C
    run_case(f"C={C} mmd_samples={mmd_samples}", make_case([S + 5, max(1, S // 3), 2], C, mmd_samples, seed=C))


@pytest.mark.gpu
def test_sample_padding():
    """Graphs of 0, 1, S−1, S and S+1 nodes in one batch: every graph below S has −1 padding, l_rv still over S."""
    C, m = 5, 4
    S = C * m
    run_case("sizes 0,1,S-1,S,S+1", make_case([0, 1, S - 1, S, S + 1, 3], C, m, seed=2))


@pytest.mark.gpu
def test_graph_ids_without_nodes():
    """Empty graph ids at the start, in the middle and at the end (equal offsets): each still adds its full l_vv."""
    run_case("empty graph ids", make_case([0, 0, 17, 0, 40, 9, 0, 0], 6, 5, seed=3))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 16])
def test_many_graphs(C):
    """B = 5000 graphs of 1–9 nodes: 5000 MMD blocks, 5000 atomics into each MMD accumulator."""
    sizes = [1 + (i * 7919) % 9 for i in range(5000)]
    run_case(f"B=5000 C={C} mmd_samples=50", make_case(sizes, C, 50, seed=C))


def _geometry(kind):
    C, m = 6, 4
    if kind == "coincident_virtual":
        case = make_case([50, 30, 12], C, m, seed=21)
        case["Xv"][1, :, 3] = case["Xv"][1, :, 1]                         # l_vv pair term 1, zero gradient
    elif kind == "sample_on_virtual":
        case = make_case([50, 30, 12], C, m, seed=22)
        for b, s, c in ((0, 0, 2), (2, 5, 0)):
            n0 = int(case["batch"].eq(b).nonzero().min())
            case["Xv"][b, :, c] = case["target"][n0 + int(case["samples"][b, s])]
    elif kind == "offset_1e4":
        case = make_case([50, 30, 12], C, m, seed=23)
        for b, shift in ((0, 1e4), (2, -1e4)):
            rows = case["batch"] == b
            case["target"][rows] += shift
            case["pred"][rows] += shift
            case["Xv"][b] += shift
    elif kind == "small_sigma":
        # σ = 1/16: a term is exp(−128·dist), so all but the pairs within ~0.7 of each other underflow to 0; every
        # virtual node sits next to one sampled target so that no entry of g_Xv is made of underflowed terms only
        case = make_case([50, 30, 12], C, m, seed=24, sigma=0.0625)
        g = torch.Generator().manual_seed(0)
        for b in range(3):
            n0 = int(case["batch"].eq(b).nonzero().min())
            for c in range(C):
                near = case["target"][n0 + int(case["samples"][b, c])]
                case["Xv"][b, :, c] = near + 0.1 * torch.randn(3, generator=g)
    elif kind == "large_sigma":
        # σ = 1024: every term ≈ 1; graphs fill half of their S slots, so l_vv/(B·C²) ≈ 2·l_rv/(B·S·C) and mmd ≈ 0
        case = make_case([C * m // 2] * 3, C, m, seed=25, sigma=1024.0)
    return case


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["coincident_virtual", "sample_on_virtual", "offset_1e4", "small_sigma",
                                  "large_sigma"])
def test_geometry_edges(kind):
    case = _geometry(kind)
    ref = ref_of(case)
    for k in ("g_pred", "g_Xv"):
        assert torch.isfinite(ref[k]).all()
    if kind == "large_sigma":
        assert abs(ref["mmd"]) <= 1e-3 * ref["mmd_scale"]
    run_case(kind, case)


@pytest.mark.gpu
@pytest.mark.parametrize("accum", [1, 3, 4])
def test_accumulation_steps(accum):
    run_case(f"accumulation_steps={accum}", make_case([300, 7, 120], 5, 10, seed=31), accum=accum)


@pytest.mark.gpu
def test_zero_weight_gives_exactly_zero_g_xv():
    case = make_case([300, 7, 120], 5, 10, seed=32, weight=0.0)
    got = fused(case)
    assert bool((got["g_Xv"] == 0).all())
    ref = ref_of(case)
    check("weight=0", got, ref, bounds_of(case, ref), skip=("g_Xv",))


@pytest.mark.gpu
def test_upstream_gradient_through_train_loss_backward():
    """(2.5·loss + (pred**2).sum()).backward(): pred.grad = 2.5·g_pred + 2·pred and Xv.grad = 2.5·g_Xv, the kernel's
    own gradients scaled in _TrainLoss.backward — and both within bounds of the float64 reference."""
    from distegnn_b200 import train_loss
    case = make_case([300, 7, 2100], 5, 10, seed=33)
    d = dev()
    p = case["pred"].to(d).requires_grad_(True)
    V = case["Xv"].to(d).requires_grad_(True)
    loss, _ = train_loss(p, case["target"].to(d), V, case["batch"].to(d), mmd_samples=case["mmd_samples"],
                         mmd_sigma=case["sigma"], mmd_weight=case["weight"], samples=case["samples"].to(d))
    g_p, g_V = torch.autograd.grad(loss, [p, V], retain_graph=True)     # the saved kernel gradients, times 1
    (2.5 * loss + (p ** 2).sum()).backward()
    assert torch.equal(V.grad, 2.5 * g_V)
    assert torch.equal(p.grad, 2.5 * g_p + 2 * p.detach())
    ref = ref_of(case)
    bd = bounds_of(case, ref, upstream=True)
    e_p = elem_err(2.5 * g_p.cpu(), 2.5 * ref["g_pred"])
    e_V = terms_err(V.grad.cpu(), 2.5 * ref["g_Xv"], 2.5 * ref["g_terms"])
    print(f"upstream 2.5: g_pred {e_p:.2e} (bound {bd['g_pred']:.2e})  g_Xv {e_V:.2e} (bound {bd['g_Xv']:.2e})")
    assert e_p <= bd["g_pred"] and e_V <= bd["g_Xv"]


@pytest.mark.gpu
def test_loc_mean_absent_or_given_on_one_rank():
    case = make_case([300, 7, 120], 5, 10, seed=34)
    ref = ref_of(case)
    bd = bounds_of(case, ref)
    lm = torch.randn(3, 3, generator=torch.Generator().manual_seed(0))
    for name, loc_mean in (("loc_mean=None", None), ("loc_mean given", lm)):
        got = fused(case, loc_mean=loc_mean)
        assert got["dev"] == 0.0
        check(name, got, ref, bd)


def run_ranks(ranks, Xv, C, S, sigma, weight, loc_means, accum=1):
    """Every rank's partials on one GPU, the packed vectors summed by hand in rank order (what the SUM all-reduce
    does), then every rank's finalize.  ranks: dicts of pred, target, batch, samples (a rank may hold no nodes)."""
    from distegnn_b200 import _lib
    from distegnn_b200._lib import check as ck, ptr
    lib, d = _lib.load(), dev()
    B, world = Xv.shape[0], len(ranks)
    npk = lib.distegnn_loss_packed_floats(B, world)
    st = torch.cuda.current_stream().cuda_stream
    Vd, bufs = Xv.to(d), []
    for r, rk in enumerate(ranks):
        n = int(rk["pred"].shape[0])
        p, t = (rk["pred"].to(d), rk["target"].to(d)) if n else (None, None)
        acc, packed, gV = torch.zeros(3, device=d), torch.zeros(npk, device=d), torch.empty(B, 3, C, device=d)
        lm = loc_means[r].to(d)
        gptr, sm = graph_offsets(rk["batch"].to(d), B), rk["samples"].to(d)
        ck(lib.distegnn_loss_partials(n, B, C, S, world, r, sigma, ptr(p), ptr(t), ptr(Vd), ptr(lm), ptr(gptr), ptr(sm),
                                      ptr(acc), ptr(packed), ptr(gV), st), "loss_partials")
        bufs.append((n, p, t, lm, acc, packed, gV))
    total = bufs[0][5].clone()
    for b in bufs[1:]:
        total += b[5]
    outs = []
    for r, (n, p, t, lm, acc, _, gV) in enumerate(bufs):
        g_pred = torch.empty_like(p) if n else None
        g_Xv, out = torch.empty(B, 3, C, device=d), torch.empty(4, device=d)
        ck(lib.distegnn_loss_finalize(n, B, C, S, world, r, sigma, weight, accum, ptr(p), ptr(t), ptr(lm), ptr(acc),
                                      ptr(total), ptr(gV), ptr(g_pred), ptr(g_Xv), ptr(out), st), "loss_finalize")
        outs.append((out, g_pred, g_Xv))
    torch.cuda.synchronize()
    return [dict(loss=float(o[0]), logged=float(o[1]), mmd=float(o[2]), dev=float(o[3]),
                 g_pred=(gp.cpu() if gp is not None else torch.zeros(0, 3)), g_Xv=gx.cpu()) for o, gp, gx in outs]


def _rank_cases(size_lists, C, m, seed, sigma=2.0, weight=0.03):
    """One case per rank with the same virtual coordinates (size_lists[r]: nodes per graph on rank r)."""
    cases = [make_case(sizes, C, m, seed=seed + r, sigma=sigma, weight=weight) for r, sizes in enumerate(size_lists)]
    for c in cases[1:]:
        c["Xv"] = cases[0]["Xv"]
    return cases


@pytest.mark.gpu
def test_world3_unequal_ranks_and_loc_mean_report():
    """world = 3 with unequal node counts (rank 1 over two node blocks); rank 2's loc_mean disagrees with rank 0's by a
    known amount, which out[3] reports on every rank."""
    C, m = 5, 6
    cases = _rank_cases([[40, 25, 300], [2100, 13, 60], [5, 0, 77]], C, m, seed=40)
    counts = [int(c["pred"].shape[0]) for c in cases]
    lm0 = torch.randn(3, 3, generator=torch.Generator().manual_seed(1))
    delta = torch.zeros(3, 3)
    delta[1, 2] = 0.0625
    lms = [lm0, lm0.clone(), lm0 + delta]
    outs = run_ranks(cases, cases[0]["Xv"], C, C * m, 2.0, 0.03, lms)
    refs = [ref_of(c, counts, r) for r, c in enumerate(cases)]
    logged = sum(r["logged"] for r in refs)
    expect_dev = float((lms[2] - lms[0]).abs().max())                    # the same float32 subtraction as the kernel
    for r, (c, got, ref) in enumerate(zip(cases, outs, refs)):
        ref = dict(ref, logged=logged)
        check(f"world=3 rank {r}", got, ref, bounds_of(c, ref, counts))
        assert got["dev"] == expect_dev


@pytest.mark.gpu
def test_world4_with_an_empty_rank():
    """world = 4, rank 2 holds no nodes (n_nodes = 0, pred and target null).  loss.cu's `n_r > 0` rule: the empty rank
    adds 0 to the loss and the logged loss and gets g_Xv = 0.  The reference differs here on purpose: its MSE over an
    empty tensor is NaN.  The other ranks match the reference with that rank's count 0."""
    C, m = 4, 5
    cases = _rank_cases([[40, 25], [2100, 13], [0, 0], [9, 70]], C, m, seed=50)
    counts = [int(c["pred"].shape[0]) for c in cases]
    assert counts[2] == 0
    lm = torch.randn(2, 3, generator=torch.Generator().manual_seed(2))
    outs = run_ranks(cases, cases[0]["Xv"], C, C * m, 2.0, 0.03, [lm] * 4)
    refs = [ref_of(c, counts, r) for r, c in enumerate(cases)]
    assert math.isnan(refs[2]["loss"])                                   # the deliberate difference
    logged = sum(r["logged"] for i, r in enumerate(refs) if i != 2)
    assert outs[2]["loss"] == 0.0 and bool((outs[2]["g_Xv"] == 0).all())
    assert scalar_err(outs[2]["logged"], logged) <= bounds_of(cases[0], refs[0], counts)["logged"]
    for r in (0, 1, 3):
        ref = dict(refs[r], logged=logged)
        check(f"world=4 rank {r}", outs[r], ref, bounds_of(cases[r], ref, counts))
        assert outs[r]["dev"] == 0.0


@pytest.mark.gpu
def test_nan_prediction_row():
    """One NaN row of pred in a batch of several graphs: loss and logged are NaN, g_pred is NaN on that row only and
    matches the reference elsewhere, g_Xv is unaffected (the MMD reads target only)."""
    case = make_case([300, 2100, 120], 5, 10, seed=60)
    row = 2300
    case["pred"][row] = math.nan
    got = fused(case)
    ref = ref_of(case)
    assert math.isnan(got["loss"]) and math.isnan(got["logged"])
    nan_rows = torch.isnan(got["g_pred"]).any(1)
    assert nan_rows.nonzero().flatten().tolist() == [row] and bool(torch.isnan(got["g_pred"][row]).all())
    keep = torch.ones(case["pred"].shape[0], dtype=torch.bool)
    keep[row] = False
    bd = bounds_of(case, ref)
    e_p = elem_err(got["g_pred"][keep], ref["g_pred"][keep])
    print(f"NaN row: g_pred on the other rows {e_p:.2e} (bound {bd['g_pred']:.2e})")
    assert e_p <= bd["g_pred"]
    check("NaN row", got, ref, bd, skip=("loss", "logged", "g_pred"))
