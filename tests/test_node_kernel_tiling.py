"""Per-node and per-graph stages on the shapes their tiling makes fragile: the tensor-core node update and embedding
prologue (node_layer_tc_kernel, embed_tc_kernel), their backward kernels (node_layer_bwd_kernel, embed_bwd_kernel, with
and without the input gradients) and the virtual update (one CTA per graph, forward and backward).

Node and embedding forward: every node-attribute / feature count, both vsum strides, node counts around one tile and far
above one tile per CTA, graph boundaries inside warps, on warps, on tiles (every tile flushes its graph sums), 1,000-node
graphs, a one-node graph in the ragged last tile, graph ids without nodes and one graph per node, isolated nodes and hubs,
rows outside the fp16 range at one encode site at a time, saturated SiLU, and the buffer contract: pre-filled vsum,
sentinel rows past N, FLAG_ZERO_AGG, in place against out of place, rerun determinism, and the data_batch validation.
Backward: at least eight tiles per CTA (the weight gradients live in registers across them), tiny and ragged node counts,
many graphs for g_vsum, hubs, no projection gradients, upstream gradients over 2^-60 … 2^60 and saturated SiLU.

Each forward case runs the production kernel, its fp32-FMA twin (tests/twin_backend.py) and the float64 restatement
(tests/shadow_backend.py); each backward case runs both entry points of the kernel against float64 autograd of the
stage (tests/test_input_grads.py InputGradShadowBackend).  Outputs are compared ROW-WISE (max |got − ref| over a row
over max |ref| of that row); three-wide coordinate rows, which are short signed sums, are judged against the largest
magnitude of the terms summed into the row instead.  Parameter gradients are compared per field, and every gradient
entry the stage does not produce must be exactly zero."""
import functools

import pytest
import torch

from distegnn_b200 import FastEGNN, _lib
from oracle import fastegnn_oracle as orc
from tests.helpers import FLOOR, check_bounds, rel, rowwise, terms_rowwise, within_rerun_bound
from tests.shadow_backend import ShadowBackend, _fields

pytestmark = pytest.mark.gpu

H, A = 64, 2
PAD = 128               # sentinel rows past N in every per-node buffer the kernels write
# Rows rescued from outside the fp16 range: the bound of test_node_kernel_tensor_core_vs_fma_twin (and TWIN_FACTOR)
RESCUE_CAP = 2e-3
LAST = _lib.FLAG_LAST


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def backend():
    from tests.twin_backend import twin_backend
    return twin_backend()


def sm_count():
    return torch.cuda.get_device_properties(dev()).multi_processor_count


def many_tiles_n(tiles_per_cta, groups=1):
    """A node count that gives every CTA (tile group) at least `tiles_per_cta` 128-node tiles and a ragged last tile."""
    return 128 * (tiles_per_cta * groups * sm_count() + 2) + 77


@functools.lru_cache(maxsize=None)
def packed(F, Na, C):
    sd = orc.init_state_dict(F, Na, A, 64, C, 2, seed=8, coord_gain=1.0)
    m = FastEGNN(hidden_nf=64, world_size=1, node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, virtual_channels=C,
                 n_layers=2)
    m.load_state_dict(sd)
    return m.to(dev()).eval()._packed_params(dev())


def K_of(C):
    return 4 + 3 * C + H * C


def fmt(errs):
    return ", ".join(f"{k} {v:.1e}" for k, v in errs.items())


def nan_rows(n, w):
    return torch.full((n, w), float("nan"), device=dev())


def padded(t):
    """t followed by PAD sentinel rows."""
    return torch.cat([t, nan_rows(PAD, t.shape[1])])


def saturated(lp, Na, C):
    """A copy of lp whose N_B1 and L_B put the pre-activations of some columns at −90 … −20 and others up to +1e4."""
    offs, _ = _lib.param_layout(A, C, Na)
    lp = lp.clone()
    g = torch.Generator().manual_seed(60)
    for name in ("N_B1", "L_B"):
        b = lp[offs[name]:offs[name] + H]
        b[:24] = -(20 + 70 * torch.rand(24, generator=g)).to(dev())
        b[24:32] = (10 ** (1 + 3 * torch.rand(8, generator=g))).to(dev())
    return lp


# ==== graph layouts ===================================================================================================
def layout_sizes(name):
    """Nodes per graph id (zeros: graph ids without nodes)."""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    if name == "inside_warps":
        return torch.randint(1, 32, (300,), generator=g)
    if name == "on_warps":
        return 32 * torch.randint(1, 4, (150,), generator=g)
    if name == "on_tiles":                  # every tile holds one graph; a CTA's consecutive tiles hold different ones
        return 128 * torch.randint(1, 4, (2 * sm_count(),), generator=g)
    if name == "thousand_node_graphs":
        return torch.randint(900, 1_101, (120,), generator=g)
    if name == "one_node_graph_in_ragged_last_tile":
        return torch.tensor([3_000, 128 * 40 + 20 - 3_000, 1])
    if name == "empty_graph_ids":
        s = torch.randint(0, 60, (200,), generator=g)
        s[::7] = 0
        s[-1] = 0
        return s
    if name == "one_graph_per_node":
        return torch.ones(3_001, dtype=torch.int64)
    raise ValueError(name)


LAYOUTS = ["inside_warps", "on_warps", "on_tiles", "thousand_node_graphs", "one_node_graph_in_ragged_last_tile",
           "empty_graph_ids", "one_graph_per_node"]


def layout_batch(name):
    sizes = layout_sizes(name)
    return torch.repeat_interleave(torch.arange(sizes.numel()), sizes), sizes.numel()


def sorted_batch(N, B, seed):
    return torch.sort(torch.randint(0, B, (N,), generator=torch.Generator().manual_seed(seed))).values


# ==== node forward ====================================================================================================
def node_inputs(batch, deg, Na, seed):
    """batch: CPU int64 sorted; deg: CPU int64 per node (agg_m, agg_x are sums over that many edges)."""
    g = torch.Generator().manual_seed(seed)
    N = batch.numel()
    rnd = lambda *s: torch.randn(*s, generator=g)
    d1 = deg.clamp(min=1).float()[:, None]
    rowptr = torch.zeros(N + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).to(torch.int32)
    x4, agg_x, tv = torch.zeros(N, 4), torch.zeros(N, 4), torch.zeros(N, 4)
    x4[:, :3], agg_x[:, :3], tv[:, :3] = rnd(N, 3), rnd(N, 3) * d1, rnd(N, 3)
    t = dict(rowptr=rowptr, batch32=batch.to(torch.int32), h=rnd(N, H), x4=x4, vel=rnd(N, 3),
             attr=rnd(N, Na) if Na else None, agg_m=rnd(N, H) * d1, agg_x=agg_x, agg_v=rnd(N, H), trans_v=tv)
    return {k: (None if v is None else v.to(dev())) for k, v in t.items()}


def node_reference(flags, inp, lp, lpn, vsum0, dims):
    """float64 restatement -> outputs, plus the magnitude of the terms of x' = x + agg_x/deg + trans_v + φ_v·vel."""
    N, B, _, C, Na = dims
    last = bool(flags & LAST)
    D = lambda t: None if t is None else t.double()
    z = lambda w: torch.zeros(N, w, dtype=torch.float64, device=dev())
    o = dict(h=z(H), x4=z(4), P=z(H), Q=z(H), Hn=z(H), loc=z(3), vsum=vsum0.double().clone())
    ShadowBackend().node_layer(dims, flags, inp["rowptr"], inp["batch32"], D(inp["h"]), D(inp["x4"]), D(inp["vel"]),
                               D(inp["attr"]), None if last else D(inp["agg_m"]), D(inp["agg_x"]),
                               None if last else D(inp["agg_v"]), D(inp["trans_v"]), lp.double(),
                               None if last else lpn.double(), o["h"], o["x4"], o["P"], o["Q"], o["Hn"],
                               o["loc"] if last else None, o["vsum"])
    f = _fields(lp.double(), A, C, Na)
    rp = inp["rowptr"].long()
    deg = (rp[1:] - rp[:-1]).clamp(min=1).double()[:, None]
    phiv = torch.nn.functional.silu(D(inp["h"]) @ f["L_W"] + f["L_B"]) @ f["L_W3"] + f["L_B3"]
    o["x_terms"] = (D(inp["x4"])[:, :3].abs() + D(inp["agg_x"])[:, :3].abs() / deg + D(inp["trans_v"])[:, :3].abs()
                    + (phiv[:, None] * D(inp["vel"])).abs())
    o["x"] = o["x4"][:, :3]
    return o


def node_run(kind, flags, inp, lp, lpn, vsum0, dims):
    """kind: 'tc' (out of place), 'tc_rerun', 'tc_inplace' (h_out = h, x4_out = x4, FLAG_ZERO_AGG, as FastEGNN._run) or
    'twin'.  Checks the buffer contract and returns the per-node outputs [:N] and vsum."""
    N = dims[0]
    last = bool(flags & LAST)
    vsum = vsum0.clone()
    keys = ("x", "loc") if last else ("h", "x", "P", "Q", "Hn")
    if kind == "twin":
        o = {k: torch.zeros(N, w, device=dev()) for k, w in (("h", H), ("x4", 4), ("P", H), ("Q", H), ("Hn", H),
                                                                ("loc", 3))}
        backend().node_layer_simt(dims, flags, inp["rowptr"], inp["batch32"], inp["h"], inp["x4"], inp["vel"],
                                  inp["attr"], None if last else inp["agg_m"], inp["agg_x"],
                                  None if last else inp["agg_v"], inp["trans_v"], lp, None if last else lpn,
                                  None if last else o["h"], o["x4"], None if last else o["P"], None if last else o["Q"],
                                  None if last else o["Hn"], o["loc"] if last else None, vsum)
        torch.cuda.synchronize()
        o["x"] = o["x4"][:, :3]
        return {**{k: o[k] for k in keys}, "vsum": vsum}
    h, x4, agg_m, agg_x = (padded(inp[k]) for k in ("h", "x4", "agg_m", "agg_x"))
    inplace = kind == "tc_inplace"
    if inplace:
        flags |= _lib.FLAG_ZERO_AGG
        h_out, x4_out = h, x4
    else:
        h_out, x4_out = nan_rows(N + PAD, H), nan_rows(N + PAD, 4)
    P, Q, Hn, loc = nan_rows(N + PAD, H), nan_rows(N + PAD, H), nan_rows(N + PAD, H), nan_rows(N + PAD, 3)
    backend().node_layer(dims, flags, inp["rowptr"], inp["batch32"], h, x4, inp["vel"], inp["attr"],
                         None if last else agg_m, agg_x, None if last else inp["agg_v"], inp["trans_v"], lp,
                         None if last else lpn, None if last else h_out, x4_out, None if last else P,
                         None if last else Q, None if last else Hn, loc if last else None, vsum)
    torch.cuda.synchronize()
    for name, t in (("h_out", h_out), ("x4_out", x4_out), ("P", P), ("Q", Q), ("Hn", Hn), ("loc_out", loc),
                    ("agg_m", agg_m), ("agg_x", agg_x)):
        assert bool(torch.isnan(t[N:]).all()), f"{kind}: {name} written past row N"
    if inplace:
        assert not agg_x[:N].any(), "FLAG_ZERO_AGG left agg_x non-zero"
        if not last:
            assert not agg_m[:N].any(), "FLAG_ZERO_AGG left agg_m non-zero"
        else:
            assert torch.equal(h[:N], inp["h"]), "h written under FLAG_LAST"
    else:
        assert torch.equal(agg_x[:N], inp["agg_x"]) and torch.equal(agg_m[:N], inp["agg_m"]), "agg_m / agg_x changed"
    if last:
        assert torch.equal(loc[:N], x4_out[:N, :3]), "loc_out differs from x4_out[:, :3]"
    else:
        assert bool(torch.isnan(loc).all()), "loc_out written without FLAG_LAST"
    o = dict(h=h_out[:N], x=x4_out[:N, :3], P=P[:N], Q=Q[:N], Hn=Hn[:N], loc=loc[:N])
    return {**{k: o[k] for k in keys}, "vsum": vsum}


def node_errors(got, ref, empty):
    e = {}
    for k, v in got.items():
        if k in ("x", "loc"):
            e[k] = terms_rowwise(v, ref["x"], ref["x_terms"])
        elif k == "vsum":
            e[k] = rowwise(v[~empty, :4], ref["vsum"][~empty, :4])
        else:
            e[k] = rowwise(v, ref[k])
    return e


def check_node(inp, B, Na, C, what, seed=0, tols=None, lps=None):
    """Flags 0 and FLAG_LAST; production kernel out of place, again, and in place, and the twin, against float64."""
    N = inp["batch32"].numel()
    dims = (N, B, A, C, Na)
    lp, lpn = lps or packed(3, Na, C)["layers"]
    vsum0 = torch.randn(B, K_of(C), generator=torch.Generator().manual_seed(seed + 1)).to(dev())
    empty = torch.bincount(inp["batch32"].long(), minlength=B) == 0
    for flags in (0, LAST):
        ref = node_reference(flags, inp, lp, lpn, vsum0, dims)
        got = {k: node_run(k, flags, inp, lp, lpn, vsum0, dims) for k in ("tc", "tc_rerun", "tc_inplace", "twin")}
        for k in ("tc", "tc_rerun", "tc_inplace", "twin"):
            v = got[k]["vsum"]
            assert torch.equal(v[:, 4:], vsum0[:, 4:]), (k, "vsum columns >= 4 changed")
            assert torch.equal(v[empty], vsum0[empty]), (k, "vsum row of a graph without nodes changed")
        for k in ("tc_rerun", "tc_inplace"):
            for f, v in got[k].items():
                if f == "vsum":
                    assert within_rerun_bound(v[:, :4], got["tc"][f][:, :4]), (k, f)
                else:
                    assert torch.equal(v, got["tc"][f]), (k, f, "not bit-identical to the out-of-place launch")
        errs = {k: node_errors(got[k], ref, empty) for k in ("tc", "twin")}
        for k in errs:
            print(f"node fwd {what} N={N} B={B} Na={Na} C={C} flags={flags} [{k}]: row-wise vs fp64 {fmt(errs[k])}")
        check_bounds(errs, tols or {})
    return errs


def random_deg(N, seed):
    return torch.randint(0, 30, (N,), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("C", [1, 16])
@pytest.mark.parametrize("Na", list(range(9)))
def test_node_fwd_attr_counts_and_channels(Na, C):
    """Every node-attribute count; C = 1 / 16 change the vsum row stride K."""
    N, B = 3_001, 5
    check_node(node_inputs(sorted_batch(N, B, Na), random_deg(N, Na), Na, seed=Na + C), B, Na, C, "attr counts",
               seed=Na)


NODE_COUNTS = {"1": lambda: 1, "2": lambda: 2, "127": lambda: 127, "128": lambda: 128, "129": lambda: 129,
               "255": lambda: 255, "257": lambda: 257, "1001": lambda: 1_001, "8_tiles_per_cta": lambda: many_tiles_n(8)}


@pytest.mark.parametrize("n_spec", list(NODE_COUNTS))
def test_node_fwd_node_counts(n_spec):
    """Fewer nodes than a tile, tile edges, and at least eight tiles per CTA with a ragged last tile."""
    N = NODE_COUNTS[n_spec]()
    B = 1 if N < 4 else 3
    check_node(node_inputs(sorted_batch(N, B, N), random_deg(N, N), 2, seed=N), B, 2, 3, f"N {n_spec}", seed=N)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_node_fwd_graph_layouts(layout):
    """Graph boundaries inside warps, on warps and on tiles (then every tile is single-graph and a CTA's consecutive
    tiles belong to different graphs, so the per-group sums are flushed on every tile), 1,000-node graphs, a one-node
    graph in the ragged last tile, graph ids without nodes (their pre-filled vsum rows stay bit-identical), B = N."""
    batch, B = layout_batch(layout)
    N = batch.numel()
    check_node(node_inputs(batch, random_deg(N, 3), 2, seed=4), B, 2, 3, layout, seed=5)


def test_node_fwd_isolated_nodes_and_hubs():
    """Degrees 0 and 1 next to hubs of 1,000 and 10,000 edges in one tile: agg_x/deg and agg_m/deg."""
    N, B = 4_000, 3
    deg = torch.randint(0, 2, (N,), generator=torch.Generator().manual_seed(6))
    deg[200:208], deg[208:216] = 10_000, 1_000
    check_node(node_inputs(sorted_batch(N, B, 6), deg, 2, seed=6), B, 2, 3, "hubs", seed=6)


RESCUE_SITES = ["h", "agg_m_deg1", "agg_m_deg1000", "agg_v", "h_prime", "attr"]


@pytest.mark.parametrize("site", RESCUE_SITES)
def test_node_fwd_fp16_range_rescue(site):
    """Every third row extreme at one encode site, so rescued and ordinary rows share every warp: h (φ_v and layer 1
    start scaled); agg_m at degree 1 (D brought to the new row scale) and at degree 1,000 (agg_m/deg back in range);
    agg_v alone (D brought to the new row scale after two in-range chunks); attr ×1e5 … 1e7 with h ordinary, so t1 and
    h' leave the range (h' is read back from h_out, which in place is h); attr ×1e2 … 1e4 with all eight attributes."""
    N, B = 6_000, 4
    Na = 8 if site == "attr" else 2
    g = torch.Generator().manual_seed(70 + RESCUE_SITES.index(site))
    deg = {"agg_m_deg1": torch.ones(N, dtype=torch.int64),
           "agg_m_deg1000": torch.full((N,), 1_000, dtype=torch.int64)}.get(site, random_deg(N, 70))
    inp = node_inputs(sorted_batch(N, B, 70), deg, Na, seed=71)
    ext = torch.arange(N) % 3 == 0
    lo, span = (2, 2) if site == "attr" else (5, 2)
    if site == "agg_m_deg1000":              # agg_m ×1e5 … 3e6 over 1,000 edges: agg_m/deg stays below the fp16 range
        inp["agg_m"], span = inp["agg_m"] / 1_000, 1.5
    scale = torch.where(ext, 10 ** (lo + span * torch.rand(N, generator=g)), torch.ones(N)).to(dev())[:, None]
    key = {"h": "h", "agg_m_deg1": "agg_m", "agg_m_deg1000": "agg_m", "agg_v": "agg_v", "h_prime": "attr",
           "attr": "attr"}[site]
    inp[key] = inp[key] * scale
    errs = check_node(inp, B, Na, 3, f"rescue {site}", seed=72, tols=dict.fromkeys(("h", "x", "P", "Q", "Hn", "loc",
                                                                                     "vsum"), RESCUE_CAP))
    print(f"rescue {site}: tensor core {fmt(errs['tc'])}; twin {fmt(errs['twin'])}")


def test_node_fwd_saturated_silu():
    """Pre-activations of 24 columns at −90 … −20 and 8 columns up to +1e4, in the node MLP and in φ_v."""
    N, B, Na, C = 3_001, 3, 2, 3
    lp, lpn = packed(3, Na, C)["layers"]
    check_node(node_inputs(sorted_batch(N, B, 80), random_deg(N, 80), Na, seed=80), B, Na, C, "saturated SiLU",
               seed=80, lps=(saturated(lp, Na, C), lpn),
               tols=dict.fromkeys(("h", "x", "P", "Q", "Hn", "loc", "vsum"), RESCUE_CAP))


# ==== embedding forward ===============================================================================================
def embed_run(kind, inp, pk, vsum0, dims, counter=None):
    N = dims[0]
    vsum = vsum0.clone()
    if kind == "twin":
        o = dict(h=torch.zeros(N, H, device=dev()), x4=torch.zeros(N, 4, device=dev()),
                 b32=torch.zeros(N, 1, dtype=torch.int32, device=dev()), P=torch.zeros(N, H, device=dev()),
                 Q=torch.zeros(N, H, device=dev()), Hn=torch.zeros(N, H, device=dev()))
        backend().embed_simt(dims, inp["feat"], inp["loc"], inp["batch"], pk["emb_wt"], pk["emb_b"], pk["layers"][0],
                             o["h"], o["x4"], o["b32"], o["P"], o["Q"], o["Hn"], vsum)
    else:
        o = dict(h=nan_rows(N + PAD, H), x4=nan_rows(N + PAD, 4),
                 b32=torch.full((N + PAD, 1), -7, dtype=torch.int32, device=dev()), P=nan_rows(N + PAD, H),
                 Q=nan_rows(N + PAD, H), Hn=nan_rows(N + PAD, H))
        backend().embed(dims, inp["feat"], inp["loc"], inp["batch"], pk["emb_wt"], pk["emb_b"], pk["layers"][0],
                        o["h"], o["x4"], o["b32"], o["P"], o["Q"], o["Hn"], vsum, counter)
    torch.cuda.synchronize()
    if kind != "twin":
        for k, t in o.items():
            past = t[N:]
            assert bool((past == -7).all() if k == "b32" else torch.isnan(past).all()), f"{k} written past row N"
        o = {k: t[:N] for k, t in o.items()}
    return dict(h=o["h"], x4=o["x4"], b32=o["b32"][:, 0], P=o["P"], Q=o["Q"], Hn=o["Hn"], vsum=vsum)


def embed_inputs(batch, F, seed):
    g = torch.Generator().manual_seed(seed)
    N = batch.numel()
    return dict(feat=(torch.randn(N, F, generator=g) * 3).to(dev()), loc=torch.randn(N, 3, generator=g).to(dev()),
                batch=batch.to(dev()))


def check_embed(inp, B, F, what, seed=0, tols=None):
    C = 3
    N = inp["batch"].numel()
    dims = (N, B, F, A, C, 0)
    pk = packed(F, 0, C)
    vsum0 = torch.randn(B, K_of(C), generator=torch.Generator().manual_seed(seed + 1)).to(dev())
    empty = torch.bincount(inp["batch"], minlength=B) == 0
    z = lambda w: torch.zeros(N, w, dtype=torch.float64, device=dev())
    ref = dict(h=z(H), x4=z(4), P=z(H), Q=z(H), Hn=z(H), vsum=vsum0.double().clone())
    b32 = torch.zeros(N, dtype=torch.int32, device=dev())
    ShadowBackend().embed(dims, inp["feat"].double(), inp["loc"].double(), inp["batch"], pk["emb_wt"].double(),
                          pk["emb_b"].double(), pk["layers"][0].double(), ref["h"], ref["x4"], b32, ref["P"], ref["Q"],
                          ref["Hn"], ref["vsum"])
    got = {k: embed_run(k, inp, pk, vsum0, dims) for k in ("tc", "tc_rerun", "twin")}
    errs = {}
    for k in ("tc", "tc_rerun", "twin"):
        o = got[k]
        assert torch.equal(o["x4"][:, :3], inp["loc"]) and not o["x4"][:, 3].any(), (k, "x4")
        assert torch.equal(o["b32"], b32), (k, "batch32")
        assert torch.equal(o["vsum"][:, 4:], vsum0[:, 4:]) and torch.equal(o["vsum"][empty], vsum0[empty]), (k, "vsum")
        if k == "tc_rerun":
            for f in ("h", "P", "Q", "Hn"):
                assert torch.equal(o[f], got["tc"][f]), (f, "rerun not bit-identical")
            assert within_rerun_bound(o["vsum"][:, :4], got["tc"]["vsum"][:, :4])
            continue
        errs[k] = {f: rowwise(o[f], ref[f]) for f in ("h", "P", "Q", "Hn")}
        errs[k]["vsum"] = rowwise(o["vsum"][~empty, :4], ref["vsum"][~empty, :4])
        print(f"embed fwd {what} N={N} B={B} F={F} [{k}]: row-wise vs fp64 {fmt(errs[k])}")
    check_bounds(errs, tols or {})
    return errs


@pytest.mark.parametrize("F", list(range(1, 17)))
def test_embed_fwd_feature_counts(F):
    N, B = 3_001, 5
    check_embed(embed_inputs(sorted_batch(N, B, F), F, seed=F), B, F, "features", seed=F)


EMBED_COUNTS = {"1": lambda: 1, "127": lambda: 127, "129": lambda: 129, "257": lambda: 257,
                "8_tiles_per_group": lambda: many_tiles_n(8, groups=2)}


@pytest.mark.parametrize("n_spec", list(EMBED_COUNTS))
def test_embed_fwd_node_counts(n_spec):
    """Fewer nodes than a tile, one and two tile groups, and at least eight tiles per tile group (two per CTA)."""
    N = EMBED_COUNTS[n_spec]()
    B = 1 if N < 4 else 3
    check_embed(embed_inputs(sorted_batch(N, B, N), 5, seed=N), B, 5, f"N {n_spec}", seed=N)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_embed_fwd_graph_layouts(layout):
    batch, B = layout_batch(layout)
    check_embed(embed_inputs(batch, 3, seed=9), B, 3, layout, seed=9)


def test_embed_fwd_h0_out_of_fp16_range():
    """Every third row of node_feat ×1e4 … 1e6: h0 leaves the fp16 range and its row is re-encoded with its own scale."""
    N, B, F = 6_000, 3, 4
    inp = embed_inputs(sorted_batch(N, B, 90), F, seed=90)
    g = torch.Generator().manual_seed(91)
    s = torch.where(torch.arange(N) % 3 == 0, 10 ** (4 + 2 * torch.rand(N, generator=g)), torch.ones(N))
    inp["feat"] = inp["feat"] * s.to(dev())[:, None]
    errs = check_embed(inp, B, F, "h0 out of range", seed=90, tols=dict.fromkeys(("h", "P", "Q", "Hn", "vsum"),
                                                                                 RESCUE_CAP))
    print(f"embed h0 out of range: tensor core {fmt(errs['tc'])}; twin {fmt(errs['twin'])}")


BATCH_DEFECTS = ["valid", "negative_ids", "ids_at_or_beyond_B", "descent_inside_a_tile", "descent_at_a_tile_boundary",
                 "descent_at_the_group_stride"]


@pytest.mark.parametrize("defect", BATCH_DEFECTS)
def test_embed_fwd_invalid_batch_ids(defect):
    """n_invalid counts exactly the entries the restatement flags (negative, >= B, smaller than their predecessor) and
    batch32 holds the ids clamped to [0, B).  Descents inside a tile, at a tile boundary, and at the first node of a
    group's second tile (the tile stride of the grid: 2 tile groups per CTA, one CTA per SM)."""
    sm = sm_count()
    N, B, F = 128 * (4 * sm + 3) + 50, 50, 3
    batch = sorted_batch(N, B, 100)
    stride = 128 * 2 * sm
    if defect == "negative_ids":
        batch[[10, 700, stride + 3]] = -1
    elif defect == "ids_at_or_beyond_B":
        batch[-3:] = torch.tensor([B, B + 1, 2 * B])
    else:
        p = {"descent_inside_a_tile": 128 * 5 + 60, "descent_at_a_tile_boundary": 128 * 7,
             "descent_at_the_group_stride": stride}.get(defect)
        if p is not None:                   # node p is the only one smaller than its predecessor
            batch[p - 1] = batch[p] + 1
    inp = embed_inputs(batch, F, seed=101)
    dims = (N, B, F, A, 3, 0)
    pk = packed(F, 0, 3)
    want, want_b32 = torch.zeros(1, dtype=torch.int64, device=dev()), torch.zeros(N, dtype=torch.int32, device=dev())
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev())
    ShadowBackend().embed(dims, inp["feat"].double(), inp["loc"].double(), inp["batch"], pk["emb_wt"].double(),
                          pk["emb_b"].double(), pk["layers"][0].double(), z(N, H), z(N, 4), want_b32, z(N, H), z(N, H),
                          z(N, H), z(B, K_of(3)), want)
    counter = torch.zeros(1, dtype=torch.int32, device=dev())
    o = embed_run("tc", inp, pk, torch.zeros(B, K_of(3), device=dev()), dims, counter)
    got, want = int(counter.item()), int(want.item())
    print(f"data_batch {defect}: n_invalid {got}, restatement {want}")
    assert got == want
    assert (want == 0) == (defect == "valid")
    assert torch.equal(o["b32"], want_b32)
    assert torch.equal(o["b32"].cpu(), batch.clamp(0, B - 1).to(torch.int32))


# ==== node backward ===================================================================================================
def node_slices(Na, C):
    """(offset, size) of every parameter-gradient field the node backward produces: this layer's, the next layer's."""
    offs, _ = _lib.param_layout(A, C, Na)
    n1 = offs["N_W1"]
    own = dict(L_W=(offs["L_W"], H * H), L_B=(offs["L_B"], H), L_W3=(offs["L_W3"], H), L_B3=(offs["L_B3"], 1),
               N_W1_h=(n1, H * H), N_W1_aggm=(n1 + H * H, H * H), N_W1_aggv=(n1 + 2 * H * H, H * H),
               N_W1_attr=(n1 + 3 * H * H, Na * H), N_B1=(offs["N_B1"], H), N_W2=(offs["N_W2"], H * H),
               N_B2=(offs["N_B2"], H))
    nxt = dict(E_W1A=(offs["E_W1A"], H * H), E_B1=(offs["E_B1"], H), E_W1B=(offs["E_W1B"], H * H),
               V_W1H=(offs["V_W1H"], H * H))
    return own, nxt


def field_errors(got, ref, slices, prefix=""):
    """Per-field relative error; a field whose reference is zero must be exactly zero, and so must every entry outside
    the listed fields."""
    errs, covered = {}, torch.zeros(got.numel(), dtype=torch.bool, device=got.device)
    for name, (o, n) in slices.items():
        if not n:
            continue
        covered[o:o + n] = True
        g, r = got[o:o + n], ref[o:o + n]
        if float(r.abs().max()) == 0.0:
            assert not g.any(), f"{prefix}{name} must be exactly zero"
            continue
        errs[prefix + name] = rel(g, r)
    assert not got[~covered].any() and not ref[~covered].any(), f"{prefix}gradient outside the stage's fields"
    return errs


def node_bwd_inputs(batch, B, deg, Na, C, seed, row_scale=None):
    """row_scale: per-node factor of every upstream gradient (then no g_vsum)."""
    g = torch.Generator().manual_seed(seed)
    N = batch.numel()
    rnd = lambda *s: torch.randn(*s, generator=g)
    rowptr = torch.zeros(N + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).to(torch.int32)
    s = torch.ones(N, 1) if row_scale is None else row_scale[:, None]
    t = dict(rowptr=rowptr, batch32=batch.to(torch.int32), h=rnd(N, H), vel=rnd(N, 3), attr=rnd(N, Na) if Na else None,
             agg_m=rnd(N, H) * deg.clamp(min=1).float()[:, None], agg_v=rnd(N, H), g_x=rnd(N, 3) * s,
             g_vsum=None if row_scale is not None else rnd(B, K_of(C)), g_h=rnd(N, H) * s, g_P=rnd(N, H) * s,
             g_Q=rnd(N, H) * s, g_Hn=rnd(N, H) * s, g_vel0=rnd(N, 3) * s, g_attr0=rnd(N, Na) * s if Na else None)
    return {k: (None if v is None else v.to(dev())) for k, v in t.items()}


def node_bwd_run(be, dt, inp, flags, lp, lpn, dims, extra, proj=True):
    """One launch (or the float64 stand-in): -> dict of every output; `extra`: the input-gradient entry point
    (g_vel / g_attr pre-filled with g_vel0 / g_attr0, accumulated onto)."""
    N, B, _, C, Na = dims
    last = bool(flags & LAST)
    c = lambda v: None if v is None else v.to(dt)
    z = lambda *s: torch.zeros(*s, dtype=dt, device=dev())
    total = lp.numel()
    o = dict(g_h=torch.full((N, H), float("nan"), dtype=dt, device=dev()), g_x=z(N, 3), g_agg_x=z(N, 4),
             g_trans_v=z(N, 4), g_agg_m=z(N, H), g_agg_v=z(N, H), g_lp=z(total), g_lpn=z(total))
    kw = {}
    if extra:
        o["g_vel"] = inp["g_vel0"].to(dt).clone()
        o["g_attr"] = None if not Na else inp["g_attr0"].to(dt).clone()
        kw = dict(g_vel=o["g_vel"], g_attr=o["g_attr"])
    up = lambda k: None if (last or not proj) else c(inp[k])
    be.node_layer_bwd(dims, flags, inp["rowptr"], inp["batch32"], c(inp["h"]), c(inp["vel"]), c(inp["attr"]),
                      None if last else c(inp["agg_m"]), None if last else c(inp["agg_v"]), c(lp),
                      None if last else c(lpn), c(inp["g_x"]), c(inp["g_vsum"]), None if last else c(inp["g_h"]),
                      up("g_P"), up("g_Q"), up("g_Hn"), o["g_h"], o["g_x"], o["g_agg_x"], o["g_trans_v"],
                      None if last else o["g_agg_m"], None if last else o["g_agg_v"], o["g_lp"],
                      None if last else o["g_lpn"], **kw)
    return o


def check_node_bwd(inp, B, Na, C, last, what, lps=None, proj=True):
    from distegnn_b200.backend import cuda_backend
    from tests.test_input_grads import InputGradShadowBackend
    N = inp["batch32"].numel()
    dims = (N, B, A, C, Na)
    flags = LAST if last else 0
    lp, lpn = lps or packed(3, Na, C)["layers"]
    be = cuda_backend()
    plain = node_bwd_run(be, torch.float32, inp, flags, lp, lpn, dims, False, proj)
    got = node_bwd_run(be, torch.float32, inp, flags, lp, lpn, dims, True, proj)
    torch.cuda.synchronize()
    for k, v in plain.items():                     # same arithmetic: per-node outputs bit for bit, atomics to rounding
        if k in ("g_lp", "g_lpn"):
            assert within_rerun_bound(got[k], v), k
        else:
            assert torch.equal(got[k], v), (k, "input-gradient entry point differs from the weights-only one")
    ref = node_bwd_run(InputGradShadowBackend(), torch.float64, inp, flags, lp, lpn, dims, True, proj)
    # terms of the three-wide rows: g_x' = g_x + g_vsum[batch, 0:3] and g_vel += φ_v·g_x'
    gterm = inp["g_x"].double().abs()
    if inp["g_vsum"] is not None:
        gterm = gterm + inp["g_vsum"][inp["batch32"].long(), :3].double().abs()
    f = _fields(lp.double(), A, C, Na)
    u = inp["h"].double() @ f["L_W"] + f["L_B"]
    phiv = torch.nn.functional.silu(u) @ f["L_W3"] + f["L_B3"]
    rp = inp["rowptr"].long()
    inv = 1.0 / (rp[1:] - rp[:-1]).clamp(min=1).double()[:, None]
    # g_φv = g_x'·vel is a three-term dot product and scales a whole row of g_u = g_φv·L_W3⊙SiLU'(u), and so the φ_v
    # part of g_h and the single entry L_B3 = Σ g_φv: those are judged against the magnitudes of the products
    gdot = (gterm * inp["vel"].double().abs()).sum(1, keepdim=True)
    su = torch.sigmoid(u)
    phi_terms = (gdot * (f["L_W3"] * su * (1 + u * (1 - su))).abs()) @ f["L_W"].abs().t()
    h_scale = torch.maximum(ref["g_h"].abs(), phi_terms)
    e = dict(g_h=terms_rowwise(got["g_h"], ref["g_h"], h_scale), g_x=terms_rowwise(got["g_x"], ref["g_x"], gterm),
             g_trans_v=terms_rowwise(got["g_trans_v"][:, :3], ref["g_trans_v"][:, :3], gterm),
             g_agg_x=terms_rowwise(got["g_agg_x"][:, :3], ref["g_agg_x"][:, :3], gterm * inv),
             g_vel=terms_rowwise(got["g_vel"], ref["g_vel"], inp["g_vel0"].double().abs() + phiv.abs()[:, None] * gterm))
    assert not got["g_agg_x"][:, 3].any() and not got["g_trans_v"][:, 3].any()
    if not last:
        e["g_agg_m"] = rowwise(got["g_agg_m"], ref["g_agg_m"])
        e["g_agg_v"] = rowwise(got["g_agg_v"], ref["g_agg_v"])
        if Na:
            e["g_attr"] = rowwise(got["g_attr"], ref["g_attr"])
    elif Na:
        assert torch.equal(got["g_attr"], inp["g_attr0"]), "g_attr changed under FLAG_LAST"
    own, nxt = node_slices(Na, C)
    e.update(field_errors(got["g_lp"], ref["g_lp"], own))
    e.update(field_errors(got["g_lpn"], ref["g_lpn"], nxt, "next."))
    o = own["L_B3"][0]
    e["L_B3"] = float((got["g_lp"][o] - ref["g_lp"][o]).abs()) / max(FLOOR, float(gdot.sum()))
    if last or not proj:
        assert not got["g_lpn"].any(), "next layer's gradient fields written without projection gradients"
    print(f"node bwd {what} N={N} B={B} Na={Na} last={last}: row-wise / per field vs fp64 {fmt(e)}")
    check_bounds({"tc": e}, {})
    return e


BWD_CASES = [(Na, last) for last in (False, True) for Na in (0, 8)]


@pytest.mark.parametrize("Na,last", BWD_CASES)
def test_node_bwd_many_tiles_per_cta(Na, last):
    """At least eight tiles per CTA and a ragged last tile: the weight gradients and column sums accumulate in registers
    over all of a CTA's tiles before the one flush."""
    N = many_tiles_n(8)
    B = N // 1_000
    check_node_bwd(node_bwd_inputs(sorted_batch(N, B, 110), B, random_deg(N, 110), Na, 3, seed=111), B, Na, 3, last,
                   "8 tiles per CTA")


@pytest.mark.parametrize("N", [1, 127, 128, 129])
@pytest.mark.parametrize("Na,last", BWD_CASES)
def test_node_bwd_small_node_counts(Na, last, N):
    B = 1 if N < 4 else 3
    check_node_bwd(node_bwd_inputs(sorted_batch(N, B, N), B, random_deg(N, N), Na, 3, seed=N), B, Na, 3, last,
                   f"N={N}")


@pytest.mark.parametrize("per_graph", [3, 1])
@pytest.mark.parametrize("Na,last", BWD_CASES)
def test_node_bwd_many_graphs(Na, last, per_graph):
    """g_vsum gathered over B = N/3 and B = N graph ids, some of them without nodes."""
    g = torch.Generator().manual_seed(120 + per_graph)
    B = 3_000 // per_graph
    sizes = torch.randint(0, 2 * per_graph + 1, (B,), generator=g)
    batch = torch.repeat_interleave(torch.arange(B), sizes)
    N = batch.numel()
    check_node_bwd(node_bwd_inputs(batch, B, random_deg(N, 121), Na, 3, seed=122), B, Na, 3, last,
                   f"{per_graph} nodes per graph")


@pytest.mark.parametrize("Na,last", BWD_CASES)
def test_node_bwd_isolated_nodes_and_hubs(Na, last):
    N, B = 4_000, 3
    deg = torch.randint(0, 2, (N,), generator=torch.Generator().manual_seed(130))
    deg[200:208], deg[208:216] = 10_000, 1_000
    check_node_bwd(node_bwd_inputs(sorted_batch(N, B, 130), B, deg, Na, 3, seed=131), B, Na, 3, last, "hubs")


@pytest.mark.parametrize("Na", [0, 8])
def test_node_bwd_without_projection_gradients(Na):
    """g_P = g_Q = g_Hn = None without FLAG_LAST: the next layer's fields stay exactly zero."""
    N, B = 3_001, 3
    check_node_bwd(node_bwd_inputs(sorted_batch(N, B, 140), B, random_deg(N, 140), Na, 3, seed=141), B, Na, 3, False,
                   "no g_P", proj=False)


@pytest.mark.parametrize("Na,last", BWD_CASES)
def test_node_bwd_upstream_gradient_range(Na, last):
    """Every upstream gradient of a node scaled by the same 2^k, k in [−60, 60] across rows."""
    N, B = 5_003, 3
    k = torch.randint(-60, 61, (N,), generator=torch.Generator().manual_seed(150)).double()
    check_node_bwd(node_bwd_inputs(sorted_batch(N, B, 150), B, random_deg(N, 150), Na, 3, seed=151,
                                   row_scale=torch.pow(2.0, k).float()), B, Na, 3, last, "2^k upstream")


@pytest.mark.parametrize("Na,last", BWD_CASES)
def test_node_bwd_saturated_silu(Na, last):
    N, B = 3_001, 3
    lp, lpn = packed(3, Na, 3)["layers"]
    check_node_bwd(node_bwd_inputs(sorted_batch(N, B, 160), B, random_deg(N, 160), Na, 3, seed=161), B, Na, 3, last,
                   "saturated SiLU", lps=(saturated(lp, Na, 3), lpn))


# ==== embedding backward ==============================================================================================
def check_embed_bwd(N, B, F, what, seed, h0_scale=None):
    from distegnn_b200.backend import cuda_backend
    from tests.test_input_grads import InputGradShadowBackend
    C = 5
    K = K_of(C)
    pk = packed(F, 0, C)
    lp0, emb_wt = pk["layers"][0], pk["emb_wt"]
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g).to(dev())
    feat = rnd(N, F)
    h0 = feat @ emb_wt + pk["emb_b"]
    if h0_scale is not None:
        h0 = h0 * h0_scale[:, None]
    gs = [rnd(N, H) for _ in range(4)]
    batch32 = sorted_batch(N, B, seed).to(torch.int32).to(dev())
    g_x0, g_vsum0 = rnd(N, 3), rnd(B, K)
    dims = (N, B, F, A, C, 0)

    def run(be, dt, extra):
        c = lambda v: v.to(dt)
        o = [torch.zeros(F, H, dtype=dt, device=dev()), torch.zeros(H, dtype=dt, device=dev()),
             torch.zeros(lp0.numel(), dtype=dt, device=dev())]
        kw = {}
        if extra:
            kw = dict(g_feat=torch.full((N, F), float("nan"), dtype=dt, device=dev()),
                      g_loc=torch.full((N, 3), float("nan"), dtype=dt, device=dev()), emb_wt=c(emb_wt), batch32=batch32,
                      g_x0=c(g_x0), g_vsum0=c(g_vsum0))
        be.embed_bwd(dims, c(feat), c(h0), c(lp0), *[c(x) for x in gs], *o, **kw)
        return o + ([kw["g_feat"], kw["g_loc"]] if extra else [])
    be = cuda_backend()
    plain, got = run(be, torch.float32, False), run(be, torch.float32, True)
    torch.cuda.synchronize()
    for a_, b_, name in zip(plain, got, ("g_emb_wt", "g_emb_b", "g_lp0")):
        assert within_rerun_bound(b_, a_), name
    ref = run(InputGradShadowBackend(), torch.float64, True)
    gterm = g_x0.double().abs() + g_vsum0[batch32.long(), :3].double().abs()
    # g_feat[r, k] = Σ_n g_h0[r, n]·emb_wt[k, n] cancels to any magnitude (with F = 1 the row is that one sum): each entry
    # is judged against the sum of the magnitudes of its terms
    f0 = _fields(lp0.double(), A, C, 0)
    g_h0 = gs[0].double() + gs[1].double() @ f0["E_W1A"].t() + gs[2].double() @ f0["E_W1B"].t() \
        + gs[3].double() @ f0["V_W1H"].t()
    feat_terms = g_h0.abs() @ emb_wt.double().abs().t()
    e = dict(g_emb_wt=rel(got[0], ref[0]), g_emb_b=rel(got[1], ref[1]),
             g_feat=terms_rowwise(got[3], ref[3], feat_terms),
             g_loc=terms_rowwise(got[4], ref[4], gterm))
    _, nxt = node_slices(0, C)
    e.update(field_errors(got[2], ref[2], nxt))
    print(f"embed bwd {what} N={N} B={B} F={F}: row-wise / per field vs fp64 {fmt(e)}")
    check_bounds({"tc": e}, {})


@pytest.mark.parametrize("F", list(range(1, 17)))
def test_embed_bwd_feature_counts(F):
    check_embed_bwd(3_001, 3, F, "features", seed=170 + F)


def test_embed_bwd_many_tiles_per_cta_and_many_graphs():
    N = many_tiles_n(8)
    check_embed_bwd(N, N // 7, 4, "8 tiles per CTA", seed=180)


def test_embed_bwd_h0_out_of_fp16_range():
    N = 5_000
    g = torch.Generator().manual_seed(190)
    s = torch.where(torch.arange(N) % 3 == 0, 10 ** (5 + 2 * torch.rand(N, generator=g)), torch.ones(N))
    check_embed_bwd(N, 3, 3, "h0 out of range", seed=191, h0_scale=s.to(dev()))


# ==== virtual update ==================================================================================================
VU_MODES = {"mid": 0, "last": LAST, "init": _lib.FLAG_INIT,
            "init_centroid": _lib.FLAG_INIT | _lib.FLAG_INIT_CENTROID, "zero_vsum": _lib.FLAG_ZERO_VSUM}
VU_B = 3_000


def vu_inputs(C, seed):
    """Packed statistics of 3,000 graphs; every 10th has count 0 (the update divides by max(n, 1))."""
    g = torch.Generator().manual_seed(seed)
    vs = torch.randn(VU_B, K_of(C), generator=g)
    vs[:, 3] = torch.randint(1, 1_000, (VU_B,), generator=g).float()
    vs[::10, 3] = 0
    return dict(vs=vs.to(dev()), Xv=torch.randn(VU_B, 3, C, generator=g).to(dev()),
                Hv=torch.randn(VU_B, C, H, generator=g).to(dev()), loc_mean=torch.randn(VU_B, 3, generator=g).to(dev()),
                gX=torch.randn(VU_B, 3, C, generator=g).to(dev()), gH=torch.randn(VU_B, C, H, generator=g).to(dev()),
                gG=torch.randn(VU_B, C, H, generator=g).to(dev()))


@pytest.mark.parametrize("mode", list(VU_MODES))
@pytest.mark.parametrize("C", list(range(1, 17)))
def test_virtual_update_fwd(C, mode):
    """Xv, Hv and the next layer's G against float64; X_0 of FLAG_INIT_CENTROID is vsum[:, :3]/max(n, 1) broadcast over
    the channels (restated here: the stand-in takes it as init_loc_mean); vsum is zeroed (FLAG_ZERO_VSUM) or kept."""
    from distegnn_b200.backend import cuda_backend
    flags = VU_MODES[mode]
    init, last = bool(flags & _lib.FLAG_INIT), bool(flags & LAST)
    pk = packed(3, 0, C)
    lp, lpn = pk["layers"]
    t = vu_inputs(C, seed=200 + C)
    loc_mean = None if mode != "init" else t["loc_mean"]
    dims = (VU_B, A, C, 0)
    vsum, Xv, Hv = t["vs"].clone(), t["Xv"].clone(), t["Hv"].clone()
    G = torch.full((VU_B, C, H), float("nan"), device=dev())
    cuda_backend().virtual_update(dims, flags, vsum, Xv, Hv, None if init else lp, None if last else lpn,
                                  None if last else G, loc_mean, pk["hv0"] if init else None)
    torch.cuda.synchronize()
    D = lambda x: x.double().clone()
    r_vsum, rX, rH, rG = D(t["vs"]), D(t["Xv"]), D(t["Hv"]), torch.zeros(VU_B, C, H, dtype=torch.float64, device=dev())
    r_loc = loc_mean
    if mode == "init_centroid":
        r_loc = t["vs"][:, :3].double() / t["vs"][:, 3:4].double().clamp(min=1)
    ShadowBackend().virtual_update(dims, flags & ~_lib.FLAG_INIT_CENTROID, r_vsum, rX, rH, None if init else lp.double(),
                                   None if last else lpn.double(), rG, None if r_loc is None else r_loc.double(),
                                   pk["hv0"].double() if init else None)
    if flags & _lib.FLAG_ZERO_VSUM:
        assert not vsum.any(), "FLAG_ZERO_VSUM left vsum non-zero"
    else:
        assert torch.equal(vsum, t["vs"]), "vsum changed"
    e = dict(Xv=rowwise(Xv.reshape(VU_B, -1), rX.reshape(VU_B, -1)))
    if last:
        assert torch.equal(Hv, t["Hv"]) and bool(torch.isnan(G).all()), "Hv / G written under FLAG_LAST"
    else:
        e["Hv"] = rowwise(Hv.reshape(VU_B * C, H), rH.reshape(VU_B * C, H))
        e["G"] = rowwise(G.reshape(VU_B * C, H), rG.reshape(VU_B * C, H))
    print(f"virtual update fwd C={C} {mode}: row-wise vs fp64 {fmt(e)}")
    check_bounds({"tc": e}, {})


@pytest.mark.parametrize("mode", ["mid", "last", "init"])
@pytest.mark.parametrize("C", list(range(1, 17)))
def test_virtual_update_bwd(C, mode):
    """g_vsum, g_Xv, g_Hv row-wise and the parameter-gradient fields (M_*, and the next layer's V_W1V, V_W1M, V_B1)
    against float64 autograd; every other entry of the gradient blocks exactly zero."""
    from distegnn_b200.backend import cuda_backend
    flags = VU_MODES[mode]
    init, last = bool(flags & _lib.FLAG_INIT), bool(flags & LAST)
    lp, lpn = packed(3, 0, C)["layers"]
    t = vu_inputs(C, seed=300 + C)
    dims = (VU_B, A, C, 0)

    def run(be, dt):
        c = lambda v: v.to(dt)
        z = lambda *s: torch.zeros(*s, dtype=dt, device=dev())
        o = dict(g_vsum=z(VU_B, K_of(C)), g_Xv=z(VU_B, 3, C), g_Hv=z(VU_B, C, H), g_lp=z(lp.numel()),
                 g_lpn=z(lp.numel()))
        be.virtual_update_bwd(dims, flags, c(t["vs"]), c(t["Xv"]), c(t["Hv"]), None if init else c(lp),
                              None if last else c(lpn), c(t["gX"]), None if last else c(t["gH"]),
                              None if last else c(t["gG"]), o["g_vsum"], o["g_Xv"], None if last else o["g_Hv"],
                              None if init else o["g_lp"], None if last else o["g_lpn"])
        return o
    got = run(cuda_backend(), torch.float32)
    torch.cuda.synchronize()
    ref = run(ShadowBackend(), torch.float64)
    offs, _ = _lib.param_layout(A, C, 0)
    own = {k: (offs[k], n) for k, n in (("M_W1", 2 * H * H), ("M_B1", H), ("M_W2", H * H), ("M_B2", H))}
    nxt = {k: (offs[k], n) for k, n in (("V_W1V", H * H), ("V_W1M", C * H), ("V_B1", H))}
    # the Σx entries of g_vsum are three-wide rows of sums over the channels that cancel (with C = 1 the gradient of
    # x̄ is one 64-term dot product of g_G with W1v_M per graph): compared over the whole block, the other columns row-wise
    e = dict(g_vsum_x=rel(got["g_vsum"][:, :3], ref["g_vsum"][:, :3]),
             g_vsum=rowwise(got["g_vsum"][:, 3:], ref["g_vsum"][:, 3:]), g_Xv=rowwise(got["g_Xv"], ref["g_Xv"]))
    if not last:
        e["g_Hv"] = rowwise(got["g_Hv"].reshape(VU_B * C, H), ref["g_Hv"].reshape(VU_B * C, H))
    e.update(field_errors(got["g_lp"], ref["g_lp"], own))
    e.update(field_errors(got["g_lpn"], ref["g_lpn"], nxt, "next."))
    print(f"virtual update bwd C={C} {mode}: row-wise / per field vs fp64 {fmt(e)}")
    check_bounds({"tc": e}, {})
