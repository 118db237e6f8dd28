"""Deterministic mode (`model.deterministic`, DESIGN §17): bitwise-reproducible forwards and rollouts.

CPU: the attribute and its plumbing into every stage, the workspace sizing, the C-ABI argument checks.  GPU: the
combine passes add exactly the specified partials in the specified order (restated in torch fp32), the outputs do not
depend on the grid, on concurrent work or on the edge capacity, the golden fixtures still pass, and rollouts (radius,
fixed graph, cutoff; eager and graphed; with a capacity overflow; differentiable) repeat bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

from distegnn_b200 import FastEGNN, _lib, differentiable_rollout, rollout, synth
from oracle import fastegnn_oracle as orc
from tests.helpers import SINGLE_CASES, golden_inputs, golden_trace, load_golden, max_abs, within_rerun_bound
from tests.shadow_backend import ShadowBackend

H, SLOT = 64, 68


def _align(b):
    return (b + 255) // 256 * 256


def _chunk_nodes(N, Cn):
    """Nodes per vsum chunk: 2^s real<->virtual tiles of 64 // C nodes, s >= 4 the smallest with at most 4096 chunks."""
    tiles, s = -(-N // (64 // Cn)), 4
    while -(-tiles // (1 << s)) > 4096:
        s += 1
    return (64 // Cn) << s


def _vsum_part(N, Cn):
    """(chunks, K, bytes) of the vsum slots."""
    K = 4 + 3 * Cn + H * Cn
    chunks = -(-N // _chunk_nodes(N, Cn))
    return chunks, K, _align(chunks * K * 4)


def _model(Cn, A, Na=2, F=3, L=3, seed=1, normalize=False, dev="cpu"):
    sd = orc.init_state_dict(F, Na, A, 64, Cn, L, seed=seed, coord_gain=0.05)
    m = FastEGNN(node_feat_nf=F, node_attr_nf=Na, edge_attr_nf=A, hidden_nf=64, virtual_channels=Cn, n_layers=L,
                 world_size=1, normalize=normalize)
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


def _inputs(sizes, A, Na=2, F=3, hub=0, max_deg=24, seed=0):
    """Graphs of the given node counts (zeros allowed), random in-graph edges (unsorted), one hub of `hub` in-edges."""
    g = torch.Generator().manual_seed(seed)
    sz = torch.tensor(sizes)
    N, B = int(sz.sum()), len(sizes)
    starts = torch.cumsum(sz, 0) - sz
    batch = torch.repeat_interleave(torch.arange(B), sz)
    pos = torch.randn(N, 3, generator=g) * 2
    rows, cols = [torch.zeros(0, dtype=torch.int64)], [torch.zeros(0, dtype=torch.int64)]
    for b, n in enumerate(sizes):
        if n == 0:
            continue
        deg = torch.randint(0, max_deg + 1, (n,), generator=g)
        if hub and b == 0:
            deg[n // 2] = hub
        r = torch.repeat_interleave(torch.arange(n), deg) + int(starts[b])
        rows.append(r)
        cols.append(torch.randint(0, n, (r.numel(),), generator=g) + int(starts[b]))
    ei = torch.stack([torch.cat(rows), torch.cat(cols)])
    ei = ei[:, torch.randperm(ei.shape[1], generator=g)]
    cnt = torch.bincount(batch, minlength=B).clamp(min=1).double()
    loc_mean = (torch.zeros(B, 3, dtype=torch.float64).index_add_(0, batch, pos.double()) / cnt[:, None]).float()
    return dict(node_feat=torch.randn(N, F, generator=g), node_loc=pos, node_vel=torch.randn(N, 3, generator=g) * 0.1,
                loc_mean=loc_mean, edge_index=ei, data_batch=batch,
                edge_attr=torch.randn(ei.shape[1], A, generator=g) if A else None,
                node_attr=torch.randn(N, Na, generator=g) if Na else None)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_attribute_defaults_off_and_documents_its_scope():
    m, _ = _model(2, 0)
    assert m.deterministic is False
    m.deterministic = True
    assert m.deterministic is True
    with pytest.raises(TypeError):
        m.deterministic = 1
    doc = type(m).deterministic.__doc__
    assert "Gradients are not covered" in doc and "bitwise" in doc
    assert not any("determin" in k for k in m.state_dict())


class _Recorder(ShadowBackend):
    """The torch stand-in, recording which stages received the deterministic workspace."""

    def __init__(self):
        super().__init__()
        self.seen = []

    def _rec(self, name, det_ws):
        self.seen.append((name, None if det_ws is None else det_ws.numel()))

    def embed(self, *a, det_ws=None, **k):
        self._rec("embed", det_ws)
        return super().embed(*a, **k)

    def edge_layer(self, *a, det_ws=None, **k):
        self._rec("edge", det_ws)
        return super().edge_layer(*a, **k)

    def virtual_layer(self, *a, det_ws=None, **k):
        self._rec("virtual", det_ws)
        return super().virtual_layer(*a, **k)

    def node_layer(self, *a, det_ws=None, **k):
        self._rec("node", det_ws)
        return super().node_layer(*a, **k)


@pytest.mark.parametrize("training", [False, True])
def test_flag_reaches_every_reducing_stage(training):
    m, _ = _model(3, 2, L=2)
    inp = _inputs([40, 25], 2)
    N, E = inp["node_loc"].shape[0], inp["edge_index"].shape[1]
    outs = []
    for det in (False, True):
        m.deterministic = det
        m._backend = be = _Recorder()
        with torch.set_grad_enabled(training):
            if training:
                m.train()
            out, X = m(**inp)
        outs.append((out.detach(), X.detach()))
        want = None if not det else _lib.deterministic_workspace_bytes(N, E, 3)
        assert be.seen == [("embed", want)] + [(s, want) for _ in range(2) for s in ("edge", "virtual", "node")]
    # the stand-in has no atomics: the plumbing changes nothing else
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_graph_cache_key_holds_the_flag():
    import inspect
    src = inspect.getsource(FastEGNN._forward_graphed)
    assert "self.deterministic" in src.split("self._graph_cache.get")[0]


@pytest.mark.parametrize("N,E,Cn", [(0, 0, 1), (1, 1, 16), (1000, 20000, 5), (64, 17, 3), (10**6, 2 * 10**7, 8),
                                    (5 * 10**6, 10**8, 1)])
def test_workspace_sizing(N, E, Cn):
    want = _vsum_part(N, Cn)[2] + _align(-(-E // 16) * SLOT * 4)
    assert _lib.deterministic_workspace_bytes(N, E, Cn) == want


def test_cabi_argument_rejection():
    lib = _lib.load()
    err = lambda: lib.distegnn_last_error().decode()
    buf = (C.c_char * 8192)()
    p = (C.addressof(buf) + 15) // 16 * 16                  # host memory: every call below fails before any launch
    nb = C.c_int64(0)
    assert lib.distegnn_deterministic_workspace_bytes(10, 10, 0, C.byref(nb)) == -1
    assert lib.distegnn_deterministic_workspace_bytes(10, 10, 17, C.byref(nb)) == -1
    assert lib.distegnn_deterministic_workspace_bytes(-1, 10, 2, C.byref(nb)) == -1
    assert lib.distegnn_deterministic_workspace_bytes(10, 10, 2, None) == -1
    N, E, Cn = 100, 1000, 2
    need = _lib.deterministic_workspace_bytes(N, E, Cn)

    def edge(ws=p, nbytes=need, A=0, row=p, agg_x=p):
        return lib.distegnn_edge_layer_fwd_det(N, E, A, Cn, 0, 0, row, p, None, p, p, p, p, p, agg_x, None, ws, nbytes,
                                               None)
    assert edge(ws=None) == -1 and "workspace" in err()
    assert edge(ws=p + 4) == -1 and "aligned" in err()
    assert edge(nbytes=need - 1) == -3 and "workspace" in err()
    assert edge(row=None) == -1 and "null" in err()
    assert edge(A=_lib.MAX_EDGE_ATTR + 1) == -1
    assert lib.distegnn_edge_combine_det(N, E, Cn, p, None, p, p, p, need - 1, None) == -3
    assert lib.distegnn_edge_combine_det(N, E, Cn, None, None, p, p, p, need, None) == -1
    assert lib.distegnn_edge_combine_det(N, E, 0, p, None, p, p, p, need, None) == -1
    vneed = _vsum_part(N, Cn)[2]

    def virt(ws=p, nbytes=vneed, vsum=p, B=3):
        return lib.distegnn_virtual_layer_fwd_det(N, B, 0, Cn, 0, 0, p, p, p, p, p, p, p, p, vsum, ws, nbytes, None)
    assert virt(ws=None) == -1
    assert virt(nbytes=vneed - 1) == -3
    assert virt(vsum=None) == -1
    assert virt(B=0) == -1
    assert lib.distegnn_vsum_combine_det(N, 3, Cn, 0, p, p, p, p, vneed - 1, None) == -3
    assert lib.distegnn_vsum_combine_det(N, 3, Cn, 0, p, p, None, p, vneed, None) == -1
    assert lib.distegnn_vsum_combine_det(N, 0, Cn, 0, p, p, p, p, vneed, None) == -1
    assert lib.distegnn_vsum_combine_det(N, 3, Cn, 0, p, p, p, None, 0, None) == -1
    assert lib.distegnn_rollout_centroid_det(N, 2, p, None, p, None) == -1 and "data_batch" in err()
    assert lib.distegnn_rollout_centroid_det(N, 1, None, None, p, None) == -1
    assert lib.distegnn_abi_version() == 3
    # the grid cap is a testing-library argument, not part of the product's ABI
    assert not hasattr(lib, "distegnn_set_deterministic_grid_cap")
    t = _testing()
    assert t.distegnn_edge_layer_fwd_det_capped(N, E, 0, Cn, 0, 0, p, p, None, p, p, p, p, p, p, None, p, need, None,
                                                -1) == -1
    assert t.distegnn_vsum_combine_det_capped(N, 3, Cn, 0, p, p, p, p, vneed - 1, None, 1) == -3


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


_CAPPED = {   # the testing library's grid-capped twins of the deterministic entry points: product arguments + max_ctas
    "distegnn_edge_layer_fwd_det": [C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_uint] + [C.c_void_p] * 11
    + [C.c_int64, C.c_void_p, C.c_int],
    "distegnn_edge_combine_det": [C.c_int64, C.c_int64, C.c_int] + [C.c_void_p] * 5 + [C.c_int64, C.c_void_p, C.c_int],
    "distegnn_virtual_layer_fwd_det": [C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint] + [C.c_void_p] * 10
    + [C.c_int64, C.c_void_p, C.c_int],
    "distegnn_vsum_combine_det": [C.c_int64, C.c_int, C.c_int, C.c_uint] + [C.c_void_p] * 4
    + [C.c_int64, C.c_void_p, C.c_int],
}


def _testing():
    import os
    lib = C.CDLL(os.path.join(os.path.dirname(_lib.LIB_PATH), "libdistegnn_b200_testing.so"))
    for name, argtypes in _CAPPED.items():
        fn = getattr(lib, name + "_capped")
        fn.argtypes, fn.restype = argtypes, C.c_int
    return lib


class _CappedLib:
    """The product library, with the deterministic entry points replaced by the testing library's twins at a grid cap."""

    def __init__(self, cap):
        self._lib, self._t, self._cap = _lib.load(), _testing(), cap

    def __getattr__(self, name):
        if name in _CAPPED:
            fn = getattr(self._t, name + "_capped")
            return lambda *a: fn(*a, self._cap)
        return getattr(self._lib, name)


def _capped_backend(cap):
    from distegnn_b200.backend import CudaBackend
    be = CudaBackend()
    be.lib = _CappedLib(cap)
    return be


def _sorted_rows(sizes_deg, extra=0, seed=0):
    """int32 destination rows, sorted: node i has sizes_deg[i] edges; `extra` garbage entries past the count."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.tensor(sizes_deg)
    row = torch.repeat_interleave(torch.arange(len(sizes_deg)), deg).int()
    N = len(sizes_deg)
    col = torch.randint(0, N, (row.numel(),), generator=g).int()
    if extra:
        row = torch.cat([row, torch.full((extra,), N - 1, dtype=torch.int32)])
        col = torch.cat([col, torch.zeros(extra, dtype=torch.int32)])
    return row, col


@pytest.mark.gpu
@pytest.mark.parametrize("A,last", [(0, False), (2, False), (8, False), (1, True)])
def test_edge_combine_adds_the_slots_in_slice_order(A, last):
    lib, d = _lib.load(), dev()
    g = torch.Generator().manual_seed(A)
    N, Cn, Na = 3000, 4, 0
    deg = torch.randint(0, 40, (N,), generator=g)
    deg[7], deg[1500], deg[2999] = 6000, 17, 33                # a hub over many slices and tiles, a ragged tail
    deg[100:140] = 0                                           # rows with no edge
    row, col = _sorted_rows(deg.tolist(), extra=77)
    nE = int(deg.sum())
    Ecap = row.numel()
    row, col = row.to(d), col.to(d)
    n_dev = torch.tensor([nE], dtype=torch.int32, device=d)
    offs, total = _lib.param_layout(A, Cn, Na)
    lp = (torch.randn(total, generator=g) * 0.1).to(d)
    x4 = torch.randn(N, 4, generator=g).to(d)
    P, Q = (torch.randn(N, H, generator=g) * 0.5).to(d), (torch.randn(N, H, generator=g) * 0.5).to(d)
    ea = torch.randn(Ecap, A, generator=g).to(d) if A else None
    nbytes = _lib.deterministic_workspace_bytes(N, Ecap, Cn)
    ws = torch.full((nbytes,), 255, dtype=torch.uint8, device=d)
    agg_m = None if last else torch.zeros(N, H, device=d)
    agg_x = torch.zeros(N, 4, device=d)
    flags = _lib.FLAG_LAST if last else 0
    args = (N, Ecap, A, Cn, Na, flags, _ptr(row), _ptr(col), _ptr(ea), _ptr(x4), _ptr(P), _ptr(Q), _ptr(lp), _ptr(agg_m),
            _ptr(agg_x), _ptr(n_dev))
    assert lib.distegnn_edge_layer_fwd_det(*args, ws.data_ptr(), nbytes, _stream()) == 0
    torch.cuda.synchronize()
    own_m = None if last else agg_m.clone().cpu()
    own_x = agg_x.clone().cpu()
    voff = _vsum_part(N, Cn)[2]
    n_sl = -(-nE // 16)
    slots = ws[voff:voff + n_sl * SLOT * 4].view(torch.float32).view(n_sl, SLOT).cpu()
    assert lib.distegnn_edge_combine_det(N, Ecap, Cn, _ptr(row), _ptr(n_dev), _ptr(agg_m), _ptr(agg_x), ws.data_ptr(),
                                         nbytes, _stream()) == 0
    torch.cuda.synchronize()
    # restate: every row = its first slice's partial + the slots of its later slices, in slice order, in fp32
    rp = torch.zeros(N + 1, dtype=torch.int64)
    rp[1:] = torch.cumsum(deg, 0)
    want_m = None if last else own_m.clone()
    want_x = own_x.clone()
    for r in range(N):
        if deg[r] == 0:
            continue
        s0, s1 = int(rp[r]) // 16, (int(rp[r + 1]) - 1) // 16
        for s in range(s0 + 1, s1 + 1):
            if not last:
                want_m[r] = want_m[r] + slots[s, :H]
            want_x[r, :3] = want_x[r, :3] + slots[s, H:H + 3]
    assert torch.equal(agg_x.cpu(), want_x)
    assert bool((agg_x.cpu()[deg == 0] == 0).all())
    for cap in (1, 7):                                         # the kernel and the combine under capped grids
        m2 = None if last else torch.zeros(N, H, device=d)
        x2 = torch.zeros(N, 4, device=d)
        t = _CappedLib(cap)
        a2 = args[:13] + (_ptr(m2), _ptr(x2), _ptr(n_dev))
        assert t.distegnn_edge_layer_fwd_det(*a2, ws.data_ptr(), nbytes, _stream()) == 0
        assert t.distegnn_edge_combine_det(N, Ecap, Cn, _ptr(row), _ptr(n_dev), _ptr(m2), _ptr(x2), ws.data_ptr(), nbytes,
                                           _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(x2, agg_x), cap
        assert last or torch.equal(m2, agg_m), cap
    if not last:
        assert torch.equal(agg_m.cpu(), want_m)
        assert bool((agg_m.cpu()[deg == 0] == 0).all())
    # and the default kernel agrees within its own run-to-run bound
    ref_m = None if last else torch.zeros(N, H, device=d)
    ref_x = torch.zeros(N, 4, device=d)
    assert lib.distegnn_edge_layer_fwd(*args[:13], _ptr(ref_m), _ptr(ref_x), _ptr(n_dev), _stream()) == 0
    torch.cuda.synchronize()
    scale = lambda t: 1e-5 * max(1.0, float(t.abs().max()))
    assert float((ref_x - agg_x).abs().max()) <= scale(ref_x)
    if not last:
        assert float((ref_m - agg_m).abs().max()) <= scale(ref_m)


def _seq_sum(rows):
    """fp32 sum of the rows in row order, starting from zero."""
    acc = np.zeros(rows.shape[1], dtype=np.float32)
    for r in rows:
        acc = (acc + r).astype(np.float32)
    return torch.from_numpy(acc)


@pytest.mark.gpu
@pytest.mark.parametrize("Cn,sizes", [(3, [5000, 1, 0, 7, 2000, 0, 3]), (1, [1] * 200 + [3000]), (16, [900, 0, 64, 65]),
                                      (5, [40] * 60), (16, [300000, 2, 70000])])
@pytest.mark.parametrize("last", [False, True])
def test_vsum_combine_adds_the_chunk_slots_in_order(Cn, sizes, last):
    lib, d = _lib.load(), dev()
    g = torch.Generator().manual_seed(Cn)
    A, Na = 0, 0
    B, N = len(sizes), sum(sizes)
    batch = torch.repeat_interleave(torch.arange(B), torch.tensor(sizes)).int().to(d)
    offs, total = _lib.param_layout(A, Cn, Na)
    lp = (torch.randn(total, generator=g) * 0.1).to(d)
    x4 = torch.randn(N, 4, generator=g).to(d)
    Hn = (torch.randn(N, H, generator=g) * 0.5).to(d)
    Xv = torch.randn(B, 3, Cn, generator=g).to(d)
    G = (torch.randn(B, Cn, H, generator=g) * 0.5).to(d)
    chunks, K, vbytes = _vsum_part(N, Cn)
    ws = torch.full((vbytes,), 255, dtype=torch.uint8, device=d)
    agg_v = None if last else torch.empty(N, H, device=d)
    trans_v = torch.empty(N, 4, device=d)
    vsum = torch.zeros(B, K, device=d)
    flags = _lib.FLAG_LAST if last else 0
    args = (N, B, A, Cn, Na, flags, _ptr(batch), _ptr(x4), _ptr(Hn), _ptr(Xv), _ptr(G), _ptr(lp), _ptr(agg_v),
            _ptr(trans_v))
    assert lib.distegnn_virtual_layer_fwd_det(*args, _ptr(vsum), ws.data_ptr(), vbytes, _stream()) == 0
    torch.cuda.synchronize()
    owner = vsum.clone().cpu()
    slots = ws.view(torch.float32)[:chunks * K].view(chunks, K).cpu()
    assert lib.distegnn_vsum_combine_det(N, B, Cn, flags, _ptr(batch), _ptr(x4), _ptr(vsum), ws.data_ptr(), vbytes,
                                         _stream()) == 0
    torch.cuda.synchronize()
    # restate: per chunk, Σx in node order; a graph = its first chunk's partial + its later chunks' partials (the
    # real<->virtual entries: the slots read above), in chunk order
    per, lo = _chunk_nodes(N, Cn), 0
    want = owner.clone()
    xs = x4.cpu().numpy()[:, :3]
    cols = slice(4, 4 + 3 * Cn) if last else slice(4, K)
    for b, n in enumerate(sizes):
        hi = lo + n
        want[b, 3] = float(n)
        if n:
            want[b, :3] = _seq_sum(xs[lo:min(hi, (lo // per + 1) * per)])
            for c in range(lo // per + 1, (hi - 1) // per + 1):
                want[b, :3] = want[b, :3] + _seq_sum(xs[c * per:min(hi, (c + 1) * per)])
                want[b, cols] = want[b, cols] + slots[c, cols]
        lo = hi
    got = vsum.cpu()
    assert torch.equal(got[:, :4], want[:, :4])
    assert torch.equal(got[:, cols], want[:, cols])
    if last:                                                   # entries the last layer does not produce: left alone
        assert torch.equal(got[:, cols.stop:], owner[:, cols.stop:])
    for cap in (1, 7):                                         # the kernel and the combine under capped grids
        v2 = torch.zeros(B, K, device=d)
        t = _CappedLib(cap)
        assert t.distegnn_virtual_layer_fwd_det(*args, _ptr(v2), ws.data_ptr(), vbytes, _stream()) == 0
        assert t.distegnn_vsum_combine_det(N, B, Cn, flags, _ptr(batch), _ptr(x4), _ptr(v2), ws.data_ptr(), vbytes,
                                           _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(v2.cpu()[:, :4], got[:, :4]), cap
        assert torch.equal(v2.cpu()[:, cols], got[:, cols]), cap
    # against the default kernel (its entries 4..K; 0..3 belong to the node kernel there)
    ref = torch.zeros(B, K, device=d)
    assert lib.distegnn_virtual_layer_fwd(*args, _ptr(ref), _stream()) == 0
    torch.cuda.synchronize()
    ref = ref.cpu()
    assert float((ref[:, cols] - got[:, cols]).abs().max()) <= 1e-5 * max(1.0, float(ref[:, cols].abs().max()))


LAYOUTS = [
    ("hub6000", dict(sizes=[3000, 500], hub=6000), 5, 2),
    ("tiny_graphs", dict(sizes=[1] * 300 + [0] * 5 + [2] * 100 + [3] * 50), 3, 1),
    ("empty_graphs", dict(sizes=[50, 0, 0, 80, 0, 1, 0]), 8, 0),
    ("many_chunks_c1", dict(sizes=[20000, 3]), 1, 2),
    ("many_chunks_c16", dict(sizes=[3000, 5000]), 16, 8),
] + [(f"C{c}_A{a}", dict(sizes=[700, 300, 1, 1200]), c, a) for c in (1, 3, 5, 8, 16) for a in (0, 1, 2, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,layout,Cn,A", LAYOUTS, ids=[x[0] for x in LAYOUTS])
def test_outputs_do_not_depend_on_the_grid_or_concurrent_work(name, layout, Cn, A):
    d = dev()
    m, _ = _model(Cn, A, dev=d)
    inp = {k: (v.to(d) if v is not None else None) for k, v in _inputs(A=A, **layout).items()}
    m.deterministic = True
    runs = []
    with torch.no_grad():
        for cap in (1, 7, None):                 # the testing library's capped twins, then the product at full grid
            m._backend = None if cap is None else _capped_backend(cap)
            runs.append(m(**inp))
        m._backend = None
        side = torch.cuda.Stream(device=d)
        big = torch.randn(6144, 6144, device=d)
        side.wait_stream(torch.cuda.current_stream(d))
        with torch.cuda.stream(side):
            for _ in range(4):
                big = big @ big * 1e-3
        runs.append(m(**inp))                    # runs while the side stream's GEMMs occupy the SMs
        torch.cuda.synchronize()
        m.deterministic = False
        ref = m(**inp)
    for i, (out, X) in enumerate(runs[1:]):
        assert torch.equal(X, runs[0][1]), (i, float((X - runs[0][1]).abs().max()))
        assert torch.equal(out, runs[0][0]), (i, float((out - runs[0][0]).abs().max()))
    out, X = runs[0]
    assert torch.isfinite(out).all()
    for a_, b_ in ((out, ref[0]), (X, ref[1])):
        assert float((a_ - b_).abs().max()) <= 1e-5 * max(1.0, float(b_.abs().max())), name


@pytest.mark.gpu
def test_captured_forward_keeps_its_workspace_when_a_larger_graph_grows_it():
    """A graphed forward captured with few edges, then a forward with more edges of the same shape (which swaps the
    shared deterministic workspace for a larger one), then memory churn over the old size: replaying the first graph
    must still write to its own workspace and give the same bits."""
    d = dev()
    m, _ = _model(5, 2, dev=d)
    m.deterministic, m.cuda_graph, m.validate_inputs = True, True, False
    few = {k: (v.to(d) if v is not None else None) for k, v in _inputs([800, 400], 2, max_deg=8, seed=1).items()}
    many = {k: (v.to(d) if v is not None else None) for k, v in _inputs([800, 400], 2, max_deg=60, seed=2).items()}
    N, E1, E2 = 1200, few["edge_index"].shape[1], many["edge_index"].shape[1]
    small = _lib.deterministic_workspace_bytes(N, E1, 5)
    assert _lib.deterministic_workspace_bytes(N, E2, 5) > small
    with torch.no_grad():
        first = [t.clone() for t in m(**few)]
        assert len(m._graph_cache) == 1
        second = [t.clone() for t in m(**many)]
        ws = next(iter(m._workspaces.values()))
        assert ws["det"].numel() >= _lib.deterministic_workspace_bytes(N, E2, 5)
        junk = [torch.full((small,), 255, dtype=torch.uint8, device=d) for _ in range(8)]   # reuse freed blocks
        again = m(**few)
        again2 = m(**many)
        torch.cuda.synchronize()
    assert len(m._graph_cache) == 2
    assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])
    assert torch.equal(again2[0], second[0]) and torch.equal(again2[1], second[1])
    assert all(bool((j == 255).all()) for j in junk)           # and nothing was written into someone else's memory


@pytest.mark.gpu
def test_outputs_do_not_depend_on_the_edge_capacity():
    from distegnn_b200.partition import radius_graph_csr
    d = dev()
    m, _ = _model(5, 2, dev=d)
    m.deterministic = True
    w = synth.WORKLOADS["fluid113k"]
    inp = {k: (v.to(d) if v is not None else None) for k, v in synth.make_partitions(w, n_nodes=6000, seed=2)[0].items()}
    inp["node_attr"] = torch.randn(inp["node_loc"].shape[0], 2, device=d)
    outs = []
    for cap in (None, 400_000, 1_000_003):
        g, ea = radius_graph_csr(inp["node_loc"], w.radius, None, edge_attr_nf=2, capacity=cap)
        a = dict(inp, edge_index=g, edge_attr=ea)
        with torch.no_grad():
            outs.append(m(**a))
    E = int(g.n_edges_dev.item()) if g.n_edges_dev is not None else g.num_edges
    assert 0 < E < 400_000
    for out, X in outs[1:]:
        assert torch.equal(out, outs[0][0]) and torch.equal(X, outs[0][1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", SINGLE_CASES)
def test_golden_fixtures_pass_the_parity_gates(name):
    """The gates of test_gpu_parity (final outputs and the per-layer h/x/Hv/X traces of the training-path forward) with
    the mode on; two runs are bitwise equal and agree with the default mode within its run-to-run bound."""
    from tests.test_gpu_parity import check_close, cuda_model, to_dev
    z, kw, sd = load_golden(name)
    inp = golden_inputs(z)
    m = cuda_model(kw, sd)
    m.deterministic = True
    with torch.no_grad():
        out, X = m(**to_dev(inp))
        out2, X2 = m(**to_dev(inp))
        m.deterministic = False
        ref, refX = m(**to_dev(inp))
    check_close(out, X, torch.from_numpy(z["out64.node_loc"]), torch.from_numpy(z["out64.virtual_loc"]),
                inp["node_loc"], name)
    assert torch.equal(out, out2) and torch.equal(X, X2)
    assert within_rerun_bound(out, ref) and within_rerun_bound(X, refX)
    # per-layer traces (one extra layer makes the last real layer's h', Hv' live)
    L = kw["n_layers"]
    trace = {k: golden_trace(z, k) for k in ("h", "x", "Hv", "X")}
    sdx = dict(sd)
    for k, v in sd.items():
        if k.startswith(f"gcl_{L - 1}."):
            sdx[k.replace(f"gcl_{L - 1}.", f"gcl_{L}.")] = v.clone()
    runs = []
    for _ in range(2):
        mt = cuda_model(dict(kw, n_layers=L + 1), sdx).train()
        mt.deterministic = True
        kept = []
        mt._keep_state = kept
        mt(**to_dev(inp))
        torch.cuda.synchronize()
        runs.append(kept[0]["layers"])
    for l in range(L):
        nxt, nxt2 = runs[0][l + 1], runs[1][l + 1]
        got = dict(h=nxt["h"], x=nxt["x4"][:, :3], Hv=nxt["Hv"].transpose(1, 2), X=nxt["Xv"])
        got2 = dict(h=nxt2["h"], x=nxt2["x4"][:, :3], Hv=nxt2["Hv"].transpose(1, 2), X=nxt2["Xv"])
        for k, g in got.items():
            r = trace[k][l]
            assert max_abs(g.cpu(), r) / max(1.0, float(r.abs().max())) <= 2e-5, (name, l, k)
            assert torch.equal(g, got2[k]), (name, l, k)
        for k in ("agg_m", "agg_x", "vsum"):
            if nxt[k] is not None:
                assert torch.equal(nxt[k], nxt2[k]), (name, l, k)


# ---- rollouts ------------------------------------------------------------------------------------------------------------
FLUID = dict(node_feat_nf=3, node_attr_nf=2, edge_attr_nf=2, virtual_channels=5, n_layers=4)


def _rollout_case(n=6000, seed=3):
    d = dev()
    w = synth.WORKLOADS["fluid113k"]
    inp = synth.make_partitions(w, n_nodes=n, seed=seed)[0]
    sd = orc.init_state_dict(3, 2, 2, 64, 5, 4, seed=1, coord_gain=0.05)
    m = FastEGNN(hidden_nf=64, world_size=1, normalize=w.normalize, **FLUID)
    m.load_state_dict(sd)
    m = m.to(d).eval()
    m.deterministic = True
    node = {k: (v.to(d) if v is not None else None) for k, v in inp.items() if k not in ("edge_index", "edge_attr")}
    return m, node, w


def _same(a, b):
    assert torch.equal(a.trajectory, b.trajectory)
    assert torch.equal(a.loc_mean, b.loc_mean)
    assert torch.equal(a.virtual_loc, b.virtual_loc)
    assert torch.equal(a.n_edges, b.n_edges)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["radius", "fixed_graph", "cutoff"])
def test_two_rollouts_are_bitwise_equal(mode):
    from distegnn_b200.partition import radius_graph_csr
    m, node, w = _rollout_case()
    kw = dict(steps=12, speed_col=0, return_trajectory=True)
    if mode == "fixed_graph":
        kw["graph"] = radius_graph_csr(node["node_loc"], w.radius, None, edge_attr_nf=2)[0]
    else:
        kw["radius"] = w.radius
    if mode == "cutoff":
        kw["cutoff_rate"] = 0.3
    with torch.no_grad():
        a = rollout(m, **node, **kw)
        b = rollout(m, **node, **kw)
    _same(a, b)


@pytest.mark.gpu
def test_graphed_rollout_equals_eager_bitwise():
    m, node, w = _rollout_case()
    with torch.no_grad():
        eager = rollout(m, **node, steps=8, radius=w.radius, speed_col=0, return_trajectory=True)
        m.cuda_graph = True
        graphed = rollout(m, **node, steps=8, radius=w.radius, speed_col=0, return_trajectory=True)
    assert graphed.replays > 0
    _same(eager, graphed)


@pytest.mark.gpu
@pytest.mark.parametrize("graphed", [False, True])
def test_overflow_rerun_equals_ample_capacity_bitwise(graphed):
    m, node, w = _rollout_case()
    m.cuda_graph = graphed
    with torch.no_grad():
        ample = rollout(m, **node, steps=6, radius=w.radius, speed_col=0, return_trajectory=True, capacity=2_000_000)
        e0 = int(ample.n_edges[0])
        small = rollout(m, **node, steps=6, radius=w.radius, speed_col=0, return_trajectory=True, capacity=e0 // 2,
                        check_every=2)
    assert small.regrowths
    _same(ample, small)


@pytest.mark.gpu
def test_differentiable_rollout_forward_equals_rollout_bitwise():
    m, node, w = _rollout_case(n=3000)
    with torch.no_grad():
        ref = rollout(m, **node, steps=5, radius=w.radius, speed_col=0, return_trajectory=True)
    res = differentiable_rollout(m, **node, steps=5, radius=w.radius, speed_col=0)
    assert torch.equal(res.trajectory.detach(), ref.trajectory)
    assert torch.equal(res.virtual_locs[-1].detach(), ref.virtual_loc)
    res2 = differentiable_rollout(m, **node, steps=5, radius=w.radius, speed_col=0)
    assert torch.equal(res2.trajectory.detach(), res.trajectory.detach())
    assert torch.equal(res2.virtual_locs.detach(), res.virtual_locs.detach())


@pytest.mark.gpu
def test_mode_off_again_gives_the_default_rollout():
    """Switching the mode off again gives the default path (within its own run-to-run bound of a det run)."""
    m, node, w = _rollout_case(n=3000)
    with torch.no_grad():
        det = rollout(m, **node, steps=3, radius=w.radius, speed_col=0, return_trajectory=True)
        m.deterministic = False
        dflt = rollout(m, **node, steps=3, radius=w.radius, speed_col=0, return_trajectory=True)
    assert float((det.trajectory - dflt.trajectory).abs().max()) <= 1e-4 * max(1.0, float(dflt.trajectory.abs().max()))


@pytest.mark.gpu
def test_two_rank_graphed_rollouts_are_bitwise_equal_on_each_rank():
    """2 ranks (2 GPUs) under torchrun, graphed, rank 0 with too small a capacity (it regrows, both ranks rerun): two
    deterministic rollouts are bitwise equal on every rank (scripts/rollout_dist_check.py --deterministic).  Skipped with
    a single GPU."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29548", os.path.join(root, "scripts", "rollout_dist_check.py"),
           "--deterministic"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    print(p.stdout[-3000:], p.stderr[-1500:])
    assert p.returncode == 0 and "ROLLOUT_DIST PASS" in p.stdout and '"repeat_bitwise_equal": [true, true]' in p.stdout
