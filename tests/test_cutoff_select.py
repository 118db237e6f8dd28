"""The edge cutoff's selection (csrc/cutoff_csr.cu, DESIGN §16) against an exact reference, on every digit pass, tie and
tile boundary of its segmented radix select.

The reference is the rule on integer keys: key = the u32 bits of the fp32 length (NaN -> 0xffffffff); per graph a stable
order by (key, candidate position); the first k_b = int(E_b·(1 − rate)) are kept; the output is in candidate order and
rowptr_out[i] = kept candidates before rowptr_in[i].  Where the layout is a star (hubs at the origin, spoke j at
(L_j, 0, 0)) every key is chosen before launch: the length is fp32 sqrt(rn(L_j²)) under any FMA contraction (the other
squares are exact zeros), which is L_j itself for L_j in [1.1e-19, 1.8e19].  Elsewhere the keys come from
`distegnn_edge_lengths_csr`, and the radius build's and the cutoff's edge_attr must equal them bit for bit.  The kept set
is also judged against float64 lengths of the fp32 positions, independently of the fp32 arithmetic.  Compared exactly:
all N+1 entries of rowptr_out, row / col / edge_attr bits of the kept edges, info[0..2], and sentinels past the kept
count (nothing written there).

CPU: the designed cases' claims (exact keys, shared prefixes, where rank k_b − 1 falls in the digit passes, tie counts,
tile positions), the restated reference against oracle/cutoff_oracle.py, and the checker rejecting wrong selections.
GPU: the cases, up to the config-5 radius graph."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from distegnn_b200 import cutoff_edges_csr, radius_graph_csr, synth
from distegnn_b200.backend import CudaBackend
from distegnn_b200.partition import RadiusGraphBuffers
from distegnn_b200.shards import CSRGraph
from oracle import cutoff_oracle as co

F32 = np.float32
TILE = 4096                    # edges per block of the histogram pass (CUT_TILE)
NAN_KEY = 0xFFFFFFFF
INF_KEY = 0x7F800000
REL = 3e-7                     # an fp32 length against the float64 length of the fp32 positions
TINY = 2.0 ** -74              # absolute slack of a length whose square underflows fp32
SENT = 0x7FA5A5A5              # pre-filled into every output buffer: no valid id, and a NaN payload no kernel writes
BIG_ID = 1 << 30               # a tail id far outside every graph: reading it would fault or show


# ---- the reference ------------------------------------------------------------------------------------------------------
def keys_of(length):
    """u32 sort keys (as int64) of fp32 lengths: the bit pattern, NaN -> 0xffffffff."""
    lf = np.asarray(length, dtype=F32)
    return np.where(np.isnan(lf), NAN_KEY, lf.view(np.uint32)).astype(np.int64)


def k_of(counts, rate):
    """int(E_b · (1 − rate)) per graph, in fp64 as Python computes it."""
    return (np.asarray(counts, dtype=np.float64) * (1.0 - rate)).astype(np.int64)


def order_of(keys, gid):
    """A stable order by (graph, key, candidate position)."""
    return np.argsort(np.asarray(gid, dtype=np.int64) << 32 | keys, kind="stable")


def select(keys, gid, B, rate, order=None):
    """bool [E]: the candidates kept."""
    order = order_of(keys, gid) if order is None else order
    counts = np.bincount(gid, minlength=B)
    start = np.cumsum(counts) - counts
    rank = np.empty(keys.shape[0], dtype=np.int64)
    rank[order] = np.arange(keys.shape[0]) - start[gid[order]]
    return rank < k_of(counts, rate)[gid]


class Case:
    """A candidate CSR graph on the host: pos fp32 [N,3], rowptr [N+1], col / row [E], batch [N] (graphs contiguous),
    and, for star layouts, the keys known before launch."""

    def __init__(self, pos, rowptr, col, batch, B, keys=None):
        self.pos = np.ascontiguousarray(pos, dtype=F32)
        self.rowptr = np.asarray(rowptr, dtype=np.int64)
        self.col = np.asarray(col, dtype=np.int32)
        self.N, self.E, self.B = self.pos.shape[0], int(self.rowptr[-1]), int(B)
        self.row = np.repeat(np.arange(self.N, dtype=np.int32), np.diff(self.rowptr))
        self.batch = np.zeros(self.N, dtype=np.int64) if batch is None else np.asarray(batch, dtype=np.int64)
        self.gid = self.batch[self.row]
        self.keys = keys


def expected(case, keys, valid, nc, cap, overflow_in, rate, order=None):
    """The reference output for the first `valid` candidates with the given keys."""
    mask = select(keys, case.gid[:valid], case.B, rate, order)
    before = np.concatenate([[0], np.cumsum(mask)])
    kept = int(mask.sum())
    return dict(mask=mask, kept=kept, rowptr=before[np.minimum(case.rowptr, valid)], row=case.row[:valid][mask],
                col=case.col[:valid][mask], keys=keys[mask], info=[kept, int(nc > cap or bool(overflow_in)), nc])


def judge(exp, got, A):
    """The device output `got` (host arrays of the pre-filled buffers) against the reference, exactly."""
    k = exp["kept"]
    rp = got["rowptr"]
    bad = np.flatnonzero(rp != exp["rowptr"])
    assert bad.size == 0, f"rowptr_out differs at {bad.size} entries, first {bad[0]}: {rp[bad[0]]} != {exp['rowptr'][bad[0]]}"
    assert got["info"][:3].tolist() == exp["info"], f"info {got['info'][:3].tolist()} != {exp['info']}"
    for name in ("row", "col"):
        bad = np.flatnonzero(got[name][:k] != exp[name])
        assert bad.size == 0, f"{name} of the kept edges differs at {bad.size} entries, first {bad[0]}"
        assert (got[name][k:] == SENT).all(), f"{name} written past the kept count"
    if A:
        ea = got["ea"]
        want = exp["keys"].astype(np.uint32).view(np.int32)
        nan = exp["keys"] == NAN_KEY
        assert (ea[:k][~nan] == want[~nan][:, None]).all(), "edge_attr bits differ from the keys"
        assert ((ea[:k][nan] & 0x7FFFFFFF) > INF_KEY).all(), "edge_attr of a NaN key is not NaN"
        assert (ea[k:] == SENT).all(), "edge_attr written past the kept count"


def judge64(case, valid, mask, keyf):
    """Independent of the fp32 arithmetic: every finite key within REL of the float64 length of the fp32 positions, and
    per graph the longest kept float64 length <= the shortest dropped one · (1 + 2·REL); NaN is the longest, lengths
    beyond the fp32 range count as inf."""
    row, col, gid = case.row[:valid], case.col[:valid], case.gid[:valid]
    p = case.pos.astype(np.float64)
    L64 = np.sqrt(((p[row] - p[col]) ** 2).sum(axis=1))
    nan = np.isnan(keyf)
    assert np.array_equal(nan, np.isnan(L64)), "NaN keys where the float64 length is not NaN (or the reverse)"
    fin = np.isfinite(keyf)
    err = np.abs(keyf[fin].astype(np.float64) - L64[fin])
    assert (err <= REL * L64[fin] + TINY).all(), f"fp32 length off float64 by {float((err / np.maximum(L64[fin], TINY)).max()):.3e}"
    v = np.where(np.isinf(keyf), np.inf, L64)
    kmax = np.full(case.B, -np.inf)
    np.maximum.at(kmax, gid[mask & ~nan], v[mask & ~nan])
    dmin = np.full(case.B, np.inf)
    np.minimum.at(dmin, gid[~mask & ~nan], v[~mask & ~nan])
    bad = np.flatnonzero(~(kmax <= dmin * (1 + 2 * REL) + TINY))
    assert bad.size == 0, f"graph {bad[0]}: kept {kmax[bad[0]]!r} > dropped {dmin[bad[0]]!r}"
    kept_nan = np.bincount(gid[mask & nan], minlength=case.B) > 0
    dropped_num = np.bincount(gid[~mask & ~nan], minlength=case.B) > 0
    assert not (kept_nan & dropped_num).any(), "a NaN kept while a number was dropped"


def got_of_mask(case, keys, valid, mask, nc, cap, overflow_in, A):
    """What a kernel that selected `mask` would leave in the pre-filled buffers (for the checker's self-test)."""
    e = expected(case, keys, valid, nc, cap, overflow_in, 0.0)
    before = np.concatenate([[0], np.cumsum(mask)])
    k = int(mask.sum())
    pad = lambda a: np.concatenate([a, np.full(cap - a.shape[0], SENT, dtype=np.int32)])
    ea = np.full((cap, A), SENT, dtype=np.int32)
    kb = keys[mask]
    ea[:k] = np.where(kb == NAN_KEY, 0x7FC00000, kb).astype(np.uint32).view(np.int32)[:, None]
    return dict(rowptr=before[np.minimum(case.rowptr, valid)], row=pad(case.row[:valid][mask]),
                col=pad(case.col[:valid][mask]), ea=ea, info=np.array([k] + e["info"][1:] + [0]))


# ---- star layouts: keys known before launch -----------------------------------------------------------------------------
def stars(L, hubs=1, mirror=False, iso=0, loop=False):
    """A batch of star graphs.  L: per graph an fp32 array of spoke offsets, or None for a graph without nodes.  Graph b:
    `hubs` coincident hubs at the origin, then its spokes at (L_j, 0, 0), then `iso` nodes without edges.  Every hub row
    holds (its self loop first if `loop`, then) one edge to every spoke in order; with `mirror` every spoke row holds one
    edge to every hub.  hubs / mirror / iso / loop: scalars or per graph."""
    B = len(L)
    nodeless = np.array([l is None for l in L])
    M = np.array([0 if l is None else len(l) for l in L], dtype=np.int64)
    per = lambda v, dt: np.broadcast_to(np.asarray(v, dtype=dt), (B,)).copy()
    H, I, mir, lp = per(hubs, np.int64), per(iso, np.int64), per(mirror, bool), per(loop, bool)
    H[nodeless] = 0
    I[nodeless] = 0
    n = H + M + I
    off = np.cumsum(n) - n
    N = int(n.sum())
    ng = np.repeat(np.arange(B), n)
    li = np.arange(N) - off[ng]
    hub = li < H[ng]
    spoke = ~hub & (li < (H + M)[ng])
    deg = np.where(hub, M[ng] + lp[ng], np.where(spoke, H[ng] * mir[ng], 0))
    rowptr = np.zeros(N + 1, dtype=np.int64)
    rowptr[1:] = np.cumsum(deg)
    row = np.repeat(np.arange(N), deg)
    q = np.arange(int(rowptr[-1])) - rowptr[row]
    g = ng[row]
    in_hub = hub[row]
    hub_col = np.where(lp[g] & (q == 0), row, off[g] + H[g] + q - lp[g])
    col = np.where(in_hub, hub_col, off[g] + q)
    x = np.zeros(N, dtype=F32)
    x[spoke] = np.concatenate([np.asarray(l, dtype=F32) for l in L if l is not None] + [np.zeros(0, F32)])
    pos = np.zeros((N, 3), dtype=F32)
    pos[:, 0] = x
    pos[~hub & ~spoke] = (0.25, 0.5, 0.75)
    d = x[np.where(in_hub, col, row)]                         # hub − spoke or spoke − hub: ±L_j, exact
    with np.errstate(over="ignore"):
        keys = keys_of(np.sqrt(d * d))                        # fp32: rn(L²), then the correctly rounded sqrt
    return Case(pos, rowptr, col, ng, B, keys)


def lengths_of_bits(bits):
    return np.asarray(bits, dtype=np.uint32).view(F32)


def distinct_lengths(rng, n):
    """n distinct fp32 lengths in [1, 2), in random order."""
    return lengths_of_bits(0x3F800000 + rng.choice(1 << 23, size=n, replace=False))


def exact_length(L):
    """fp32 sqrt(rn(L²)) == L bit for bit."""
    L = np.asarray(L, dtype=F32)
    return np.array_equal(np.sqrt(L * L).view(np.uint32), L.view(np.uint32))


def rate_for(k, E):
    rate = 1 - (k + 0.5) / E
    assert int(E * (1 - rate)) == k
    return rate


# ---- 1. digit passes ----------------------------------------------------------------------------------------------------
PREFIX = {1: 0x3F, 2: 0x3F8A, 3: 0x3F8A5B}       # keys sharing their top 1, 2 or 3 bytes
DIGIT_TARGETS = ("first", "last", "single", "bin0", "bin255", "lane7", "lane8", "k1", "kEm1")
SINGLE_BIN, WIDE_BIN = 131, 64


def digit_case(p, seed=0):
    """One star graph of 50,000 edges (13 tiles) whose keys share their top p bytes; the next digit (pass p) spreads over
    the 256 bins with bins 0, 7, 8, 255 and WIDE_BIN well filled, SINGLE_BIN holding one key and a few bins empty.
    Returns (case, {target: k})."""
    rng = np.random.default_rng(100 + p)
    E = 50_000
    h = rng.integers(0, 360, size=256)
    h[rng.choice(256, size=12, replace=False)] = 0
    h[[0, 7, 8, 255, WIDE_BIN]] = (300, 250, 250, 300, 280)
    h[SINGLE_BIN] = 1
    h[200] = 0
    h[200] = E - h.sum()
    assert h[200] > 0
    shift = 24 - 8 * p
    digit = np.repeat(np.arange(256), h)
    low = rng.integers(0, 1 << shift, size=E) if shift else np.zeros(E, dtype=np.int64)
    bits = (PREFIX[p] << (shift + 8)) | (digit << shift) | low
    L = lengths_of_bits(rng.permutation(bits))
    c = np.concatenate([[0], np.cumsum(h)])                    # keys with digit < b
    k = dict(first=c[WIDE_BIN] + 1, last=c[WIDE_BIN + 1], single=c[SINGLE_BIN] + 1, bin0=h[0] // 2 + 1,
             bin255=c[255] + h[255] // 2 + 1, lane7=c[8], lane8=c[8] + 1, k1=1, kEm1=E - 1)
    return stars([L]), {t: int(v) for t, v in k.items()}


def radix_trace(keys, k):
    """Per digit pass over one graph's keys: (bin, rank within the bin, histogram) of rank k − 1."""
    r, sel, out = k - 1, np.asarray(keys, dtype=np.int64), []
    for p in range(4):
        d = (sel >> (24 - 8 * p)) & 255
        h = np.bincount(d, minlength=256)
        c = np.cumsum(h)
        b = int(np.searchsorted(c, r, side="right"))
        r -= int(c[b] - h[b])
        out.append((b, r, h))
        sel = sel[d == b]
    return out


def digit_claim(target, trace, p, k, E):
    b, left, h = trace[p]
    return {"first": left == 0 and h[b] >= 2, "last": left == h[b] - 1 and h[b] >= 2, "single": h[b] == 1,
            "bin0": b == 0 and 0 < left < h[0] - 1, "bin255": b == 255 and 0 < left < h[255] - 1,
            "lane7": b == 7 and left == h[7] - 1 and h[8] > 0, "lane8": b == 8 and left == 0 and h[7] > 0,
            "k1": k == 1, "kEm1": k == E - 1}[target]


# ---- 2. ties at the threshold -------------------------------------------------------------------------------------------
TIE_L = F32(1.5)
TIE_NEED = ("one", "half", "all_but_one")


def tie_case(boundaries, seed=0):
    """A star graph of 3 coincident hubs and 6,000 spokes with mirror edges (36,000 edges, 9 tiles); 40 spokes at TIE_L,
    so 240 equal keys on the three hub rows and 40 spoke rows.  `boundaries`: small graphs before and after it, so tiles
    holding ties also hold graph boundaries (the global histogram path).  Returns (case, main graph id)."""
    rng = np.random.default_rng(seed)
    L = distinct_lengths(rng, 6000)
    L = L[L != TIE_L]
    L[rng.choice(L.shape[0], size=40, replace=False)] = TIE_L
    if not boundaries:
        return stars([L], hubs=3, mirror=True), 0
    return stars([distinct_lengths(rng, 1500), L, distinct_lengths(rng, 700)], hubs=[1, 3, 1], mirror=[False, True, False]), 1


def tie_k(case, g, need):
    keys = case.keys[case.gid == g]
    less, ties = int((keys < keys_of(TIE_L)).sum()), int((keys == keys_of(TIE_L)).sum())
    return less + {"one": 1, "half": ties // 2, "all_but_one": ties - 1}[need], less, ties


# ---- 3. tiles and graph layouts -----------------------------------------------------------------------------------------
def boundary_case(seed=0):
    """Star graphs starting on a tile start, at t0 + 1 and at t1 − 1 of tiles 1..6, with graphs without nodes first,
    last, consecutive and on tile boundaries, and graphs with nodes but no edges on tile boundaries."""
    rng = np.random.default_rng(seed)
    starts = sorted({t * TILE + o for t in range(1, 7) for o in (0, 1, TILE - 1)} | {7 * TILE + 2, 7 * TILE + 3})
    sizes = np.diff([0] + starts + [7 * TILE + 900])
    lens = np.split(distinct_lengths(rng, int(sizes.sum())), np.cumsum(sizes)[:-1])
    L = [None, None]
    for i, l in enumerate(lens):
        L.append(l)
        if i in (0, 3):
            L += [None, None, None]                           # consecutive graphs without nodes, on a tile start
        if i in (6, 9):
            L += [np.zeros(0, F32), None]                     # a hub without edges, then no nodes, on a tile start
    L.append(None)
    return stars(L, iso=[i % 3 for i in range(len(L))])


def tiny_graphs_case(seed=0):
    """Hundreds of tiny graphs with distinct keys inside one tile, between a full tile and a larger graph."""
    rng = np.random.default_rng(seed)
    sizes = [TILE] + list(rng.integers(0, 11, size=350)) + [3000]
    lens = np.split(distinct_lengths(rng, int(sum(sizes))), np.cumsum(sizes)[:-1])
    return stars(lens), len(sizes)


def long_graph_case(seed=0):
    """One graph over 301 tiles between one-edge graphs."""
    rng = np.random.default_rng(seed)
    sizes = [1, 1, 301 * TILE - 5, 1, 1, 1]
    lens = np.split(distinct_lengths(rng, int(sum(sizes))), np.cumsum(sizes)[:-1])
    return stars(lens)


def many_graphs_case(B=100_000, seed=0):
    """B graphs: 0–30 spokes, every 20th without nodes, every 7th with two hubs and mirror edges (ties across rows)."""
    rng = np.random.default_rng(seed)
    m = rng.integers(0, 31, size=B)
    lens = np.split(lengths_of_bits(0x3F800000 + rng.integers(0, 1 << 23, size=int(m.sum()))), np.cumsum(m)[:-1])
    L = [None if b % 20 == 0 else l for b, l in enumerate(lens)]
    two = np.arange(B) % 7 == 0
    return stars(L, hubs=np.where(two, 2, 1), mirror=two)


# ---- 4. count extremes --------------------------------------------------------------------------------------------------
COUNT_RATES = (0.0, 1.0, 2.0 ** -52, 1 - 2.0 ** -52, 1 / 3, 0.1, 0.3, 0.7, 0.9)
# edge counts where E·(1 − rate) is an integer in decimal but one fp64 rounding away from it (none for 0.1 below 2000)
NEAR_INT = {r: [E for E in range(1, 1000) if (E * (1 - Fraction(s))).denominator == 1
                and E * (1 - r) != E * (1 - Fraction(s))][:6] for r, s in ((0.3, "0.3"), (0.7, "0.7"), (0.9, "0.9"))}


def count_case(seed=0):
    """Graphs of 0–40 edges, of 99–101 and 4095–4097 edges, and of the NEAR_INT edge counts; graphs without nodes
    between them."""
    rng = np.random.default_rng(seed)
    sizes = list(range(41)) + [99, 100, 101, 4095, 4096, 4097] + sorted({E for v in NEAR_INT.values() for E in v})
    rng.shuffle(sizes)
    lens = np.split(distinct_lengths(rng, int(sum(sizes))), np.cumsum(sizes)[:-1])
    L = []
    for i, l in enumerate(lens):
        L += [l] + ([None] if i % 9 == 4 else [])
    return stars(L, loop=False)


# ---- 5. special lengths -------------------------------------------------------------------------------------------------
L_MIN = np.nextafter(F32(2.0 ** -75), F32(1))             # the smallest offset whose square does not underflow to 0
KEY_MIN = int(keys_of(np.sqrt(L_MIN * L_MIN)))            # the smallest non-zero key a length can have
SPECIAL_CLASS = {"zero": 0, "underflow": 0, "smallest": KEY_MIN, "inf": INF_KEY, "nan": NAN_KEY}


def special_case(seed=0):
    """Graphs of 40 edges each (one hub), whose threshold at rate 0.5 (k = 20) falls inside one class of special keys:
    zero from a self loop and coincident spokes; zero from offsets below 2^-75; the smallest non-zero key; +inf from
    |x| ≈ 3e38; NaN from a NaN coordinate.  Then a keep-none graph of one zero-length edge, one of one self loop, and a
    graph of only NaN edges (kept whole at rate 0).  Returns (case, [class of each graph])."""
    rng = np.random.default_rng(seed)
    r = lambda n: 1 + rng.random(n).astype(F32)
    shuf = lambda *a: rng.permutation(np.concatenate([np.asarray(x, dtype=F32) for x in a]))
    nan = F32(np.nan)
    L = [shuf(np.zeros(24), r(15)),                                                   # + the self loop: 25 zeros
         shuf(rng.choice([1e-23, -1e-23, 5e-24, -2e-23, 2.0 ** -76], size=22), np.zeros(3), r(15)),
         shuf(np.zeros(10), np.full(20, L_MIN), -np.full(4, L_MIN), r(6)),
         shuf(r(10), rng.choice([3e38, -3.2e38, 3.4e38], size=25), np.full(5, nan)),
         shuf(r(10), np.full(30, nan)),
         np.zeros(1, F32), np.zeros(0, F32), np.full(3, nan)]
    classes = ["zero", "underflow", "smallest", "inf", "nan", "none", "none", "all_nan"]
    return stars(L, loop=[True, False, False, False, False, False, True, False]), classes


# ---- 6. device counts ---------------------------------------------------------------------------------------------------
def count_dev_case(seed=0):
    """Three mirrored stars (hub rows of 3,000 edges, 3 hubs) and one plain one, about 21,500 edges; the last node has a
    NaN coordinate and no edges (a capacity tail pointing at it must never be read)."""
    rng = np.random.default_rng(seed)
    L = [distinct_lengths(rng, 3000), distinct_lengths(rng, 200), distinct_lengths(rng, 400), distinct_lengths(rng, 900)]
    case = stars(L, hubs=[3, 2, 3, 1], mirror=[True, True, True, False], iso=[0, 0, 0, 1])
    case.pos[-1] = np.nan
    return case


def device_counts(case):
    """n_edges_dev values: mid-row, on a row boundary inside a graph, on a tile boundary, and 0."""
    rp = case.rowptr
    starts = np.concatenate([[0], np.cumsum(np.bincount(case.batch, minlength=case.B))])
    first_rows = set(starts.tolist())
    inner = [int(rp[i]) for i in range(1, case.N) if i not in first_rows and 0 < rp[i] < case.E and rp[i] % TILE]
    mid_row = int(rp[1]) + 17
    assert rp[1] < mid_row < rp[2]
    return dict(mid_row=mid_row, row_boundary=inner[len(inner) // 2], tile=2 * TILE, zero=0)


# ---- CPU ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [1, 2, 3])
def test_digit_case_claims(p):
    case, ks = digit_case(p)
    E = case.E
    L = case.pos[1:, 0]
    assert E == 50_000 and -(-E // TILE) == 13
    assert exact_length(L) and np.array_equal(np.sort(case.keys), np.sort(keys_of(L)))
    shift = 32 - 8 * p
    assert (case.keys >> shift == PREFIX[p]).all(), "the keys share their top p bytes"
    for target in DIGIT_TARGETS:
        k = ks[target]
        tr = radix_trace(case.keys, k)
        assert all(int((tr[q][2] > 0).sum()) == 1 for q in range(p)), "passes before p see one bucket"
        assert int((tr[p][2] > 0).sum()) > 200, "pass p decides"
        assert digit_claim(target, tr, p, k, E), target
        assert int(E * (1 - rate_for(k, E))) == k


@pytest.mark.parametrize("boundaries", [False, True], ids=["one_graph", "boundaries"])
def test_tie_case_claims(boundaries):
    case, g = tie_case(boundaries)
    assert exact_length(case.pos[:, 0])
    T = int(keys_of(TIE_L))
    tie = np.flatnonzero((case.keys == T) & (case.gid == g))
    assert tie.size == 240
    assert len(set((tie // TILE).tolist())) >= 3 and len(set(case.row[tie].tolist())) >= 40
    tiles_with_boundary = set()
    gs = np.concatenate([[0], np.cumsum(np.bincount(case.gid, minlength=case.B))])
    for s in gs[1:-1]:
        tiles_with_boundary.add(int(s) // TILE)
    if boundaries:
        assert tiles_with_boundary & set((tie // TILE).tolist()), "ties in a tile holding a graph boundary"
        assert set((tie // TILE).tolist()) - tiles_with_boundary, "and ties in a tile inside the graph"
    for need in TIE_NEED:
        k, less, ties = tie_k(case, g, need)
        keys = case.keys[case.gid == g]
        assert np.sort(keys)[k - 1] == T and k - less == {"one": 1, "half": 120, "all_but_one": 239}[need]
        assert ties == 240


def test_layout_case_claims():
    case = boundary_case()
    gs = np.concatenate([[0], np.cumsum(np.bincount(case.gid, minlength=case.B))])
    E_b = np.diff(gs)
    starts = set(gs[:-1][E_b > 0].tolist())
    for t in range(1, 7):
        assert {t * TILE, t * TILE + 1, (t + 1) * TILE - 1} <= starts
    nodes = np.bincount(case.batch, minlength=case.B)
    assert nodes[0] == 0 and nodes[1] == 0 and nodes[-1] == 0
    assert any(nodes[i] == nodes[i + 1] == 0 and gs[i] % TILE == 0 and 0 < gs[i] < case.E for i in range(2, case.B - 1))
    assert any(nodes[i] > 0 and E_b[i] == 0 and gs[i] % TILE == 0 and 0 < gs[i] < case.E for i in range(case.B))
    assert exact_length(case.pos[:, 0])
    tiny, Bt = tiny_graphs_case()
    gs = np.concatenate([[0], np.cumsum(np.bincount(tiny.gid, minlength=tiny.B))])
    inside = [b for b in range(1, Bt - 1) if gs[b] // TILE == 1 and gs[b + 1] <= 2 * TILE]
    assert len(inside) == Bt - 2 and len(np.unique(tiny.keys)) == tiny.E
    big = long_graph_case()
    E_b = np.bincount(big.gid, minlength=big.B)
    assert E_b.tolist()[:2] == [1, 1] and E_b[2] >= 300 * TILE and E_b.tolist()[3:] == [1, 1, 1]


def test_count_case_claims():
    case = count_case()
    E_b = np.bincount(case.gid, minlength=case.B)
    assert (np.bincount(case.batch, minlength=case.B) == 0).any()
    for r in COUNT_RATES:
        k = k_of(E_b, r)
        assert (k == np.array([int(E * (1 - r)) for E in E_b])).all()
    for r, Es in NEAR_INT.items():
        assert Es and set(Es) <= set(E_b.tolist()), r
    assert int(10 * (1 - 0.9)) == 0 and int(10 * (1 - 0.7)) == 3 and 10 in E_b
    seen = set()
    for r in COUNT_RATES:
        k = k_of(E_b, r)
        big = E_b >= 3
        seen |= {c for c, m in (("0", k == 0), ("1", k == 1), ("E-1", k == E_b - 1), ("E", k == E_b)) if (m & big).any()}
    assert seen == {"0", "1", "E-1", "E"}


def test_special_case_claims():
    case, classes = special_case()
    E_b = np.bincount(case.gid, minlength=case.B)
    k = k_of(E_b, 0.5)
    for b, cls in enumerate(classes):
        keys = case.keys[case.gid == b]
        if cls in SPECIAL_CLASS:
            T = np.sort(keys)[k[b] - 1]
            less, ties = int((keys < T).sum()), int((keys == T).sum())
            assert E_b[b] == 40 and T == SPECIAL_CLASS[cls] and 0 < k[b] - less < ties, cls
        elif cls == "none":
            assert E_b[b] == 1 and k[b] == 0 and (keys == 0).all()
        else:
            assert (keys == NAN_KEY).all() and k_of(E_b[b], 0.0) == E_b[b]
    und = case.gid == 1
    assert ((case.keys[und] == 0) & (np.abs(case.pos[case.col[und], 0]) > 0)).sum() >= 20, "zeros from underflow"
    assert (case.row[case.gid == 0] == case.col[case.gid == 0]).sum() == 1, "a self loop"


def test_device_count_claims():
    case = count_dev_case()
    n = device_counts(case)
    rp = case.rowptr
    assert not np.isin(n["mid_row"], rp) and n["tile"] % TILE == 0 and n["tile"] < case.E
    i = int(np.searchsorted(rp, n["row_boundary"]))
    assert rp[i] == n["row_boundary"] and case.batch[i] == case.batch[i - 1], "a row boundary inside a graph"
    assert np.isnan(case.pos[-1]).all() and rp[-1] == rp[-2]


def _random_lengths_case(rng):
    """Random graphs (with graphs without nodes and without edges) and lengths drawn with ties, 0, inf and NaN."""
    B = int(rng.integers(1, 12))
    nodes = rng.integers(0, 6, size=B)
    nodes[rng.random(B) < 0.2] = 0
    N = max(int(nodes.sum()), 1)
    nodes[-1] += N - int(nodes.sum())
    batch = np.repeat(np.arange(B), nodes)
    deg = rng.integers(0, 9, size=N)
    rowptr = np.concatenate([[0], np.cumsum(deg)])
    E = int(rowptr[-1])
    pool = np.array([0, 0.5, 0.5, 1, 2, np.inf, np.nan, 3], dtype=F32)
    length = np.where(rng.random(E) < 0.6, rng.choice(pool, size=E), rng.random(E).astype(F32)).astype(F32)
    col = rng.integers(0, N, size=E)
    return Case(np.zeros((N, 3)), rowptr, col, batch, B, keys_of(length)), length


def test_reference_agrees_with_the_oracle():
    rng = np.random.default_rng(0)
    for _ in range(300):
        case, length = _random_lengths_case(rng)
        rate = float(rng.choice([0.0, 1.0, 0.5, 1 / 3, 0.1, 0.9, float(rng.random())]))
        valid = int(rng.integers(0, case.E + 1))
        rp = np.minimum(case.rowptr, valid)
        orp, orow, ocol, olen, omask = co.cutoff_csr(rp, case.row[:valid], case.col[:valid], None, rate, case.batch,
                                                      case.B, lengths=length[:valid])
        e = expected(case, case.keys[:valid], valid, valid, case.E, 0, rate)
        assert np.array_equal(e["mask"], omask) and np.array_equal(e["rowptr"], orp)
        assert np.array_equal(e["row"], orow) and np.array_equal(e["col"], ocol)
        assert np.array_equal(keys_of(olen), e["keys"])


def test_checker_rejects_wrong_selections():
    """The exact checker passes the reference and fails one tie too few, ties broken in reverse order and NaN sorted
    first; the float64 check fails NaN sorted first as well."""
    case, _ = special_case()
    tcase, g = tie_case(True)
    for c, rate in ((case, 0.5), (tcase, rate_for(tie_k(tcase, g, "half")[0], int((tcase.gid == g).sum())))):
        keys, valid, A = c.keys, c.E, 2
        keyf = lengths_of_bits(np.where(keys == NAN_KEY, 0x7FC00000, keys))
        exp = expected(c, keys, valid, valid, c.E, 0, rate)
        judge(exp, got_of_mask(c, keys, valid, exp["mask"], valid, c.E, 0, A), A)
        judge64(c, valid, exp["mask"], keyf)
        kept = exp["mask"]
        T = np.zeros(c.B, dtype=np.int64)
        np.maximum.at(T, c.gid[kept], keys[kept])
        at_T = kept & (keys == T[c.gid])
        tie_graphs = [b for b in range(c.B) if 0 < at_T[c.gid == b].sum() < ((keys == T[b]) & (c.gid == b)).sum()]
        assert tie_graphs
        b = tie_graphs[0]
        ties = np.flatnonzero((keys == T[b]) & (c.gid == b))
        need = int(at_T[c.gid == b].sum())
        few = kept.copy()
        few[ties[need - 1]] = False
        rev = kept.copy()
        rev[ties] = False
        rev[ties[-need:]] = True
        nan_first = select(np.where(keys == NAN_KEY, 0, keys + 1), c.gid, c.B, rate)
        wrong = [few, rev] + ([nan_first] if (keys == NAN_KEY).any() else [])
        for m in wrong:
            assert not np.array_equal(m, kept)
            with pytest.raises(AssertionError):
                judge(exp, got_of_mask(c, keys, valid, m, valid, c.E, 0, A), A)
        if (keys == NAN_KEY).any():
            with pytest.raises(AssertionError, match="NaN kept"):
                judge64(c, valid, nan_first, keyf)


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


_BACKEND = []


def backend():
    if not _BACKEND:
        _BACKEND.append(CudaBackend())
    return _BACKEND[0]


def upload(case, n_valid=None, capacity=None, tail=None, overflow_in=0):
    """The case as a device CSRGraph (+ pos, batch): edge arrays of `capacity` entries (default E; a shorter capacity
    truncates, a longer one pads with `tail`), entries from n_valid on replaced by `tail`, count on the device."""
    d = dev()
    cap = case.E if capacity is None else capacity
    row = np.full(cap, tail if tail is not None else SENT, dtype=np.int64)
    col = row.copy()
    m = min(cap, case.E)
    row[:m], col[:m] = case.row[:m], case.col[:m]
    if n_valid is not None and tail is not None:
        row[n_valid:], col[n_valid:] = tail, tail
    t32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int32)).to(d)
    g = CSRGraph(t32(case.rowptr), t32(col), t32(row))
    if n_valid is not None:
        g.n_edges_dev = t32([n_valid])
    if overflow_in:
        g.info = t32([n_valid if n_valid is not None else case.E, 1, 0, 0])
    pos = torch.from_numpy(case.pos).to(d)
    batch = torch.from_numpy(case.batch).to(d) if case.B > 1 else None
    return g, pos, batch


def buffers(N, cap, A):
    return RadiusGraphBuffers(N, cap, A, dev(), table_cells=27)


def device_keys(g, pos):
    """The library's own fp32 lengths (distegnn_edge_lengths_csr) of g's candidates, as keys; nothing may be written at
    or past the device count."""
    cap = g.num_edges
    ea = torch.full((cap, 1), SENT, dtype=torch.int32, device=pos.device)
    backend().edge_lengths(g.rows(), g.col, pos, g.n_edges_dev, ea.view(torch.float32))
    bits = ea[:, 0].cpu().numpy()
    nc = int(g.n_edges_dev[0]) if g.n_edges_dev is not None else int(g.rowptr[-1])
    valid = max(0, min(nc, cap))
    assert (bits[valid:] == SENT).all(), "distegnn_edge_lengths_csr wrote at or past n_edges_dev"
    keyf = bits[:valid].view(F32)
    return keys_of(keyf), keyf, valid, nc


def fetch(out, A):
    ea = out.edge_attr.view(torch.int32).cpu().numpy() if A else None
    return dict(rowptr=out.rowptr.cpu().numpy().astype(np.int64), row=out.row.cpu().numpy(), col=out.col.cpu().numpy(),
                ea=ea, info=out.info.cpu().numpy())


def check_cut(case, rate, dg=None, A=2, out=None, order=None, overflow_in=0):
    """One cutoff of the device graph dg = (CSRGraph, pos, batch) (default: the whole case) into pre-filled buffers,
    judged exactly against the reference on the device keys and against float64.  Returns the host outputs."""
    g, pos, batch = upload(case) if dg is None else dg
    keys, keyf, valid, nc = device_keys(g, pos)
    if case.keys is not None:
        bad = np.flatnonzero(keys != case.keys[:valid])
        assert bad.size == 0, f"{bad.size} device keys differ from the designed ones, first at {bad[0]}"
    cap = g.num_edges
    if out is None:
        out = buffers(case.N, cap, A)
    for t in (out.rowptr, out.row, out.col, out.info):
        t.fill_(SENT)
    if A:
        out.edge_attr.view(torch.int32).fill_(SENT)
    res, ea = cutoff_edges_csr(g, pos, rate, batch, case.B, A, out=out)
    assert res is out.graph and (ea is None) == (A == 0)
    got = fetch(out, A)
    exp = expected(case, keys, valid, nc, cap, overflow_in, rate, order)
    judge(exp, got, A)
    judge64(case, valid, exp["mask"], keyf)
    return got


def same(a, b):
    return all((a[k] is None and b[k] is None) or np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.gpu
@pytest.mark.parametrize("p", [1, 2, 3])
def test_digit_passes(p):
    case, ks = digit_case(p)
    dg = upload(case)
    for target in DIGIT_TARGETS:
        check_cut(case, rate_for(ks[target], case.E), dg=dg)


@pytest.mark.gpu
@pytest.mark.parametrize("boundaries", [False, True], ids=["one_graph", "boundaries"])
@pytest.mark.parametrize("need", TIE_NEED)
def test_ties_at_the_threshold(boundaries, need):
    case, g_main = tie_case(boundaries)
    k, _, _ = tie_k(case, g_main, need)
    check_cut(case, rate_for(k, int((case.gid == g_main).sum())))


@pytest.mark.gpu
def test_tile_boundaries_and_empty_graphs():
    case = boundary_case()
    dg = upload(case)
    for rate in (0.5, 0.3, 0.77, 0.0, 1.0):
        check_cut(case, rate, dg=dg)


@pytest.mark.gpu
def test_hundreds_of_tiny_graphs_in_one_tile():
    case, _ = tiny_graphs_case()
    dg = upload(case)
    for rate in (0.5, 0.3, 0.9):
        check_cut(case, rate, dg=dg)


@pytest.mark.gpu
def test_a_graph_over_300_tiles_next_to_one_edge_graphs():
    case = long_graph_case()
    dg = upload(case)
    order = order_of(case.keys, case.gid)
    for rate in (0.5, 0.37, 2.0 ** -52):
        check_cut(case, rate, dg=dg, order=order)


@pytest.mark.gpu
def test_100k_graphs():
    case = many_graphs_case()
    dg = upload(case)
    order = order_of(case.keys, case.gid)
    for rate in (0.5, 0.3):
        check_cut(case, rate, dg=dg, order=order)


@pytest.mark.gpu
def test_count_extremes_in_one_batch():
    case = count_case()
    dg = upload(case)
    for rate in COUNT_RATES:
        check_cut(case, rate, dg=dg)


@pytest.mark.gpu
def test_special_lengths():
    case, _ = special_case()
    dg = upload(case)
    for rate in (0.5, 0.0, 1.0, 0.25, 0.75, 0.95):
        check_cut(case, rate, dg=dg)


@pytest.mark.gpu
@pytest.mark.parametrize("tail", ["nan_node", "far_id"])
def test_device_count_and_capacity_tail(tail):
    case = count_dev_case()
    tid = case.N - 1 if tail == "nan_node" else BIG_ID
    for what, n in device_counts(case).items():
        dg = upload(case, n_valid=n, tail=tid)
        check_cut(case, 0.5, dg=dg)
        dg = upload(case, n_valid=n, capacity=case.E + 777, tail=tid)   # capacity past the CSR's end
        check_cut(case, 0.4, dg=dg)


@pytest.mark.gpu
def test_overflowed_candidates_and_count_only_graphs():
    case = count_dev_case()
    cap = case.E - 1000
    dg = upload(case, n_valid=case.E, capacity=cap)             # count > capacity: the first cap candidates
    got = check_cut(case, 0.5, dg=dg)
    assert got["info"][1] == 1 and got["info"][2] == case.E
    dg = upload(case, n_valid=cap - 5, capacity=cap, overflow_in=1)    # flagged by the candidate build
    got = check_cut(case, 0.5, dg=dg, overflow_in=1)
    assert got["info"][1] == 1
    dg = upload(case, n_valid=case.E, capacity=0)               # capacity 0: a count-only graph
    got = check_cut(case, 0.5, dg=dg, A=2)
    assert (got["rowptr"] == 0).all() and got["info"][:3].tolist() == [0, 1, case.E]
    # an overflowed radius build
    x = torch.from_numpy(np.random.default_rng(3).random((3000, 3), dtype=np.float32)).to(dev())
    full, _ = radius_graph_csr(x, 0.1, edge_attr_nf=0)
    E = full.num_edges
    cg, _ = radius_graph_csr(x, 0.1, edge_attr_nf=0, capacity=E // 2)
    rc = Case(x.cpu().numpy(), full.rowptr.cpu().numpy(), full.col.cpu().numpy(), None, 1)
    assert torch.equal(cg.col, full.col[:E // 2]) and torch.equal(cg.rowptr, full.rowptr)
    got = check_cut(rc, 0.5, dg=(cg, x, None), overflow_in=1)
    assert got["info"][:3].tolist()[1:] == [1, E]


@pytest.mark.gpu
def test_reruns_and_buffer_reuse():
    a = count_dev_case(seed=1)
    b = count_dev_case(seed=2)
    assert (a.N, a.B, a.E) == (b.N, b.B, b.E) and not np.array_equal(a.keys, b.keys)
    out = buffers(a.N, a.E, 2)
    ga = upload(a)
    gb = upload(b, n_valid=b.E - 3000, tail=BIG_ID)
    first = check_cut(a, 0.5, ga, out=out)
    ws = out.cut_ws
    reused = check_cut(b, 0.5, gb, out=out)
    assert out.cut_ws is ws, "the workspace keyed by (B, capacity) is reused"
    fresh = check_cut(b, 0.5, gb)
    assert same(reused, fresh)
    assert same(check_cut(b, 0.5, gb, out=out), reused) and same(check_cut(a, 0.5, ga, out=out), first)


@pytest.mark.gpu
@pytest.mark.parametrize("A", [0, 1, 8])
def test_edge_attr_widths(A):
    case, g_main = tie_case(True)
    check_cut(case, rate_for(tie_k(case, g_main, "half")[0], int((case.gid == g_main).sum())), A=A)
    check_cut(special_case()[0], 0.5, A=A)


def _radius_case(x, r, batch, B, A):
    """A radius graph as a Case, after checking its edge_attr against distegnn_edge_lengths_csr bit for bit."""
    g, ea = radius_graph_csr(x, r, batch, n_graphs=B, edge_attr_nf=A)
    bits = ea.view(torch.int32).cpu().numpy()
    keys, keyf, _, _ = device_keys(g, x)
    assert (bits == keyf.view(np.int32)[:, None]).all(), "the radius build's edge_attr differs from the length kernel"
    case = Case(x.cpu().numpy(), g.rowptr.cpu().numpy(), g.col.cpu().numpy(),
                None if batch is None else batch.cpu().numpy(), B)
    return case, g, keys


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0.0, 1e3, -1e3, 1e4, -1e4])
def test_general_positions_three_lengths_agree(offset):
    """Radius candidates at general positions: the radius build's edge_attr, the length kernel and the cutoff's kept
    edge_attr are one fp32 length bit for bit; at ±1e4 the fp32 grid makes many exact ties."""
    rng = np.random.default_rng(int(abs(offset)) + (offset < 0))
    sizes = [1700, 1, 0, 2299]
    x = torch.from_numpy((rng.random((sum(sizes), 3)) + offset).astype(F32)).to(dev())
    batch = torch.repeat_interleave(torch.arange(4), torch.tensor(sizes)).to(dev())
    case, g, _ = _radius_case(x, 0.08, batch, 4, 2)
    for rate in (0.5, 0.25, 0.9):
        check_cut(case, rate, dg=(g, x, batch))


@pytest.mark.gpu
def test_config5_radius_graph():
    """BASELINE config 5: 1M nodes, r = 0.075, about 20.6M candidates, at rates 0.25, 0.5 and 0.75."""
    w = synth.WORKLOADS["synth1m"]
    x = torch.from_numpy(synth.make_points(w, 0, w.n_nodes)["pos"]).to(dev())
    case, g, keys = _radius_case(x, w.radius, None, 1, 1)
    assert case.E > 20_000_000
    order = order_of(keys, case.gid)
    out = buffers(case.N, case.E, 1)
    for rate in (0.25, 0.5, 0.75):
        check_cut(case, rate, dg=(g, x, None), A=1, out=out, order=order)


@pytest.mark.gpu
def test_nbody_250_complete_graphs():
    B, n = 250, 100
    x = torch.randn(B * n, 3, generator=torch.Generator().manual_seed(0))
    i, j = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    keep = i != j
    ei = torch.cat([torch.stack([i[keep], j[keep]]) + n * b for b in range(B)], 1)
    g, _ = CSRGraph.from_edge_index(ei.to(dev()), B * n)
    batch = torch.arange(B).repeat_interleave(n)
    case = Case(x.numpy(), g.rowptr.cpu().numpy(), g.col.cpu().numpy(), batch.numpy(), B)
    x, batch = x.to(dev()), batch.to(dev())
    order = order_of(device_keys(g, x)[0], case.gid)
    for rate in (0.25, 0.5, 0.75):
        check_cut(case, rate, dg=(g, x, batch), order=order)
