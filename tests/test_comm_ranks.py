"""The virtual-node exchange (csrc/comm.cuh) with W ranks on one GPU, against rank-order sums and float64.

All W ranks run in one cooperative launch of the testing library (csrc/testing/comm_ranks.cu): every CTA of every rank
is resident at once, so ranks that spin on each other's flags always progress.  The device code is the product's, so
these tests reach what a world of 1 never runs: the reduction over several ranks, the parity double buffer, the per-slot
epochs, the segment each push targets, the write-back of the summed vsum and DESIGN §5's claim that every rank ends with
the same bits.

The reference of an all-reduce is the fp32 sum in rank order, ((x0 + x1) + x2) + …, which is bit for bit what every
rank must produce.  The inputs are built so that other summation orders give other bits (checked on the CPU); at W = 2
every order gives the same bits, because fp32 addition is commutative, so the order is only tested at W >= 3.  The fused
update is compared with float64 run on that fp32 sum, and bitwise with the single-rank kernel run on it."""
import ctypes as C

import numpy as np
import pytest
import torch

from distegnn_b200 import _lib
from tests.helpers import check_bounds, rowwise
from tests.shadow_backend import ShadowBackend
from tests.twin_backend import TESTING_LIB_PATH

_i32, _i64, _u32, _u64, _vp = C.c_int, C.c_int64, C.c_uint, C.c_uint64, C.c_void_p
SIGNATURES = {
    "distegnn_comm_init": [_i32, _i32, _i32, _i32, C.POINTER(_vp), _vp],
    "distegnn_comm_handle_bytes": [],
    "distegnn_comm_set_timeout_ms": [_vp, _i64],
    "distegnn_comm_status": [_vp, C.POINTER(_i32)],
    "distegnn_comm_destroy": [_vp],
    "distegnn_comm_connect_local": [_vp, _i32],
    "distegnn_comm_ranks_capacity": [C.POINTER(_i32), C.POINTER(_i32)],
    "distegnn_allreduce_packed_ranks": [_vp, _i32, _vp, _i64, _i32, _i32, _i64, _u64, _vp],
    "distegnn_virtual_update_fwd_ranks": [_vp, _i32, _i32, _i32, _i32, _i32, _u32] + [_vp] * 8 + [_i64, _u64, _vp],
}
PAUSE_SEEDED, PAUSE_ONE_SLOW_RANK = 0, 1
EINVAL = -1
H, A = 64, 2
PAD = 37                # sentinel floats past `count` in every buffer
SENTINEL = -1234.5
TIMEOUT_MS = 1000
ORDER_WORLDS = [3, 4, 8, 16]        # worlds at which the summation order shows in the bits
_t = None


def tlib():
    global _t
    if _t is None:
        lib = C.CDLL(TESTING_LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            getattr(lib, name).argtypes = argtypes
            getattr(lib, name).restype = C.c_int
        lib.distegnn_last_error.argtypes = []
        lib.distegnn_last_error.restype = C.c_char_p
        _t = lib
    return _t


def last_error():
    return tlib().distegnn_last_error().decode()


def parray(values):
    """A C array of pointers (ints, tensors or None)."""
    vals = [v.data_ptr() if isinstance(v, torch.Tensor) else v for v in values]
    return (_vp * max(16, len(vals)))(*vals)          # null past the given entries


def stride_of(slot_floats):
    return (slot_floats + 3) // 4 * 4


def K_of(C_):
    return 4 + 3 * C_ + H * C_


# ==== host references ===================================================================================================
def rank_order(xs):
    """fp32 sum over axis 0 in rank order: ((x0 + x1) + x2) + …"""
    s = xs[0].astype(np.float32)
    for x in xs[1:]:
        s = s + x.astype(np.float32)
    return s


def tree_sum(xs):
    if len(xs) == 1:
        return xs[0].astype(np.float32)
    h = len(xs) // 2
    return tree_sum(xs[:h]) + tree_sum(xs[h:])


def other_orders(xs):
    """The summation orders a wrong reduction would use: reversed, each 'own rank first' rotation, a pairwise tree."""
    W = len(xs)
    out = {"reversed": rank_order(xs[::-1]), "tree": tree_sum(xs)}
    for k in range(1, W):
        out[f"rotation {k}"] = rank_order(np.concatenate([xs[k:], xs[:k]]))
    return out


def rank_inputs(W, n, seed):
    """[W, n] fp32: mixed signs; per element a scale 2^e with e in [-21, 21] and per rank 2^[-3, 3] around it, so the
    magnitudes span 2^±24 and the W terms of an element are close enough for every rounding to matter."""
    rng = np.random.default_rng(seed)
    e = rng.integers(-21, 22, n)[None, :] + rng.integers(-3, 4, (W, n))
    x = rng.choice([-1.0, 1.0], (W, n)) * rng.uniform(1.0, 2.0, (W, n)) * np.exp2(e)
    return x.astype(np.float32)


def check_sum(got, xs, what):
    """got [n] must be the rank-order fp32 sum of xs [W, n] bit for bit; the float64 sum is printed beside it."""
    want = rank_order(xs)
    bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} sums differ from the rank-order sum, first [{bad[0]}]: " \
                          f"{got[bad[0]]!r} != {want[bad[0]]!r}"
    f64 = xs.astype(np.float64).sum(0)
    bound = len(xs) * 2.0 ** -24 * np.abs(xs.astype(np.float64)).sum(0)
    err = np.abs(want.astype(np.float64) - f64)
    assert (err <= bound).all()
    return float((err / np.maximum(bound, 1e-300)).max())


# ==== CPU: the inputs tell the orders apart; argument checks ==========================================================
@pytest.mark.parametrize("W", ORDER_WORLDS)
def test_inputs_tell_summation_orders_apart(W):
    xs = rank_inputs(W, 4096, seed=W)
    want = rank_order(xs)
    assert np.abs(xs).max() <= 2.0 ** 25 and np.abs(xs).min() >= 2.0 ** -24
    for name, other in other_orders(xs).items():
        frac = float((other.view(np.int32) != want.view(np.int32)).mean())
        assert frac >= 0.25, f"W={W}: the {name} order gives the rank-order bits on {1 - frac:.0%} of the elements"


def test_two_ranks_sum_alike_in_every_order():
    """Why the order is only tested at W >= 3: x0 + x1 == x1 + x0 in fp32, bit for bit."""
    xs = rank_inputs(2, 4096, seed=2)
    want = rank_order(xs)
    for other in other_orders(xs).values():
        assert np.array_equal(other.view(np.int32), want.view(np.int32))


def test_argument_checks_without_a_device():
    t = tlib()
    nulls = parray([None] * 16)
    one = (C.c_int * 1)()

    def vu(comms=nulls, world=2, B=3, C_=4, pause=0):
        return t.distegnn_virtual_update_fwd_ranks(comms, world, B, A, C_, 0, 0, nulls, nulls, nulls, None, None, nulls,
                                                   None, None, pause, 0, None)

    def ar(comms=nulls, world=2, bufs=nulls, count=4, calls=1, schedule=PAUSE_SEEDED, pause=0):
        return t.distegnn_allreduce_packed_ranks(comms, world, bufs, count, calls, schedule, pause, 0, None)

    for call, msg in [
        (lambda: t.distegnn_comm_connect_local(None, 2), "null comms"),
        (lambda: t.distegnn_comm_connect_local(nulls, 0), "world size outside"),
        (lambda: t.distegnn_comm_connect_local(nulls, 17), "world size outside"),
        (lambda: t.distegnn_comm_connect_local(nulls, 2), "null communicator"),
        (lambda: t.distegnn_comm_ranks_capacity(None, one), "null pointer"),
        (lambda: ar(comms=None), "null pointer"),
        (lambda: ar(bufs=None), "null pointer"),
        (lambda: ar(world=0), "world size outside"),
        (lambda: ar(world=17), "world size outside"),
        (lambda: ar(count=-1), "negative count"),
        (lambda: ar(calls=-1), "negative count or calls"),
        (lambda: ar(pause=-1), "negative pause"),
        (lambda: ar(schedule=2), "unknown pause schedule"),
        (lambda: ar(), "null buffer"),
        (lambda: vu(comms=None), "null pointer"),
        (lambda: vu(world=0), "world size outside"),
        (lambda: vu(world=17), "world size outside"),
        (lambda: vu(pause=-5), "negative pause"),
        (lambda: vu(C_=17), "virtual_channels"),
        (lambda: vu(B=-1), "bad size"),
        (lambda: vu(), "null pointer"),
    ]:
        assert call() == EINVAL and msg in last_error(), (msg, last_error())


# ==== GPU harness =====================================================================================================
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def stream():
    return torch.cuda.current_stream(dev()).cuda_stream


class Ranks:
    """W communicators of this process, connected to each other's segments; destroyed on exit."""

    def __init__(self, W, max_slots, slot_floats, connect=True):
        self.W, self.max_slots, self.stride = W, max_slots, stride_of(slot_floats)
        self.handles = []
        t = tlib()
        try:
            for r in range(W):
                self.handles.append(self.make(r, W, max_slots, slot_floats))
            if connect:
                assert t.distegnn_comm_connect_local(self.array(), W) == 0, last_error()
        except BaseException:
            self.destroy()
            raise

    @staticmethod
    def make(rank, world, max_slots, slot_floats):
        t = tlib()
        h = _vp()
        handle = (C.c_ubyte * t.distegnn_comm_handle_bytes())()
        assert t.distegnn_comm_init(rank, world, max_slots, slot_floats, C.byref(h), handle) == 0, last_error()
        assert t.distegnn_comm_set_timeout_ms(h, TIMEOUT_MS) == 0
        return h

    def array(self):
        return parray([h.value for h in self.handles])

    def statuses(self):
        out = []
        for h in self.handles:
            v = C.c_int(-1)
            assert tlib().distegnn_comm_status(h, C.byref(v)) == 0, last_error()
            out.append(v.value)
        return out

    def destroy(self):
        torch.cuda.synchronize()
        for h in self.handles:
            tlib().distegnn_comm_destroy(h)
        self.handles = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.destroy()

    def packed(self, bufs, count, calls=1, schedule=PAUSE_SEEDED, max_pause_ns=0, seed=0):
        return tlib().distegnn_allreduce_packed_ranks(self.array(), self.W, parray(bufs), count, calls, schedule,
                                                      max_pause_ns, seed, stream())

    def update(self, dims, flags, vsum, Xv, Hv, lp, lpn, G, loc=None, hv0=None, max_pause_ns=0, seed=0):
        B, A_, C_, Na = dims
        return tlib().distegnn_virtual_update_fwd_ranks(
            self.array(), self.W, B, A_, C_, Na, flags, parray(vsum), parray(Xv), parray(Hv),
            None if lp is None else lp.data_ptr(), None if lpn is None else lpn.data_ptr(), parray(G),
            None if loc is None else loc.data_ptr(), None if hv0 is None else hv0.data_ptr(), max_pause_ns, seed,
            stream())

    def check_status(self):
        torch.cuda.synchronize()
        assert self.statuses() == [0] * self.W, f"a wait timed out: statuses {self.statuses()}"


def with_sentinel(x):
    """A device copy of the fp32 vector x followed by PAD sentinel floats."""
    return torch.cat([torch.from_numpy(x), torch.full((PAD,), SENTINEL)]).to(dev())


def check_sentinel(buf, count, what):
    tail = buf[count:].cpu()
    assert torch.equal(tail, torch.full((PAD,), SENTINEL)), f"{what}: written past count"


# ==== GPU: rank-order sums ============================================================================================
SLOT_FLOATS = [1, 3, 4, 5] + [4 + 67 * c for c in (1, 3, 4, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("slot_floats", SLOT_FLOATS)
@pytest.mark.parametrize("W", [2, 3, 4, 5, 8, 16])
def test_rank_order_sums(W, slot_floats):
    """Every rank's buffer is the rank-order fp32 sum bit for bit, at counts around one slot and around the capacity;
    nothing past `count` is written."""
    max_slots = 5
    stride = stride_of(slot_floats)
    cap = max_slots * stride
    counts = sorted({1, stride - 1, stride, stride + 1, cap - 1, cap} - {0})
    worst = 0.0
    with Ranks(W, max_slots, slot_floats) as R:
        for i, count in enumerate(counts):
            xs = rank_inputs(W, count, seed=1000 * W + 10 * slot_floats + i)
            bufs = [with_sentinel(xs[r]) for r in range(W)]
            assert R.packed(bufs, count) == 0, last_error()
            R.check_status()
            for r in range(W):
                worst = max(worst, check_sum(bufs[r][:count].cpu().numpy(), xs, f"W={W} count={count} rank {r}"))
                check_sentinel(bufs[r], count, f"W={W} count={count} rank {r}")
    print(f"W={W} slot_floats={slot_floats} counts {counts}: bitwise rank-order sums; rank-order vs float64 at most "
          f"{worst:.2f} of W·u·Σ|x|")


# ==== GPU: consecutive calls under skew ===============================================================================
SCHEDULES = {"none": (PAUSE_SEEDED, 0), "random_50us": (PAUSE_SEEDED, 50_000),
             "one_slow_rank": (PAUSE_ONE_SLOW_RANK, 50_000)}


@pytest.mark.gpu
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("W", [2, 3, 8, 16])
def test_consecutive_calls_under_skew(W, schedule):
    """Nine calls in one launch, then launches whose counts shrink and grow, so that some slots skip calls and the
    per-slot epochs (and parities) diverge; the ranks drift by the pause schedule.  Every call is checked."""
    kind, max_ns = SCHEDULES[schedule]
    max_slots, slot_floats = 6, 29
    stride = stride_of(slot_floats)
    cap = max_slots * stride
    with Ranks(W, max_slots, slot_floats) as R:
        for launch, (calls, count) in enumerate([(9, cap), (4, stride + 5), (7, cap - 3), (2, 1)]):
            xs = rank_inputs(W, calls * count, seed=7 * W + launch)
            bufs = [with_sentinel(xs[r]) for r in range(W)]
            assert R.packed(bufs, count, calls, kind, max_ns, seed=launch) == 0, last_error()
            R.check_status()
            for r in range(W):
                got = bufs[r][:calls * count].cpu().numpy()
                for c in range(calls):
                    s = slice(c * count, (c + 1) * count)
                    check_sum(got[s], xs[:, s], f"launch {launch} call {c} rank {r}")
                check_sentinel(bufs[r], calls * count, f"launch {launch} rank {r}")


# ==== GPU: the fused update ===========================================================================================
VU_MODES = {"mid": 0, "last": _lib.FLAG_LAST, "init": _lib.FLAG_INIT,
            "init_centroid": _lib.FLAG_INIT | _lib.FLAG_INIT_CENTROID, "zero_vsum": _lib.FLAG_ZERO_VSUM}


def partial_stats(W, B, C_, seed):
    """[W, B, K] per-rank statistics: integral counts, graphs absent from some ranks (count and sums 0) and graph 0
    absent from all of them (total count 0: the update divides by max(n, 1))."""
    rng = np.random.default_rng(seed)
    n = rng.integers(1, 500, (W, B)).astype(np.float32)
    n[rng.random((W, B)) < 0.3] = 0
    n[:, 0] = 0
    vs = (rng.standard_normal((W, B, K_of(C_))) * np.sqrt(np.maximum(n, 1))[..., None]).astype(np.float32)
    vs[:, :, 0:3] += rng.standard_normal((W, B, 3)).astype(np.float32) * n[..., None]
    vs[:, :, 3] = n
    vs[n == 0] = 0
    return vs


def run_update(R, C_, flags, vs, state, pk, max_pause_ns=20_000, seed=0):
    """The fused update on all ranks from per-rank statistics vs [W, B, K] and the replicated state (Xv, Hv)."""
    W, B = vs.shape[0], vs.shape[1]
    init, last = bool(flags & _lib.FLAG_INIT), bool(flags & _lib.FLAG_LAST)
    lp, lpn = pk["layers"]
    vsum = [torch.from_numpy(vs[r]).to(dev()) for r in range(W)]
    Xv = [state["Xv"].clone() for _ in range(W)]
    Hv = [state["Hv"].clone() for _ in range(W)]
    G = [torch.full((B, C_, H), float("nan"), device=dev()) for _ in range(W)]
    loc = state["loc"] if flags == _lib.FLAG_INIT else None
    rc = R.update((B, A, C_, 0), flags, vsum, Xv, Hv, None if init else lp, None if last else lpn,
                  [None] * W if last else G, loc, pk["hv0"] if init else None, max_pause_ns, seed)
    assert rc == 0, last_error()
    R.check_status()
    return dict(vsum=vsum, Xv=Xv, Hv=Hv, G=G, loc=loc)


def single_rank_update(C_, flags, summed, state, pk):
    """The product kernel without a communicator on the rank-order sum: what every rank must compute."""
    from distegnn_b200.backend import cuda_backend
    B = summed.shape[0]
    init, last = bool(flags & _lib.FLAG_INIT), bool(flags & _lib.FLAG_LAST)
    lp, lpn = pk["layers"]
    vsum = torch.from_numpy(summed).to(dev())
    Xv, Hv = state["Xv"].clone(), state["Hv"].clone()
    G = torch.full((B, C_, H), float("nan"), device=dev())
    cuda_backend().virtual_update((B, A, C_, 0), flags, vsum, Xv, Hv, None if init else lp, None if last else lpn,
                                  None if last else G, state["loc"] if flags == _lib.FLAG_INIT else None,
                                  pk["hv0"] if init else None)
    torch.cuda.synchronize()
    return Xv, Hv, G


def check_update(out, vs, flags, state, pk, C_, what):
    """vsum: the rank-order sum bit for bit (or zeros under FLAG_ZERO_VSUM); Xv, Hv, G: equal on all ranks and equal to
    the single-rank kernel on the rank-order sum; against float64 row-wise."""
    W, B = vs.shape[0], vs.shape[1]
    last, init = bool(flags & _lib.FLAG_LAST), bool(flags & _lib.FLAG_INIT)
    summed = rank_order(vs)
    for r in range(W):
        v = out["vsum"][r].cpu().numpy()
        if flags & _lib.FLAG_ZERO_VSUM:
            assert not v.any(), f"{what}: FLAG_ZERO_VSUM left vsum of rank {r} non-zero"
        else:
            check_sum(v.reshape(-1), vs.reshape(W, -1), f"{what}: vsum of rank {r}")
    for name in ("Xv", "Hv") + (() if last else ("G",)):
        for r in range(1, W):
            assert torch.equal(out[name][r], out[name][0]), f"{what}: {name} of rank {r} differs from rank 0"
    Xs, Hs, Gs = single_rank_update(C_, flags, summed, state, pk)
    assert torch.equal(out["Xv"][0], Xs) and torch.equal(out["Hv"][0], Hs), f"{what}: not the single-rank update"
    if not last:
        assert torch.equal(out["G"][0], Gs), f"{what}: G is not the single-rank update's"
    # float64 on the fp32 rank-order sum
    lp, lpn = pk["layers"]
    D = lambda x: x.double().clone()
    s64 = torch.from_numpy(summed).double().to(dev())
    rX, rH, rG = D(state["Xv"]), D(state["Hv"]), torch.zeros(B, C_, H, dtype=torch.float64, device=dev())
    r_loc = out["loc"]
    if flags & _lib.FLAG_INIT_CENTROID:
        r_loc = s64[:, :3] / s64[:, 3:4].clamp(min=1)
    ShadowBackend().virtual_update((B, A, C_, 0), flags & ~_lib.FLAG_INIT_CENTROID, s64.clone(), rX, rH,
                                   None if init else lp.double(), None if last else lpn.double(), rG,
                                   None if r_loc is None else r_loc.double(), pk["hv0"].double() if init else None)
    e = dict(Xv=rowwise(out["Xv"][0].reshape(B, -1), rX.reshape(B, -1)))
    if last:
        assert all(torch.equal(h, state["Hv"]) for h in out["Hv"]), f"{what}: Hv written under FLAG_LAST"
        assert all(bool(torch.isnan(g).all()) for g in out["G"]), f"{what}: G written under FLAG_LAST"
    else:
        e["Hv"] = rowwise(out["Hv"][0].reshape(B * C_, H), rH.reshape(B * C_, H))
        e["G"] = rowwise(out["G"][0].reshape(B * C_, H), rG.reshape(B * C_, H))
    check_bounds({"tc": e}, {})
    return e


def update_state(B, C_, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(Xv=torch.randn(B, 3, C_, generator=g).to(dev()), Hv=torch.randn(B, C_, H, generator=g).to(dev()),
                loc=torch.randn(B, 3, generator=g).to(dev()))


def packed_params(C_):
    from tests.test_node_kernel_tiling import packed
    return packed(3, 0, C_)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(VU_MODES))
@pytest.mark.parametrize("C_", list(range(1, 17)))
@pytest.mark.parametrize("W", [3, 8])
def test_fused_update_vs_float64(W, C_, mode):
    B = 24
    flags = VU_MODES[mode]
    pk = packed_params(C_)
    vs = partial_stats(W, B, C_, seed=100 * W + C_)
    state = update_state(B, C_, seed=C_)
    with Ranks(W, B, K_of(C_)) as R:
        out = run_update(R, C_, flags, vs, state, pk, seed=C_)
        e = check_update(out, vs, flags, state, pk, C_, f"W={W} C={C_} {mode}")
    print(f"fused update W={W} C={C_} {mode}: ranks bitwise equal; row-wise vs fp64 "
          + ", ".join(f"{k} {v:.1e}" for k, v in e.items()))


@pytest.mark.gpu
@pytest.mark.parametrize("C_", [3, 4, 16])
def test_packed_calls_and_fused_updates_share_slots(C_):
    """The model's layout: max_slots = B, slot_floats = K; the backward's g_vsum exchange is one packed call of B·K
    floats, which with C mod 4 != 0 cuts slots across graph rows and leaves the last slots without a call."""
    W, B = 3, 10
    K = K_of(C_)
    pk = packed_params(C_)
    state = update_state(B, C_, seed=40 + C_)
    with Ranks(W, B, K) as R:
        for step, flags in enumerate([0, _lib.FLAG_ZERO_VSUM, _lib.FLAG_INIT, 0]):
            vs = partial_stats(W, B, C_, seed=500 + 10 * C_ + step)
            out = run_update(R, C_, flags, vs, state, pk, seed=step)
            check_update(out, vs, flags, state, pk, C_, f"C={C_} step {step} update")
            if not flags & _lib.FLAG_INIT:
                state = dict(state, Xv=out["Xv"][0].clone(), Hv=out["Hv"][0].clone())
            xs = rank_inputs(W, B * K, seed=600 + 10 * C_ + step)
            bufs = [with_sentinel(xs[r]) for r in range(W)]
            assert R.packed(bufs, B * K, 1, PAUSE_SEEDED, 20_000, seed=step) == 0, last_error()
            R.check_status()
            for r in range(W):
                check_sum(bufs[r][:B * K].cpu().numpy(), xs, f"C={C_} step {step} packed, rank {r}")
                check_sentinel(bufs[r], B * K, f"C={C_} step {step} packed, rank {r}")


# ==== GPU: capacity edges =============================================================================================
def capacity():
    p, u = C.c_int(0), C.c_int(0)
    assert tlib().distegnn_comm_ranks_capacity(C.byref(p), C.byref(u)) == 0, last_error()
    return p.value, u.value


@pytest.mark.gpu
@pytest.mark.parametrize("C_", [3, 4])
def test_sixteen_ranks_at_the_largest_grid(C_):
    """W = 16 at the most graphs whose CTAs are co-resident, with B = max_slots, and K = stride (C = 4) or K < stride
    (C = 3); one graph more is refused with DISTEGNN_EINVAL and launches nothing."""
    W = 16
    _, ctas = capacity()
    B = ctas // W
    assert B >= 1
    pk = packed_params(C_)
    state = update_state(B, C_, seed=70)
    vs = partial_stats(W, B, C_, seed=71 + C_)
    with Ranks(W, B, K_of(C_)) as R:
        assert R.stride == K_of(C_) if C_ == 4 else R.stride > K_of(C_)
        out = run_update(R, C_, 0, vs, state, pk)
        check_update(out, vs, 0, state, pk, C_, f"W=16 B={B}")
    vs1 = partial_stats(W, B + 1, C_, seed=72)
    state1 = update_state(B + 1, C_, seed=73)
    with Ranks(W, B + 1, K_of(C_)) as R:
        vsum = [torch.from_numpy(vs1[r]).to(dev()) for r in range(W)]
        Xv = [state1["Xv"].clone() for _ in range(W)]
        Hv = [state1["Hv"].clone() for _ in range(W)]
        G = [torch.zeros(B + 1, C_, H, device=dev()) for _ in range(W)]
        lp, lpn = pk["layers"]
        assert R.update((B + 1, A, C_, 0), 0, vsum, Xv, Hv, lp, lpn, G) == EINVAL
        assert "do not fit" in last_error(), last_error()
        R.check_status()
        assert all(torch.equal(v.cpu(), torch.from_numpy(vs1[r])) for r, v in enumerate(vsum)), "launched anyway"
    print(f"W=16: {B} graphs per rank at C={C_} ({ctas} co-resident CTAs), {B + 1} refused")


@pytest.mark.gpu
def test_sixteen_ranks_packed_at_the_largest_grid():
    """W = 16 at the most slots whose CTAs are co-resident; one slot more is refused and launches nothing."""
    W, slot_floats = 16, 67
    ctas, _ = capacity()
    slots = ctas // W
    with Ranks(W, slots + 1, slot_floats) as R:
        count = slots * R.stride
        xs = rank_inputs(W, count, seed=81)
        bufs = [with_sentinel(xs[r]) for r in range(W)]
        assert R.packed(bufs, count, 1, PAUSE_SEEDED, 10_000, seed=2) == 0, last_error()
        R.check_status()
        for r in range(W):
            check_sum(bufs[r][:count].cpu().numpy(), xs, f"W=16 {slots} slots, rank {r}")
        xs = rank_inputs(W, count + 1, seed=82)
        bufs = [with_sentinel(xs[r]) for r in range(W)]
        assert R.packed(bufs, count + 1) == EINVAL and "do not fit" in last_error(), last_error()
        R.check_status()
        assert all(torch.equal(b[:count + 1].cpu(), torch.from_numpy(xs[r])) for r, b in enumerate(bufs))
    print(f"W=16 packed: {slots} slots per rank ({ctas} co-resident CTAs), {slots + 1} refused")


# ==== GPU: the twins are the product at W = 1 =========================================================================
class _Handle:
    def __init__(self, h):
        self.handle = h


@pytest.mark.gpu
def test_twins_are_the_product_at_world_1():
    from distegnn_b200.backend import cuda_backend
    be = cuda_backend()
    C_, B = 5, 7
    K = K_of(C_)
    with Ranks(1, B, K) as R:
        comm = _Handle(R.handles[0])
        for count in (1, K, K + 1, B * R.stride):
            x = rank_inputs(1, count, seed=count)[0]
            a, b = torch.from_numpy(x).to(dev()), torch.from_numpy(x).to(dev())
            be.allreduce_packed(comm, a)
            assert R.packed([b], count) == 0, last_error()
            R.check_status()
            assert torch.equal(a, b) and torch.equal(a.cpu(), torch.from_numpy(x))
        pk = packed_params(C_)
        lp, lpn = pk["layers"]
        for mode, flags in VU_MODES.items():
            init, last = bool(flags & _lib.FLAG_INIT), bool(flags & _lib.FLAG_LAST)
            vs = partial_stats(1, B, C_, seed=90)
            state = update_state(B, C_, seed=91)
            out = run_update(R, C_, flags, vs, state, pk, max_pause_ns=0)
            vsum = torch.from_numpy(vs[0]).to(dev())
            Xv, Hv = state["Xv"].clone(), state["Hv"].clone()
            G = torch.full((B, C_, H), float("nan"), device=dev())
            be.virtual_update((B, A, C_, 0), flags, vsum, Xv, Hv, None if init else lp, None if last else lpn,
                              None if last else G, state["loc"] if flags == _lib.FLAG_INIT else None,
                              pk["hv0"] if init else None, comm)
            R.check_status()
            for name, want in (("vsum", vsum), ("Xv", Xv), ("Hv", Hv), ("G", G)):
                got = out[name][0]
                assert torch.equal(got.nan_to_num(7.0), want.nan_to_num(7.0)), (mode, name)


# ==== GPU: connect_local rejects what it must =========================================================================
@pytest.mark.gpu
def test_connect_local_rejects():
    t = tlib()
    made = []

    def comm(rank, world, max_slots=4, slot_floats=8):
        made.append(Ranks.make(rank, world, max_slots, slot_floats))
        return made[-1]

    def rejects(handles, world, msg):
        assert t.distegnn_comm_connect_local(parray([h.value for h in handles]), world) == EINVAL
        assert msg in last_error(), last_error()

    try:
        w3 = [comm(r, 3) for r in range(3)]
        rejects(w3[:2], 2, "another world size")
        rejects(w3, 4, "another world size")
        rejects(w3, 0, "world size outside")
        rejects(w3, 17, "world size outside")
        rejects([w3[0], w3[1], w3[1]], 3, "duplicate rank")
        rejects([comm(0, 2), comm(1, 2, max_slots=5)], 2, "unequal max_slots")
        rejects([comm(0, 2), comm(1, 2, slot_floats=9)], 2, "unequal slot stride")
        # a refused connect leaves every communicator unconnected: the right set connects afterwards, once
        assert t.distegnn_comm_connect_local(parray([h.value for h in w3]), 3) == 0, last_error()
        rejects(w3, 3, "already connected")
        rejects([comm(0, 2), w3[1]], 2, "already connected")
        # a stride rounded up to the same multiple of 4 is the same stride: these connect
        assert t.distegnn_comm_connect_local(parray([comm(0, 2, slot_floats=5).value,
                                                     comm(1, 2, slot_floats=8).value]), 2) == 0, last_error()
        if torch.cuda.device_count() >= 2:
            a = comm(0, 2)
            with torch.cuda.device(1):
                b = comm(1, 2)
            rejects([a, b], 2, "different devices")
    finally:
        torch.cuda.synchronize()
        for h in made:
            t.distegnn_comm_destroy(h)
