"""The N-body dataset on the device: the reference's charged-particle generator (dataset_generation/nbody), isolated
bodies, sticks and hinges, written as the files `frames.load_nbody` and `main.py --trajectory` read (DESIGN §25).

    python -m distegnn_b200.nbody --num-train 5000 --num-valid 2000 --num-test 2000 --n_isolated 100 --seed 43 \\
        --path data/nbody

Initial conditions are drawn on the host with numpy, the reference's calls in the reference's order, from one stream
per system: RandomState(MT19937(SeedSequence([seed, split, s]))) with split 0 / 1 / 2 for train / valid / test.  The
simulation runs in fp64 on the device (csrc/nbody.cu, distegnn_nbody_simulate) in a fixed arithmetic order, so its bits
do not depend on how the systems or the steps are chunked.  Sticks (two bodies at a fixed distance) and hinges (three
bodies, two rigid arms sharing a joint) come from `generate_dataset(..., n_stick=, n_hinge=)`; their initial state is
the reference's `initialize` on the host, their step the restated `update` on the device
(distegnn_nbody_simulate_objects).
"""
from __future__ import annotations

import argparse
import json
import os
import pickle
import time
from dataclasses import dataclass
from typing import Any, Iterable, List, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib

SPLITS = ("train", "valid", "test")
CHARGE_TYPES = [1.0, -1.0]
LOC_STD, VEL_NORM = 1.0, 0.5
EPS = 1e-6                              # physical_objects.py:3, the tolerance of the end-of-run check


def tag_of(n_isolated: int, clusters: int = 1, suffix: str = "", *, n_stick: int = 0, n_hinge: int = 0) -> str:
    """The reference's file tag: `_charged{n_isolated}_{n_stick}_{n_hinge}_{clusters}{suffix}`
    (generate_dataset.py:51-53)."""
    return f"_charged{n_isolated}_{n_stick}_{n_hinge}_{clusters}{suffix}"


def system_rng(seed: int, split: int, s: int) -> np.random.RandomState:
    """The numpy stream of system s of split `split`."""
    return np.random.RandomState(np.random.MT19937(np.random.SeedSequence([seed, split, s])))


def _one_system(rs: np.random.RandomState, n: int, clusters: int):
    # system.py:23-60, the same calls in the same order; the object-selection draws that follow (:66-90) are made by
    # _select_objects when there are sticks or hinges; for isolated bodies alone they only permute them and are skipped
    loc_std = LOC_STD * (float(n) / 5.) ** (1 / 3) + 0.1
    charges = rs.choice(CHARGE_TYPES, size=(n, 1))
    if clusters == 1:
        centres = np.array([0.0, 0.0, 0.0])
    elif clusters == 3:
        centres = rs.uniform(low=-10 * clusters, high=10 * clusters, size=(clusters, 3))
    else:
        centres = rs.uniform(low=-3 * clusters, high=3 * clusters, size=(clusters, 3))
    if clusters == 1:
        # choice(1) takes nothing from the stream and randn carries its spare Gaussian across calls, so one draw gives
        # the per-body loop's bits (tests/test_nbody_gen.py)
        X = rs.randn(n, 3) * loc_std + centres[0]
    else:
        X = np.zeros((n, 3))
        for i in range(n):
            c = rs.choice(clusters)
            X[i] = rs.randn(3) * loc_std + centres[c]
    V = rs.randn(n, 3)
    V = V / np.sqrt((V ** 2).sum(axis=-1)).reshape(-1, 1) * VEL_NORM
    return X, V, charges


def _check_counts(n_isolated: int, clusters: int, n_stick: int = 0, n_hinge: int = 0) -> None:
    if clusters not in (1, 3, 10):
        raise ValueError(f"clusters must be 1, 3 or 10 (got {clusters})")
    if n_stick < 0 or n_hinge < 0:
        raise ValueError(f"n_stick and n_hinge must be >= 0 (got {n_stick}, {n_hinge})")
    if n_stick == 0 and n_hinge == 0 and n_isolated < 2:
        raise ValueError(f"n_isolated must be >= 2 (got {n_isolated}): the force-size check needs a pair of bodies")
    if n_isolated < 0:
        raise ValueError(f"n_isolated must be >= 0 (got {n_isolated})")


def n_bodies(n_isolated: int, n_stick: int = 0, n_hinge: int = 0) -> int:
    """Bodies per system: n_isolated + 2·n_stick + 3·n_hinge (system.py:20)."""
    return n_isolated + 2 * n_stick + 3 * n_hinge


@dataclass
class Objects:
    """The sticks and hinges of S systems: body tables in the reference's object order (within a kind the draw order,
    within an object its `node_idx` order) and the state each object carries from step to step.  Host numpy arrays
    from `initial_conditions`; `to(device)` gives the tensors `advance` takes."""
    isolated: Any           # int32 [S, n_isolated]: the isolated bodies in draw order (configuration() only)
    sticks: Any             # int32 [S, n_stick, 2]
    hinges: Any             # int32 [S, n_hinge, 3]
    stick_state: Any        # float64 [S, n_stick, 9]: xc, vc, wc (centre, its velocity, angular velocity)
    hinge_state: Any        # float64 [S, n_hinge, 6]: w1, w2 (the arms' angular velocities)
    stick_length: Any       # float64 [S, n_stick]: the lengths `check` holds the sticks to
    hinge_length: Any       # float64 [S, n_hinge, 2]: the arms' lengths

    def configuration(self, s: int) -> dict:
        """System s's `System.configuration()`: {"Isolated": [[i], ...], "Stick": [[i, j], ...], "Hinge": [...]},
        kinds without objects left out."""
        cfg = {}
        for kind, tab, k in (("Isolated", self.isolated, 1), ("Stick", self.sticks, 2), ("Hinge", self.hinges, 3)):
            tab = np.asarray(tab[s].cpu() if torch.is_tensor(tab) else tab[s]).reshape(-1, k)
            if len(tab):
                cfg[kind] = [[int(b) for b in row] for row in tab]
        return cfg

    def to(self, device: Union[str, torch.device]) -> "Objects":
        """Contiguous tensors on `device` (tables int32, the rest float64); the states are copies."""
        conv = lambda a, dt: torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a, dtype=dt).to(
            device).contiguous().clone()
        return Objects(conv(self.isolated, torch.int32), conv(self.sticks, torch.int32), conv(self.hinges, torch.int32),
                       conv(self.stick_state, torch.float64), conv(self.hinge_state, torch.float64),
                       conv(self.stick_length, torch.float64), conv(self.hinge_length, torch.float64))


def _select_objects(rs: np.random.RandomState, n: int, counts: Sequence[int]) -> List[np.ndarray]:
    # system.py:66-90: each object draws `choice(rest, size=k, replace=False)`, which legacy numpy makes as
    # rest[permutation(len(rest))[:k]]; rest stays ascending as the reference's list comprehension keeps it, but is
    # an array here (O(n) per draw, not O(n²))
    rest = np.arange(n)
    picks = []
    for k in counts:
        j = rs.permutation(len(rest))[:k]
        picks.append(rest[j])
        rest = np.delete(rest, j)
    return picks


def _projection(va, vb):
    return np.dot(va, vb.T) / np.dot(vb, vb.T) * vb      # physical_objects.py:6-7


def _stick_initialize(X, V, idx):
    # physical_objects.py:72-99 (Stick.initialize), the same numpy calls; returns (xc, vc, wc, length)
    x, v = X[idx], V[idx]
    x0, x1 = x[0], x[1]
    v0, v1 = v[0], v[1]
    m0, m1 = 1., 1.
    d = x1 - x0
    v0_pro, v1_pro = _projection(v0, d), _projection(v1, d)
    v0_vert, v1_vert = v0 - v0_pro, v1 - v1_pro
    average_v_pro = (v0_pro + v1_pro) / 2
    v0, v1 = v0_vert + average_v_pro, v1_vert + average_v_pro
    xc = (m0 * x0 + m1 * x1) / (m0 + m1)
    vc = (m0 * v0 + m1 * v1) / (m0 + m1)
    relative_v0, relative_v1 = v0 - vc, v1 - vc
    r0, r1 = x0 - xc, x1 - xc
    w0, w1 = np.cross(r0, relative_v0) / np.dot(r0, r0.T), np.cross(r1, relative_v1) / np.dot(r1, r1.T)
    if not np.sum(np.abs(w0 - w1)) < 1e-5:
        raise ValueError(f"stick {list(idx)}: the two bodies' angular velocities differ by {np.sum(np.abs(w0 - w1))} "
                         "(the reference asserts < 1e-5)")
    X[idx[0]], X[idx[1]] = x0, x1
    V[idx[0]], V[idx[1]] = v0, v1
    return xc, vc, w0, np.sqrt(np.sum(d ** 2))


def _hinge_initialize(X, V, idx):
    # physical_objects.py:162-184 (Hinge.initialize), the same numpy calls; returns (w1, w2, length1, length2)
    x, v = X[idx], V[idx]
    x0, x1, x2 = x[0], x[1], x[2]
    v0, v1, v2 = v[0], v[1], v[2]
    d1, d2 = x1 - x0, x2 - x0
    v0_pro1, v0_pro2 = _projection(v0, d1), _projection(v0, d2)
    v1_pro, v2_pro = _projection(v1, d1), _projection(v2, d2)
    v1_vert, v2_vert = v1 - v1_pro, v2 - v2_pro
    v1, v2 = v0_pro1 + v1_vert, v0_pro2 + v2_vert
    r1, r2 = x1 - x0, x2 - x0
    v01, v02 = v1 - v0, v2 - v0
    w1, w2 = np.cross(r1, v01) / np.dot(r1, r1.T), np.cross(r2, v02) / np.dot(r2, r2.T)
    X[idx[0]], X[idx[1]], X[idx[2]] = x0, x1, x2
    V[idx[0]], V[idx[1]], V[idx[2]] = v0, v1, v2
    return w1, w2, np.sqrt(np.sum(d1 ** 2)), np.sqrt(np.sum(d2 ** 2))


def _one_system_objects(rs: np.random.RandomState, ni: int, ns: int, nh: int, clusters: int):
    X, V, charges = _one_system(rs, n_bodies(ni, ns, nh), clusters)
    picks = _select_objects(rs, len(X), [1] * ni + [2] * ns + [3] * nh)
    ss, sl = np.zeros((ns, 9)), np.zeros(ns)
    hs, hl = np.zeros((nh, 6)), np.zeros((nh, 2))
    for o, idx in enumerate(picks[ni:ni + ns]):
        xc, vc, wc, sl[o] = _stick_initialize(X, V, idx)
        ss[o] = np.concatenate([xc, vc, wc])
    for o, idx in enumerate(picks[ni + ns:]):
        w1, w2, hl[o, 0], hl[o, 1] = _hinge_initialize(X, V, idx)
        hs[o] = np.concatenate([w1, w2])
    tab = lambda p, k: np.array(p, dtype=np.int32).reshape(-1, k)
    return X, V, charges, tab(picks[:ni], 1).reshape(-1), tab(picks[ni:ni + ns], 2), tab(picks[ni + ns:], 3), ss, hs, \
        sl, hl


def initial_conditions(n_isolated: int, clusters: int, seed: int, split: int,
                       systems: Union[int, Iterable[int]], *, n_stick: int = 0, n_hinge: int = 0):
    """Host arrays (x [S,n,3], v [S,n,3], charges [S,n,1]), float64, of the systems `systems` (a count means
    range(count)) of split `split` (0 train, 1 valid, 2 test), n = n_isolated + 2·n_stick + 3·n_hinge.  With sticks or
    hinges, (x, v, charges, Objects): the reference's object selection and `initialize`, bitwise, with x and v the
    adjusted state."""
    _check_counts(n_isolated, clusters, n_stick, n_hinge)
    ids = range(systems) if isinstance(systems, int) else list(systems)
    if n_stick == 0 and n_hinge == 0:
        out = [_one_system(system_rng(seed, split, s), n_isolated, clusters) for s in ids]
        if not out:
            z = np.zeros((0, n_isolated, 3))
            return z, z.copy(), np.zeros((0, n_isolated, 1))
        return tuple(np.stack(a) for a in zip(*out))
    n = n_bodies(n_isolated, n_stick, n_hinge)
    out = [_one_system_objects(system_rng(seed, split, s), n_isolated, n_stick, n_hinge, clusters) for s in ids]
    shapes = [(n, 3), (n, 3), (n, 1), (n_isolated,), (n_stick, 2), (n_hinge, 3), (n_stick, 9), (n_hinge, 6),
              (n_stick,), (n_hinge, 2)]
    arrs = [np.stack(a) if out else np.zeros((0,) + sh) for a, sh in zip(zip(*out) if out else shapes, shapes)]
    for i in (3, 4, 5):
        arrs[i] = arrs[i].astype(np.int32)
    return arrs[0], arrs[1], arrs[2], Objects(*arrs[3:])


def n_frames(length: int, sample_freq: int) -> int:
    """Frames recorded in `length` steps: steps t with t % sample_freq == 0."""
    return len(range(0, length, sample_freq))


def _status_message(status: torch.Tensor) -> Optional[str]:
    st = status.cpu()
    bad = torch.nonzero(st >= 0).flatten().tolist()
    if not bad:
        return None
    head = ", ".join(f"system {s} at step {int(st[s])}" for s in bad[:5])
    return (f"{len(bad)} system(s) failed the reference's force-size check (an off-diagonal |q_i q_j / l2^1.5| not above "
            f"1e-10: a coincident, too close or too far pair): {head}{' ...' if len(bad) > 5 else ''}")


def _check_objects(o: Objects, S: int, dev: torch.device) -> None:
    ns, nh = o.sticks.shape[1], o.hinges.shape[1]
    for t, name, shape, dtype in ((o.sticks, "sticks", (S, ns, 2), torch.int32),
                                  (o.hinges, "hinges", (S, nh, 3), torch.int32),
                                  (o.stick_state, "stick_state", (S, ns, 9), torch.float64),
                                  (o.hinge_state, "hinge_state", (S, nh, 6), torch.float64)):
        if not torch.is_tensor(t) or t.dtype != dtype or t.device != dev or not t.is_contiguous() or t.shape != shape:
            raise ValueError(f"objects.{name} must be a contiguous {dtype} tensor {list(shape)} on {dev} (Objects.to)")


def advance(x: torch.Tensor, v: torch.Tensor, q: torch.Tensor, status: torch.Tensor, first_step: int, n_steps: int,
            sample_freq: int = 100, dt: float = 1e-3, *, objects: Optional[Objects] = None):
    """Steps first_step .. first_step + n_steps − 1 of the device state (x, v [S,n,3], q [S,n], status [S] int64, all
    contiguous on one device; x, v and status updated in place).  Returns (frames_x, frames_v) [S,R,n,3]: the steps of
    the range with t % sample_freq == 0, in order.  `objects` (Objects.to(device), with sticks or hinges): their
    states are updated in place too; a table entry out of range or naming a body twice raises ValueError (this reads
    a device counter, so it synchronises)."""
    S, n = x.shape[0], x.shape[1]
    for t, name in ((x, "x"), (v, "v"), (q, "q")):
        if t.dtype != torch.float64 or not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous float64 CUDA tensor")
    if x.shape != (S, n, 3) or v.shape != x.shape or q.shape != (S, n):
        raise ValueError(f"x, v must be [S,n,3] and q [S,n]; got {tuple(x.shape)}, {tuple(v.shape)}, {tuple(q.shape)}")
    if status.dtype != torch.int64 or status.shape != (S,) or status.device != x.device:
        raise ValueError("status must be int64 [S] on the state's device")
    if sample_freq < 1:
        raise ValueError(f"sample_freq must be >= 1 (got {sample_freq})")
    end = first_step + n_steps
    R = len(range((first_step + sample_freq - 1) // sample_freq * sample_freq, end, sample_freq))
    fx = torch.empty((S, R, n, 3), dtype=torch.float64, device=x.device)
    fv = torch.empty_like(fx)
    dt = float(dt)
    max_f = 0.1 / dt                    # system.py:15, on the host
    lib = _lib.load()
    if objects is not None and (objects.sticks.shape[1] or objects.hinges.shape[1]):
        _check_objects(objects, S, x.device)
        ns, nh = objects.sticks.shape[1], objects.hinges.shape[1]
        nbytes = _lib.C.c_int64()
        _lib.check(lib.distegnn_nbody_objects_workspace_bytes(S, n, _lib.C.byref(nbytes)),
                   "distegnn_nbody_objects_workspace_bytes")
        ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=x.device)
        invalid = torch.zeros(1, dtype=torch.int64, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(lib.distegnn_nbody_simulate_objects(
                S, n, ns, nh, first_step, n_steps, sample_freq, dt, max_f, _lib.ptr(x), _lib.ptr(v), _lib.ptr(q),
                _lib.ptr(objects.sticks), _lib.ptr(objects.hinges), _lib.ptr(objects.stick_state),
                _lib.ptr(objects.hinge_state), _lib.ptr(fx), _lib.ptr(fv), _lib.ptr(status), _lib.ptr(invalid),
                _lib.ptr(ws), nbytes.value, _lib.stream_ptr(x.device)), "distegnn_nbody_simulate_objects")
        bad = int(invalid.item()) if S and n_steps else 0
        if bad:
            raise ValueError(f"{bad} object table entries are out of [0, {n}) or name a body another entry names")
        return fx, fv
    with torch.cuda.device(x.device):
        _lib.check(lib.distegnn_nbody_simulate(S, n, first_step, n_steps, sample_freq, dt, max_f, _lib.ptr(x),
                                               _lib.ptr(v), _lib.ptr(q), _lib.ptr(fx), _lib.ptr(fv), _lib.ptr(status),
                                               _lib.stream_ptr(x.device)), "distegnn_nbody_simulate")
    return fx, fv


def constraint_violations(x, v, objects: Objects) -> np.ndarray:
    """System.check() (physical_objects.py:147-158, 237-253) of the state x, v [S,n,3]: bool [S], True where a stick
    or arm length is not within EPS of its initial value or the velocities of its two ends do not project equally
    onto it (NaN fails)."""
    x, v = (np.asarray(a.cpu() if torch.is_tensor(a) else a, dtype=np.float64) for a in (x, v))
    tab = lambda a: np.asarray(a.cpu() if torch.is_tensor(a) else a)
    S = np.arange(x.shape[0])[:, None]
    proj = lambda va, vb: (np.sum(va * vb, -1) / np.sum(vb * vb, -1))[..., None] * vb
    bad = np.zeros(x.shape[0], dtype=bool)
    arms = [(tab(objects.sticks)[..., 0], tab(objects.sticks)[..., 1], tab(objects.stick_length))]
    hg, hl = tab(objects.hinges), tab(objects.hinge_length)
    arms += [(hg[..., 0], hg[..., 1], hl[..., 0]), (hg[..., 0], hg[..., 2], hl[..., 1])]
    with np.errstate(all="ignore"):
        for a, b, length in arms:
            if a.shape[1] == 0:
                continue
            d = x[S, b] - x[S, a]
            ok = np.abs(np.sqrt(np.sum(d ** 2, -1)) - length) < EPS
            ok &= np.sum(np.abs(proj(v[S, a], d) - proj(v[S, b], d)), -1) < EPS
            bad |= ~ok.all(1)
    return bad


def simulate(x0: torch.Tensor, v0: torch.Tensor, charges: torch.Tensor, length: int, sample_freq: int = 100,
             dt: float = 1e-3, box_size: Optional[float] = None, *, objects: Optional[Objects] = None):
    """`length` steps of the systems from (x0, v0) [S,n,3] and charges [S,n] or [S,n,1], float64 on one CUDA device.
    Returns (frames_x, frames_v [S,T,n,3], status [S]) with T = n_frames(length, sample_freq) and status −1 for every
    system.  Raises ValueError naming the first failing systems and steps where the reference would abort: the
    force-size check, or with `box_size` a final position outside [−box_size, box_size].  `objects` (from
    initial_conditions; not modified) adds the sticks and hinges and the reference's end-of-run check: every stick and
    arm within 1e-6 of its initial length, with equal velocity projections at its two ends."""
    if length < 1:
        raise ValueError(f"length must be >= 1 (got {length})")
    x, v = x0.contiguous().clone(), v0.contiguous().clone()
    q = charges.reshape(charges.shape[0], -1).contiguous()
    status = torch.full((x.shape[0],), -1, dtype=torch.int64, device=x.device)
    dev_obj = objects.to(x.device) if objects is not None else None
    fx, fv = advance(x, v, q, status, 0, length, sample_freq, dt, objects=dev_obj)
    msg = _status_message(status)
    if msg:
        raise ValueError(msg)
    if box_size is not None:
        out = torch.nonzero(~((x <= box_size) & (x >= -box_size)).flatten(1).all(1)).flatten().tolist()
        if out:
            raise ValueError(f"{len(out)} system(s) end outside the box [-{box_size}, {box_size}]: systems "
                             f"{out[:5]}{' ...' if len(out) > 5 else ''}")
    if objects is not None:
        out = np.nonzero(constraint_violations(x, v, objects))[0].tolist()
        if out:
            raise ValueError(f"{len(out)} system(s) fail the reference's end-of-run check (a stick or hinge arm off its "
                             f"length or with unequal end velocities along it by 1e-6 or more): systems "
                             f"{out[:5]}{' ...' if len(out) > 5 else ''}")
    return fx, fv, status


def meta_path(path: str, tag: str) -> str:
    return os.path.join(path, f"nbody_meta{tag}.json")


def meta_rollout_tau(path: str, delta: int, tag: str = tag_of(100)) -> Optional[float]:
    """Δ·sample_freq·dt, the time between frames f and f + Δ of the N-body files under `path` (from their
    nbody_meta file), or None when there is no meta file."""
    p = meta_path(path, tag)
    if not os.path.exists(p):
        return None
    with open(p) as f:
        m = json.load(f)
    return float(delta) * int(m["sample_freq"]) * float(m["dt"])


def generate_dataset(path: str, num_train: int = 10000, num_valid: int = 2000, num_test: int = 2000,
                     length: int = 5000, length_test: int = 5000, sample_freq: int = 100, n_isolated: int = 5,
                     clusters: int = 1, seed: int = 42, suffix: str = "", box_size: Optional[float] = None,
                     dt: float = 1e-3, chunk: Optional[int] = None, device: Union[str, torch.device] = "cuda",
                     verbose: bool = False, *, n_stick: int = 0, n_hinge: int = 0) -> dict:
    """Write loc_{split}{tag}.npy, vel_… (float64 [S,T,n,3]) and charges_… ([S,n,1]) of every split with systems, and
    nbody_meta{tag}.json, under `path`; tag = tag_of(n_isolated, clusters, suffix, n_stick=, n_hinge=) and n =
    n_isolated + 2·n_stick + 3·n_hinge.  With sticks or hinges also cfg_{split}{tag}.pkl: the reference's tuple of
    one `System.configuration()` dict per system, the only record of which bodies are joined.  `chunk` systems at a
    time (default: about 1 GB of frames per chunk, several waves of CTAs at 100 bodies).  Returns the file paths and
    seconds spent on host initial conditions, on the device (simulation, CUDA events) and on copying out and
    writing."""
    _check_counts(n_isolated, clusters, n_stick, n_hinge)
    n = n_bodies(n_isolated, n_stick, n_hinge)
    constrained = n_stick > 0 or n_hinge > 0
    for k, val in (("num_train", num_train), ("num_valid", num_valid), ("num_test", num_test)):
        if val < 0:
            raise ValueError(f"{k} must be >= 0 (got {val})")
    if length < 1 or length_test < 1 or sample_freq < 1:
        raise ValueError("length, length_test and sample_freq must be >= 1")
    dev = torch.device(device)
    tag = tag_of(n_isolated, clusters, suffix, n_stick=n_stick, n_hinge=n_hinge)
    os.makedirs(path, exist_ok=True)
    stats = {"files": [], "init_s": 0.0, "simulate_s": 0.0, "write_s": 0.0}
    for split, (part, num) in enumerate(zip(SPLITS, (num_train, num_valid, num_test))):
        L = length_test if part == "test" else length
        T = n_frames(L, sample_freq)
        per = chunk or max(1, (1 << 30) // (2 * T * n * 3 * 8))
        names = {k: os.path.join(path, f"{k}_{part}{tag}.npy") for k in ("loc", "vel", "charges")}
        loc = np.lib.format.open_memmap(names["loc"], mode="w+", dtype=np.float64, shape=(num, T, n, 3))
        vel = np.lib.format.open_memmap(names["vel"], mode="w+", dtype=np.float64, shape=(num, T, n, 3))
        chg = np.lib.format.open_memmap(names["charges"], mode="w+", dtype=np.float64, shape=(num, n, 1))
        cfgs = []
        for lo in range(0, num, per):
            hi = min(num, lo + per)
            t0 = time.perf_counter()
            x0, v0, q, *objs = initial_conditions(n_isolated, clusters, seed, split, range(lo, hi), n_stick=n_stick,
                                                  n_hinge=n_hinge)
            objects = objs[0] if objs else None
            if objects is not None:
                cfgs += [objects.configuration(s) for s in range(hi - lo)]
            t1 = time.perf_counter()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            with torch.cuda.device(dev):
                ev[0].record()
                try:
                    fx, fv, _ = simulate(torch.from_numpy(x0).to(dev), torch.from_numpy(v0).to(dev),
                                         torch.from_numpy(q).to(dev), L, sample_freq, dt, box_size, objects=objects)
                except ValueError as e:
                    raise ValueError(f"{part} systems {lo}..{hi - 1}: {e}") from None
                ev[1].record()
            t2 = time.perf_counter()
            loc[lo:hi] = fx.cpu().numpy()
            vel[lo:hi] = fv.cpu().numpy()
            chg[lo:hi] = q
            t3 = time.perf_counter()
            stats["init_s"] += t1 - t0
            stats["simulate_s"] += ev[0].elapsed_time(ev[1]) / 1e3
            stats["write_s"] += t3 - t2
            if verbose:
                print(f"{part}: systems {lo}..{hi - 1} of {num} done", flush=True)
        for a in (loc, vel, chg):
            a.flush()
        del loc, vel, chg
        stats["files"] += list(names.values())
        if constrained:
            name = os.path.join(path, f"cfg_{part}{tag}.pkl")
            with open(name, "wb") as f:
                pickle.dump(tuple(cfgs), f)
            stats["files"].append(name)
    meta = {"dt": dt, "sample_freq": sample_freq, "length": length, "length_test": length_test, "seed": seed,
            "num_train": num_train, "num_valid": num_valid, "num_test": num_test, "n_isolated": n_isolated,
            "n_stick": n_stick, "n_hinge": n_hinge, "clusters": clusters, "box_size": box_size, "suffix": suffix}
    with open(meta_path(path, tag), "w") as f:
        json.dump(meta, f, indent=1)
    stats["files"].append(meta_path(path, tag))
    return stats


def _parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m distegnn_b200.nbody",
        description="Generate the charged N-body dataset (isolated bodies) on the GPU: loc_/vel_/charges_{split}"
                    "_charged{n}_0_0_{clusters}{suffix}.npy and nbody_meta_....json under --path.  The reference's "
                    "edges_*.npy and cfg_*.pkl are not written: no loader of the reference or of this project reads "
                    "them.")
    p.add_argument("--path", type=str, default="data", help="directory to write")
    p.add_argument("--num-train", type=int, default=10000, help="training systems")
    p.add_argument("--num-valid", type=int, default=2000, help="validation systems")
    p.add_argument("--num-test", type=int, default=2000, help="test systems")
    p.add_argument("--length", type=int, default=5000, help="steps of a training / validation trajectory")
    p.add_argument("--length_test", type=int, default=5000, help="steps of a test trajectory")
    p.add_argument("--sample-freq", type=int, default=100, help="record every this many steps")
    p.add_argument("--n_isolated", type=int, default=5, help="bodies per system")
    p.add_argument("--n_stick", type=int, default=0, help="accepted only as 0 here; sticks are generated by "
                   "distegnn_b200.nbody.generate_dataset(n_stick=...)")
    p.add_argument("--n_hinge", type=int, default=0, help="accepted only as 0 here; hinges are generated by "
                   "distegnn_b200.nbody.generate_dataset(n_hinge=...)")
    p.add_argument("--clusters", type=int, default=1, help="Gaussian clusters of initial positions: 1, 3 or 10")
    p.add_argument("--seed", type=int, default=42, help="seed of the per-system random streams")
    p.add_argument("--suffix", type=str, default="", help="appended to the file tag")
    p.add_argument("--box_size", type=float, default=None, help="fail when a final position leaves [-box, box]")
    return p


def main(argv: Optional[Sequence[str]] = None) -> dict:
    a = _parser().parse_args(argv)
    if a.n_stick != 0 or a.n_hinge != 0:
        raise SystemExit("--n_stick and --n_hinge: the command line generates isolated bodies only (both must be 0); "
                         "sticks and hinges come from distegnn_b200.nbody.generate_dataset(n_stick=..., n_hinge=...)")
    try:
        stats = generate_dataset(a.path, a.num_train, a.num_valid, a.num_test, a.length, a.length_test, a.sample_freq,
                                 a.n_isolated, a.clusters, a.seed, a.suffix, a.box_size, verbose=True)
    except ValueError as e:
        raise SystemExit(f"nbody: {e}")
    print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}, indent=1))
    return stats


if __name__ == "__main__":
    main()
