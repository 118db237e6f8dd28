"""Sticks and hinges in the N-body generator (distegnn_b200.nbody, csrc/nbody.cu: distegnn_nbody_simulate_objects,
DESIGN §25).

CPU: initial conditions, object selection, object state and configuration() bitwise equal to the reference `System`
(tests/golden/nbody_constrained_reference.npz, recorded by oracle/make_golden_nbody_constrained.py); the float64 oracle
(oracle/nbody_constrained_oracle.py) against the reference's steps; its sincos and 3×3 solve; the collinear case;
argument and C-ABI checks.  GPU: the kernels bitwise equal to the oracle on both paths, in chunks, with planted tables,
the invalid-table counter and an end-to-end run through generate_dataset, load_nbody, FrameLoader and main.py."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from distegnn_b200 import nbody
from oracle import nbody_constrained_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "nbody_constrained_reference.npz")
STEPPED = ["s1", "h1", "s5", "i5s3h2", "i10s5h3c3", "s20h20", "i6s4h3c10"]
DT = 1e-3


def same_bits(a, b):
    """Bitwise equality of float64 arrays, any NaN equal to any NaN."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape:
        return False
    return bool(((a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))).all())


def _golden(name):
    z = np.load(GOLDEN)
    k = name + "_"
    return z, k, [int(c) for c in z[k + "counts"]]


def _orc_args(z, k):
    return (z[k + "sticks"][None], z[k + "hinges"][None], z[k + "stick_state"][None], z[k + "hinge_state"][None])


# ----------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", STEPPED + ["init_n1035"])
def test_initial_conditions_objects_match_reference_bits(name):
    z, k, (ni, ns, nh, c) = _golden(name)
    x, v, q, ob = nbody.initial_conditions(ni, c, 43, 0, [0], n_stick=ns, n_hinge=nh)
    assert same_bits(x[0], z[k + "X"]) and same_bits(v[0], z[k + "V"]) and same_bits(q[0], z[k + "charges"])
    for key in ("isolated", "sticks", "hinges"):
        assert np.array_equal(getattr(ob, key)[0], z[k + key]) and getattr(ob, key).dtype == np.int32
    for key in ("stick_state", "hinge_state", "stick_length", "hinge_length"):
        assert same_bits(getattr(ob, key)[0], z[k + key]), key
    cfg = ob.configuration(0)
    want = {kind: z[k + key].tolist() for kind, key in (("Isolated", "isolated"), ("Stick", "sticks"),
                                                         ("Hinge", "hinges")) if z[k + key].size}
    want["Isolated"] = [[i] for i in z[k + "isolated"].tolist()] if ni else None
    assert cfg == {kk: vv for kk, vv in want.items() if vv is not None}
    assert list(cfg) == [kind for kind, m in (("Isolated", ni), ("Stick", ns), ("Hinge", nh)) if m]


def test_isolated_only_calls_unchanged():
    a = nbody.initial_conditions(7, 3, 5, 1, 4)
    b = nbody.initial_conditions(7, 3, 5, 1, 4, n_stick=0, n_hinge=0)
    assert len(a) == len(b) == 3 and all(same_bits(p, q) for p, q in zip(a, b))
    assert nbody.tag_of(100) == "_charged100_0_0_1" and nbody.tag_of(7, 10, "_x") == "_charged7_0_0_10_x"
    assert nbody.tag_of(0, 1, n_stick=5) == "_charged0_5_0_1"
    assert nbody.tag_of(5, 3, "_y", n_stick=3, n_hinge=2) == "_charged5_3_2_3_y"


def test_objects_streams_are_per_system_and_chunkable():
    x, v, q, ob = nbody.initial_conditions(3, 1, 9, 2, 5, n_stick=2, n_hinge=2)
    x2, v2, q2, ob2 = nbody.initial_conditions(3, 1, 9, 2, [4, 1], n_stick=2, n_hinge=2)
    assert same_bits(x[[4, 1]], x2) and same_bits(v[[4, 1]], v2) and same_bits(q[[4, 1]], q2)
    assert np.array_equal(ob.sticks[[4, 1]], ob2.sticks) and same_bits(ob.hinge_state[[4, 1]], ob2.hinge_state)
    assert x.shape == (5, 13, 3) and ob.sticks.shape == (5, 2, 2) and ob.hinges.shape == (5, 2, 3)
    for s in range(5):              # every body exactly once
        bodies = np.concatenate([ob.isolated[s], ob.sticks[s].ravel(), ob.hinges[s].ravel()])
        assert sorted(bodies.tolist()) == list(range(13))
    assert not nbody.constraint_violations(x, v, ob).any()
    empty = nbody.initial_conditions(0, 1, 0, 0, 0, n_stick=1)
    assert empty[0].shape == (0, 2, 3) and empty[3].sticks.shape == (0, 1, 2)


@pytest.mark.parametrize("name", STEPPED)
def test_oracle_matches_reference_steps(name):
    """The oracle and the reference differ in the order of the force sums (within 1e-12·max|F| per step, as
    test_nbody_gen shows), of np.dot / np.matmul against the fixed dot, in sin / cos (<= 1 ulp) and the 3×3 solve
    (np.linalg.inv, within a few ulp for eigenvalues in [1, 3]).  Each of these perturbs a step's state by a few ulp of
    the state's scale; the step is well conditioned over 50 steps (a 1-ulp perturbation of a 5/3/2 system grows by
    less than 10× over 1,000 steps).  Bounds, with scale = max(1, max|X|): 1e-13·scale after one step and 1e-12·scale
    after 50 (observed: at most 4e-15 and 4e-13 unscaled)."""
    z, k, _ = _golden(name)
    X, V, q = z[k + "X"][None], z[k + "V"][None], z[k + "charges"][None]
    scale = max(1.0, np.abs(X).max())
    F, bad = orc.nbody_oracle.forces(X, q.reshape(1, -1))
    assert not bad.any()
    assert np.abs(np.clip(F, -100.0, 100.0)[0] - z[k + "F0"]).max() <= 1e-12 * max(1.0, np.abs(z[k + "F0"]).max())
    for steps, tag, bound in ((1, "1", 1e-13), (50, "50", 1e-12)):
        x, v, _, _, st, ss, hs = orc.simulate(X, V, q, *_orc_args(z, k), steps, dt=DT)
        assert (st == -1).all()
        for got, want in ((x[0], z[k + "X" + tag]), (v[0], z[k + "V" + tag]), (ss[0], z[k + "stick_state" + tag]),
                          (hs[0], z[k + "hinge_state" + tag])):
            assert np.abs(got - want).max(initial=0.0) <= bound * scale, (steps, np.abs(got - want).max())
    assert int(z[k + "check50"]) == 1


def test_collinear_system_goes_nan_and_fails_at_step_one():
    """Every position and velocity on the x axis: zero torque, wc = 0, a 0/0 rotation axis and NaN positions after
    step 0, so the force-size check fails at step 1, as in the reference (`fail1`)."""
    z, k, _ = _golden("collinear")
    X, V, q = z[k + "X"][None], z[k + "V"][None], z[k + "charges"][None]
    assert (z[k + "stick_state"][:, 6:] == 0).all() and (z[k + "hinge_state"] == 0).all()
    x, v, _, _, st, ss, hs = orc.simulate(X, V, q, *_orc_args(z, k), 1, dt=DT)
    assert same_bits(x[0], z[k + "X1"]) and np.isnan(x).any() and (st == -1).all()
    assert np.array_equal(np.isnan(v[0]), np.isnan(z[k + "V1"]))
    *_, st2, _, _ = orc.simulate(X, V, q, *_orc_args(z, k), 2, dt=DT)
    assert st2[0] == 1 and int(z[k + "fail1"]) == 1


def test_sincos_within_one_ulp():
    rng = np.random.default_rng(0)
    t = np.concatenate([rng.uniform(-1, 1, 200_000) * 10.0 ** rng.integers(-8, 7, 200_000),
                        rng.uniform(-orc.SINCOS_RANGE, orc.SINCOS_RANGE, 100_000),
                        np.nextafter(np.arange(1, 100_000) * (np.pi / 2), np.inf), [0.0, -0.0, 1e-300, np.pi / 4]])
    s, c = orc.sincos(t)
    for got, want in ((s, np.sin(t)), (c, np.cos(t))):
        ulp = np.spacing(np.maximum(np.abs(got), np.abs(want)))
        assert (np.abs(got - want) <= ulp).all()
    s, c = orc.sincos(np.array([np.inf, -np.inf, np.nan]))
    assert np.isnan(s).all() and np.isnan(c).all()


def test_solve3_agrees_with_inverse():
    rng = np.random.default_rng(1)
    e1, e2 = (u / np.linalg.norm(u, axis=1, keepdims=True) for u in rng.standard_normal((2, 5000, 3)))
    A = np.eye(3) + e1[:, :, None] * e1[:, None] + e2[:, :, None] * e2[:, None]
    b = rng.standard_normal((5000, 3)) * 10.0 ** rng.integers(-3, 4, (5000, 1))
    want = np.einsum("nij,nj->ni", np.linalg.inv(A), b)
    assert (np.abs(orc.solve3(A, b) - want).max(1) <= 1e-14 * np.abs(b).max(1)).all()


def test_planted_length_violation_is_reported():
    x, v, q, ob = nbody.initial_conditions(2, 1, 3, 0, 3, n_stick=2, n_hinge=1)
    assert not nbody.constraint_violations(x, v, ob).any()
    x2 = x.copy()
    x2[1, ob.sticks[1, 0, 1]] += 1e-5
    assert nbody.constraint_violations(x2, v, ob).tolist() == [False, True, False]
    v2 = v.copy()
    v2[2, ob.hinges[2, 0, 2]] += 1e-3 * (x[2, ob.hinges[2, 0, 2]] - x[2, ob.hinges[2, 0, 0]])
    assert nbody.constraint_violations(x, v2, ob).tolist() == [False, False, True]


def test_argument_validation():
    with pytest.raises(ValueError, match="n_stick"):
        nbody.initial_conditions(5, 1, 0, 0, 1, n_stick=-1)
    with pytest.raises(ValueError, match="n_isolated"):
        nbody.initial_conditions(-1, 1, 0, 0, 1, n_stick=2)
    with pytest.raises(ValueError, match="n_isolated"):
        nbody.initial_conditions(1, 1, 0, 0, 1)
    with pytest.raises(ValueError, match="clusters"):
        nbody.generate_dataset("unused", num_train=1, n_isolated=0, n_stick=1, clusters=4)
    nbody.initial_conditions(0, 1, 0, 0, 1, n_stick=1)       # n = 2: enough for the force check
    with pytest.raises(SystemExit, match="generate_dataset"):
        nbody.main(["--n_stick", "1", "--path", "unused"])
    assert "generate_dataset(n_hinge" in nbody._parser().format_help()


def test_c_entry_point_rejects_bad_arguments():
    from distegnn_b200 import _lib
    lib = _lib.load()
    call = lambda S, n, ns, nh, sf=1, dt=1e-3, ws=0: lib.distegnn_nbody_simulate_objects(
        S, n, ns, nh, 0, 1, sf, dt, 100.0, *([None] * 12), ws, None)
    for args, msg in (((1, 5, 0, 0), b"no sticks or hinges"), ((1, 5, -1, 1), b"n_sticks or n_hinges < 0"),
                      ((1, 4, 1, 1), b"2 * n_sticks + 3 * n_hinges"), ((1, 4, 1, 0, 0), b"sample_freq"),
                      ((1, 4, 1, 0, 1, float("nan")), b"dt"), ((1, 4, 1, 0), b"null")):
        assert call(*args) == -1 and msg in lib.distegnn_last_error(), (args, lib.distegnn_last_error())
    assert call(0, 4, 1, 0) == 0
    nbytes = _lib.C.c_int64()
    assert lib.distegnn_nbody_objects_workspace_bytes(7, 1024, _lib.C.byref(nbytes)) == 0 and nbytes.value == 0
    assert lib.distegnn_nbody_objects_workspace_bytes(7, 1025, _lib.C.byref(nbytes)) == 0
    assert nbytes.value >= 7 * 1025 * (24 + 4) + 7 * 4
    assert lib.distegnn_nbody_objects_workspace_bytes(-1, 5, _lib.C.byref(nbytes)) == -1


def test_main_nbody_tag(tmp_path):
    import main
    cfg = {"data": {"dataset_name": "nbody_100", "frame_0": 30, "frame_T": 40, "nbody_tag": "charged0_5_0_1"}}
    assert main.nbody_tag(cfg) == "charged0_5_0_1" and main.nbody_tag({"data": {}}) == "charged100_0_0_1"
    (tmp_path / "loc_valid_charged0_5_0_1.npy").write_bytes(b"")
    assert main.split_files(str(tmp_path), "nbody", "valid", "charged0_5_0_1") != []
    assert main.split_files(str(tmp_path), "nbody", "valid") == []
    with open(nbody.meta_path(str(tmp_path), "_charged0_5_0_1"), "w") as f:
        json.dump({"dt": 1e-3, "sample_freq": 50}, f)
    import argparse
    args = argparse.Namespace(trajectory=str(tmp_path), rollout_steps=2, rollout_tau=None)
    assert main.rollout_args(args, cfg, 0) == ("nbody", 2, 0.5)


# ----------------------------------------------------------------------------------------------------------- GPU
def _device_run(x, v, q, ob, steps, sample_freq, chunks=None, sys_chunks=None):
    """advance() over step ranges and system ranges; host (x, v, frames_x, frames_v, status, stick_state,
    hinge_state)."""
    dev = torch.device("cuda:0")
    S = x.shape[0]
    bounds, sys_bounds = chunks or [0, steps], sys_chunks or [0, S]
    parts = []
    for a, b in zip(sys_bounds[:-1], sys_bounds[1:]):
        sub = nbody.Objects(*(f[a:b] for f in (ob.isolated, ob.sticks, ob.hinges, ob.stick_state, ob.hinge_state,
                                               ob.stick_length, ob.hinge_length))).to(dev)
        xd, vd = (torch.from_numpy(np.ascontiguousarray(t[a:b])).to(dev) for t in (x, v))
        qd = torch.from_numpy(np.ascontiguousarray(q[a:b].reshape(b - a, -1))).to(dev)
        st = torch.full((b - a,), -1, dtype=torch.int64, device=dev)
        fx, fv = [], []
        for t0, t1 in zip(bounds[:-1], bounds[1:]):
            f = nbody.advance(xd, vd, qd, st, t0, t1 - t0, sample_freq, objects=sub)
            fx.append(f[0].cpu().numpy()), fv.append(f[1].cpu().numpy())
        parts.append((xd.cpu().numpy(), vd.cpu().numpy(), np.concatenate(fx, 1), np.concatenate(fv, 1),
                      st.cpu().numpy(), sub.stick_state.cpu().numpy(), sub.hinge_state.cpu().numpy()))
    return tuple(np.concatenate(p, 0) for p in zip(*parts))


def _check_against_oracle(x, v, q, ob, steps, sample_freq, **kw):
    got = _device_run(x, v, q, ob, steps, sample_freq, **kw)
    want = orc.simulate(x, v, q, ob.sticks, ob.hinges, ob.stick_state, ob.hinge_state, steps, sample_freq)
    want = want[:4] + (want[4],) + want[5:]
    for name, g, w in zip(("x", "v", "frames_x", "frames_v", "status", "stick_state", "hinge_state"), got, want):
        assert same_bits(g, w), f"{name}: max |device − oracle| {np.nanmax(np.abs(g - w)) if g.shape == w.shape else g.shape}"
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("ni,ns,nh,S,sample_freq,clusters,steps", [
    (0, 1, 0, 3, 1, 1, 40), (0, 0, 1, 1, 7, 3, 60), (1, 2, 0, 257, 7, 10, 30), (0, 1, 5, 3, 100, 1, 230),
    (5, 3, 2, 257, 7, 3, 30), (0, 20, 20, 3, 7, 1, 50), (15, 1, 0, 3, 1, 10, 25),
    (994, 6, 6, 1, 7, 10, 15),                                # n = 1,024: the CTA path's largest
    (1000, 5, 5, 1, 7, 1, 15), (1250, 50, 50, 3, 1, 3, 12),   # n = 1,025 and 1,500: tiled
    (0, 512, 0, 1, 7, 10, 10), (0, 0, 500, 1, 7, 1, 10),      # every body constrained, both paths
])
def test_kernel_bitwise_equals_oracle(ni, ns, nh, S, sample_freq, clusters, steps):
    x, v, q, ob = nbody.initial_conditions(ni, clusters, 11, 0, S, n_stick=ns, n_hinge=nh)
    got = _check_against_oracle(x, v, q, ob, steps, sample_freq)
    assert (got[4] == -1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [100, 1100])
def test_planted_tables_across_warps_tiles_and_ctas(n):
    """Objects whose bodies are as far apart as the system allows: the first and last bodies, and bodies on both
    sides of every warp (32) and tile (256) boundary; several systems share a CTA at n = 100."""
    x, v, q = nbody.initial_conditions(n, 1, 4, 0, 5)
    last, tile = n - 1, min(256, n // 2)
    sticks = np.array([[0, last], [31, 32], [tile - 1, tile], [63, last - 1]], dtype=np.int32)
    hinges = np.array([[last - 2, 1, 33], [64, tile + 1, 95]], dtype=np.int32)
    assert len(set(sticks.ravel()) | set(hinges.ravel())) == 14
    S = x.shape[0]
    ob = nbody.Objects(np.zeros((S, 0), np.int32), np.repeat(sticks[None], S, 0), np.repeat(hinges[None], S, 0),
                       np.zeros((S, 4, 9)), np.zeros((S, 2, 6)), np.zeros((S, 4)), np.zeros((S, 2, 2)))
    for s in range(S):
        for o, idx in enumerate(sticks):
            xc, vc, wc, ob.stick_length[s, o] = nbody._stick_initialize(x[s], v[s], idx)
            ob.stick_state[s, o] = np.concatenate([xc, vc, wc])
        for o, idx in enumerate(hinges):
            w1, w2, l1, l2 = nbody._hinge_initialize(x[s], v[s], idx)
            ob.hinge_state[s, o], ob.hinge_length[s, o] = np.concatenate([w1, w2]), (l1, l2)
    _check_against_oracle(x, v, q, ob, 20, 7)


@pytest.mark.gpu
@pytest.mark.parametrize("n_iso", [5, 1030])
def test_chunks_repeat_and_collinear(n_iso):
    x, v, q, ob = nbody.initial_conditions(n_iso, 10, 3, 2, 5, n_stick=3, n_hinge=2)
    one = _device_run(x, v, q, ob, 30, 7)
    chunked = _device_run(x, v, q, ob, 30, 7, chunks=[0, 1, 7, 8, 20, 30], sys_chunks=[0, 2, 3, 5])
    again = _device_run(x, v, q, ob, 30, 7)
    for a, b, c in zip(one, chunked, again):
        assert same_bits(a, b) and same_bits(a, c)
    fx, fv, st = nbody.simulate(*(torch.from_numpy(a).cuda() for a in (x, v, q)), 30, 7, objects=ob)
    assert same_bits(fx.cpu().numpy(), one[2]) and same_bits(fv.cpu().numpy(), one[3])
    # the collinear fixture: NaN after step 0 on the device too, and the force check fails at step 1
    z, k, _ = _golden("collinear")
    X, V, Q = z[k + "X"][None], z[k + "V"][None], z[k + "charges"][None]
    col = nbody.Objects(z[k + "isolated"][None].astype(np.int32), *(z[k + key][None] for key in (
        "sticks", "hinges", "stick_state", "hinge_state", "stick_length", "hinge_length")))
    got = _check_against_oracle(X, V, Q, col, 3, 1)
    assert same_bits(got[2][0, 0], z[k + "X1"]) and got[4][0] == 1
    with pytest.raises(ValueError, match="system 0 at step 1"):
        nbody.simulate(*(torch.from_numpy(a).cuda() for a in (X, V, Q)), 3, 1, objects=col)


@pytest.mark.gpu
@pytest.mark.parametrize("n_iso", [5, 1030])
def test_invalid_tables_are_counted(n_iso):
    x, v, q, ob = nbody.initial_conditions(n_iso, 1, 0, 0, 3, n_stick=2, n_hinge=1)
    n = x.shape[1]
    bad = nbody.Objects(*(np.array(f) for f in (ob.isolated, ob.sticks, ob.hinges, ob.stick_state, ob.hinge_state,
                                                ob.stick_length, ob.hinge_length)))
    bad.sticks[1, 0, 1] = n                 # out of range
    bad.hinges[2, 0, 2] = bad.sticks[2, 1, 0]     # a body named twice: both entries count
    bad.sticks[0, 1, 0] = -3
    dev = torch.device("cuda:0")
    xd, vd = torch.from_numpy(x).to(dev), torch.from_numpy(v).to(dev)
    st = torch.full((3,), -1, dtype=torch.int64, device=dev)
    with pytest.raises(ValueError, match="4 object table entries"):
        nbody.advance(xd, vd, torch.from_numpy(q.reshape(3, -1)).to(dev), st, 0, 5, 1, objects=bad.to(dev))
    assert same_bits(xd.cpu().numpy(), x) and same_bits(vd.cpu().numpy(), v)    # invalid systems do not move
    with pytest.raises(ValueError, match="must be a contiguous"):
        nbody.advance(xd, vd, torch.from_numpy(q.reshape(3, -1)).to(dev), st, 0, 5, 1, objects=ob)


@pytest.mark.gpu
def test_planted_length_violation_raises():
    x, v, q, ob = nbody.initial_conditions(5, 1, 0, 0, 2, n_stick=3, n_hinge=2)
    args = [torch.from_numpy(a).cuda() for a in (x, v, q)]
    nbody.simulate(*args, 20, 7, objects=ob)
    ob.stick_length[1, 2] += 1e-5
    with pytest.raises(ValueError, match=r"end-of-run check.*systems \[1\]"):
        nbody.simulate(*args, 20, 7, objects=ob)


@pytest.mark.gpu
def test_generate_dataset_constrained_end_to_end(tmp_path):
    import yaml
    from distegnn_b200.frames import FrameLoader, load_nbody, sample_list
    data = tmp_path / "nbody"
    ni, ns, nh = 5, 3, 2
    stats = nbody.generate_dataset(str(data), num_train=10, num_valid=4, num_test=4, length=1100, length_test=1100,
                                   n_isolated=ni, seed=43, chunk=3, n_stick=ns, n_hinge=nh)
    tag = "_charged5_3_2_1"
    for part, S in (("train", 10), ("valid", 4), ("test", 4)):
        loc = np.load(data / f"loc_{part}{tag}.npy")
        vel = np.load(data / f"vel_{part}{tag}.npy")
        assert loc.shape == vel.shape == (S, 11, 17, 3)
        assert np.load(data / f"charges_{part}{tag}.npy").shape == (S, 17, 1)
        assert not (data / f"edges_{part}{tag}.npy").exists()
        with open(data / f"cfg_{part}{tag}.pkl", "rb") as f:
            cfg = pickle.load(f)
        _, _, _, ob = nbody.initial_conditions(ni, 1, 43, ("train", "valid", "test").index(part), S, n_stick=ns,
                                               n_hinge=nh)
        assert isinstance(cfg, tuple) and len(cfg) == S and all(cfg[s] == ob.configuration(s) for s in range(S))
        for t in range(loc.shape[1]):           # every recorded frame keeps the constraints
            assert not nbody.constraint_violations(loc[:, t], vel[:, t], ob).any(), (part, t)
    x, v, q, ob = nbody.initial_conditions(ni, 1, 43, 1, [3], n_stick=ns, n_hinge=nh)
    _, _, fx, fv, *_ = orc.simulate(x, v, q, ob.sticks, ob.hinges, ob.stick_state, ob.hinge_state, 201, 100)
    assert same_bits(np.load(data / f"loc_valid{tag}.npy")[3, :3], fx[0])
    assert same_bits(np.load(data / f"vel_valid{tag}.npy")[3, :3], fv[0])
    meta = json.load(open(data / f"nbody_meta{tag}.json"))
    assert (meta["n_stick"], meta["n_hinge"], meta["n_isolated"]) == (3, 2, 5) and len(stats["files"]) == 13
    traj = load_nbody(str(data), "train", tag[1:])
    ld = FrameLoader(traj, sample_list(traj, frame_0=3, delta_t=5), delta_t=5, radius=-1, batch_size=4,
                     device=torch.device("cuda:0"))
    assert len(list(ld)) == 2                   # 10 systems in batches of 4, the partial batch dropped
    with open(os.path.join(ROOT, "config", "nbody_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["log"] = dict(cfg.get("log") or {}, log_dir=str(tmp_path / "logs"))
    cfg["data"].update(frame_0=3, frame_T=8, nbody_tag=tag[1:])
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--config_path", str(p), "--trajectory",
                        str(data), "--epochs", "1", "--batch_size", "4"], capture_output=True, text=True, timeout=900,
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
