"""Record tests/golden/nbody_constrained_reference.npz from the reference's N-body `System` with sticks and hinges
(dataset_generation/nbody/system.py, physical_objects.py), unmodified, so that tests compare distegnn_b200.nbody's
constrained systems against the reference where the reference is not installed.

    python oracle/make_golden_nbody_constrained.py REFERENCE_ROOT      # the root of a checkout of the reference

Each case sets the global numpy state to the state of system 0 of split 0 with seed 43 (distegnn_b200.nbody.system_rng)
and builds `System(n_isolated, n_stick, n_hinge, clusters)`.  Keys {case}_{name}:
  X, V, charges                     the initial state, after the objects' `initialize`
  isolated [ni], sticks [ns,2], hinges [nh,3]     `configuration()`, in object order
  stick_state [ns,9] (xc, vc, wc), stick_length [ns], hinge_state [nh,6] (w1, w2), hinge_length [nh,2]
  F0                                `compute_F` of the initial state (clamped)
  X1, V1, stick_state1, hinge_state1        after one `simulate_one_step`; likewise X50, ... after 50
  check50                           1 when `System.check()` passes after 50 steps
The case `init_n1035` records the initial state only.  The case `collinear` plants a system with every position and
velocity on the x axis, re-runs the objects' own `initialize` on it and records one step; its key `fail1` is 1 when
the reference's force-size assertion fails at step 1.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "nbody_constrained_reference.npz")
SEED, SPLIT, SYSTEM = 43, 0, 0
# name: (n_isolated, n_stick, n_hinge, clusters, steps recorded)
CASES = {
    "s1": (0, 1, 0, 1, 50), "h1": (0, 0, 1, 1, 50), "s5": (0, 5, 0, 1, 50), "i5s3h2": (5, 3, 2, 1, 50),
    "i10s5h3c3": (10, 5, 3, 3, 50), "s20h20": (0, 20, 20, 1, 50), "i6s4h3c10": (6, 4, 3, 10, 50),
    "init_n1035": (1000, 10, 5, 1, 0),
}


def _record(out, k, sy, steps):
    from physical_objects import Hinge, Stick
    objs = sy.physical_objects

    def state(tag):
        st = [o for o in objs if isinstance(o, Stick)]
        hg = [o for o in objs if isinstance(o, Hinge)]
        out[k + "stick_state" + tag] = np.array([np.concatenate([o.xc, o.vc, o.wc]) for o in st]).reshape(-1, 9)
        out[k + "hinge_state" + tag] = np.array([np.concatenate([o.w1, o.w2]) for o in hg]).reshape(-1, 6)
        if tag == "":
            out[k + "stick_length"] = np.array([o.length for o in st], dtype=np.float64)
            out[k + "hinge_length"] = np.array([[o.length1, o.length2] for o in hg], dtype=np.float64).reshape(-1, 2)

    cfg = sy.configuration()
    out[k + "isolated"] = np.array(cfg.get("Isolated", []), dtype=np.int64).reshape(-1)
    out[k + "sticks"] = np.array(cfg.get("Stick", []), dtype=np.int64).reshape(-1, 2)
    out[k + "hinges"] = np.array(cfg.get("Hinge", []), dtype=np.int64).reshape(-1, 3)
    out[k + "X"], out[k + "V"], out[k + "charges"] = sy.X.copy(), sy.V.copy(), sy.charges.copy()
    state("")
    if steps == 0:
        return
    out[k + "F0"] = sy.compute_F(sy.X, sy.V)
    for t in range(steps):
        sy.simulate_one_step()
        if t == 0:
            out[k + "X1"], out[k + "V1"] = sy.X.copy(), sy.V.copy()
            state("1")
    if steps == 1:
        return
    out[k + "X50"], out[k + "V50"] = sy.X.copy(), sy.V.copy()
    state("50")
    try:
        sy.check()
        out[k + "check50"] = np.array(1)
    except AssertionError:
        out[k + "check50"] = np.array(0)


def main(ref_root: str) -> None:
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ref_root, "dataset_generation", "nbody"))
    if "tqdm" not in sys.modules:            # the reference imports tqdm for progress bars only
        stub = types.ModuleType("tqdm")
        stub.tqdm = lambda it, **k: it
        sys.modules["tqdm"] = stub
    from system import System
    from distegnn_b200.nbody import system_rng
    out = {}
    for name, (ni, ns, nh, c, steps) in CASES.items():
        np.random.set_state(system_rng(SEED, SPLIT, SYSTEM).get_state())
        sy = System(n_isolated=ni, n_stick=ns, n_hinge=nh, clusters=c)
        out[name + "_counts"] = np.array([ni, ns, nh, c])
        _record(out, name + "_", sy, steps)
    # collinear: one isolated body, one stick, one hinge, all on the x axis; every angular velocity is exactly 0
    np.random.set_state(system_rng(SEED, SPLIT, SYSTEM).get_state())
    sy = System(n_isolated=1, n_stick=1, n_hinge=1, clusters=1)
    X, V = sy.X.copy(), sy.V.copy()
    X[:, 1:] = 0.0
    V[:, 1:] = 0.0
    for o in sy.physical_objects:
        X, V = o.initialize(X, V)
    sy.X, sy.V = X, V
    k = "collinear_"
    out["collinear_counts"] = np.array([1, 1, 1, 1])
    _record(out, k, sy, 1)
    try:
        sy.simulate_one_step()
        out[k + "fail1"] = np.array(0)
    except AssertionError:
        out[k + "fail1"] = np.array(1)
    np.savez_compressed(OUT, **out)
    print(OUT, len(out), "arrays")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
