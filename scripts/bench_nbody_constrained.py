"""Time N-body generation with sticks and hinges (distegnn_b200.nbody, DESIGN §25) on the GPU against isolated-only
runs at the same body count, and write one JSON report.

    python scripts/bench_nbody_constrained.py --out profiles/nbody_constrained_h100.json [--quick]

Workloads (each through generate_dataset into a temporary directory):
  run_sh_sticks   the reference's run.sh stick line: 0 isolated / 5 sticks / 0 hinges (n = 10), 5,000 / 2,000 / 2,000
                  systems × 5,000 steps, CTA path
  cta_s20h20      0 / 20 / 20 (n = 100), 2,000 systems × 5,000 steps, CTA path
  tiled_n1035     1,000 / 10 / 5 in 10 clusters (n = 1,035), 100 systems × 500 steps, tiled path
Each is also run with n isolated bodies and no objects (same systems, steps and clusters).  Reported: host set-up
seconds (initial conditions: draws, object selection, `initialize`), device seconds (CUDA events around simulate(); for
constrained runs this includes the end-of-run check, which reads the final state back to the host), write seconds, and
the constrained / isolated device-time ratio.  The reference's cost, measured on one core of a CPU host with numpy, is
recorded beside them (REFERENCE_MS_PER_STEP).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from distegnn_b200 import nbody  # noqa: E402

WORKLOADS = {
    "run_sh_sticks": dict(num_train=5000, num_valid=2000, num_test=2000, length=5000, length_test=5000, n_isolated=0,
                          n_stick=5, n_hinge=0, clusters=1, seed=43),
    "cta_s20h20": dict(num_train=2000, num_valid=0, num_test=0, length=5000, length_test=5000, n_isolated=0,
                       n_stick=20, n_hinge=20, clusters=1, seed=43),
    "tiled_n1035": dict(num_train=100, num_valid=0, num_test=0, length=500, length_test=500, n_isolated=1000,
                        n_stick=10, n_hinge=5, clusters=10, seed=43),
}
QUICK = {"run_sh_sticks": dict(num_train=50, num_valid=20, num_test=20, length=500, length_test=500),
         "cta_s20h20": dict(num_train=20, length=500, length_test=500),
         "tiled_n1035": dict(num_train=4, length=20, length_test=20)}
# the reference System, ms per step on one CPU core (numpy): ni/ns/nh -> ms
REFERENCE_MS_PER_STEP = {"0/5/0": 1.0, "5/3/2": 1.4, "10/5/3": 2.1, "0/20/20": 11.9}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(kw):
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        st = nbody.generate_dataset(d, sample_freq=100, **kw)
        wall = time.perf_counter() - t0
    return {"wall_s": round(wall, 3), "host_init_s": round(st["init_s"], 3), "device_s": round(st["simulate_s"], 4),
            "write_s": round(st["write_s"], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="JSON report path (default: print only)")
    ap.add_argument("--quick", action="store_true", help="small sizes: a rehearsal, not a measurement")
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nbody_constrained needs a CUDA device")
    names = a.only.split(",") if a.only else list(WORKLOADS)
    for n_iso in (4, 1030):         # warm-up: module load and first launches of both paths, both entry points
        x, v, q, ob = nbody.initial_conditions(n_iso, 1, 0, 0, 2, n_stick=1, n_hinge=1)
        nbody.simulate(*(torch.from_numpy(t).cuda() for t in (x, v, q)), 3, 1, objects=ob)
        nbody.simulate(*(torch.from_numpy(t).cuda() for t in (x, v, q)), 3, 1)
    torch.cuda.synchronize()
    rep = {"card": card(), "quick": a.quick, "reference_ms_per_step_cpu": REFERENCE_MS_PER_STEP, "results": []}
    for name in names:
        kw = dict(WORKLOADS[name], **(QUICK[name] if a.quick else {}))
        n = nbody.n_bodies(kw["n_isolated"], kw["n_stick"], kw["n_hinge"])
        iso = dict(kw, n_isolated=n, n_stick=0, n_hinge=0)
        c, i = run(kw), run(iso)
        steps = (kw["num_train"] + kw["num_valid"]) * kw["length"] + kw["num_test"] * kw["length_test"]
        r = {"workload": name, **kw, "n_bodies": n, "system_steps": steps, "constrained": c, "isolated": i,
             "device_ratio": round(c["device_s"] / i["device_s"], 3),
             "host_init_ratio": round(c["host_init_s"] / max(i["host_init_s"], 1e-9), 3),
             "device_us_per_system_step": round(c["device_s"] / steps * 1e6, 4)}
        print(json.dumps(r), flush=True)
        rep["results"].append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)
    print(json.dumps({"card": rep["card"]}))


if __name__ == "__main__":
    main()
