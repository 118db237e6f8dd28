"""Training through K-step rollouts (DESIGN §26): the stepped fused loss (`train_loss` on [K,N,3] inputs, the *_steps
entry points of csrc/loss.cu) against a float64 restatement and against K one-step calls, and `main.py --train_rollout K`
in both training loops.

The stepped restatement is `tests/test_loss_kernel.reference` per step, combined as (1/K)·Σ_t; on the CPU it is checked
against oracle/train_loss_oracle.py (the per-step restatement of utils/train.py:98-147), on the GPU the kernels are
checked against it with test_loss_kernel's element-wise bounds, widened by the one rounding of the 1/K scaling and the K
additions of the step means."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from distegnn_b200.loss import graph_offsets
from oracle import train_loss_oracle as tlo
from tests import test_loss_kernel as tlk
from tests.test_loss_kernel import (bounds, elem_err, gamma, make_case, scalar_err, terms_err)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatement of the stepped loss
# ---------------------------------------------------------------------------------------------------------------------

def stepped_case(sizes, C, mmd_samples, K, seed, **kw):
    """K one-step cases on the same graphs (sizes), each with its own positions, virtual coordinates and samples."""
    steps = [make_case(sizes, C, mmd_samples, seed=seed + 1000 * t, **kw) for t in range(K)]
    st = lambda k: torch.stack([c[k] for c in steps])
    return dict(steps=steps, pred=st("pred"), target=st("target"), Xv=st("Xv"), samples=st("samples"),
                batch=steps[0]["batch"], C=C, S=steps[0]["S"], mmd_samples=mmd_samples, sigma=steps[0]["sigma"],
                weight=steps[0]["weight"], K=K)


def stepped_reference(case, node_counts=None, rank=0, accum=1):
    """loss = (1/K)·Σ_t ℓ_t, logged and mmd the step means, g_pred [K,N,3] and g_Xv [K,B,3,C] = (1/K)·the step's
    one-step gradient; the per-step references ride along for the bounds."""
    K = case["K"]
    refs = [tlk.ref_of(c, node_counts, rank, accum) for c in case["steps"]]
    return dict(loss=sum(r["loss"] for r in refs) / K, logged=sum(r["logged"] for r in refs) / K,
                mmd=sum(r["mmd"] for r in refs) / K, g_pred=torch.stack([r["g_pred"] for r in refs]) / K,
                g_Xv=torch.stack([r["g_Xv"] for r in refs]) / K, g_terms=torch.stack([r["g_terms"] for r in refs]) / K,
                steps=refs, logged_steps=[r["logged"] for r in refs], mmd_steps=[r["mmd"] for r in refs])


def stepped_bounds(case, ref, node_counts=None, upstream=False):
    """test_loss_kernel.bounds of every step; loss / mmd: Σ_t of each step's absolute bound over K, plus the K − 1
    additions and the 1/K product (γ_{K+1}) of the step mean; logged: the largest step bound plus γ_{K+1}; gradients:
    the largest step bound plus one more rounding (coef·(1/K))."""
    K = case["K"]
    counts = node_counts or [case["pred"].shape[1]]
    per = [bounds(r, counts, case["C"], case["S"], case["Xv"].shape[1], case["weight"], world=len(counts),
                  upstream=upstream) for r in ref["steps"]]
    mean = gamma(K + 1)
    out = {}
    # logged is the sum over the ranks of positive terms: each step's relative bound holds for the step mean too
    out["logged"] = max(b["logged"] for b in per) + mean
    for k, scale in (("loss", None), ("mmd", "mmd_scale")):
        mag = [abs(r[k]) if scale is None else r[scale] for r in ref["steps"]]
        absolute = sum(b[k] * m for b, m in zip(per, mag)) / K + mean * sum(abs(r[k]) for r in ref["steps"]) / K
        denom = abs(ref[k]) if scale is None else sum(mag) / K
        out[k] = absolute / max(denom, 1e-300)
    out["g_pred"] = max(b["g_pred"] for b in per) + gamma(1)
    out["g_Xv"] = max(b["g_Xv"] for b in per) + gamma(1)
    return out


def check_stepped(name, got, ref, bd):
    errs = dict(loss=scalar_err(got["loss"], ref["loss"]),
                logged=scalar_err(got["logged"], ref["logged"]),
                mmd=scalar_err(got["mmd"], ref["mmd"], sum(r["mmd_scale"] for r in ref["steps"]) / len(ref["steps"])),
                g_pred=elem_err(got["g_pred"], ref["g_pred"]),
                g_Xv=terms_err(got["g_Xv"], ref["g_Xv"], ref["g_terms"]))
    print(f"{name}: " + "  ".join(f"{k} {v:.2e} (bound {bd[k]:.2e})" for k, v in errs.items()))
    bad = {k: (v, bd[k]) for k, v in errs.items() if not v <= bd[k]}
    assert not bad, (name, bad)


def _oracle_stepped(case, node_counts, rank, accum):
    """oracle/train_loss_oracle.py once per step, combined as (1/K)·Σ_t: loss, logged, g_pred, g_Xv."""
    K = case["K"]
    p = case["pred"].double().requires_grad_(True)
    V = case["Xv"].double().requires_grad_(True)
    loss, logged = 0.0, 0.0
    for t in range(K):
        smp = [row[row >= 0].long() for row in case["samples"][t]]
        l_t, lg_t = tlo.train_loss(p[t], case["target"][t].double(), V[t], case["batch"], smp, node_counts=node_counts,
                                   rank=rank, sigma=case["sigma"], weight=case["weight"],
                                   samples_per_channel=case["mmd_samples"], accumulation_steps=accum)
        loss, logged = loss + l_t / K, logged + float(lg_t) / K
    gp, gV = torch.autograd.grad(loss, [p, V])
    return float(loss.detach()), logged, gp, gV


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [1, 2, 5])
@pytest.mark.parametrize("layout", ["one_rank", "world3_rank1"])
def test_stepped_restatement_matches_the_per_step_oracle(K, layout):
    """The stepped float64 restatement agrees with oracle/train_loss_oracle.py run once per step within 1e-12."""
    case = stepped_case([0, 3, 19, 20, 21, 40], 4, 5, K, seed=11, sigma=1.5, weight=0.05)
    n = int(case["pred"].shape[1])
    counts, rank, accum = ([n], 0, 1) if layout == "one_rank" else ([17, n, 123], 1, 3)
    ref = stepped_reference(case, counts, rank, accum)
    loss, logged, gp, gV = _oracle_stepped(case, counts, rank, accum)
    assert scalar_err(ref["loss"], loss) <= 1e-12
    assert scalar_err(ref["logged"], logged) <= 1e-12
    assert elem_err(ref["g_pred"], gp) <= 1e-12
    assert terms_err(ref["g_Xv"], gV, ref["g_terms"]) <= 1e-12


def _main(args, **env):
    return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), *args], capture_output=True, text=True,
                          timeout=600, cwd=ROOT, env=dict(os.environ, **env))


def _walk(rng, T, n, step):
    x0 = rng.uniform(0.2, 0.8, (1, n, 3))
    return (x0 + np.cumsum(step * rng.standard_normal((T, n, 3)), 0)).astype(np.float32)


def _water(d, sizes, T=10, seed=0, step=0.01):
    rng = np.random.default_rng(seed)
    for k, n in enumerate(sizes):
        np.savez(str(d / f"water_{k}.npz"), position=_walk(rng, T, n, step), particle_type=rng.integers(1, 9, n))


def _water_cfg(tmp_path, data, **data_kw):
    import yaml
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"].update(node_feat_nf=2, node_attr_nf=1)
    cfg["data"].update(dict(dataset_name="Water3D", inner_radius=0.3, max_samples=8, split_mode="random", delta_t=2,
                            batch_size=2), **data_kw)
    cfg["log"] = {"log_dir": str(tmp_path / "logs"), "test_interval": 1}
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    return str(p), cfg


def _nbody_files(d, S=3, T=41, n=5, seed=0):
    """The reference's N-body file layout, random walks (the CLI checks read shapes only)."""
    rng = np.random.default_rng(seed)
    for part in ("train", "valid", "test"):
        loc = np.cumsum(rng.standard_normal((S, T, n, 3)), 1)
        np.save(d / f"loc_{part}_charged100_0_0_1.npy", loc)
        np.save(d / f"vel_{part}_charged100_0_0_1.npy", np.gradient(loc, axis=1))
        np.save(d / f"charges_{part}_charged100_0_0_1.npy", rng.choice([-1.0, 1.0], (S, n, 1)))


def test_main_rejects_bad_train_rollout_before_cuda_work(tmp_path):
    """Exit code 2 and a message, with no CUDA device visible: K < 1, no --trajectory, Water-3D scenes too short for K
    steps of delta_t frames, N-body files whose frame_0 cannot hold K steps, and no rollout time step."""
    data = tmp_path / "water"
    for part in ("train", "valid", "test"):
        (data / part).mkdir(parents=True)
        _water(data / part, [20, 30], T=10)
    cfg, _ = _water_cfg(tmp_path, data)
    base = ["--config_path", cfg, "--trajectory", str(data)]
    nb = tmp_path / "nbody"
    nb.mkdir()
    _nbody_files(nb)
    nb_cfg = os.path.join(ROOT, "config", "nbody_fastegnn.yaml")           # frame_0 30, frame_T 40: one step fits
    for args, msg in ((base + ["--train_rollout", "0"], ">= 1"), (base + ["--train_rollout", "-3"], ">= 1"),
                      (["--config_path", cfg, "--train_rollout", "2"], "used with --trajectory"),
                      (base + ["--train_rollout", "5", "--epochs", "1"], "cannot hold 5 step(s)"),
                      (["--config_path", nb_cfg, "--trajectory", str(nb), "--train_rollout", "2"], "horizon=2"),
                      (["--config_path", nb_cfg, "--trajectory", str(nb), "--train_rollout", "1"], "--rollout_tau")):
        r = _main(args, CUDA_VISIBLE_DEVICES="")
        assert r.returncode == 2 and msg in r.stdout and r.stdout.startswith("--train_rollout"), (args, r.stdout,
                                                                                                  r.stderr[-2000:])
        assert "CUDA" not in r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the stepped kernels
# ---------------------------------------------------------------------------------------------------------------------

def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (no fallback)"
    return torch.device("cuda:0")


def fused_stepped(case, accum=1, loc_mean=None):
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
                logged_steps=info["logged_steps"].cpu(), mmd_steps=info["mmd_steps"].cpu(),
                dev=float(info["loc_mean_dev"]), g_pred=p.grad.cpu(), g_Xv=V.grad.cpu(), info=info)


SHAPES = {   # name: (graph sizes, C, mmd_samples)
    "B1_C1": ([300], 1, 7),
    "B3_C3_fewer_nodes_than_S": ([40, 5, 2], 3, 10),
    "B3_C8_beyond_one_cta": ([2047, 2, 2100], 8, 50),
    "B250_C16": ([1 + (i * 7919) % 60 for i in range(250)], 16, 3),
    "B3_C16_S_above_threads": ([500, 30, 900], 16, 50),
}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("K", [1, 2, 5])
def test_stepped_loss_against_float64(K, shape):
    sizes, C, m = SHAPES[shape]
    case = stepped_case(sizes, C, m, K, seed=7 + K)
    accum = 2 if K == 2 else 1
    ref = stepped_reference(case, accum=accum)
    got = fused_stepped(case, accum)
    check_stepped(f"K={K} {shape}", got, ref, stepped_bounds(case, ref))
    for t in range(K):                                                    # the per-step values of info
        assert scalar_err(float(got["logged_steps"][t]), ref["logged_steps"][t]) <= 1e-5
        assert scalar_err(float(got["mmd_steps"][t]), ref["mmd_steps"][t], ref["steps"][t]["mmd_scale"]) <= 1e-5


def run_ranks_stepped(ranks, Xv, C, S, sigma, weight, loc_means, K, accum=1):
    """test_loss_kernel.run_ranks through the *_steps entry points: every rank's partials on one GPU, the packed vectors
    summed in rank order, every rank's finalize."""
    from distegnn_b200 import _lib
    from distegnn_b200._lib import check as ck, ptr
    lib, d = _lib.load(), dev()
    B, world = Xv.shape[1], len(ranks)
    npk = lib.distegnn_loss_packed_floats_steps(K, B, world)
    assert npk == 1 + K + world * 3 * B
    st = torch.cuda.current_stream().cuda_stream
    Vd, bufs = Xv.to(d).contiguous(), []
    for r, rk in enumerate(ranks):
        n = int(rk["pred"].shape[1])
        p, t = (rk["pred"].to(d).contiguous(), rk["target"].to(d).contiguous()) if n else (None, None)
        acc, packed, gV = torch.zeros(3 * K, device=d), torch.zeros(npk, device=d), torch.empty(K, B, 3, C, device=d)
        lm = loc_means[r].to(d)
        gptr, sm = graph_offsets(rk["batch"].to(d), B), rk["samples"].to(d).contiguous()
        ck(lib.distegnn_loss_partials_steps(K, n, B, C, S, world, r, sigma, ptr(p), ptr(t), ptr(Vd), ptr(lm), ptr(gptr),
                                            ptr(sm), ptr(acc), ptr(packed), ptr(gV), st), "loss_partials_steps")
        bufs.append((n, p, t, lm, acc, packed, gV))
    total = bufs[0][5].clone()
    for b in bufs[1:]:
        total += b[5]
    outs = []
    for r, (n, p, t, lm, acc, _, gV) in enumerate(bufs):
        g_pred = torch.empty_like(p) if n else None
        g_Xv, out, out_steps = torch.empty(K, B, 3, C, device=d), torch.empty(4, device=d), torch.empty(2 * K, device=d)
        ck(lib.distegnn_loss_finalize_steps(K, n, B, C, S, world, r, sigma, weight, accum, ptr(p), ptr(t), ptr(lm),
                                            ptr(acc), ptr(total), ptr(gV), ptr(g_pred), ptr(g_Xv), ptr(out),
                                            ptr(out_steps), st), "loss_finalize_steps")
        outs.append((out, g_pred, g_Xv))
    torch.cuda.synchronize()
    return [dict(loss=float(o[0]), logged=float(o[1]), mmd=float(o[2]), dev=float(o[3]),
                 g_pred=(gp.cpu() if gp is not None else torch.zeros(K, 0, 3)), g_Xv=gx.cpu()) for o, gp, gx in outs]


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 5])
def test_stepped_world3_unequal_ranks_and_loc_mean_report(K):
    """test_loss_kernel's world = 3 layout, K steps: every rank against the float64 restatement, the loc_mean
    deviation reported once."""
    C, m = 5, 6
    cases = [stepped_case(s, C, m, K, seed=40 + r, sigma=2.0, weight=0.03)
             for r, s in enumerate([[40, 25, 300], [2100, 13, 60], [5, 0, 77]])]
    for c in cases[1:]:
        c["Xv"] = cases[0]["Xv"]
        for t in range(K):
            c["steps"][t]["Xv"] = cases[0]["steps"][t]["Xv"]
    counts = [int(c["pred"].shape[1]) for c in cases]
    lm0 = torch.randn(3, 3, generator=torch.Generator().manual_seed(1))
    delta = torch.zeros(3, 3)
    delta[1, 2] = 0.0625
    lms = [lm0, lm0.clone(), lm0 + delta]
    outs = run_ranks_stepped(cases, cases[0]["Xv"], C, C * m, 2.0, 0.03, lms, K)
    refs = [stepped_reference(c, counts, r) for r, c in enumerate(cases)]
    logged = sum(r["logged"] for r in refs)
    for r, (c, got, ref) in enumerate(zip(cases, outs, refs)):
        ref = dict(ref, logged=logged)
        check_stepped(f"K={K} world=3 rank {r}", got, ref, stepped_bounds(c, ref, counts))
        assert got["dev"] == float((lms[2] - lms[0]).abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 3])
def test_stepped_world4_with_an_empty_rank(K):
    C, m = 4, 5
    cases = [stepped_case(s, C, m, K, seed=50 + r, sigma=2.0, weight=0.03)
             for r, s in enumerate([[40, 25], [2100, 13], [0, 0], [9, 70]])]
    for c in cases[1:]:
        c["Xv"] = cases[0]["Xv"]
        for t in range(K):
            c["steps"][t]["Xv"] = cases[0]["steps"][t]["Xv"]
    counts = [int(c["pred"].shape[1]) for c in cases]
    lm = torch.randn(2, 3, generator=torch.Generator().manual_seed(2))
    outs = run_ranks_stepped(cases, cases[0]["Xv"], C, C * m, 2.0, 0.03, [lm] * 4, K)
    refs = [stepped_reference(c, counts, r) for r, c in enumerate(cases)]
    logged = sum(r["logged"] for i, r in enumerate(refs) if i != 2)
    assert outs[2]["loss"] == 0.0 and bool((outs[2]["g_Xv"] == 0).all())
    for r in (0, 1, 3):
        ref = dict(refs[r], logged=logged)
        check_stepped(f"K={K} world=4 rank {r}", outs[r], ref, stepped_bounds(cases[r], ref, counts))


# loss.cu adds its partial sums with atomics in no fixed order, so two runs of the same call can differ in the last bits
# wherever an atomic sum has three or more addends.  This shape has none: one node block (the SSE is one block tree and
# one atomic), two graphs (two atomics per MMD accumulator) and C = 1, S = 2 (the one virtual node's gradient gets the
# two sample terms only; its pair with itself is at distance 0).  There every output is a fixed function of the inputs.
ORDER_FREE = ([700, 900], 1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["order_free", "B3_C8_beyond_one_cta", "B250_C16"])
def test_k1_is_bitwise_the_one_step_call(shape):
    """[1,N,3] inputs run the one-step arithmetic: with the same samples, the same bits as the [N,3] call — loss,
    logged, mmd, g_pred and g_Xv on the order-free shape, and g_pred and the loc_mean report on every shape (no atomic
    in them).  With default samples both draw the same randperms from the global generator."""
    sizes, C, m = ORDER_FREE if shape == "order_free" else SHAPES[shape]
    case = stepped_case(sizes, C, m, 1, seed=3)
    lm = torch.ones(len(sizes), 3)
    one = tlk.fused(case["steps"][0], accum=2, loc_mean=lm)
    st = fused_stepped(case, accum=2, loc_mean=lm)
    exact = ("loss", "logged", "mmd", "dev") if shape == "order_free" else ("dev",)
    for k in exact:
        assert st[k] == one[k] and math.copysign(1, st[k]) == math.copysign(1, one[k]), k
    assert torch.equal(st["g_pred"][0], one["g_pred"])
    if shape == "order_free":
        again = tlk.fused(case["steps"][0], accum=2, loc_mean=lm)        # the shape is order-free: runs agree
        assert torch.equal(again["g_Xv"], one["g_Xv"]) and again["loss"] == one["loss"]
        assert torch.equal(st["g_Xv"][0], one["g_Xv"])
        assert float(st["logged_steps"][0]) == one["logged"] and float(st["mmd_steps"][0]) == one["mmd"]
    from distegnn_b200 import train_loss
    d = dev()
    c = case["steps"][0]
    args = dict(mmd_samples=m, mmd_sigma=c["sigma"], mmd_weight=c["weight"], node_counts=sizes)
    torch.manual_seed(5)
    _, i1 = train_loss(c["pred"].to(d), c["target"].to(d), c["Xv"].to(d), c["batch"].to(d), **args)
    torch.manual_seed(5)
    _, ik = train_loss(case["pred"].to(d), case["target"].to(d), case["Xv"].to(d), case["batch"].to(d), **args)
    assert ik["samples"].shape == (1,) + tuple(i1["samples"].shape) and torch.equal(ik["samples"][0], i1["samples"])


@pytest.mark.gpu
def test_k_steps_equal_the_mean_of_k_one_step_calls_and_cost_one_collective(monkeypatch):
    """K = 4: g_pred is bitwise (1/K)·Σ_t of the one-step calls' (1/4 scales exactly); g_Xv, the loss and logged agree
    within twice the float64 bounds (each side's atomic sums round in their own order); and the call issues ONE
    collective where K one-step calls issue K (world_size 2 through a counting stand-in for the all-reduce that adds an
    identical rank's vector)."""
    import torch.distributed as dist
    from distegnn_b200 import train_loss
    K = 4
    sizes, C, m = SHAPES["B3_C8_beyond_one_cta"]
    case = stepped_case(sizes, C, m, K, seed=9)
    calls = []

    def fake_all_reduce(t, op=None, group=None):
        calls.append(int(t.numel()))
        t.mul_(2.0)                                                  # rank 1 sends the same vector
    monkeypatch.setattr(dist, "all_reduce", fake_all_reduce)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    d = dev()
    kw = dict(world_size=2, mmd_samples=m, mmd_sigma=case["sigma"], mmd_weight=case["weight"])
    p = case["pred"].to(d).requires_grad_(True)
    V = case["Xv"].to(d).requires_grad_(True)
    loss, info = train_loss(p, case["target"].to(d), V, case["batch"].to(d), samples=case["samples"].to(d), **kw)
    loss.backward()
    assert calls == [1 + K + 2 * 3 * len(sizes)]
    calls.clear()
    p1 = case["pred"].to(d).requires_grad_(True)
    V1 = case["Xv"].to(d).requires_grad_(True)
    tot, logged = 0.0, 0.0
    for t in range(K):
        l_t, i_t = train_loss(p1[t], case["target"][t].to(d), V1[t], case["batch"].to(d),
                              samples=case["samples"][t].to(d), **kw)
        tot, logged = tot + l_t / K, logged + float(i_t["logged"]) / K
    tot.backward()
    assert len(calls) == K
    assert torch.equal(p.grad, p1.grad)
    n = int(case["pred"].shape[1])
    ref = stepped_reference(case, [n, n], 0)                              # the stand-in's world: two equal ranks
    bd = stepped_bounds(case, ref, [n, n])
    e_V = terms_err(V.grad.cpu(), V1.grad.cpu(), ref["g_terms"])
    e_l = scalar_err(float(loss), float(tot))
    e_g = scalar_err(float(info["logged"]), logged)
    print(f"K={K} stepped vs mean of one-step calls: g_Xv {e_V:.2e} (2x bound {2 * bd['g_Xv']:.2e})  loss {e_l:.2e} "
          f"(2x bound {2 * bd['loss']:.2e})  logged {e_g:.2e} (2x bound {2 * bd['logged']:.2e})")
    assert e_V <= 2 * bd["g_Xv"] and e_l <= 2 * bd["loss"] and e_g <= 2 * bd["logged"]


@pytest.mark.gpu
def test_noise_shifts_every_step_target_by_the_input_noise(tmp_path):
    """--train_noise with K steps: FrameLoader adds each node's ε_x to its position and to every one of its K target
    rows, so the noisy targets of every step are the clean ones shifted by the input's shift."""
    from distegnn_b200.frames import FrameLoader, load_scenes, sample_list
    _water(tmp_path, [40, 30], T=12)
    traj = load_scenes(sorted(str(p) for p in tmp_path.glob("*.npz")), "water3d")
    samples = sample_list(traj, seed=0, max_frame=2)
    kw = dict(delta_t=2, radius=0.2, batch_size=2, seed=3, device=dev(), horizon=4)
    (ck, cx), = list(FrameLoader(traj, samples[:2], **kw))
    (nk, nx), = list(FrameLoader(traj, samples[:2], noise=(1e-2, 1e-2), **kw))
    eps = (nk["node_loc"] - ck["node_loc"]).double()
    assert float(eps.abs().max()) > 1e-3
    for t in range(4):
        shift = (nx["targets"][t] - cx["targets"][t]).double()
        assert float((shift - eps).abs().max()) <= 4e-7, t                 # two fp32 roundings of coordinates ≲ 1


# ---------------------------------------------------------------------------------------------------------------------
# GPU: main.py --train_rollout
# ---------------------------------------------------------------------------------------------------------------------

def _water_data(tmp_path):
    data = tmp_path / "data"
    for part, sizes, seed in (("train", [60, 50, 40], 1), ("valid", [45, 35], 2), ("test", [55], 3)):
        (data / part).mkdir(parents=True)
        _water(data / part, sizes, T=14, seed=seed)
    return data


@pytest.mark.gpu
def test_train_rollout_1_gives_the_one_step_gradients(tmp_path):
    """One FrameLoader batch, the same weights and MMD samples: the K = 1 rollout loss's parameter gradients are within
    1e-5 of the one-step path's, relative in the norm over all parameters (the backward kernels' atomic sums round in
    their own order in each run)."""
    import main
    data = _water_data(tmp_path)
    _, cfg = _water_cfg(tmp_path, data)
    d = dev()
    torch.manual_seed(0)
    model = main.get_model(cfg, 1).to(d)
    _, lds = main.frame_loaders(str(data), cfg, 1, 0, d, None, parts=("train",))
    kw, ex = next(iter(lds["train"]))
    one = main.trajectory_loss(cfg, model, 1, False)
    roll = main.trajectory_rollout_loss(cfg, model, 1, False, lds["train"], "water3d", 2.0, 1)
    grads = []
    for loss_of in (one, roll):
        model.zero_grad()
        torch.manual_seed(123)                                          # the same randperm draws
        loss, info = loss_of(kw, ex, 2)
        loss.backward()
        grads.append([p.grad.detach().clone() for p in model.parameters()])
    a, b = (torch.cat([g.double().reshape(-1) for g in gs]) for gs in grads)
    rel = float((a - b).norm() / a.norm())
    worst = max(float((x - y).abs().max() / x.abs().max().clamp(min=1e-30)) for x, y in zip(*grads))
    print(f"--train_rollout 1 vs one-step: parameter gradients {rel:.2e} relative (norm over all parameters), largest "
          f"per-tensor max-relative difference {worst:.2e}")
    assert rel <= 1e-5


def _read_log(out):
    with open(os.path.join(out, "log", "log.json")) as f:
        return json.load(f)


@pytest.mark.gpu
def test_main_fits_nbody_on_three_step_rollouts_and_resumes(tmp_path):
    """N-body files written by distegnn_b200.nbody, --epochs 2 --train_rollout 3 with accumulation_steps 2: best and
    last checkpoints, train.train_rollout in their config, valid/test losses that are the one-step losses of the stored
    weights, the train line marked as a rollout mean; then a resume from last_model.pth to epoch 3."""
    import yaml
    import main
    from distegnn_b200 import nbody
    data = tmp_path / "nbody"
    nbody.generate_dataset(str(data), num_train=12, num_valid=4, num_test=4, length=4100, length_test=4100,
                           n_isolated=100, seed=5)
    with open(os.path.join(ROOT, "config", "nbody_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(frame_0=0, frame_T=10, batch_size=4)
    cfg["train"] = dict(cfg.get("train") or {}, accumulation_steps=2)
    cfg["log"] = dict(cfg.get("log") or {}, log_dir=str(tmp_path / "logs"), test_interval=1)
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    base = [sys.executable, os.path.join(ROOT, "main.py"), "--config_path", str(p), "--trajectory", str(data)]
    r = subprocess.run(base + ["--epochs", "2", "--train_rollout", "3"], capture_output=True, text=True, timeout=900,
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "avg loss" in r.stdout and "(mean over 3 rollout steps)" in r.stdout, r.stdout[-2000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("logs and checkpoints: ")][0]
    out = line.split(": ", 1)[1]
    best, log, c = _read_log(out)
    assert log["epochs"] == [1, 2] and c["train"]["train_rollout"] == 3
    sd_dir = os.path.join(out, "state_dict")
    last = torch.load(os.path.join(sd_dir, "last_model.pth"), map_location="cpu")
    assert os.path.exists(os.path.join(sd_dir, "best_model.pth")) and last["epoch"] == 2
    assert last["config"]["train"]["train_rollout"] == 3
    # the stored valid / test losses: the one-step logged MSE of the stored weights
    d = dev()
    model = main.get_model(c, 1).to(d)
    model.load_state_dict(last["model_state_dict"])
    model.eval()
    loss_of = main.trajectory_loss(c, model, 1, False)
    rate = float(c["data"].get("cutoff_rate", 0.0))
    for part in ("valid", "test"):
        _, lds = main.frame_loaders(str(data), c, 1, 0, d, rate, parts=(part,))
        tot, graphs = 0.0, 0
        with torch.no_grad():
            for kw, ex in lds[part]:
                tot += float(loss_of(kw, ex)[1]["logged"]) * ex["n_graphs"]
                graphs += ex["n_graphs"]
        assert last[f"loss_{part}"] == pytest.approx(tot / graphs, rel=1e-4), part
    r = subprocess.run(base + ["--epochs", "3", "--train_rollout", "3", "--checkpoint",
                               os.path.join(sd_dir, "last_model.pth")], capture_output=True, text=True, timeout=900,
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "resuming after epoch 2" in r.stdout and "train epoch: 3" in r.stdout, r.stdout[-2000:]


@pytest.mark.gpu
def test_main_water_radius_with_train_noise(tmp_path):
    """A Water-3D-style .npz set (radius graph rebuilt every step) with --train_noise: trajectory_run trains on 2-step
    rollouts and evaluates one-step."""
    data = _water_data(tmp_path)
    cfg, _ = _water_cfg(tmp_path, data)
    r = _main(["--config_path", cfg, "--trajectory", str(data), "--train_steps", "3", "--train_rollout", "2",
               "--train_noise", "1e-3,1e-3"])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "train step 3: 2-step rollout mean MSE" in r.stdout and "evaluation over" in r.stdout, r.stdout[-2000:]


@pytest.mark.gpu
def test_two_gpu_train_rollout_under_torchrun():
    """2 ranks (2 GPUs) under torchrun: K = 1 gradients after the rank sum match the DDP one-step path within 1e-5, and
    K = 3 leaves the same parameters on both ranks after an optimiser step (scripts/train_rollout_dist_check.py).
    Skipped with a single GPU."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29561", os.path.join(ROOT, "scripts", "train_rollout_dist_check.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    print(p.stdout[-3000:], p.stderr[-1500:])
    assert p.returncode == 0 and "TRAIN_ROLLOUT_DIST PASS" in p.stdout
