"""main.fit: the reference's epoch loop (utils/train.py:17-289, DESIGN §24).  On the CPU with a torch stand-in model and
list loaders: best selection, early stopping, the evaluation interval, gradient accumulation, the cosine schedule, the
clip condition, the checkpoint and log.json layout, a bitwise resume, two gloo ranks and the CLI's rejections.  On the
device: `main.py --trajectory DIR --epochs E` end to end on Water-3D scenes."""
import json
import math
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.multiprocessing as mp

import main
from tests.test_frames import _water

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT_KEYS = {"epoch", "model_state_dict", "optimizer_state_dict", "scheduler_state_dict", "loss_train", "loss_valid",
             "loss_test", "config"}


# ---- stand-ins ----------------------------------------------------------------------------------------------------
class ListLoader:
    """FrameLoader's interface over a list of (kw, ex) batches: a same-seed shuffle whose `batches()` draws one epoch's
    order, as iterating does; `orders` records the order of every iteration."""

    def __init__(self, items, shuffle=False, seed=0):
        self.items, self.shuffle, self.orders = items, shuffle, []
        self.generator = torch.Generator().manual_seed(seed)

    def __len__(self):
        return len(self.items)

    def batches(self):
        n = len(self.items)
        return torch.randperm(n, generator=self.generator).tolist() if self.shuffle else list(range(n))

    def __iter__(self):
        order = self.batches()
        self.orders.append(order)
        return iter([self.items[i] for i in order])


def _batches(n, seed, graphs=2):
    g = torch.Generator().manual_seed(seed)
    return [({"x": torch.randn(6, 3, generator=g)}, {"y": torch.randn(6, 3, generator=g), "n_graphs": graphs})
            for _ in range(n)]


def _loaders(n_train=5, n_eval=2, seed=0):
    return {"train": ListLoader(_batches(n_train, 1), shuffle=True, seed=seed), "valid": ListLoader(_batches(n_eval, 2)),
            "test": ListLoader(_batches(n_eval, 3, graphs=3))}


def net(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(3, 8), torch.nn.Tanh(), torch.nn.Linear(8, 3))


def mse_loss(model):
    """MSE plus a term on rows drawn from the global generator, as the MMD draws its samples."""
    def loss_of(kw, ex, accumulation_steps):
        pred = model(kw["x"])
        mse = ((pred - ex["y"]) ** 2).mean()
        idx = torch.randperm(pred.shape[0])[:2]
        return (mse + 1e-2 * (pred[idx] ** 2).mean()) / accumulation_steps, {"logged": mse.detach()}
    return loss_of


def scripted(model, valid, test=None):
    """A loss whose logged value on the valid (test) split is valid[k] (test[k]) at the k-th evaluation."""
    calls = {"valid": 0, "test": 0}
    inner = mse_loss(model)

    def loss_of(kw, ex, accumulation_steps):
        loss, info = inner(kw, ex, accumulation_steps)
        tag = ex.get("tag")
        if tag is not None:
            seq = valid if tag == "valid" else (test or valid)
            info = {"logged": torch.tensor(seq[calls[tag]])}
            calls[tag] += 1
        return loss, info
    return loss_of


def _tagged_loaders(n_train=3):
    lds = _loaders(n_train, 1)
    for tag in ("valid", "test"):
        for _, ex in lds[tag].items:
            ex["tag"] = tag
    return lds


def _cfg(tmp_path, **train):
    return {"model": {"model_name": "FastEGNN"}, "data": {"dataset_name": "Fluid113K"},
            "train": dict({"accumulation_steps": 1}, **train), "log": {"log_dir": str(tmp_path), "test_interval": 1}}


def _fit(tmp_path, cfg, epochs, model=None, loaders=None, loss_of=None, opt=None, scheduler=None, start=0, **kw):
    model = model if model is not None else net()
    opt = opt if opt is not None else torch.optim.Adam(model.parameters(), lr=1e-2)
    loaders = loaders if loaders is not None else _loaders()
    loss_of = loss_of if loss_of is not None else mse_loss(model)
    out = str(tmp_path / "run")
    best, log = main.fit(model, opt, scheduler, loaders, loss_of, cfg, epochs, start, out_dir=out, **kw)
    return best, log, out


def _ck(out, which):
    return torch.load(os.path.join(out, "state_dict", f"{which}_model.pth"), weights_only=True)


def _log(out):
    with open(os.path.join(out, "log", "log.json")) as f:
        return json.load(f)


# ---- the loop on the CPU ------------------------------------------------------------------------------------------
def test_best_is_a_strictly_lower_valid_loss(tmp_path):
    model = net()
    best, log, out = _fit(tmp_path, _cfg(tmp_path), 5, model=model, loaders=_tagged_loaders(),
                          loss_of=scripted(model, [3.0, 2.0, 2.0, 1.5, 1.5], [9.0, 8.0, 7.0, 6.0, 5.0]))
    assert best["epoch_index"] == 4 and best["loss_valid"] == 1.5 and best["loss_test"] == 6.0
    assert _ck(out, "best")["epoch"] == 4 and _ck(out, "last")["epoch"] == 5
    assert log["epochs"] == [1, 2, 3, 4, 5] and log["loss"] == [9.0, 8.0, 7.0, 6.0, 5.0]
    model = net()
    best, _, out = _fit(tmp_path, _cfg(tmp_path), 3, model=model, loaders=_tagged_loaders(),
                        loss_of=scripted(model, [3.0, 2.0, 2.0]))
    assert best["epoch_index"] == 2 and _ck(out, "best")["epoch"] == 2 and _ck(out, "best")["loss_valid"] == 2.0


def test_early_stop_fires_at_the_first_eval_epoch_past_n(tmp_path):
    model = net()
    best, log, _ = _fit(tmp_path, _cfg(tmp_path, early_stop=2), 10, model=model, loaders=_tagged_loaders(),
                        loss_of=scripted(model, [3.0, 2.0, 2.5, 2.6, 2.7, 2.8]))
    assert best["epoch_index"] == 2 and best["early_stop"] == 4 and len(log["loss_train"]) == 4
    # interval 2, N = 1: epoch 3 is past N but not an evaluation epoch; the stop waits for epoch 4
    model = net()
    cfg = _cfg(tmp_path, early_stop=1)
    cfg["log"]["test_interval"] = 2
    best, log, _ = _fit(tmp_path, cfg, 10, model=model, loaders=_tagged_loaders(), loss_of=scripted(model, [2.0, 3.0]))
    assert best["epoch_index"] == 2 and best["early_stop"] == 4 and len(log["loss_train"]) == 4
    model = net()                                             # no early_stop: never
    best, log, _ = _fit(tmp_path, _cfg(tmp_path), 6, model=model, loaders=_tagged_loaders(),
                        loss_of=scripted(model, [1.0, 2.0, 3.0, 4.0, 5.0, 6.0]))
    assert "early_stop" not in best and len(log["loss_train"]) == 6


def test_test_interval_is_honoured(tmp_path):
    cfg = _cfg(tmp_path)
    cfg["log"]["test_interval"] = 3
    lds = _loaders()
    best, log, out = _fit(tmp_path, cfg, 7, loaders=lds)
    assert log["epochs"] == [3, 6] and len(log["loss_train"]) == 7 and len(log["loss"]) == 2
    assert len(lds["valid"].orders) == len(lds["test"].orders) == 2 and len(lds["train"].orders) == 7
    assert _ck(out, "last")["epoch"] == 6 and best["epoch_index"] in (3, 6)


def test_epoch_loss_is_graph_weighted(tmp_path):
    lds = _loaders(n_train=3, n_eval=2)
    lds["valid"].items[1][1]["n_graphs"] = 5
    model = net()
    _, log, out = _fit(tmp_path, _cfg(tmp_path), 1, model=model, loaders=lds)
    with torch.no_grad():
        m = [float(((model(kw["x"]) - ex["y"]) ** 2).mean()) for kw, ex in lds["valid"].items]
    assert _ck(out, "last")["loss_valid"] == pytest.approx((2 * m[0] + 5 * m[1]) / 7, rel=1e-12)


def test_accumulation_steps_and_the_dropped_remainder(tmp_path):
    A, n = 2, 5
    model, ref = net(), net()
    lds = _loaders(n_train=n)
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    steps = []
    opt.register_step_pre_hook(lambda *_: steps.append(1))
    _fit(tmp_path, _cfg(tmp_path, accumulation_steps=A), 2, model=model, loaders=lds, opt=opt)
    assert len(steps) == 2 * (n // A)
    # the same by hand: a step after every A-th batch; the fifth batch's gradient is dropped by the next zero_grad
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1)
    loss_of = mse_loss(ref)
    net()                                                      # the global generator as fit found it
    for order in lds["train"].orders:
        ropt.zero_grad()
        for step, i in enumerate(order):
            kw, ex = lds["train"].items[i]
            loss_of(kw, ex, A)[0].backward()
            if (step + 1) % A == 0:
                ropt.step()
                ropt.zero_grad()
        with torch.no_grad():                                  # the evaluation's draws on the global generator
            for tag in ("valid", "test"):
                for kw, ex in lds[tag].items:
                    loss_of(kw, ex, 1)
    for a, b in zip(model.parameters(), ref.parameters()):
        assert torch.equal(a, b)


def test_cosine_schedule_is_cosine_annealing_lr(tmp_path):
    E, n, A, lr = 3, 5, 2, 1e-2
    cfg = _cfg(tmp_path, accumulation_steps=A, scheduler="cosine", learning_rate=lr, weight_decay=1e-12)
    model = net()
    opt, sched = main.optimizer_of(model, cfg, E, n)
    assert isinstance(opt, torch.optim.Adam) and opt.defaults["weight_decay"] == 1e-12
    assert isinstance(sched, torch.optim.lr_scheduler.CosineAnnealingLR)
    assert sched.T_max == E * n // A == 7 and sched.eta_min == 1e-8
    seen = []
    opt.register_step_pre_hook(lambda o, *_: seen.append(o.param_groups[0]["lr"]))
    _fit(tmp_path, cfg, E, model=model, loaders=_loaders(n_train=n), opt=opt, scheduler=sched)
    want = [1e-8 + (lr - 1e-8) * (1 + math.cos(math.pi * t / 7)) / 2 for t in range(E * (n // A))]
    assert seen == pytest.approx(want, rel=1e-12, abs=1e-15)
    for value in ("None", None, "step"):
        assert main.optimizer_of(net(), _cfg(tmp_path, scheduler=value), E, n)[1] is None


def test_clip_runs_exactly_under_the_reference_condition(tmp_path, monkeypatch):
    def cfg(name, model="FastEGNN"):
        c = _cfg(tmp_path)
        c["data"]["dataset_name"], c["model"]["model_name"] = name, model
        return c
    assert main.reference_clips(cfg("LargeFluid"), 1) and main.reference_clips(cfg("Fluid113K"), 2)
    assert not main.reference_clips(cfg("Fluid113K"), 1) and not main.reference_clips(cfg("largefluid"), 1)
    assert not main.reference_clips(cfg("LargeFluid", "FastRF"), 1) and not main.reference_clips(cfg("Water3D"), 1)
    calls = []
    monkeypatch.setattr(torch.nn.utils, "clip_grad_norm_", lambda p, max_norm: calls.append(max_norm))
    _fit(tmp_path, cfg("Fluid113K"), 2)
    assert calls == []
    _fit(tmp_path, cfg("LargeFluid"), 2)
    assert calls == [0.3] * 10


def test_checkpoints_and_log_json_have_the_reference_layout(tmp_path):
    cfg = _cfg(tmp_path, early_stop=50)
    model = net()
    best, log, out = _fit(tmp_path, cfg, 3, model=model)
    for which in ("best", "last"):
        ck = _ck(out, which)
        assert set(ck) == CKPT_KEYS and ck["scheduler_state_dict"] is None and ck["config"] == cfg
        assert list(ck["model_state_dict"]) == list(model.state_dict())
        assert set(ck["optimizer_state_dict"]) == {"state", "param_groups"}
    assert _ck(out, "last")["epoch"] == 3
    for k, v in _ck(out, "last")["model_state_dict"].items():
        assert torch.equal(v, model.state_dict()[k])
    b, lg, c = _log(out)
    assert set(b) == {"epoch_index", "loss_valid", "loss_test", "loss_train", "time_cost"} and b["time_cost"] > 0
    assert set(lg) == {"epochs", "loss", "loss_train"} and lg == log and c == cfg
    assert {k: v for k, v in b.items() if k != "time_cost"} == {k: v for k, v in best.items() if k != "time_cost"}


def test_resume_is_bitwise(tmp_path):
    cfg = _cfg(tmp_path, accumulation_steps=2, scheduler="cosine", learning_rate=1e-2)

    def run(epochs, model, start=0, state=None):
        lds = _loaders(n_train=5, seed=4)
        opt, sched = main.optimizer_of(model, cfg, 4, len(lds["train"]))
        if state is not None:
            model.load_state_dict(state["model_state_dict"])
            opt.load_state_dict(state["optimizer_state_dict"])
            sched.load_state_dict(state["scheduler_state_dict"])
        _, _, out = _fit(tmp_path / f"{start}_{epochs}", cfg, epochs, model=model, loaders=lds, opt=opt,
                         scheduler=sched, start=start)
        return opt, sched, lds["train"].orders, out

    straight = net(1)
    torch.manual_seed(7)                                   # the stand-in's draws, as the MMD's, use the global generator
    opt_a, sched_a, orders_a, _ = run(4, straight)
    first, resumed = net(1), net(2)                        # both built before the runs: construction draws
    torch.manual_seed(7)
    _, _, orders_b, out = run(2, first)
    opt_b, sched_b, orders_c, _ = run(4, resumed, start=2, state=_ck(out, "last"))
    for a, b in zip(straight.parameters(), resumed.parameters()):
        assert torch.equal(a, b)
    sa, sb = opt_a.state_dict(), opt_b.state_dict()
    for k in sa["state"]:
        for name in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sa["state"][k][name], sb["state"][k][name]), (k, name)
    assert opt_a.param_groups[0]["lr"] == opt_b.param_groups[0]["lr"] and sched_a.last_epoch == sched_b.last_epoch == 8
    assert orders_a == orders_b + orders_c and len(orders_c) == 2


def _gloo_rank(rank, world, port, root, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        model = net()
        # rank 0's valid loss stops improving after epoch 2; rank 1's keeps improving
        seq = [3.0, 2.0, 2.5, 2.6, 2.7, 2.8, 2.9, 3.0] if rank == 0 else [8.0, 7.0, 6.0, 5.0, 4.0, 3.0, 2.0, 1.0]
        cfg = {"model": {"model_name": "FastEGNN"}, "data": {"dataset_name": "Fluid113K"},
               "train": {"early_stop": 2}, "log": {"test_interval": 1}}
        lds = _tagged_loaders()
        opt = torch.optim.Adam(model.parameters(), lr=1e-2)
        best, log = main.fit(model, opt, None, lds, scripted(model, seq), cfg, 8, world_size=world, rank=rank,
                             out_dir=os.path.join(root, f"rank{rank}"))
        q.put((rank, len(lds["train"].orders), best, log))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_stop_at_rank_0s_epoch_and_only_rank_0_writes(tmp_path):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_rank, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    [p.start() for p in procs]
    res = dict((r, rest) for r, *rest in [q.get(timeout=120) for _ in procs])
    [p.join(timeout=60) for p in procs]
    assert res[0][0] == res[1][0] == 4
    assert res[0][1]["early_stop"] == 4 and res[1][1] is None and res[1][2] is None
    assert os.path.exists(tmp_path / "rank0" / "state_dict" / "best_model.pth")
    assert not os.path.exists(tmp_path / "rank1")


def test_checkpoint_loads_into_fastegnn_and_the_reference_module(tmp_path):
    from distegnn_b200 import FastEGNN
    kw = dict(node_feat_nf=2, node_attr_nf=1, edge_attr_nf=2, hidden_nf=64, virtual_channels=3, world_size=1,
              n_layers=2)
    torch.manual_seed(0)
    model = FastEGNN(**kw)

    def loss_of(_kw, ex, accumulation_steps):                  # no CPU forward: a loss on the weights themselves
        loss = sum((p ** 2).sum() for p in model.parameters()) * 1e-3
        return loss / accumulation_steps, {"logged": loss.detach()}

    _, _, out = _fit(tmp_path, _cfg(tmp_path), 2, model=model, loss_of=loss_of)
    sd = _ck(out, "best")["model_state_dict"]
    fresh = FastEGNN(**kw)
    assert list(sd) == list(fresh.state_dict())
    fresh.load_state_dict(sd)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, model.state_dict()[k]), k
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("the reference module is not installed (oracle/build_ref.py)")
    ref = ref_loader.load_reference()(**kw)
    ref.load_state_dict(sd)                                    # strict: the same keys and shapes


# ---- the CLI -------------------------------------------------------------------------------------------------------
def _main(args, timeout=600, **env):
    return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), *args], capture_output=True, text=True,
                          timeout=timeout, cwd=ROOT, env=dict(os.environ, **env))


def test_main_rejects_bad_epochs_before_cuda_work(tmp_path):
    cfg = os.path.join(ROOT, "config", "largefluid_distegnn.yaml")
    for part in ("train", "valid"):
        (tmp_path / part).mkdir()
        _water(tmp_path / part, [20])
    base = ["--config_path", cfg, "--trajectory", str(tmp_path)]
    for args, msg in ((["--config_path", cfg, "--epochs", "3"], "used with --trajectory"),
                      (base + ["--epochs", "3", "--train_steps", "2"], "used without --train_steps"),
                      (base + ["--epochs", "0"], ">= 1"), (base + ["--epochs", "-2"], ">= 1"),
                      (base + ["--epochs", "3"], "has no test")):
        r = _main(args, CUDA_VISIBLE_DEVICES="")
        assert r.returncode == 2 and msg in r.stdout and r.stdout.startswith("--epochs"), (args, r.stdout, r.stderr)
        assert "CUDA" not in r.stderr
    (tmp_path / "valid" / "water_0.npz").unlink()
    (tmp_path / "test").mkdir()
    _water(tmp_path / "test", [20])
    r = _main(base + ["--epochs", "3"], CUDA_VISIBLE_DEVICES="")
    assert r.returncode == 2 and "has no valid" in r.stdout and "CUDA" not in r.stderr, r.stdout


def test_main_no_longer_warns_about_early_stop_with_epochs(tmp_path):
    """The warning is printed before the CUDA check, so both runs below get as far as it without a GPU."""
    cfg = os.path.join(ROOT, "config", "largefluid_distegnn.yaml")
    for part in ("train", "valid", "test"):
        (tmp_path / part).mkdir()
        _water(tmp_path / part, [20])
    base = ["--config_path", cfg, "--trajectory", str(tmp_path), "--early_stop", "5"]
    r = _main(base + ["--epochs", "2", "--wandb"], CUDA_VISIBLE_DEVICES="")
    assert "--wandb accepted" in r.stdout and "--early_stop" not in r.stdout, r.stdout
    r = _main(base + ["--train_steps", "2"], CUDA_VISIBLE_DEVICES="")
    assert "--early_stop accepted" in r.stdout, r.stdout


# ---- on the device ------------------------------------------------------------------------------------------------
def _water_run(tmp_path, **train):
    import yaml
    data = tmp_path / "data"
    for part, sizes, seed in (("train", [60, 50, 40], 1), ("valid", [45, 35], 2), ("test", [55], 3)):
        (data / part).mkdir(parents=True)
        _water(data / part, sizes, seed=seed)
    with open(os.path.join(ROOT, "config", "largefluid_distegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"].update(node_feat_nf=2, node_attr_nf=1)
    cfg["data"].update(dataset_name="Water3D", inner_radius=0.3, max_samples=8, split_mode="random", delta_t=2,
                       batch_size=2)
    cfg["train"] = dict(accumulation_steps=2, **train)
    cfg["log"] = {"log_dir": str(tmp_path / "logs"), "test_interval": 1}
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    return str(data), str(p), cfg


def _run_dir(tmp_path, stdout):
    line = [ln for ln in stdout.splitlines() if ln.startswith("logs and checkpoints: ")]
    assert len(line) == 1, stdout
    d = line[0].split(": ", 1)[1]
    assert d.startswith(str(tmp_path / "logs"))
    return d


def _split_loss(cfg, data, sd, part):
    """Σ logged · graphs / Σ graphs over `part` with the weights `sd`, recomputed through FrameLoader + train_loss."""
    dev = torch.device("cuda", 0)
    model = main.get_model(cfg, 1).to(dev)
    model.load_state_dict(sd)
    model.eval()
    loss_of = main.trajectory_loss(cfg, model, 1, False)
    _, lds = main.frame_loaders(data, cfg, 1, 0, dev, None, parts=(part,))
    tot, graphs = 0.0, 0
    with torch.no_grad():
        for kw, ex in lds[part]:
            tot += float(loss_of(kw, ex)[1]["logged"]) * ex["n_graphs"]
            graphs += ex["n_graphs"]
    return tot / graphs


@pytest.mark.gpu
def test_main_trains_three_epochs_and_writes_the_reference_checkpoints(tmp_path):
    from distegnn_b200 import FastEGNN
    data, cfg_path, cfg = _water_run(tmp_path, scheduler="cosine")
    r = _main(["--config_path", cfg_path, "--trajectory", data, "--epochs", "3", "--rollout_steps", "2"])
    assert r.returncode == 0, r.stderr[-3000:]
    out = _run_dir(tmp_path, r.stdout)
    assert os.path.basename(out).startswith("Water3D_random_FastEGNN_0.075_0.3_1_5_")
    best, log, c = _log(out)
    assert log["epochs"] == [1, 2, 3] and len(log["loss_train"]) == 3 and c["log"]["exp_name"] == os.path.basename(out)
    ck, last = _ck(out, "best"), _ck(out, "last")
    assert set(ck) == set(last) == CKPT_KEYS and last["epoch"] == 3 and ck["epoch"] == best["epoch_index"]
    _, lds = main.frame_loaders(data, c, 1, 0, torch.device("cuda", 0), None, parts=("train",))
    assert ck["scheduler_state_dict"]["T_max"] == 3 * len(lds["train"]) // 2
    m = cfg["model"]
    fresh = FastEGNN(node_feat_nf=2, node_attr_nf=1, edge_attr_nf=m["edge_attr_nf"], hidden_nf=m["hidden_nf"],
                     virtual_channels=m["virtual_channels"], world_size=1, n_layers=m["n_layers"])
    assert list(ck["model_state_dict"]) == list(fresh.state_dict())
    fresh.load_state_dict(ck["model_state_dict"])
    # the stored losses are the logged MSE (no MMD draw in it) of the stored weights
    for part in ("valid", "test"):
        want = _split_loss(c, data, ck["model_state_dict"], part)
        assert ck[f"loss_{part}"] == pytest.approx(want, rel=1e-4), part
    assert "rollout step 2" in r.stdout and "best model restored" in r.stdout, r.stdout


@pytest.mark.gpu
def test_best_epoch_is_the_argmin_of_the_valid_losses(tmp_path):
    data, _, cfg = _water_run(tmp_path)
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = main.get_model(cfg, 1).to(dev)
    _, lds = main.frame_loaders(data, cfg, 1, 0, dev, None, parts=("train", "valid", "test"))
    inner = main.trajectory_loss(cfg, model, 1, False)
    opt, sched = main.optimizer_of(model, cfg, 4, len(lds["train"]))
    seen, vals = [], []

    def recording(kw, ex, accumulation_steps):              # every batch's logged MSE, in the loop's order
        loss, info = inner(kw, ex, accumulation_steps)
        seen.append((model.training, ex["n_graphs"], info["logged"]))
        return loss, info

    best, log = main.fit(model, opt, sched, lds, recording, cfg, 4, out_dir=str(tmp_path / "run"))
    nv, nt, ntr = len(lds["valid"]), len(lds["test"]), len(lds["train"])
    per_epoch = ntr + nv + nt
    assert len(seen) == 4 * per_epoch
    for e in range(4):
        rows = seen[e * per_epoch + ntr:e * per_epoch + ntr + nv]
        assert not any(t for t, _, _ in rows)
        vals.append(sum(float(v) * g for _, g, v in rows) / sum(g for _, g, _ in rows))
    assert best["epoch_index"] == 1 + min(range(4), key=lambda e: vals[e])
    assert _log(str(tmp_path / "run"))[0]["epoch_index"] == best["epoch_index"]
    assert best["loss_valid"] == pytest.approx(min(vals), rel=1e-12)


@pytest.mark.gpu
def test_resume_on_the_device_continues_the_run(tmp_path):
    data, cfg_path, cfg = _water_run(tmp_path)
    straight = _main(["--config_path", cfg_path, "--trajectory", data, "--epochs", "4"])
    assert straight.returncode == 0, straight.stderr[-3000:]
    first = _main(["--config_path", cfg_path, "--trajectory", data, "--epochs", "2"])
    assert first.returncode == 0, first.stderr[-3000:]
    ck = os.path.join(_run_dir(tmp_path, first.stdout), "state_dict", "last_model.pth")
    second = _main(["--config_path", cfg_path, "--trajectory", data, "--epochs", "4", "--checkpoint", ck])
    assert second.returncode == 0, second.stderr[-3000:]
    assert "resuming after epoch 2" in second.stdout, second.stdout
    a, b = _ck(_run_dir(tmp_path, straight.stdout), "last"), _ck(_run_dir(tmp_path, second.stdout), "last")
    assert a["epoch"] == b["epoch"] == 4
    assert _log(_run_dir(tmp_path, second.stdout))[1]["epochs"] == [3, 4]
    dev = torch.device("cuda", 0)
    _, lds = main.frame_loaders(data, cfg, 1, 0, dev, None, parts=("train",))
    steps = lambda c: {float(s["step"]) for s in c["optimizer_state_dict"]["state"].values()}
    assert steps(a) == steps(b) == {4 * (len(lds["train"]) // 2)}    # accumulation 2
    for k, v in a["model_state_dict"].items():             # the backward's float atomics: not bitwise
        w = b["model_state_dict"][k]
        assert float((v - w).abs().max()) <= 1e-4 * max(1.0, float(v.abs().max())), k
    # per-epoch train batches: the resumed loader continues the uninterrupted order
    _, lds = main.frame_loaders(data, cfg, 1, 0, dev, None, parts=("train",))
    orders = [lds["train"].batches() for _ in range(4)]
    _, lds = main.frame_loaders(data, cfg, 1, 0, dev, None, parts=("train",))
    for _ in range(2):
        lds["train"].batches()
    assert [lds["train"].batches() for _ in range(2)] == orders[2:] and orders[2:] != orders[:2]


@pytest.mark.gpu
def test_early_stop_ends_the_run_once_valid_stops_improving(tmp_path):
    data, cfg_path, _ = _water_run(tmp_path)
    r = _main(["--config_path", cfg_path, "--trajectory", data, "--epochs", "6", "--early_stop", "1", "--lr", "10"])
    assert r.returncode == 0, r.stderr[-3000:]
    best, log, c = _log(_run_dir(tmp_path, r.stdout))
    assert c["train"]["early_stop"] == 1 and c["train"]["learning_rate"] == 10
    assert best["early_stop"] == best["epoch_index"] + 1 < 6
    assert len(log["loss_train"]) == best["early_stop"] and f"Early stopped! Epoch: {best['early_stop']}" in r.stdout
