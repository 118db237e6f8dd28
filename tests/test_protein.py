"""The protein dataset (distegnn_b200/protein.py, the `protein` recipe of distegnn_b200/frames.py, main.py's protein
path): DCD and PSF readers against files written here per the CHARMM formats, the backbone selection, the sample
ranges, and on the device FrameLoader's protein batches against the reference's lines restated in
oracle/protein_oracle.py."""
import math
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

import main
from distegnn_b200.frames import PROTEIN_SPLITS, FrameLoader, check_samples, sample_list
from distegnn_b200.protein import (AtomSelection, backbone_index, cubic_edge, find_files, load_protein, read_dcd,
                                   read_psf)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_FULL = PROTEIN_SPLITS["test"][1] - 1 + 15 + 1          # the last test sample (4170) and its target at delta_t = 15


# ---- fixtures: files written per the formats ------------------------------------------------------------------------
def write_dcd(path, pos, order="<", cells=None, namnf=0, dim4=False, wide=False, nset=None, cut=0,
              title=("REMARKS written by tests/test_protein.py", "REMARKS second title line")):
    """A CHARMM-format DCD (ICNTRL[19] = 24): every record framed by its length (4 or, `wide`, 8 bytes), in `order`."""
    def rec(payload):
        m = struct.pack(order + ("q" if wide else "i"), len(payload))
        return m + payload + m
    T, n, _ = pos.shape
    icntrl = [T if nset is None else nset, 1, 1, T, 0, 0, 0, 0, namnf]
    tail = [1 if cells is not None else 0, 1 if dim4 else 0, 0, 0, 0, 0, 0, 0, 0, 24]
    parts = [rec(b"CORD" + struct.pack(order + "9i", *icntrl) + struct.pack(order + "f", 0.0489) +
                 struct.pack(order + "10i", *tail)),
             rec(struct.pack(order + "i", len(title)) + b"".join(t.encode().ljust(80) for t in title)),
             rec(struct.pack(order + "i", n))]
    if namnf:
        parts.append(rec(struct.pack(order + f"{n - namnf}i", *range(1, n - namnf + 1))))
    for t in range(T):
        if cells is not None:
            parts.append(rec(struct.pack(order + "6d", *cells[t])))
        for c in range(3):
            parts.append(rec(struct.pack(order + f"{n}f", *pos[t, :, c].tolist())))
        if dim4:
            parts.append(rec(struct.pack(order + f"{n}f", *([0.0] * n))))
    data = b"".join(parts)
    with open(path, "wb") as f:
        f.write(data[:len(data) - cut])
    return str(path)


# (resname, atom names) of the fixture: a chain with HSD and HSE, a C-terminus with OT1/OT2, a ligand whose atoms are
# named CA and C, a water and an ion
RESIDUES = [("MET", ["N", "HT1", "CA", "CB", "C", "O"]), ("HSD", ["N", "HN", "CA", "CB", "ND1", "C", "O"]),
            ("GLY", ["N", "HN", "CA", "HA1", "C", "O"]), ("HSE", ["N", "HN", "CA", "CB", "NE2", "C", "O"]),
            ("ALA", ["N", "HN", "CA", "CB", "C", "O"]), ("LYS", ["N", "HN", "CA", "CB", "NZ", "C", "OT1", "OT2"]),
            ("LIG", ["CA", "C", "O1"]), ("TIP3", ["OH2", "H1", "H2"]), ("SOD", ["SOD"])]


def fixture_atoms(repeat=1):
    """(names, resnames, resids) of RESIDUES' protein part `repeat` times, then the rest, and the backbone indices."""
    prot, rest = RESIDUES[:6], RESIDUES[6:]
    names, resnames, resids, want = [], [], [], []
    resid = 0
    for k in range(repeat):
        for j, (rn, atoms) in enumerate(prot):
            if k < repeat - 1 and j == len(prot) - 1:        # a C-terminus only at the end of the chain
                atoms = [a for a in atoms if a != "OT2"]
                atoms = [a if a != "OT1" else "O" for a in atoms]
            resid += 1
            for a in atoms:
                if a in ("N", "CA", "C", "O"):
                    want.append(len(names))
                names.append(a), resnames.append(rn), resids.append(resid)
    for rn, atoms in rest:
        resid += 1
        for a in atoms:
            names.append(a), resnames.append(rn), resids.append(resid)
    return names, resnames, resids, np.array(want, dtype=np.int64)


def write_psf(path, names, resnames, resids, charges, ext=False):
    """A CHARMM PSF: the standard (I8,1X,A4,...) or the EXT (I10,1X,A8,...) atom line layout."""
    lines = ["PSF EXT CMAP" if ext else "PSF", "", "       2 !NTITLE", "* protein fixture", "* second line", "",
             f"{len(names):8d} !NATOM"]
    for k, (a, rn, ri, q) in enumerate(zip(names, resnames, resids, charges)):
        seg = "PROT"
        if ext:
            lines.append(f"{k + 1:10d} {seg:<8s} {ri:<8d} {rn:<8s} {a:<8s} {a[:6]:<6s} {q:14.6f}{12.011:14.4f}{0:8d}")
        else:
            lines.append(f"{k + 1:8d} {seg:<4s} {ri:<4d} {rn:<4s} {a:<4s} {a[:4]:<4s} {q:14.6f}{12.011:14.4f}{0:12d}")
    lines += ["", f"{0:8d} !NBOND: bonds", ""]
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return str(path)


def spread_positions(n, T, seed=0, r=10.0, gap=0.2, side=30.0, jitter=0.01):
    """[T, n, 3] float32 Å: a fixed configuration with no pair distance in [r − gap, r + gap], each frame with its own
    N(0, jitter²) displacement.  A pair's distance moves by at most the sum of its two displacements, which stays
    below gap unless one exceeds 10·jitter: no frame has a pair near r."""
    rng = np.random.default_rng(seed)
    base = np.zeros((0, 3))
    while len(base) < n:
        c = rng.random(3) * side
        if (np.abs(np.linalg.norm(base - c, axis=1) - r) > gap).all():
            base = np.concatenate([base, c[None]])
    return (base[None] + rng.normal(0, jitter, (T, n, 3))).astype(np.float32)


def write_protein(d, T=T_FULL, repeat=1, seed=0, cells=None, **kw):
    """`d`/prot.psf and `d`/prot.dcd; returns (positions [T, N, 3], charges [N], backbone indices)."""
    names, resnames, resids, want = fixture_atoms(repeat)
    rng = np.random.default_rng(seed + 1)
    charges = np.round(rng.uniform(-0.6, 0.6, len(names)), 2)
    pos = spread_positions(len(names), T, seed=seed)
    os.makedirs(d, exist_ok=True)
    write_psf(os.path.join(d, "prot.psf"), names, resnames, resids, charges)
    write_dcd(os.path.join(d, "prot.dcd"), pos, cells=cells, **kw)
    return pos, charges, want


# ---- DCD -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ["<", ">"])
@pytest.mark.parametrize("with_cell", [False, True])
@pytest.mark.parametrize("T", [1, 5])
def test_dcd_returns_what_was_written(tmp_path, order, with_cell, T):
    rng = np.random.default_rng(T)
    n = 7
    pos = rng.normal(0, 20, (T, n, 3)).astype(np.float32)
    cells = rng.uniform(30, 60, (T, 6)) if with_cell else None
    d = read_dcd(write_dcd(tmp_path / "a.dcd", pos, order=order, cells=cells))
    assert (d.n_atoms, d.n_frames, d.nset, d.istart, d.nsavc) == (n, T, T, 1, 1)
    assert d.title == ["REMARKS written by tests/test_protein.py", "REMARKS second title line"]
    assert d.positions.shape == (T, n, 3) and np.array_equal(np.asarray(d.positions), pos)
    assert np.array_equal(d.positions[T - 1], pos[T - 1])
    assert np.shares_memory(d.positions, d.memmap) and not d.positions.flags.writeable     # a view, no copy
    if with_cell:
        assert np.array_equal(np.asarray(d.unit_cell), cells)
    else:
        assert d.unit_cell is None


def test_dcd_frame_count_is_the_file_size(tmp_path):
    pos = np.ones((4, 3, 3), np.float32)
    assert read_dcd(write_dcd(tmp_path / "a.dcd", pos, nset=0)).n_frames == 4


def test_dcd_rejects_what_it_cannot_read(tmp_path):
    pos = np.arange(2 * 5 * 3, dtype=np.float32).reshape(2, 5, 3)
    cases = [(dict(namnf=2), "fixed atoms"), (dict(dim4=True), "4-D"), (dict(wide=True), "8-byte record markers"),
             (dict(wide=True, order=">"), "8-byte record markers"), (dict(cut=6), "truncated: the last frame"),
             (dict(nset=3), "truncated: the header counts 3 frames")]
    for k, (kw, msg) in enumerate(cases):
        with pytest.raises(ValueError, match=msg):
            read_dcd(write_dcd(tmp_path / f"bad{k}.dcd", pos, **kw))
    (tmp_path / "junk.dcd").write_bytes(b"\x00" * 200)
    with pytest.raises(ValueError, match="not a DCD"):
        read_dcd(str(tmp_path / "junk.dcd"))


def test_cubic_edge(tmp_path):
    pos = np.zeros((3, 2, 3), np.float32)
    cube = [[40.0, 90.0, 40.0, 90.0, 90.0, 40.0]] * 3
    assert cubic_edge(read_dcd(write_dcd(tmp_path / "c.dcd", pos, cells=np.array(cube))), range(3)) == 40.0
    cosines = [[40.0, 0.0, 40.0, 0.0, 0.0, 40.0]] * 3                     # newer CHARMM writes the angles' cosines
    assert cubic_edge(read_dcd(write_dcd(tmp_path / "k.dcd", pos, cells=np.array(cosines))), range(3)) == 40.0
    for k, cells in enumerate(([[40.0, 90.0, 41.0, 90.0, 90.0, 40.0]] * 3,
                               [[40.0, 60.0, 40.0, 90.0, 90.0, 40.0]] * 3,
                               cube[:2] + [[41.0, 90.0, 41.0, 90.0, 90.0, 41.0]])):
        with pytest.raises(ValueError, match="not one cubic cell"):
            cubic_edge(read_dcd(write_dcd(tmp_path / f"n{k}.dcd", pos, cells=np.array(cells))), range(3))
    with pytest.raises(ValueError, match="no unit cell"):
        cubic_edge(read_dcd(write_dcd(tmp_path / "none.dcd", pos)), range(3))


# ---- PSF and the selection --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ext", [False, True])
def test_psf_layouts_and_the_backbone_selection(tmp_path, ext):
    names, resnames, resids, want = fixture_atoms()
    charges = np.linspace(-0.9, 0.9, len(names)).round(4)
    psf = read_psf(write_psf(tmp_path / "a.psf", names, resnames, resids, charges, ext=ext))
    assert psf.names.tolist() == names and psf.resnames.tolist() == resnames
    assert np.array_equal(psf.charges, charges)
    ix = backbone_index(psf)
    # N CA C O of MET, HSD, GLY, HSE, ALA; N CA C of the C-terminal LYS (OT1/OT2 are not O); not the ligand's CA, C
    assert ix.tolist() == [0, 2, 4, 5, 6, 8, 11, 12, 13, 15, 17, 18, 19, 21, 24, 25, 26, 28, 30, 31, 32, 34, 37]
    assert ix.tolist() == want.tolist()


def test_psf_rejects_malformed_files(tmp_path):
    (tmp_path / "a.psf").write_text("not a psf\n")
    with pytest.raises(ValueError, match="not a PSF"):
        read_psf(str(tmp_path / "a.psf"))
    (tmp_path / "b.psf").write_text("PSF\n\n       3 !NATOM\n       1 P 1 ALA N N -0.3 14.0 0\n")
    with pytest.raises(ValueError, match="counts 3 atoms"):
        read_psf(str(tmp_path / "b.psf"))
    (tmp_path / "c.psf").write_text("PSF\n\n       1 !NATOM\n       1 P 1 ALA N N\n")
    with pytest.raises(ValueError, match="malformed atom line"):
        read_psf(str(tmp_path / "c.psf"))


def test_load_protein_selects_lazily_and_takes_the_charges(tmp_path):
    pos, charges, want = write_protein(str(tmp_path), T=6)
    files = find_files(str(tmp_path))
    assert [os.path.basename(f) for f in files] == ["prot.psf", "prot.dcd"]
    bb = load_protein(files).scenes[0]
    assert isinstance(bb.position, AtomSelection) and bb.position.shape == (6, len(want), 3)
    assert np.array_equal(bb.position[3], pos[3][want]) and np.array_equal(np.asarray(bb.position), pos[:, want])
    assert np.array_equal(bb.static[:, 0], charges[want].astype(np.float32))
    every = load_protein(files, backbone=False).scenes[0]
    assert isinstance(every.position, np.ndarray) and not every.position.flags.owndata     # the DCD's view
    assert np.array_equal(np.asarray(every.position), pos) and np.array_equal(every.static[:, 0],
                                                                             charges.astype(np.float32))
    # an .npz scene with position and charges, for converted data
    z = tmp_path / "npz"
    z.mkdir()
    np.savez(z / "adk.npz", position=pos[:, want], charges=charges[want])
    sc = load_protein(find_files(str(z))).scenes[0]
    assert np.array_equal(np.asarray(sc.position), pos[:, want]) and np.array_equal(bb.static, sc.static)
    # the PSF and the DCD must agree; a directory holds one trajectory
    write_dcd(tmp_path / "prot.dcd", pos[:, :5])
    with pytest.raises(ValueError, match="atoms"):
        load_protein(files)
    write_dcd(tmp_path / "other.dcd", pos)
    with pytest.raises(ValueError, match="2 .dcd files"):
        find_files(str(tmp_path))
    assert find_files(str(tmp_path / "nothing")) == []


# ---- samples ---------------------------------------------------------------------------------------------------------
def test_sample_ranges_and_their_frames(tmp_path):
    write_protein(str(tmp_path))
    traj = load_protein(find_files(str(tmp_path)))
    got = {p: sample_list(traj, delta_t=15, split=p, max_samples=10) for p in ("train", "valid", "test")}
    assert [len(got[p]) for p in ("train", "valid", "test")] == [2481, 827, 863]            # max_samples ignored
    assert got["train"][0] == (0, 0) and got["train"][-1] == (0, 2480)
    assert got["valid"][0] == (0, 2481) and got["valid"][-1] == (0, 3307)
    assert got["test"][0] == (0, 3308) and got["test"][-1] == (0, 4170)
    assert traj.scenes[0].n_frames == 4186                # frame 4170 + 15 = 4185, the last one the test split reads
    with pytest.raises(ValueError, match="split="):
        sample_list(traj, delta_t=15)
    with pytest.raises(ValueError, match=r"sample \(0, 4170\)"):
        sample_list(traj, delta_t=16, split="test")


def test_a_short_trajectory_is_rejected_naming_the_sample(tmp_path):
    write_protein(str(tmp_path), T=4000)
    traj = load_protein(find_files(str(tmp_path)))
    assert len(sample_list(traj, delta_t=15, split="train")) == 2481
    with pytest.raises(ValueError, match=r"sample \(0, 3985\): frames 3985..4000 fall outside scene 0 of 4000"):
        sample_list(traj, delta_t=15, split="test")
    with pytest.raises(ValueError, match=r"sample \(0, 3308\)"):
        check_samples(traj, [(0, 3308)], delta_t=700)


# ---- main.py without a GPU -------------------------------------------------------------------------------------------
def _cfg(tmp_path, **data):
    with open(os.path.join(ROOT, "config", "protein_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"].update(data)
    cfg["log"]["log_dir"] = str(tmp_path / "logs")
    p = tmp_path / "cfg.yaml"
    with open(p, "w") as f:
        yaml.safe_dump(cfg, f)
    return str(p), cfg


def _main(args, **env):
    return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), *args], capture_output=True, text=True,
                          timeout=900, cwd=ROOT, env=dict(os.environ, **env))


def test_the_config_picks_the_protein_recipe():
    with open(os.path.join(ROOT, "config", "protein_fastegnn.yaml")) as f:
        cfg = yaml.safe_load(f)
    assert main.recipe_of_config(cfg) == ("protein", 0, 15)
    assert main.recipe_of_config({"data": {"dataset_name": "Protein_AdK"}})[0] == "protein"
    assert main.recipe_of_config({"data": {"dataset_name": "mystery"}})[0] == "largefluid"     # unchanged
    d = cfg["data"]
    assert (d["radius"], d["batch_size"], d["cutoff_rate"], cfg["model"]["virtual_channels"]) == (10, 5, 0.0, 3)
    assert cfg["train"]["mmd"] == {"sigma": 1.0, "weight": 0.5, "samples": 3}
    assert (cfg["model"]["node_feat_nf"], cfg["model"]["node_attr_nf"]) == (2, 0)


def test_main_exits_2_before_cuda_work(tmp_path):
    cfg, _ = _cfg(tmp_path)
    data = tmp_path / "data"
    data.mkdir()
    base = ["--config_path", cfg, "--trajectory", str(data), "--epochs", "2"]
    r = _main(base, CUDA_VISIBLE_DEVICES="")                                       # neither file
    assert r.returncode == 2 and "no protein trajectory" in r.stdout and "CUDA" not in r.stderr, (r.stdout, r.stderr)
    write_protein(str(data), T=4000)
    os.remove(data / "prot.psf")                                                   # a DCD without its PSF
    r = _main(base, CUDA_VISIBLE_DEVICES="")
    assert r.returncode == 2 and "no protein trajectory" in r.stdout, r.stdout
    write_protein(str(data), T=4000)                                              # too short for the test split
    r = _main(base, CUDA_VISIBLE_DEVICES="")
    assert r.returncode == 2 and "sample (0, 3985)" in r.stdout and "CUDA" not in r.stderr, (r.stdout, r.stderr)
    os.remove(data / "prot.dcd")                                                   # a PSF without its DCD
    r = _main(base, CUDA_VISIBLE_DEVICES="")
    assert r.returncode == 2 and "no protein trajectory" in r.stdout, r.stdout


def test_main_rejects_test_trans_without_a_cubic_cell(tmp_path):
    data = tmp_path / "data"
    write_protein(str(data))
    cfg, c = _cfg(tmp_path, test_trans=True)
    r = _main(["--config_path", cfg, "--trajectory", str(data), "--epochs", "2"], CUDA_VISIBLE_DEVICES="")
    assert r.returncode == 2 and "test_trans needs a cubic unit cell" in r.stdout and "no unit cell" in r.stdout, \
        r.stdout
    assert "CUDA" not in r.stderr
    cells = np.tile([50.0, 90.0, 50.0, 90.0, 90.0, 50.0], (T_FULL, 1))
    cells[3500, 2] = 51.0                                                          # one test frame is not cubic
    write_protein(str(data), cells=cells)
    r = _main(["--config_path", cfg, "--trajectory", str(data), "--epochs", "2"], CUDA_VISIBLE_DEVICES="")
    assert r.returncode == 2 and "not one cubic cell" in r.stdout, r.stdout
    cells[3500, 2] = 50.0
    write_protein(str(data), cells=cells)
    assert main.protein_test_transform(str(data), c) == dict(translate=25.0)
    c["data"]["test_rot"] = True
    assert main.protein_test_transform(str(data), c) == dict(rotate=True, translate=25.0)


# ---- on the device -----------------------------------------------------------------------------------------------------
def _ulps(a, b):
    ia, ib = a.contiguous().view(torch.int32).long(), b.contiguous().view(torch.int32).long()
    assert bool(((a >= 0) == (b >= 0)).all())
    return int((ia - ib).abs().max()) if a.numel() else 0


@pytest.mark.gpu
@pytest.mark.parametrize("backbone,rate", [(True, 0.0), (False, 0.0), (True, 0.5)])
def test_batches_match_the_reference_lines(tmp_path, backbone, rate):
    from oracle import protein_oracle as po
    pos, charges, want = write_protein(str(tmp_path), repeat=3)
    ix = want if backbone else np.arange(pos.shape[1])
    traj = load_protein(find_files(str(tmp_path)), backbone=backbone)
    r, dt = 10.0, 15
    samples = sample_list(traj, delta_t=dt, split="test")[-10:]          # the last test samples: frames up to 4185
    ld = FrameLoader(traj, samples, delta_t=dt, radius=r, batch_size=5, device=torch.device("cuda:0"),
                     cutoff_rate=rate)
    n = 0
    for b0, (kw, ex) in enumerate(ld):
        assert ex["node_counts"] == [len(ix)] * 5
        E = int(kw["edge_index"].rowptr[-1])
        row, col = kw["edge_index"].rows()[:E].long().cpu(), kw["edge_index"].col[:E].long().cpu()
        for b in range(5):
            t = samples[b0 * 5 + b][1]
            p64 = pos[t][ix].astype(np.float64)
            dist = np.linalg.norm(p64[:, None] - p64[None], axis=-1)
            assert np.abs(dist - r).min() > 1e-4 * r                   # no pair near r: the edge sets must be equal
            w = po.sample(pos, charges, ix, t, dt, r, rate)
            lo, hi = ex["ptr"][b], ex["ptr"][b + 1]
            assert torch.equal(kw["node_loc"][lo:hi].cpu(), w["pos"])
            assert torch.equal(kw["node_vel"][lo:hi].cpu(), w["vel"])
            assert torch.equal(kw["node_attr"][lo:hi].cpu(), w["attr"])
            assert torch.equal(ex["target"][lo:hi].cpu(), w["target"])
            assert _ulps(kw["node_feat"][lo:hi].cpu(), w["x"]) <= 1
            whole = torch.from_numpy(p64).mean(0)
            assert float((kw["loc_mean"][b].cpu().double() - whole).abs().max()) <= 1e-6 * float(whole.abs().max())
            m = (row >= lo) & (row < hi)
            mine = set(zip((row[m] - lo).tolist(), (col[m] - lo).tolist()))
            theirs = set(zip(w["edge_index"][0].tolist(), w["edge_index"][1].tolist()))
            if rate == 0:
                assert mine == theirs
            else:                       # kept sets may differ only among edges tied with the longest kept one (§16)
                ei = w["edge_index"]
                thr = float((w["pos"][ei[0]] - w["pos"][ei[1]]).norm(dim=1).max())
                for a, c in mine ^ theirs:
                    assert abs(float((w["pos"][a] - w["pos"][c]).norm()) - thr) <= 1e-6 * thr
                assert len(mine) == len(theirs)
            n += 1
    assert n == 10


def _split_loss(cfg, data, sd, part):
    dev = torch.device("cuda", 0)
    model = main.get_model(cfg, 1).to(dev)
    model.load_state_dict(sd)
    model.eval()
    loss_of = main.trajectory_loss(cfg, model, 1, False)
    _, lds = main.frame_loaders(data, cfg, 1, 0, dev, 0.0, parts=(part,))
    tot, graphs = 0.0, 0
    with torch.no_grad():
        for kw, ex in lds[part]:
            tot += float(loss_of(kw, ex)[1]["logged"]) * ex["n_graphs"]
            graphs += ex["n_graphs"]
    return tot / graphs


@pytest.mark.gpu
def test_main_trains_two_epochs_and_rolls_out(tmp_path):
    data = tmp_path / "data"
    write_protein(str(data), repeat=3)
    cfg_path, cfg = _cfg(tmp_path)
    cfg["log"]["test_interval"] = 1
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)
    r = _main(["--config_path", cfg_path, "--trajectory", str(data), "--epochs", "2", "--rollout_steps", "3"])
    assert r.returncode == 0, r.stderr[-3000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("logs and checkpoints: ")]
    out = line[0].split(": ", 1)[1]
    assert os.path.basename(out).startswith("protein_FastEGNN_10_0.000_3_1_")
    for f in ("state_dict/best_model.pth", "state_dict/last_model.pth", "log/log.json"):
        assert os.path.exists(os.path.join(out, f)), f
    ck = torch.load(os.path.join(out, "state_dict", "best_model.pth"), map_location="cpu")
    want = _split_loss(ck["config"], str(data), ck["model_state_dict"], "valid")
    assert ck["loss_valid"] == pytest.approx(want, rel=1e-4)
    steps = [ln for ln in r.stdout.splitlines() if ln.startswith("[protein] rollout step ")]
    assert len(steps) == 3 and all(math.isfinite(float(s.rsplit("MSE ", 1)[1])) for s in steps), r.stdout


@pytest.mark.gpu
def test_the_rotated_test_split_gives_the_same_loss(tmp_path):
    data = tmp_path / "data"
    cells = np.tile([60.0, 90.0, 60.0, 90.0, 90.0, 60.0], (T_FULL, 1))
    write_protein(str(data), repeat=3, cells=cells)
    _, cfg = _cfg(tmp_path)
    torch.manual_seed(0)
    sd = main.get_model(cfg, 1).state_dict()
    plain = _split_loss(cfg, str(data), sd, "test")
    moved = {}
    for key, extra in (("rot", dict(test_rot=True)), ("rot+trans", dict(test_rot=True, test_trans=True))):
        c = dict(cfg, data=dict(cfg["data"], **extra))
        _, lds = main.frame_loaders(str(data), c, 1, 0, torch.device("cuda", 0), 0.0, parts=("test",))
        assert lds["test"].transform == ((True, 0.0) if key == "rot" else (True, 30.0))
        moved[key] = _split_loss(c, str(data), sd, "test")
    for key, v in moved.items():
        assert abs(v - plain) <= 1e-4 * plain, (key, v, plain)
