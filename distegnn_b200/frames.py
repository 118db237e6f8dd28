"""Training batches from raw simulation frames, assembled on the device as each batch is needed.

The reference builds its samples once on the host and caches them as pickled PyG `Data` lists
(datasets/process_dataset.py).  Here the trajectories stay in host memory (memory-mapped), only the frames a batch
needs cross PCIe, and the per-sample arithmetic, the split and the graph run on the device:

    traj = load_scenes(sorted(glob("water3d/train/*.npz")), "water3d")     # or load_nbody(dir, "train")
    samples = sample_list(traj, seed=0, max_samples=1000, delta_t=1)       # the reference's frame draws, seeded
    loader = FrameLoader(traj, samples, delta_t=1, radius=0.035, cutoff_rate=0.5, batch_size=1, shuffle=True,
                         device="cuda:0")
    for kwargs, extras in loader:                                           # as ShardLoader yields them
        loc_pred, X = model(**kwargs)
        loss, _ = train_loss(loc_pred, extras["target"], X, kwargs["data_batch"], node_counts=extras["node_counts"], ...)

Recipes (the reference's per-sample lines, restated exactly; `s` the scene's static column):

    nbody       (:61-115)   x = loc[f0], target = loc[fT], v = vel[f0], feat = [‖v‖, q / max q], attr = q
    water3d     (:239-277, :334-347)  x = pos[f], target = pos[f+Δ], v = pos[f+1] − pos[f], feat = [‖v‖, type / max type],
                attr = type
    largefluid  (:480-557)  x = pos[f], target = pos[f+Δ], v = vel[f], feat = [viscosity, mass, ‖vel[f]‖],
                attr = [viscosity, mass]
    protein     (:142-198)  Water-3D's columns with the charge q in place of the type: feat = [‖v‖, q / max q], attr = q

`loc_mean` and the max are taken over the whole scene before any split (distribute_graphs.py:32; :346 then :348).  The
graph: a radius graph per sample (of this rank's nodes) with `radius_graph_csr`, or for `radius` None / < 0 the fully
connected graph (:97-99, built once per node-count tuple and kept), then `cutoff_rate` > 0 keeps the shortest edges of
every graph (:103, `cutoff_edges_csr`).  `edge_attr` is the length in every column (:104).

Input layout.  N-body: the reference's own `loc_*.npy`, `vel_*.npy` [S,T,n,3] and `charges_*.npy` [S,n,1].  Water-3D and
Fluid113K: one `.npz` per scene holding `position` [T,n,3], optionally `velocity` [T,n,3], and the static fields
(`particle_type` [n], or `viscosity` and `mass` [n]).  Uncompressed `.npz` members (np.savez) are memory-mapped.
Protein: one trajectory, a CHARMM PSF and DCD (or one `.npz` with `position` and `charges`), read by
`distegnn_b200.protein.load_protein` (DESIGN §27).

Training noise (DESIGN §22).  `FrameLoader(..., noise=(σ_x, σ_v))` trains on a perturbed input state, so that the model
sees inputs like the slightly wrong ones it feeds itself in a rollout (GNS's input noise):

    train = FrameLoader(traj, samples, ..., shuffle=True, noise=(3e-4, 3e-4))            # clean valid loader: no noise

Every node gets x + ε_x, v + ε_v (‖v‖ of the noisy v) and every target row + ε_x, so the displacement to learn stays the
recorded one; loc_mean is the whole-scene mean of the noisy positions and the graph is built on them.  The split is the
clean frame's.  ε is a pure function of (noise_seed, epoch, sample index, scene node), generated inside the assembly
kernels: every rank, world size, batch size and order sees the same noise for the same node.  The epoch is the number of
earlier `batches()` calls (every iteration draws one).

Rotated and translated evaluation splits (DESIGN §23).  `FrameLoader(..., rotate=True, translate=S)` gives every sample a
rigid transform, R Haar-uniform on SO(3) and t ~ N(0, S²·I), applied to every staged position (R·x + t) and velocity
(R·v) before the recipe's arithmetic, for measuring that test error does not depend on the frame (the reference's
`test_rot` / `test_trans`):

    valid = FrameLoader(traj, samples, ..., rotate=True, translate=1.0)                 # a fixed copy of the split

(R, t) is a pure function of (transform_seed, sample index), independent of the epoch, generated inside the assembly
kernels; the split is the untransformed frame's and the graph is built on the transformed positions.
"""
from __future__ import annotations

import random
import struct
import zipfile
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr
from .loader import n_batches, sampler_batches, staged
from .partition import cutoff_edges_csr, node_chunks, radius_graph_csr
from .shards import CSRGraph

Tensor = torch.Tensor


@dataclass(frozen=True)
class Recipe:
    name: str
    code: int                   # DISTEGNN_FRAMES_* of include/distegnn_b200.h
    static_keys: Tuple[str, ...]
    needs_velocity: bool        # vel[f] is read from the data (False: pos[f+1] − pos[f])
    node_feat_nf: int
    node_attr_nf: int
    max_frame: Optional[int]    # the reference's randint(0, max_frame) ...
    per_scene: Optional[int]    # ... drawn this many times per scene


RECIPES = {
    "nbody": Recipe("nbody", _lib.FRAMES_NBODY, ("charges",), True, 2, 1, None, None),
    "water3d": Recipe("water3d", _lib.FRAMES_WATER3D, ("particle_type",), False, 2, 1, 250, 15),          # :245
    "largefluid": Recipe("largefluid", _lib.FRAMES_LARGEFLUID, ("viscosity", "mass"), True, 3, 2, 50, 16),  # :499
    "protein": Recipe("protein", _lib.FRAMES_WATER3D, ("charges",), False, 2, 1, None, None),
}

# the protein recipe's samples: every frame of a fixed range of its one trajectory, per split (:205-209)
PROTEIN_SPLITS = {"train": (0, 2481), "valid": (2481, 2481 + 827), "test": (2481 + 827, 2481 + 827 + 863)}


def recipe_of(name: str) -> Recipe:
    if name not in RECIPES:
        raise ValueError(f"unknown recipe {name!r} ({'|'.join(RECIPES)})")
    return RECIPES[name]


class Scene:
    """One trajectory: `position` [T,n,3] and `velocity` [T,n,3] or None (memory-mapped numpy arrays, read a frame at a
    time), `static` float32 [n,S] (the recipe's static columns, in memory)."""

    def __init__(self, position, velocity, static: np.ndarray, name: str = ""):
        self.position, self.velocity, self.static, self.name = position, velocity, static, name

    @property
    def n_frames(self) -> int:
        return int(self.position.shape[0])

    @property
    def n_nodes(self) -> int:
        return int(self.position.shape[1])


class Trajectories:
    """The scenes of one dataset split, checked against a recipe."""

    def __init__(self, scenes: Sequence[Scene], recipe: str):
        self.recipe = recipe_of(recipe)
        self.scenes = list(scenes)
        if not self.scenes:
            raise ValueError("no scenes")
        for sc in self.scenes:
            _check_scene(sc, self.recipe)

    def __len__(self) -> int:
        return len(self.scenes)


def _check_scene(sc: Scene, rc: Recipe) -> None:
    p = sc.position
    if p.ndim != 3 or p.shape[2] != 3 or p.shape[0] < 1 or p.shape[1] < 1:
        raise ValueError(f"{sc.name}: position must be [T>=1, n>=1, 3], got {tuple(p.shape)}")
    if rc.needs_velocity:
        if sc.velocity is None:
            raise ValueError(f"{sc.name}: recipe {rc.name!r} needs velocities")
        if tuple(sc.velocity.shape) != tuple(p.shape):
            raise ValueError(f"{sc.name}: velocity shape {tuple(sc.velocity.shape)} != position shape {tuple(p.shape)}")
    if sc.static.shape != (p.shape[1], len(rc.static_keys)) or sc.static.dtype != np.float32:
        raise ValueError(f"{sc.name}: static fields must be float32 [{p.shape[1]}, {len(rc.static_keys)}], "
                         f"got {sc.static.dtype} {tuple(sc.static.shape)}")


def _npz_members(path: str) -> Dict[str, np.ndarray]:
    """The arrays of an .npz: stored (uncompressed) members memory-mapped read-only, compressed ones read in full."""
    out = {}
    with zipfile.ZipFile(path) as zf, open(path, "rb") as f:
        for info in zf.infolist():
            name = info.filename[:-4] if info.filename.endswith(".npy") else info.filename
            if info.compress_type == zipfile.ZIP_STORED:
                f.seek(info.header_offset)
                head = f.read(30)
                nlen, xlen = struct.unpack("<HH", head[26:30])       # local file header: name and extra lengths
                f.seek(info.header_offset + 30 + nlen + xlen)
                major, _ = np.lib.format.read_magic(f)
                rd = np.lib.format.read_array_header_1_0 if major == 1 else np.lib.format.read_array_header_2_0
                shape, fortran, dtype = rd(f)
                if not fortran and not dtype.hasobject and int(np.prod(shape)) > 0:
                    out[name] = np.memmap(path, dtype=dtype, mode="r", offset=f.tell(), shape=shape)
                    continue
            with zf.open(info) as m:
                out[name] = np.lib.format.read_array(m)
    return out


def _static(fields: Dict[str, np.ndarray], rc: Recipe, n: int, where: str) -> np.ndarray:
    cols = []
    for k in rc.static_keys:
        if k not in fields:
            raise ValueError(f"{where}: missing {k!r} (recipe {rc.name!r} needs {', '.join(rc.static_keys)})")
        a = np.asarray(fields[k])
        if a.shape not in ((n,), (n, 1)):
            raise ValueError(f"{where}: {k} must be [{n}] or [{n},1], got {a.shape}")
        cols.append(a.reshape(n).astype(np.float32))           # the reference's .float()
    return np.ascontiguousarray(np.stack(cols, axis=1))


def load_scenes(paths: Sequence[str], recipe: str) -> Trajectories:
    """One .npz per scene (Water-3D: `position`, `particle_type`; Fluid113K: `position`, `velocity`, `viscosity`,
    `mass`)."""
    rc = recipe_of(recipe)
    if rc.name == "protein":
        raise ValueError("unknown recipe 'protein' for a list of .npz scenes: the protein recipe is one trajectory, "
                         "read by distegnn_b200.protein.load_protein")
    scenes = []
    for p in paths:
        z = _npz_members(p)
        if "position" not in z:
            raise ValueError(f"{p}: missing 'position'")
        pos = z["position"]
        if pos.ndim != 3:
            raise ValueError(f"{p}: position must be [T,n,3], got {pos.shape}")
        scenes.append(Scene(pos, z.get("velocity"), _static(z, rc, pos.shape[1], p), name=str(p)))
    return Trajectories(scenes, recipe)


def load_nbody(directory: str, partition: str = "train", tag: str = "charged100_0_0_1") -> Trajectories:
    """The reference's N-body files as they are (process_dataset.py:75-84): `loc_{partition}_{tag}.npy`,
    `vel_...` [S,T,n,3] and `charges_...` [S,n,1]; every system is a scene."""
    import os
    name = lambda k: os.path.join(directory, f"{k}_{partition}_{tag}.npy")
    loc = np.load(name("loc"), mmap_mode="r")
    vel = np.load(name("vel"), mmap_mode="r")
    charges = np.load(name("charges"))
    if loc.ndim != 4 or loc.shape[3] != 3 or vel.shape != loc.shape:
        raise ValueError(f"N-body loc / vel must be [S,T,n,3] alike, got {loc.shape} / {vel.shape}")
    if charges.shape[:2] != (loc.shape[0], loc.shape[2]) or charges.size != loc.shape[0] * loc.shape[2]:
        raise ValueError(f"N-body charges must be [S,n,1] = [{loc.shape[0]},{loc.shape[2]},1], got {charges.shape}")
    rc = RECIPES["nbody"]
    return Trajectories([Scene(loc[s], vel[s], _static({"charges": charges[s]}, rc, loc.shape[2], f"system {s}"),
                               name=f"system {s}") for s in range(loc.shape[0])], "nbody")


def sample_list(traj: Trajectories, seed: int = 0, max_samples: Optional[int] = None, delta_t: int = 1,
                frame_0: int = 0, frames_per_scene: Optional[int] = None,
                max_frame: Optional[int] = None, split: Optional[str] = None) -> List[Tuple[int, int]]:
    """The reference's samples as (scene, frame) pairs.  N-body: every system at `frame_0`, the first `max_samples`
    (:81).  Water-3D / Fluid113K: scene by scene, min(frames_per_scene, max_samples − drawn) frames `randint(0,
    max_frame)` (:245, :499: 15 of [0, 250], 16 of [0, 50]) from `random.Random(seed)` — the reference's distribution
    (its thread pool makes its exact set irreproducible).  Protein: every frame of `PROTEIN_SPLITS[split]` of its one
    scene, in order (:205-211; `max_samples` does not apply, as in the reference).  Raises if a sample's frames fall
    outside its scene."""
    rc = traj.recipe
    cap = len(traj) * 10 ** 9 if max_samples is None else int(max_samples)
    if rc.name == "protein":
        if split not in PROTEIN_SPLITS:
            raise ValueError(f"the protein recipe's samples need split= one of {', '.join(PROTEIN_SPLITS)} (got {split!r})")
        if len(traj) != 1:
            raise ValueError(f"the protein recipe reads one trajectory (got {len(traj)} scenes)")
        out = [(0, t) for t in range(*PROTEIN_SPLITS[split])]
    elif rc.max_frame is None:
        out = [(s, int(frame_0)) for s in range(min(len(traj), cap))]
    else:
        per = rc.per_scene if frames_per_scene is None else int(frames_per_scene)
        hi = rc.max_frame if max_frame is None else int(max_frame)
        rng = random.Random(seed)
        out = []
        for s in range(len(traj)):
            out += [(s, rng.randint(0, hi)) for _ in range(min(per, cap - len(out)))]
    check_samples(traj, out, delta_t)
    return out


def check_samples(traj: Trajectories, samples: Sequence[Tuple[int, int]], delta_t: int, horizon: int = 1) -> None:
    """Raise ValueError naming the first sample whose frames f, f+1 (Water-3D's velocity) or f + tΔ for t = 1..horizon
    fall outside its scene."""
    if not isinstance(horizon, int) or isinstance(horizon, bool) or horizon < 1:
        raise ValueError(f"horizon must be an int >= 1 (got {horizon!r})")
    need_next = not traj.recipe.needs_velocity                   # v = pos[f+1] − pos[f]
    for s, f in samples:
        if not 0 <= s < len(traj):
            raise ValueError(f"sample ({s}, {f}): no scene {s} (there are {len(traj)})")
        T = traj.scenes[s].n_frames
        ends = (f + delta_t, f + horizon * delta_t)
        last = max(*ends, f + 1 if need_next else f)
        if f < 0 or min(ends) < 0 or last >= T:
            fit = (T - 1 - f) // delta_t if delta_t > 0 and 0 <= f < T else 0
            more = "" if horizon == 1 else \
                f"; horizon={horizon} needs frame {f + horizon * delta_t}, and only {max(fit, 0)} step(s) of {delta_t} " \
                f"frames fit after frame {f} (at most horizon {max(fit, 0)})"
            raise ValueError(f"sample ({s}, {f}): frames {f}..{last} fall outside scene {s} of {T} frames "
                             f"(delta_t={delta_t}){more}")


def _check_noise(noise) -> Optional[Tuple[float, float]]:
    """FrameLoader's `noise` as (σ_x, σ_v) floats, or None for no noise (None or (0, 0)); ValueError otherwise."""
    if noise is None:
        return None
    if isinstance(noise, (str, bytes)):
        raise ValueError(f"noise must be (sigma_x, sigma_v) or None (got {noise!r})")
    try:
        sx, sv = (float(v) for v in noise)
    except (TypeError, ValueError):
        raise ValueError(f"noise must be (sigma_x, sigma_v) or None (got {noise!r})") from None
    if not (np.isfinite(sx) and np.isfinite(sv) and sx >= 0 and sv >= 0):
        raise ValueError(f"noise sigmas must be finite and >= 0 (got {noise!r})")
    return None if sx == 0 and sv == 0 else (sx, sv)


def _check_transform(rotate, translate) -> Optional[Tuple[bool, float]]:
    """FrameLoader's `rotate`, `translate` as (rotate, translate), or None for no transform (False, 0); ValueError
    otherwise."""
    if not isinstance(rotate, (bool, np.bool_)):
        raise ValueError(f"rotate must be True or False (got {rotate!r})")
    if isinstance(translate, (str, bytes, bool)):
        raise ValueError(f"translate must be a finite number >= 0 (got {translate!r})")
    try:
        t = float(translate)
    except (TypeError, ValueError):
        raise ValueError(f"translate must be a finite number >= 0 (got {translate!r})") from None
    if not (np.isfinite(t) and t >= 0):
        raise ValueError(f"translate must be a finite number >= 0 (got {translate!r})")
    return None if not rotate and t == 0 else (bool(rotate), t)


def complete_graph_edges(n: int) -> Tensor:
    """The reference's fully connected edge list (process_dataset.py:98): [[i, j] for i for j if i != j], int64 [2,E]."""
    i = torch.arange(n).repeat_interleave(max(n - 1, 0))
    j = torch.arange(n).repeat(n, 1)[~torch.eye(n, dtype=torch.bool)]
    return torch.stack([i, j])


class FrameLoader:
    """Iterate over (scene, frame) samples in batches, the reference's way (same-seed `RandomSampler`, `drop_last`), each
    batch assembled on the device from the raw frames.  Yields `(forward_kwargs, extras)` as `ShardLoader` does.

    traj, samples   a `Trajectories` and its (scene, frame) list (`sample_list`)
    delta_t         target frame offset (N-body: frame_T − frame_0)
    radius          radius of the graph (per partition: the reference's inner_radius); None or < 0 = fully connected
    world_size, rank, split_mode   this rank's share of every sample: "random" (a randperm chunk from a generator seeded
                    per sample, `sample_generator(i)`, identical on every rank), "kmeans", "spectral" or "metis" (labels
                    computed from the sample's frame on first use and cached; spectral: world_size <= 16; metis: on the
                    graph of radius `outer_radius`); every rank needs nodes of every sample, else ValueError
    outer_radius    the radius of the graph the metis split partitions (the reference's outer_radius; split_mode="metis"
                    with world_size > 1 needs it)
    cutoff_rate     > 0: keep the int(E_b·(1 − rate)) shortest edges of every graph
    capacity        None: exact graph allocation (the edge counts are read back every batch).  K: edge buffers of K
                    entries and no host synchronisation at all; `check()` raises if a batch overflowed them
    horizon         K >= 1 target frames per sample: extras["targets"] float32 [K,M,3] holds this rank's nodes at frames
                    f + tΔ, t = 1..K (targets[0] is extras["target"] itself), for `rollout(targets=...)` or a loss on a
                    differentiable rollout.  2 + K frames per sample are staged; K = 1 stages and launches as without it
    noise           (σ_x, σ_v), finite and >= 0: training noise on positions (and every target row) and velocities (module
                    docstring, DESIGN §22).  None or (0, 0): no noise, the same launches as without the argument
    noise_seed      the noise's seed, an int in [0, 2^64) (default `seed`)
    rotate, translate   an evaluation split in another frame (module docstring, DESIGN §23): every sample gets a
                    rotation (Haar-uniform; rotate=True) and a translation translate·N(0, I) (translate finite and >= 0),
                    a function of (transform_seed, sample index) only.  False, 0: the same launches as without them.
                    Not combined with `noise` (ValueError)
    transform_seed  the transform's seed, an int in [0, 2^64) (default `seed`)
    """

    def __init__(self, traj: Trajectories, samples: Sequence[Tuple[int, int]], delta_t: int = 1,
                 radius: Optional[float] = None, batch_size: int = 1, shuffle: bool = False, seed: int = 0,
                 drop_last: bool = True, device=None, prefetch: int = 2, world_size: int = 1, rank: int = 0,
                 split_mode: str = "random", split_seed: Optional[int] = None, cutoff_rate: float = 0.0,
                 capacity: Optional[int] = None, edge_attr_nf: int = 2, loop: bool = False, horizon: int = 1,
                 noise: Optional[Tuple[float, float]] = None, noise_seed: Optional[int] = None,
                 rotate: bool = False, translate: float = 0.0, transform_seed: Optional[int] = None,
                 outer_radius: Optional[float] = None):
        self.traj, self.samples, self.delta_t = traj, [(int(s), int(f)) for s, f in samples], int(delta_t)
        check_samples(traj, self.samples, self.delta_t, horizon)
        self.horizon = horizon
        if world_size < 1 or not 0 <= rank < world_size:
            raise ValueError(f"rank {rank} outside world_size {world_size}")
        if world_size > 1 and split_mode not in ("random", "kmeans", "spectral", "metis"):
            raise ValueError(f"unsupported split_mode {split_mode!r} (random|kmeans|spectral|metis)")
        if world_size > 1 and split_mode == "spectral" and world_size > 16:
            raise ValueError(f"split_mode='spectral' splits into at most 16 parts (world_size {world_size})")
        if world_size > 1 and split_mode == "metis" and outer_radius is None:
            raise ValueError("split_mode='metis' needs outer_radius (the radius of the graph METIS partitions)")
        self.outer_radius = None if outer_radius is None else float(outer_radius)
        self.radius = None if radius is None or radius < 0 else float(radius)
        self.batch_size, self.shuffle, self.drop_last = int(batch_size), shuffle, drop_last
        self.device = torch.device(device) if device is not None else None
        self.prefetch = int(prefetch)
        self.world_size, self.rank, self.split_mode = int(world_size), int(rank), split_mode
        self.split_seed = int(seed if split_seed is None else split_seed)
        self.cutoff_rate, self.capacity, self.edge_attr_nf, self.loop = float(cutoff_rate), capacity, edge_attr_nf, loop
        self.generator = torch.Generator()
        self.generator.manual_seed(seed)
        self._kmeans: Dict[int, Tuple[Tensor, List[int]]] = {}
        self._complete: Dict[Tuple[int, ...], CSRGraph] = {}
        self._overflow: Optional[Tensor] = None
        self.noise = _check_noise(noise)
        self.noise_seed = int(seed if noise_seed is None else noise_seed)
        if self.noise is not None:
            if not 0 <= self.noise_seed < 1 << 64:
                raise ValueError(f"noise_seed must be an int in [0, 2^64) (got {self.noise_seed})")
            if len(self.samples) >= 1 << 32:
                raise ValueError(f"training noise numbers samples with 32 bits: {len(self.samples)} samples are too many")
        self.transform = _check_transform(rotate, translate)
        self.transform_seed = int(seed if transform_seed is None else transform_seed)
        if self.transform is not None:
            if self.noise is not None:
                raise ValueError("noise and a rigid transform (rotate / translate) cannot be combined: the noise is for "
                                 "training, the transform for evaluation splits")
            if not 0 <= self.transform_seed < 1 << 64:
                raise ValueError(f"transform_seed must be an int in [0, 2^64) (got {self.transform_seed})")
            if len(self.samples) >= 1 << 32:
                raise ValueError(f"the rigid transform numbers samples with 32 bits: {len(self.samples)} samples are "
                                 "too many")
        self.epoch = 0

    def __len__(self) -> int:
        return n_batches(len(self.samples), self.batch_size, self.drop_last)

    def batches(self) -> List[List[int]]:
        """The next epoch's batches of sample indices (advances the sampler's generator and `epoch`, as iterating
        does)."""
        out = sampler_batches(len(self.samples), self.batch_size, self.shuffle, self.generator, self.drop_last)
        self.epoch += 1
        return out

    # ---- partitions ----------------------------------------------------------------------------------------------
    def sample_generator(self, i: int) -> torch.Generator:
        """The generator of sample i's random split: the same on every rank, independent of the batch order."""
        return torch.Generator().manual_seed((self.split_seed * 1_000_003 + int(i)) % (1 << 63))

    def partition(self, i: int) -> Tuple[Optional[Tensor], List[int]]:
        """Sample i's node list on this rank (host int32, scene-local, in the reference's order; None = all nodes) and
        every rank's node count."""
        s, f = self.samples[i]
        n = self.traj.scenes[s].n_nodes
        if self.world_size == 1:
            return None, [n]
        if self.split_mode in ("kmeans", "spectral", "metis"):
            if i not in self._kmeans:
                if self.device is None or self.device.type != "cuda":
                    raise _lib.DistEGNNError(f"split_mode={self.split_mode!r} runs on a CUDA device")
                pos = torch.from_numpy(np.array(self.traj.scenes[s].position[f], dtype=np.float32))
                chunks = node_chunks(n, self.world_size, self.split_mode, pos=pos.to(self.device),
                                     outer_radius=self.outer_radius)
                counts = [int(c.numel()) for c in chunks]
                self._check_counts(i, counts)
                self._kmeans[i] = (chunks[self.rank].to("cpu", torch.int32), counts)
            return self._kmeans[i]
        chunks = node_chunks(n, self.world_size, "random", generator=self.sample_generator(i))
        counts = [int(c.numel()) for c in chunks]
        self._check_counts(i, counts)
        return chunks[self.rank].to(torch.int32), counts

    def _check_counts(self, i: int, counts: List[int]) -> None:
        if min(counts) == 0:
            s, f = self.samples[i]
            raise ValueError(f"sample {i} (scene {s}, frame {f}): a {self.split_mode} split over {self.world_size} ranks "
                             f"leaves a rank without nodes ({counts}); every graph needs nodes on every rank")

    # ---- staging (host) ------------------------------------------------------------------------------------------
    def _host_batch(self, idx: Sequence[int], epoch: int = 0) -> Dict[str, object]:
        rc = self.traj.recipe
        pin = self.device is not None and self.device.type == "cuda"
        scenes = [self.traj.scenes[self.samples[i][0]] for i in idx]
        ns = [sc.n_nodes for sc in scenes]
        N = sum(ns)
        frames = torch.empty(2 + self.horizon, N, 3, dtype=torch.float32, pin_memory=pin)
        statics = torch.empty(N, len(rc.static_keys), dtype=torch.float32, pin_memory=pin)
        fr, st = frames.numpy(), statics.numpy()
        parts, counts, off = [], [], 0
        for i, sc, n in zip(idx, scenes, ns):
            f = self.samples[i][1]
            fr[0, off:off + n] = sc.position[f]
            fr[1, off:off + n] = sc.velocity[f] if rc.needs_velocity else sc.position[f + 1]
            for t in range(1, self.horizon + 1):                 # pos[f + tΔ]
                fr[1 + t, off:off + n] = sc.position[f + t * self.delta_t]
            st[off:off + n] = sc.static
            chunk, cnt = self.partition(i)
            parts.append(chunk)
            counts.append(cnt[self.rank])
            off += n
        B = len(idx)
        noisy = self.noise is not None or self.transform is not None
        meta = torch.empty(2 * B + 2 + (B if noisy else 0), dtype=torch.int64, pin_memory=pin)
        meta[:B + 1] = torch.tensor([0] + list(np.cumsum(ns)), dtype=torch.int64)
        meta[B + 1:2 * B + 2] = torch.tensor([0] + list(np.cumsum(counts)), dtype=torch.int64)
        if noisy:                                                # the samples' indices: the noise's / transform's
            meta[2 * B + 2:] = torch.tensor(list(idx), dtype=torch.int64)
        host = dict(frames=frames, statics=statics, meta=meta, n_frame=N, node_counts=counts, epoch=epoch)
        if self.world_size > 1:
            index = torch.empty(sum(counts), dtype=torch.int32, pin_memory=pin)
            torch.cat(parts, out=index)
            host["index"] = index
        return host

    # ---- assembly + graph (device, on the staging stream) ----------------------------------------------------------
    def _complete_graph(self, counts: Tuple[int, ...], dev) -> CSRGraph:
        if counts not in self._complete:
            eis, off = [], 0
            for m in counts:
                eis.append(complete_graph_edges(m) + off)
                off += m
            g, _ = CSRGraph.from_edge_index(torch.cat(eis, 1).to(dev), off)
            g._checked = True
            self._complete[counts] = g
        return self._complete[counts]

    def complete_graph(self, counts: Sequence[int]) -> CSRGraph:
        """The fully connected graph of a batch with these per-graph node counts (kept per tuple; the candidates of a
        fully connected recipe's cutoff, e.g. for `rollout(graph=..., cutoff_rate=...)`)."""
        return self._complete_graph(tuple(int(c) for c in counts), self.device)

    def _to_device(self, host: Dict[str, object]) -> Tuple[Dict[str, object], Dict[str, object]]:
        rc, dev, A = self.traj.recipe, self.device, self.edge_attr_nf
        counts: List[int] = host["node_counts"]
        B, M = len(counts), sum(counts)
        frames = host["frames"].to(dev, non_blocking=True)
        statics = host["statics"].to(dev, non_blocking=True)
        meta = host["meta"].to(dev, non_blocking=True)
        index = host["index"].to(dev, non_blocking=True) if "index" in host else None
        f32 = dict(dtype=torch.float32, device=dev)
        feat, loc, vel = torch.empty(M, rc.node_feat_nf, **f32), torch.empty(M, 3, **f32), torch.empty(M, 3, **f32)
        K = self.horizon
        attr, targets = torch.empty(M, rc.node_attr_nf, **f32), torch.empty(K, M, 3, **f32)
        target = targets[0]
        batch = torch.empty(M, dtype=torch.int64, device=dev)
        loc_mean, scene_max = torch.empty(B, 3, **f32), torch.empty(B, **f32)
        scene_ptr, out_ptr = meta[:B + 1], meta[B + 1:2 * B + 2]
        with torch.cuda.device(dev):
            if self.noise is not None:
                check(_lib.load().distegnn_frames_assemble_noise(
                    rc.code, B, host["n_frame"], M, K, ptr(frames), ptr(statics), ptr(scene_ptr), ptr(out_ptr),
                    ptr(index), ptr(feat), ptr(loc), ptr(vel), ptr(attr), ptr(targets), ptr(batch), ptr(loc_mean),
                    ptr(scene_max), ptr(meta[2 * B + 2:]), self.noise_seed, host["epoch"] % (1 << 32), self.noise[0],
                    self.noise[1], _lib.stream_ptr(dev)), "frames_assemble_noise")
            elif self.transform is not None:
                check(_lib.load().distegnn_frames_assemble_transform(
                    rc.code, B, host["n_frame"], M, K, ptr(frames), ptr(statics), ptr(scene_ptr), ptr(out_ptr),
                    ptr(index), ptr(feat), ptr(loc), ptr(vel), ptr(attr), ptr(targets), ptr(batch), ptr(loc_mean),
                    ptr(scene_max), ptr(meta[2 * B + 2:]), self.transform_seed, int(self.transform[0]),
                    self.transform[1], _lib.stream_ptr(dev)), "frames_assemble_transform")
            else:
                check(_lib.load().distegnn_frames_assemble(
                    rc.code, B, host["n_frame"], M, ptr(frames), ptr(statics), ptr(scene_ptr), ptr(out_ptr),
                    ptr(index), ptr(feat), ptr(loc), ptr(vel), ptr(attr), ptr(target), ptr(batch), ptr(loc_mean),
                    ptr(scene_max), _lib.stream_ptr(dev)), "frames_assemble")
                if K > 1:
                    check(_lib.load().distegnn_frames_targets(B, host["n_frame"], M, K, ptr(frames), ptr(scene_ptr),
                                                              ptr(out_ptr), ptr(index), ptr(targets),
                                                              _lib.stream_ptr(dev)), "frames_targets")
        graph, edge_attr = self._graph(loc, batch, tuple(counts))
        kwargs = dict(node_feat=feat, node_loc=loc, node_vel=vel, loc_mean=loc_mean, edge_index=graph,
                      data_batch=batch, edge_attr=edge_attr, node_attr=attr)
        ptr_ = [0] + np.cumsum(counts).tolist()
        extras = dict(target=target, targets=targets, ptr=ptr_, n_graphs=B, node_counts=list(counts),
                      scene_max=scene_max)
        return kwargs, extras

    def _graph(self, loc: Tensor, batch: Tensor, counts: Tuple[int, ...]) -> Tuple[CSRGraph, Optional[Tensor]]:
        dev, A, B, rate = loc.device, self.edge_attr_nf, len(counts), self.cutoff_rate
        if self.radius is None:                                  # fully connected: fixed topology, fresh lengths
            cand = self._complete_graph(counts, dev)
            if rate > 0:
                g, ea = cutoff_edges_csr(cand, loc, rate, batch, B, A,
                                         capacity=cand.num_edges if self.capacity is not None else None)
            else:
                g, ea = cand, torch.empty(cand.num_edges, A, dtype=torch.float32, device=dev)
                with torch.cuda.device(dev):
                    check(_lib.load().distegnn_edge_lengths_csr(cand.num_edges, A, ptr(cand.row), ptr(cand.col),
                                                                ptr(loc), None, ptr(ea), _lib.stream_ptr(dev)),
                          "edge_lengths_csr")
        else:
            g, ea = radius_graph_csr(loc, self.radius, batch, loop=self.loop, edge_attr_nf=A, capacity=self.capacity,
                                     n_graphs=B, cutoff_rate=rate)
        if g.n_edges_dev is None:
            g._checked = True                                    # built on the device: valid by construction
        elif g.info is not None:
            if self._overflow is None:
                self._overflow = torch.zeros(1, dtype=torch.int32, device=dev)
            torch.maximum(self._overflow, g.info[1:2], out=self._overflow)
        return g, ea

    def __iter__(self):
        if self.device is None or self.device.type != "cuda":
            raise _lib.DistEGNNError("FrameLoader assembles batches on a CUDA device (no CPU path)")
        epoch = self.epoch                                       # this epoch's number, fixed before the order is drawn
        yield from staged(self.batches(), lambda idx: self._host_batch(idx, epoch), self._to_device, self.device,
                          self.prefetch)

    def check(self) -> None:
        """Capacity mode: raise if any batch's graph outgrew `capacity` since the last check (one host read)."""
        if self._overflow is None:
            return
        torch.cuda.synchronize(self.device)
        if int(self._overflow.item()):
            self._overflow.zero_()
            raise RuntimeError(f"FrameLoader: a batch's graph outgrew the capacity {self.capacity}; its edges are "
                               "incomplete — pass a larger capacity, or None for exact allocation")
