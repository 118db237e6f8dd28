"""The protein dataset's files, read without MDAnalysis: a CHARMM/NAMD DCD trajectory and a CHARMM PSF topology.

The reference reads the AdK equilibrium trajectory that MDAnalysisData fetches (`adk4AKE.psf`,
`1ake_007-nowater-core-dt240ps.dcd`) through `MDAnalysis.Universe` and keeps the `backbone` atoms
(datasets/process_dataset.py:142-147).  Here:

    traj = load_protein(find_files("adk_equilibrium"), backbone=True)     # a frames.Trajectories of one scene
    samples = sample_list(traj, delta_t=15, split="train")                # every frame of [0, 2481)

DCD (the CHARMM binary layout, as CHARMM and NAMD write it; every record is a 4-byte length, the payload and the length
again, in the byte order the first marker (84) shows):
    84 | "CORD" | 20 int32 ICNTRL | 84              NSET = ICNTRL[0], NAMNF (fixed atoms) = [8], unit cell flag = [10],
                                                    4-D flag = [11], CHARMM version = [19] (0: X-PLOR, no cell, no 4-D)
    4 + 80·NTITLE | NTITLE | NTITLE × 80 bytes | ..  the title
    4 | NATOM | 4
    per frame: [48 | 6 float64 | 48] X Y Z           the unit cell (CHARMM's A, γ, B, β, α, C) if flagged; then one
                                                    record of NATOM float32 per coordinate
The frame count comes from the file size, as MDAnalysis counts it.  `positions` is a read-only [T, NATOM, 3] view over
the memory map (the X, Y and Z records of a frame are 4·NATOM + 8 bytes apart), so a batch reads only its frames.
Fixed atoms, 4-D coordinates, 8-byte record markers and a truncated file raise ValueError.

PSF: the `!NATOM` section, one line per atom `id segid resid resname name type charge mass imove`, in the standard
(I8, A4 fields) and the `EXT` (I10, A8 fields) layouts alike; the fields are read by whitespace.
"""
from __future__ import annotations

import glob
import os
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from .frames import Scene, Trajectories, _npz_members, _static, RECIPES

# MDAnalysis's `backbone` keyword: these atom names in residues of its protein residue list (core/selection.py,
# BackboneSelection and ProteinSelection): the CHARMM, PDB, GROMACS and AMBER names of the amino acids
BACKBONE_NAMES = frozenset({"N", "CA", "C", "O"})
PROTEIN_RESIDUES = frozenset({
    "ALA", "ARG", "ASN", "ASP", "CYS", "GLN", "GLU", "GLY", "HSD", "HSE", "HSP", "ILE", "LEU", "LYS", "MET", "PHE",
    "PRO", "SER", "THR", "TRP", "TYR", "VAL", "ALAD", "HIS", "MSE",
    "ARGN", "ASPH", "CYS2", "CYSH", "QLN", "PGLU", "GLUH", "HIS1", "HISD", "HISE", "HISH", "LYSH",
    "ASN1", "CYS1", "HISA", "HISB", "HIS2",
    "HID", "HIE", "HIP", "ORN", "DAB", "LYN", "HYP", "CYM", "CYX", "ASH", "GLH", "ACE", "NME",
    "NALA", "NGLY", "NSER", "NTHR", "NLEU", "NILE", "NVAL", "NASN", "NGLN", "NARG", "NHID", "NHIE", "NHIP", "NTRP",
    "NPHE", "NTYR", "NGLU", "NASP", "NLYS", "NPRO", "NCYS", "NCYX", "NMET", "CALA", "CGLY", "CSER", "CTHR", "CLEU",
    "CILE", "CVAL", "CASF", "CASN", "CGLN", "CARG", "CHID", "CHIE", "CHIP", "CTRP", "CPHE", "CTYR", "CGLU", "CASP",
    "CLYS", "CPRO", "CCYS", "CCYX", "CMET", "CME", "ASF"})


@dataclass
class DCD:
    """An opened DCD file.  `positions` float32 [T, n, 3] and `unit_cell` float64 [T, 6] (CHARMM order A, γ, B, β, α,
    C) or None are read-only views over `memmap`, one record per frame; nothing is read until indexed."""
    path: str
    n_atoms: int
    n_frames: int
    nset: int                   # the header's frame count (MDAnalysis, like this reader, counts frames by file size)
    istart: int
    nsavc: int
    title: List[str]
    memmap: np.memmap
    positions: np.ndarray
    unit_cell: Optional[np.ndarray]


def read_dcd(path: str) -> DCD:
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        head = f.read(min(size, 1 << 16))
    if len(head) < 92:
        raise ValueError(f"{path}: {len(head)} bytes, too short for a DCD header")
    order = next((e for e in "<>" if int(np.frombuffer(head, e + "i4", 1, 0)[0]) == 84), None)
    if order is None:
        if head[8:12] == b"CORD" and any(int(np.frombuffer(head, e + "i8", 1, 0)[0]) == 84 for e in "<>"):
            raise ValueError(f"{path}: 8-byte record markers are not supported (write the DCD with 4-byte markers)")
        raise ValueError(f"{path}: not a DCD file (the first record marker is not 84 in either byte order)")
    if head[4:8] != b"CORD":
        if head[8:12] == b"CORD":
            raise ValueError(f"{path}: 8-byte record markers are not supported (write the DCD with 4-byte markers)")
        raise ValueError(f"{path}: not a coordinate DCD (no 'CORD' tag)")
    i4 = np.dtype(order + "i4")
    icntrl = np.frombuffer(head, i4, 20, 8).astype(np.int64)
    if int(np.frombuffer(head, i4, 1, 88)[0]) != 84:
        raise ValueError(f"{path}: malformed header record (its closing marker is not 84)")
    charmm = icntrl[19] != 0
    has_cell, dim4, namnf = bool(charmm and icntrl[10]), bool(charmm and icntrl[11]), int(icntrl[8])
    if namnf > 0:
        raise ValueError(f"{path}: {namnf} fixed atoms (NAMNF > 0) are not supported: such a file stores only the free "
                         "atoms after its first frame")
    if dim4:
        raise ValueError(f"{path}: 4-D coordinates are not supported")

    def record(off, what):                      # (payload offset, payload length) of the record at `off`
        if off + 4 > len(head):
            raise ValueError(f"{path}: truncated in the {what} record")
        n = int(np.frombuffer(head, i4, 1, off)[0])
        if n < 0 or off + 8 + n > len(head) or int(np.frombuffer(head, i4, 1, off + 4 + n)[0]) != n:
            raise ValueError(f"{path}: malformed {what} record")
        return off + 4, n

    t_off, t_len = record(92, "title")
    ntitle = int(np.frombuffer(head, i4, 1, t_off)[0])
    if t_len != 4 + 80 * ntitle:
        raise ValueError(f"{path}: malformed title record ({ntitle} lines in {t_len} bytes)")
    title = [head[t_off + 4 + 80 * k:t_off + 84 + 80 * k].decode("latin-1").rstrip("\x00 ") for k in range(ntitle)]
    a_off, a_len = record(t_off + t_len + 4, "atom count")
    if a_len != 4:
        raise ValueError(f"{path}: malformed atom count record")
    n = int(np.frombuffer(head, i4, 1, a_off)[0])
    if n < 1:
        raise ValueError(f"{path}: {n} atoms")
    first = a_off + 8                             # the first frame's first record
    fields = [("cm0", i4), ("cell", order + "f8", (6,)), ("cm1", i4)] if has_cell else []
    for c in "xyz":                               # a record: its length, NATOM float32, its length
        fields += [(c + "0", i4), (c + "1", order + "f4", (n,)), (c + "2", i4)]
    frame = np.dtype(fields)
    T, rest = divmod(size - first, frame.itemsize)
    if rest:
        raise ValueError(f"{path}: truncated: the last frame has {rest} of {frame.itemsize} bytes")
    if T < 1 or T < icntrl[0]:
        raise ValueError(f"{path}: truncated: the header counts {int(icntrl[0])} frames, the file holds {T}")
    mm = np.memmap(path, dtype=frame, mode="r", offset=first, shape=(T,))
    for t in sorted({0, T - 1}):                  # the record layout, checked on the first and the last frame
        if has_cell and not int(mm["cm0"][t]) == int(mm["cm1"][t]) == 48:
            raise ValueError(f"{path}: frame {t}: malformed unit-cell record")
        for c in "xyz":
            if not int(mm[c + "0"][t]) == int(mm[c + "2"][t]) == 4 * n:
                raise ValueError(f"{path}: frame {t}: malformed {c.upper()} record (the file is not a {n}-atom DCD "
                                 "with the header's unit-cell flag)")
    pos = np.lib.stride_tricks.as_strided(mm["x1"], shape=(T, n, 3), strides=(frame.itemsize, 4, 4 * n + 8),
                                          writeable=False)
    return DCD(path, n, int(T), int(icntrl[0]), int(icntrl[1]), int(icntrl[2]), title, mm, pos,
               mm["cell"] if has_cell else None)


def cubic_edge(dcd: DCD, frames: Sequence[int]) -> float:
    """The edge of the DCD's unit cell over `frames`, which must be one cubic cell (A = B = C, the angles 90° or their
    cosines 0, as CHARMM and NAMD write them); ValueError otherwise."""
    if dcd.unit_cell is None:
        raise ValueError(f"{dcd.path} has no unit cell")
    c = np.asarray(dcd.unit_cell[np.asarray(frames, dtype=np.int64)], dtype=np.float64)
    a = c[:, [0, 2, 5]]
    ang = c[:, [1, 3, 4]]
    if not ((a == a[0, 0]).all() and a[0, 0] > 0 and ((ang == 90.0) | (ang == 0.0)).all()):
        raise ValueError(f"{dcd.path}: the unit cell is not one cubic cell over frames {frames[0]}..{frames[-1]} "
                         f"(first A, γ, B, β, α, C = {c[0].tolist()})")
    return float(a[0, 0])


@dataclass
class PSF:
    """A PSF's atoms: names, residue names (str arrays) and charges (float64), in file order."""
    names: np.ndarray
    resnames: np.ndarray
    charges: np.ndarray


def read_psf(path: str) -> PSF:
    with open(path, "r", encoding="latin-1") as f:
        lines = f.read().splitlines()
    body = [ln for ln in lines if ln.strip()]
    if not body or not body[0].split()[0] == "PSF":
        raise ValueError(f"{path}: not a PSF file (no 'PSF' header line)")
    at = next((k for k, ln in enumerate(lines) if "!NATOM" in ln), None)
    if at is None:
        raise ValueError(f"{path}: no !NATOM section")
    try:
        n = int(lines[at].split()[0])
    except ValueError:
        raise ValueError(f"{path}: malformed !NATOM line {lines[at]!r}") from None
    rows = lines[at + 1:at + 1 + n]
    if len(rows) < n:
        raise ValueError(f"{path}: !NATOM counts {n} atoms, the file has {len(rows)} lines after it")
    names, resnames, charges = [], [], np.empty(n, dtype=np.float64)
    for k, ln in enumerate(rows):
        f = ln.split()
        try:
            if len(f) < 8:
                raise ValueError
            charges[k] = float(f[6])
        except ValueError:
            raise ValueError(f"{path}: malformed atom line {at + 2 + k}: {ln!r}") from None
        resnames.append(f[3])
        names.append(f[4])
    return PSF(np.array(names, dtype=str), np.array(resnames, dtype=str), charges)


def backbone_index(psf: PSF) -> np.ndarray:
    """MDAnalysis's `select_atoms('backbone').ix`: atoms named N, CA, C or O in protein residues, ascending, int64."""
    sel = np.isin(psf.names, list(BACKBONE_NAMES)) & np.isin(psf.resnames, list(PROTEIN_RESIDUES))
    return np.flatnonzero(sel).astype(np.int64)


class AtomSelection:
    """`positions[:, index]` as an array-like [T, len(index), 3] that gathers one frame's atoms when indexed, so a
    selection copies the frames a batch reads and nothing else."""

    def __init__(self, positions: np.ndarray, index: np.ndarray):
        self.positions, self.index = positions, index
        self.shape = (positions.shape[0], len(index), positions.shape[2])
        self.ndim, self.dtype = 3, positions.dtype

    def __getitem__(self, f):
        return np.take(self.positions[f], self.index, axis=-2)

    def __array__(self, dtype=None, copy=None):
        out = self[:]
        return out if dtype is None else out.astype(dtype)


def find_files(directory: str) -> List[str]:
    """The protein trajectory in `directory`: [psf, dcd] (one *.psf and one *.dcd, e.g. the adk_equilibrium folder
    MDAnalysisData writes), else [npz] (one *.npz scene with `position` [T,n,3] and `charges` [n]); [] if neither.
    ValueError if the directory holds several candidates of a kind."""
    psf, dcd = (sorted(glob.glob(os.path.join(directory, f"*.{e}"))) for e in ("psf", "dcd"))
    npz = sorted(glob.glob(os.path.join(directory, "*.npz")))
    for kind, found in (("psf", psf), ("dcd", dcd), ("npz", npz)):
        if len(found) > 1:
            raise ValueError(f"{directory}: {len(found)} .{kind} files ({', '.join(map(os.path.basename, found))}); "
                             "keep one protein trajectory per directory")
    if psf and dcd:
        return psf + dcd
    if npz and not (psf or dcd):
        return npz
    return []


def load_protein(files: Sequence[str], backbone: bool = True) -> Trajectories:
    """The protein recipe's one-scene `Trajectories` of `find_files`' list.  PSF + DCD: the backbone atoms
    (`backbone_index`, ascending) or all atoms, their charges from the PSF.  An .npz scene holds the atoms to use
    (`backbone` does not apply to it)."""
    rc = RECIPES["protein"]
    if len(files) == 1 and files[0].endswith(".npz"):
        z = _npz_members(files[0])
        if "position" not in z:
            raise ValueError(f"{files[0]}: missing 'position'")
        pos = z["position"]
        if pos.ndim != 3:
            raise ValueError(f"{files[0]}: position must be [T,n,3], got {pos.shape}")
        return Trajectories([Scene(pos, None, _static(z, rc, pos.shape[1], files[0]), name=files[0])], "protein")
    psf_path = next((p for p in files if p.endswith(".psf")), None)
    dcd_path = next((p for p in files if p.endswith(".dcd")), None)
    if psf_path is None or dcd_path is None or len(files) != 2:
        raise ValueError(f"a protein trajectory is one .psf and one .dcd, or one .npz (got {list(files)})")
    psf, dcd = read_psf(psf_path), read_dcd(dcd_path)
    if len(psf.charges) != dcd.n_atoms:
        raise ValueError(f"{psf_path} has {len(psf.charges)} atoms, {dcd_path} {dcd.n_atoms}")
    if backbone:
        ix = backbone_index(psf)
        if len(ix) == 0:
            raise ValueError(f"{psf_path}: no backbone atoms (N, CA, C, O of protein residues)")
        pos = AtomSelection(dcd.positions, ix)
    else:
        ix, pos = np.arange(dcd.n_atoms), dcd.positions
    static = np.ascontiguousarray(psf.charges[ix].astype(np.float32).reshape(-1, 1))    # the reference's .float()
    return Trajectories([Scene(pos, None, static, name=dcd_path)], "protein")
