"""Torsion fingerprint deviation (TFD) matrices between the conformers of each molecule on the GPU (RDKit
``TorsionFingerprints.GetTFDMatrix``; reference: ``nvmolkit/tfd.py:126-195``).

Two layers:

* :func:`tfd_torsions` builds the flat, per-molecule torsion tables (:class:`TFDTorsions`) on the host through the RDKit
  ``Mol`` accessors, once per set of molecules and options; they can be passed back to every later call.
* :func:`GetTFDMatrices` / :func:`GetTFDMatrix` compute the matrices with ``b200mol_tfd_matrices`` (a feature pass over
  (conformer, torsion) and a tiled pair pass, ``csrc/tfd.cu``), from RDKit conformers, from an on-device
  :class:`~nvmolkit_b200.types.Device3DResult` (``EmbedMolecules(output=DEVICE)``), or from a :class:`FlatTFDMolecules`.

Torsion tables restate the reference (``src/tfd/tfd_common.cpp``): non-ring bonds whose two atoms both have heavy
neighbours carry a torsion (:145-236); triple-bond ends and allene centres cannot be its middle atoms, and with
``ignoreColinearBonds=False`` the torsion walks out along the chain; the end atoms are chosen by symmetry invariants
(one neighbour; all neighbours if their invariants are equal; the odd one of three; else the smallest invariant);
``maxDev="spec"`` gives 90 / 60 / 30 / 180 by the symmetry case (:328-428); every ring is one torsion over its consecutive
quartets with maxDev ``180 exp(-0.025 (n - 14)^2)`` (180 from n = 14). Weights (:439-512): the central bond is the
bond of the two non-terminal atoms with the smallest spread of topological distances; ``beta = -ln 0.1 / (dmax / 2)^2``;
a non-ring torsion weighs ``exp(-beta d^2)`` with d its distance to the central bond (+1, 0 for the central bond
itself), a ring ``exp(-beta dbar^2) n / 2``.

``dmax`` is the largest distance from the central atom to a bond between two non-terminal atoms. RDKit before 2026.03.1
tested the END atom twice (``_calculateBeta``), so it also counts bonds whose begin atom is terminal; that older rule is
the one that reproduces the reference's weight known answers (``tests/test_tfd_cpu.cpp:173-205``, e.g. CCCCC {1, 0.1};
the newer rule gives {1, 1e-4}). :func:`tfd_torsions` uses the rule of the RDKit it runs against (``rdkit.__version__``;
the newer rule when no version is given).
"""

from __future__ import annotations

import math
import re
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._hostutil import device_conformer_order
from nvmolkit_b200._interop import require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.types import Device3DResult

SINGLE, SYMMETRIC, RING = 0, 1, 2  # B200MOL_TFD_* of include/b200mol.h
MAX_ATOMS = 32767  # quartets hold int16 atom indices
_RETURN_TYPES = ("list", "numpy", "tensor")


@dataclass
class TFDTorsions:
    """Flat per-molecule torsion tables in the layout of ``b200mol_tfd_matrices``: torsions of molecule m are
    ``[tors_start[m], tors_start[m+1])``, torsion t owns quartets ``[quartet_start[t], quartet_start[t+1])`` of
    ``quartets`` (molecule-local atom indices), with ``type`` (SINGLE / SYMMETRIC / RING), ``weight`` and ``maxdev``
    (degrees)."""

    tors_start: np.ndarray  # int32 [nMols+1]
    quartet_start: np.ndarray  # int32 [nTors+1]
    quartets: np.ndarray  # int16 [nQ, 4]
    type: np.ndarray  # uint8 [nTors]
    weight: np.ndarray  # float64 [nTors]
    maxdev: np.ndarray  # float64 [nTors]

    def __post_init__(self):
        self.tors_start = np.ascontiguousarray(self.tors_start, np.int32)
        self.quartet_start = np.ascontiguousarray(self.quartet_start, np.int32)
        self.quartets = np.ascontiguousarray(self.quartets, np.int16).reshape(-1, 4)
        self.type = np.ascontiguousarray(self.type, np.uint8)
        self.weight = np.ascontiguousarray(self.weight, np.float64)
        self.maxdev = np.ascontiguousarray(self.maxdev, np.float64)
        n_tors = len(self.type)
        if (len(self.tors_start) < 1 or self.tors_start[0] != 0 or self.tors_start[-1] != n_tors
                or np.any(np.diff(self.tors_start) < 0)):
            raise ValueError("tors_start must rise from 0 to the number of torsions")
        if (len(self.quartet_start) != n_tors + 1 or self.quartet_start[0] != 0
                or self.quartet_start[-1] != len(self.quartets) or np.any(np.diff(self.quartet_start) < 1)):
            raise ValueError("quartet_start must rise from 0 to the number of quartets, at least one per torsion")
        if len(self.weight) != n_tors or len(self.maxdev) != n_tors:
            raise ValueError("weight and maxdev need one entry per torsion")

    @property
    def n_mols(self) -> int:
        return len(self.tors_start) - 1

    @classmethod
    def from_lists(cls, per_mol: Sequence[Sequence[tuple]]) -> "TFDTorsions":
        """``per_mol[m]`` = list of ``(quartets [[i, j, k, l], ...], type, weight, maxdev)``."""
        ts, qs, qa, ty, w, md = [0], [0], [], [], [], []
        for tors in per_mol:
            for quartets, typ, weight, maxdev in tors:
                qa.extend(list(q) for q in quartets)
                qs.append(len(qa))
                ty.append(typ)
                w.append(weight)
                md.append(maxdev)
            ts.append(len(ty))
        return cls(np.array(ts), np.array(qs), np.array(qa, np.int16).reshape(-1, 4), np.array(ty, np.uint8),
                   np.array(w, np.float64), np.array(md, np.float64))

    def molecule(self, m: int) -> List[tuple]:
        """The torsions of molecule m as ``(quartets, type, weight, maxdev)`` tuples."""
        out = []
        for t in range(int(self.tors_start[m]), int(self.tors_start[m + 1])):
            q = self.quartets[self.quartet_start[t]:self.quartet_start[t + 1]]
            out.append(([tuple(int(v) for v in r) for r in q], int(self.type[t]), float(self.weight[t]), float(self.maxdev[t])))
        return out


# ---------------------------------------------------------------------------------------------------------- host tables
def _legacy_beta_rule() -> bool:
    """True when the RDKit in use predates 2026.03.1 (its _calculateBeta tests the end atom twice)."""
    try:
        import rdkit
    except ImportError:
        return False
    version = getattr(rdkit, "__version__", None)
    if not version:
        return False
    nums = [int(x) for x in re.findall(r"\d+", str(version))[:3]] + [0, 0, 0]
    return tuple(nums[:3]) < (2026, 3, 1)


def _heavy(atom, exclude: int = -1) -> List[int]:
    return [n.GetIdx() for n in atom.GetNeighbors() if n.GetAtomicNum() != 1 and n.GetIdx() != exclude]


def _torsion_bonds(mol, ignore_colinear: bool):
    """(a1, a2, nb1, nb2) of every bond that carries a torsion (reference src/tfd/tfd_common.cpp:145-236)."""
    n = mol.GetNumAtoms()
    flag = [False] * n  # cannot be a middle atom: triple-bond ends, allene centres
    for b in mol.GetBonds():
        if b.GetBondTypeAsDouble() == 3.0:
            flag[b.GetBeginAtomIdx()] = flag[b.GetEndAtomIdx()] = True
    for a in mol.GetAtoms():
        if a.GetAtomicNum() == 6 and sum(1 for b in a.GetBonds() if b.GetBondTypeAsDouble() == 2.0) == 2:
            flag[a.GetIdx()] = True
    ring = mol.GetRingInfo()
    done, out = set(), []
    for b in mol.GetBonds():
        if ring.NumBondRings(b.GetIdx()) > 0:
            continue
        a1, a2 = b.GetBeginAtomIdx(), b.GetEndAtomIdx()
        nb1, nb2 = _heavy(mol.GetAtomWithIdx(a1), a2), _heavy(mol.GetAtomWithIdx(a2), a1)
        if b.GetIdx() in done or not nb1 or not nb2:
            continue
        done.add(b.GetIdx())
        if not (flag[a1] or flag[a2]):
            out.append((a1, a2, nb1, nb2))
            continue
        if ignore_colinear:
            continue

        def walk(a, nb):  # move the middle atom out along a chain of colinear atoms
            for _ in range(n):
                if len(nb) != 1 or not flag[a]:
                    break
                old, a = a, nb[0]
                step = mol.GetBondBetweenAtoms(old, a)
                if step is None:
                    break
                nb = _heavy(mol.GetAtomWithIdx(a), old)
                done.add(step.GetIdx())
            return a, nb

        a1, nb1 = walk(a1, nb1)
        a2, nb2 = walk(a2, nb2)
        if nb1 and nb2:
            out.append((a1, a2, nb1, nb2))
    return out


def _invariants(mol, radius: int) -> List[int]:
    """Radius-`radius` Morgan environment code of each atom (RDKit's Morgan generator); atom degree for radius 0."""
    if radius <= 0:
        return [a.GetDegree() for a in mol.GetAtoms()]
    from rdkit.Chem import rdFingerprintGenerator

    gen = rdFingerprintGenerator.GetMorganGenerator(radius=radius, countSimulation=False, includeChirality=False,
                                                    useBondTypes=True, onlyNonzeroInvariants=False,
                                                    includeRedundantEnvironments=True)
    ao = rdFingerprintGenerator.AdditionalOutput()
    ao.AllocateBitInfoMap()
    gen.GetSparseCountFingerprint(mol, additionalOutput=ao)
    inv = [0] * mol.GetNumAtoms()
    for bit, hits in ao.GetBitInfoMap().items():
        for atom, r in hits:
            if r == radius:
                inv[atom] = int(bit)
    return inv


def _pick(nbrs: List[int], inv: List[int]) -> List[int]:
    if len(nbrs) == 1 or all(inv[a] == inv[nbrs[0]] for a in nbrs):
        return list(nbrs)
    if len(nbrs) == 3:
        a, b, c = (inv[x] for x in nbrs)
        if a == b and a != c:
            return [nbrs[2]]
        if a == c and a != b:
            return [nbrs[1]]
        if b == c and a != b:
            return [nbrs[0]]
    return [min(nbrs, key=lambda x: inv[x])]  # (first of equal minima)


def _ring_maxdev(n: int) -> float:
    return 180.0 if n >= 14 else 180.0 * math.exp(-0.025 * (n - 14) ** 2)


def _weights(mol, bonds, bond_rings, legacy_beta: bool) -> List[float]:
    """Reference src/tfd/tfd_common.cpp:248-323 (central bond, beta) and :439-512 (weights)."""
    from rdkit import Chem

    n_tors = len(bonds) + len(bond_rings)
    if n_tors == 0:
        return []
    dist = np.asarray(Chem.GetDistanceMatrix(mol), np.float64)
    n = mol.GetNumAtoms()
    heavy_deg = [len(_heavy(a)) for a in mol.GetAtoms()]
    spread = []
    for i in range(n):
        if heavy_deg[i] < 2:
            continue
        row = np.delete(dist[i], i)
        mean = row.sum() / len(row)
        spread.append((math.sqrt(max(0.0, float((row * row).sum()) / len(row) - mean * mean)), i))
    spread.sort()
    aid1 = aid2 = -1
    if spread:
        for _, i in spread[1:]:
            if mol.GetBondBetweenAtoms(spread[0][1], i) is not None:
                aid1, aid2 = spread[0][1], i
                break
    if aid1 < 0:
        return [1.0] * n_tors
    dmax = 0.0
    for b in mol.GetBonds():
        i, j = b.GetBeginAtomIdx(), b.GetEndAtomIdx()
        begin_ok = heavy_deg[j] > 1 if legacy_beta else heavy_deg[i] > 1
        if begin_ok and heavy_deg[j] > 1:
            dmax = max(dmax, dist[aid1, i], dist[aid1, j])
    half = dmax / 2.0 if dmax / 2.0 >= 1e-6 else 1.0
    beta = -math.log(0.1) / (half * half)

    def to_central(i, j):
        return min(dist[aid1, i], dist[aid1, j], dist[aid2, i], dist[aid2, j]) + 1.0

    w = []
    for a1, a2, _, _ in bonds:
        d = 0.0 if {a1, a2} == {aid1, aid2} else to_central(a1, a2)
        w.append(math.exp(-beta * d * d))
    by_idx = {b.GetIdx(): (b.GetBeginAtomIdx(), b.GetEndAtomIdx()) for b in mol.GetBonds()}
    for ring in bond_rings:
        dbar = sum(to_central(*by_idx[k]) for k in ring) / len(ring)
        w.append(math.exp(-beta * dbar * dbar) * len(ring) / 2.0)
    return w


def _molecule_torsions(mol, use_weights: bool, spec: bool, radius: int, ignore_colinear: bool, legacy_beta: bool):
    bonds = _torsion_bonds(mol, ignore_colinear)
    inv = _invariants(mol, radius)
    tors = []
    for a1, a2, nb1, nb2 in bonds:
        d1, d2 = _pick(nb1, inv), _pick(nb2, inv)
        quartets = [(x, a1, a2, y) for x in d1 for y in d2]
        maxdev = 180.0
        if spec and len(quartets) > 1:
            if len(d1) == 1:
                maxdev = 90.0 if len(nb2) == 2 else 60.0
            elif len(d2) == 1:
                maxdev = 90.0 if len(nb1) == 2 else 60.0
            elif len(nb1) == 2 and len(nb2) == 2:
                maxdev = 90.0
            elif len(nb1) == 3 and len(nb2) == 3:
                maxdev = 60.0
            else:
                maxdev = 30.0
        tors.append([quartets, SYMMETRIC if len(quartets) > 1 else SINGLE, 1.0, maxdev])
    ring_info = mol.GetRingInfo()
    atom_rings = list(ring_info.AtomRings())
    for ring in atom_rings:
        k = len(ring)
        quartets = [(ring[i], ring[(i + 1) % k], ring[(i + 2) % k], ring[(i + 3) % k]) for i in range(k)]
        tors.append([quartets, RING if k > 1 else SINGLE, 1.0, _ring_maxdev(k)])
    if use_weights:
        bond_rings = list(ring_info.BondRings()) if atom_rings else []
        for t, w in zip(tors, _weights(mol, bonds, bond_rings, legacy_beta)):
            t[2] = w
    return [tuple(t) for t in tors]


def _check_options(maxDev: str, return_type: str) -> None:
    if maxDev not in ("equal", "spec"):
        raise ValueError(f"maxDev must be 'equal' or 'spec', got {maxDev!r}")
    if return_type not in _RETURN_TYPES:
        raise ValueError(f"Invalid return_type {return_type!r}. Must be 'list', 'numpy', or 'tensor'.")


def tfd_torsions(mols, useWeights: bool = True, maxDev: str = "equal", symmRadius: int = 2,
                 ignoreColinearBonds: bool = True) -> TFDTorsions:
    """Torsion tables of RDKit molecules (read through the ``Mol`` accessors), built once and reusable."""
    _check_options(maxDev, "list")
    legacy = _legacy_beta_rule()
    per_mol = []
    for i, mol in enumerate(mols):
        if mol is None:
            raise ValueError(f"Molecule at index {i} is None")
        if mol.GetNumAtoms() > MAX_ATOMS:
            raise ValueError(f"Molecule at index {i} has {mol.GetNumAtoms()} atoms; at most {MAX_ATOMS} are supported")
        per_mol.append(_molecule_torsions(mol, bool(useWeights), maxDev == "spec", int(symmRadius),
                                          bool(ignoreColinearBonds), legacy))
    return TFDTorsions.from_lists(per_mol)


# ------------------------------------------------------------------------------------------------------------- device
@dataclass
class FlatTFDMolecules:
    """Torsion tables plus coordinates, the seam below RDKit: conformer c of the whole batch owns rows
    ``[conf_atom_start[c], conf_atom_start[c+1])`` of ``xyz`` (float64 [atoms, 3], host or CUDA); the conformers of
    molecule m are ``[mol_conf_start[m], mol_conf_start[m+1])``, in matrix order."""

    torsions: TFDTorsions
    xyz: object
    conf_atom_start: np.ndarray
    mol_conf_start: np.ndarray
    atom_counts: np.ndarray

    @classmethod
    def from_coordinates(cls, torsions: TFDTorsions, coords: Sequence[Sequence[np.ndarray]]) -> "FlatTFDMolecules":
        """``coords[m]`` = the conformers of molecule m, each [nAtoms, 3] (or one [C, nAtoms, 3] array)."""
        if len(coords) != torsions.n_mols:
            raise ValueError(f"{len(coords)} coordinate sets for {torsions.n_mols} molecules")
        blocks, cas, mcs, counts = [], [0], [0], []
        for m, confs in enumerate(coords):
            arr = [np.asarray(c, np.float64).reshape(-1, 3) for c in confs]
            n_atoms = int(confs.shape[1]) if isinstance(confs, np.ndarray) and confs.ndim == 3 else (len(arr[0]) if arr else 0)
            if any(len(a) != n_atoms for a in arr):
                raise ValueError(f"molecule {m}: conformers with different atom counts")
            counts.append(n_atoms)
            for a in arr:
                blocks.append(a)
                cas.append(cas[-1] + len(a))
            mcs.append(mcs[-1] + len(arr))
        xyz = np.concatenate(blocks) if blocks else np.zeros((0, 3))
        return cls(torsions, xyz, np.array(cas, np.int32), np.array(mcs, np.int32), np.array(counts, np.int64))


def _check_quartets(tors: TFDTorsions, atom_counts: Sequence[int]) -> None:
    for m, n in enumerate(atom_counts):
        if int(n) > MAX_ATOMS:
            raise ValueError(f"Molecule at index {m} has {int(n)} atoms; at most {MAX_ATOMS} are supported")
        q0, q1 = tors.quartet_start[tors.tors_start[m]], tors.quartet_start[tors.tors_start[m + 1]]
        q = tors.quartets[q0:q1]
        if len(q) and (q.min() < 0 or q.max() >= int(n)):
            raise ValueError(f"molecule {m}: torsion atom index outside its {int(n)} atoms")


def _split(out: torch.Tensor, counts: np.ndarray, return_type: str, stream):
    sizes = counts * (counts - 1) // 2
    starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    if return_type == "tensor":
        return [out[int(starts[m]):int(starts[m + 1])] for m in range(len(counts))]
    with torch.cuda.device(out.device), stream_ctx(stream):  # ordered after the kernels on the caller's stream
        host = out.cpu().numpy()  # the one device-to-host copy of "numpy" / "list" (synchronises that stream)
    if return_type == "numpy":
        return [host[starts[m]:starts[m + 1]].copy() for m in range(len(counts))]
    return [host[starts[m]:starts[m + 1]].tolist() for m in range(len(counts))]


def _run(tors: TFDTorsions, counts: np.ndarray, conf_order: Optional[torch.Tensor], conf_atom_start: torch.Tensor,
         xyz: torch.Tensor, stream) -> torch.Tensor:
    counts = np.asarray(counts, np.int64)
    mcs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    total = int((counts * (counts - 1) // 2).sum())
    out = torch.empty(total, dtype=torch.float32, device=xyz.device)
    _lib.call("b200mol_tfd_matrices", len(counts), mcs.ctypes.data, conf_order.data_ptr() if conf_order is not None else None,
              conf_atom_start.data_ptr(), xyz.data_ptr(), tors.tors_start.ctypes.data, tors.quartet_start.ctypes.data,
              tors.quartets.ctypes.data, tors.type.ctypes.data, tors.weight.ctypes.data, tors.maxdev.ctypes.data,
              out.data_ptr() if total else None, stream_ptr(stream))
    return out


def GetTFDMatrices(mols, useWeights: bool = True, maxDev: str = "equal", symmRadius: int = 2,
                   ignoreColinearBonds: bool = True, return_type: str = "list", *, coordinates: Optional[Device3DResult] = None,
                   torsions: Optional[TFDTorsions] = None, stream: Optional[torch.cuda.Stream] = None):
    """TFD matrix of every molecule: RDKit's lower triangle (for I in 0..C-1, J < I), as a list of Python float lists
    (``"list"``), float32 NumPy arrays (``"numpy"``) or per-molecule views of one float32 CUDA buffer (``"tensor"``,
    no copy).

    ``mols`` is a list of RDKit molecules or a :class:`FlatTFDMolecules`. With RDKit molecules the coordinates are their
    conformers (each molecule needs at least one), or ``coordinates``: a :class:`Device3DResult` whose molecule m pairs
    with ``mols[m]``, read on the device, conformers in ``conf_indices`` order (its conformer table is copied to the
    host once to plan the call). ``torsions`` reuses tables from :func:`tfd_torsions`; the torsion options are then
    those the tables were built with. Molecules with fewer than two conformers get an empty matrix, molecules without
    torsions zeros. Runs on ``stream`` (default: the current stream); ``"list"`` and ``"numpy"`` copy the result to
    the host at the end.
    """
    _check_options(maxDev, return_type)
    if isinstance(mols, FlatTFDMolecules):
        flat = mols
        tors = flat.torsions
        counts = np.diff(np.asarray(flat.mol_conf_start, np.int64))
        if len(counts) != tors.n_mols or len(flat.atom_counts) != tors.n_mols:
            raise ValueError("FlatTFDMolecules: torsion tables and coordinates describe different molecule counts")
        _check_quartets(tors, flat.atom_counts)
        if tors.n_mols == 0:
            return []
        stream_ptr(stream)  # (rejects a bad stream argument before any device work)
        require_cuda()
        dev = flat.xyz.device if isinstance(flat.xyz, torch.Tensor) and flat.xyz.is_cuda else torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev), stream_ctx(stream):
            xyz = torch.as_tensor(flat.xyz, dtype=torch.float64).to(dev).contiguous()
            cas = torch.from_numpy(np.ascontiguousarray(flat.conf_atom_start, np.int32)).to(dev)
            out = _run(tors, counts, None, cas, xyz, stream)
        return _split(out, counts, return_type, stream)

    mols = list(mols)
    for i, mol in enumerate(mols):
        if mol is None:
            raise ValueError(f"Molecule at index {i} is None")
    atom_counts = [m.GetNumAtoms() for m in mols]
    for i, n in enumerate(atom_counts):
        if n > MAX_ATOMS:
            raise ValueError(f"Molecule at index {i} has {n} atoms; at most {MAX_ATOMS} are supported")
    if coordinates is None:
        for i, mol in enumerate(mols):
            if len(mol.GetConformers()) == 0:
                raise ValueError(f"Molecule at index {i} has no conformers")
    elif not isinstance(coordinates, Device3DResult):
        raise TypeError(f"coordinates must be a Device3DResult, got {type(coordinates).__name__}")
    elif coordinates.n_mols != len(mols):
        raise ValueError(f"coordinates hold {coordinates.n_mols} molecules, mols has {len(mols)}")
    if torsions is not None and torsions.n_mols != len(mols):
        raise ValueError(f"torsions describe {torsions.n_mols} molecules, mols has {len(mols)}")
    tors = torsions if torsions is not None else tfd_torsions(mols, useWeights, maxDev, symmRadius, ignoreColinearBonds)
    _check_quartets(tors, atom_counts)
    if not mols:
        return []
    if coordinates is None:
        confs = [[np.asarray(c.GetPositions(), np.float64) for c in mol.GetConformers()] for mol in mols]
        flat = FlatTFDMolecules.from_coordinates(tors, confs)
        return GetTFDMatrices(flat, return_type=return_type, stream=stream)

    xyz = coordinates.values.torch()
    dev = xyz.device
    order, counts, starts_t = device_conformer_order(coordinates, atom_counts)
    stream_ptr(stream)
    require_cuda()
    with torch.cuda.device(dev), stream_ctx(stream):
        d_order = torch.from_numpy(order).to(dev)
        cas = starts_t.to(device=dev, dtype=torch.int32).contiguous()
        out = _run(tors, counts, d_order, cas, xyz.to(torch.float64).contiguous(), stream)
    return _split(out, counts, return_type, stream)


def GetTFDMatrix(mol, useWeights: bool = True, maxDev: str = "equal", symmRadius: int = 2,
                 ignoreColinearBonds: bool = True, return_type: str = "list", *, coordinates: Optional[Device3DResult] = None,
                 torsions: Optional[TFDTorsions] = None, stream: Optional[torch.cuda.Stream] = None):
    """The TFD matrix of one molecule's conformers (:func:`GetTFDMatrices` of ``[mol]``)."""
    return GetTFDMatrices([mol], useWeights, maxDev, symmRadius, ignoreColinearBonds, return_type,
                          coordinates=coordinates, torsions=torsions, stream=stream)[0]
