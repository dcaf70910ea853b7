"""Conformer RMSD matrices on the GPU (RDKit ``AllChem.GetConformerRMSMatrix``; reference:
``nvmolkit/conformerRmsd.py``).

:func:`GetConformerRMSMatrix` / :func:`GetConformerRMSMatrixBatch` keep the reference's names, arguments, return types
and errors. They compute with ``b200mol_conformer_rmsd`` (``csrc/conformer_rmsd.cu``): every pair's 3x3 covariance is a
block of one fp64 tensor-core Gram product per molecule, and the best superposition follows in closed form. Coordinates
come from the molecules' RDKit conformers or, with ``coordinates=``, from an on-device
:class:`~nvmolkit_b200.types.Device3DResult` (``EmbedMolecules(output=DEVICE)``), so conformers can stay on the GPU from
embedding through minimisation and this matrix to :func:`nvmolkit_b200.clustering.butina`.

Semantics:

* The RMSD uses every atom of the molecule, or with ``atomIds`` the listed atoms only (RDKit's ``atomIds``).
* ``prealigned=False``: the RMSD after the best proper rigid superposition (rotation and translation, no reflection),
  ``sqrt(max(0, Ga + Gb - 2 (s1 + s2 + sign(det H) s3)) / n)`` on centred coordinates. RDKit's own function first aligns
  every conformer to conformer 0 in place; here the input coordinates are never modified.
* ``prealigned=True``: ``sqrt(sum |a - b|^2 / n)`` on the coordinates as given.
* Per molecule with C conformers: a float64 vector of C(C-1)/2 values, pair (i, j), i > j, at ``i(i-1)/2 + j``; fewer
  than two conformers give an empty vector. Results are bitwise repeatable, and a molecule's matrix does not depend on
  the other molecules of the batch.

:func:`GetAllConformerBestRMS` / :func:`GetAllConformerBestRMSBatch` follow RDKit's ``rdMolAlign.GetAllConformerBestRMS``:
pair (i, j), i > j, is the minimum over atom mappings of the RMSD between conformer i's probe atoms and conformer j's
mapped atoms (``b200mol_conformer_rmsd_mapped``: one tensor-core product per mapping, the minimum taken in the
epilogue), so that symmetric molecules (a ring flip, a tert-butyl rotation, a carboxylate's two oxygens) are not
counted as different conformers. The mappings come from ``map`` or from the molecule's matches onto itself
(:func:`nvmolkit_b200.rdkit_adapter.self_matches`).

Differences from RDKit's ``GetAllConformerBestRMS``:

* It returns :class:`AsyncGpuResult` lower triangles like the matrix calls, where RDKit returns a tuple of floats.
* ``numThreads`` is accepted and ignored; a non-empty ``weights`` is refused (weighted RMSD is not computed).
* ``prealigned=True`` (not in RDKit's signature) gives the symmetrised RMSD without alignment, RDKit's ``CalcRMS``.
* The self matches with ``symmetrizeConjugatedTerminalGroups`` are a restatement of RDKit's symmetrised query
  (:func:`~nvmolkit_b200.rdkit_adapter.self_matches`); without RDKit present, it has not been checked against RDKit.
* The input coordinates are never modified.
"""

from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._hostutil import device_conformer_order
from nvmolkit_b200._interop import require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult

__all__ = ["GetConformerRMSMatrix", "GetConformerRMSMatrixBatch", "GetAllConformerBestRMS", "GetAllConformerBestRMSBatch"]


def _check_stream(stream) -> None:
    if stream is not None and not isinstance(stream, torch.cuda.Stream):
        raise TypeError(f"stream must be a torch.cuda.Stream or None, got {type(stream).__name__}")


def pair_offsets(conf_counts) -> np.ndarray:
    """int64 start of each molecule's lower triangle in the concatenated output, plus the total at the end."""
    counts = np.asarray(conf_counts, np.int64)
    return np.concatenate([[0], np.cumsum(counts * (counts - 1) // 2)]).astype(np.int64)


def _check_atoms(atom_counts: np.ndarray, conf_counts: np.ndarray) -> None:
    bad = np.nonzero((conf_counts > 0) & (atom_counts == 0))[0]
    if len(bad):
        raise ValueError(f"mol at index {int(bad[0])} has conformers but no atoms")


class MapTables:
    """Flat mapping tables of ``b200mol_conformer_rmsd_mapped``: molecule m holds ``count[m]`` mappings of ``length[m]``
    atoms in ``atoms[start[m]:start[m + 1]]``, the probe list P first, then the reference lists Q_1 .. Q_K."""

    def __init__(self, lists):
        """``lists[m]``: ``(P, Q)``, P of L atoms and Q a K x L array of reference lists."""
        self.count = np.array([len(q) for _, q in lists], np.int32)
        self.length = np.array([len(p) for p, _ in lists], np.int32)
        self.start = np.concatenate([[0], np.cumsum((self.count.astype(np.int64) + 1) * self.length)]).astype(np.int64)
        blocks = [np.concatenate([np.asarray(p, np.int64), np.asarray(q, np.int64).reshape(-1)]) for p, q in lists]
        self.atoms = np.concatenate(blocks).astype(np.int16) if blocks else np.zeros(0, np.int16)


def _check_list(ids, n: int, what: str) -> np.ndarray:
    arr = np.asarray(ids)
    if arr.ndim != 1 or len(arr) == 0 or not np.issubdtype(arr.dtype, np.integer):
        raise ValueError(f"{what} must be a non-empty list of atom indices")
    arr = arr.astype(np.int64)
    if arr.min() < 0 or arr.max() >= n:
        raise ValueError(f"{what} holds an atom index outside [0, {n})")
    if len(np.unique(arr)) != len(arr):
        raise ValueError(f"{what} holds an atom index twice")
    return arr


def _atom_ids_lists(atomIds, n: int, what: str):
    ids = np.arange(n, dtype=np.int64) if atomIds is None else _check_list(list(atomIds), n, what)
    return ids, ids[None, :]


def _map_lists(mapping, n: int, what: str, n_ref: Optional[int] = None, order: bool = False):
    """GetBestRMS's ``map`` (mappings of (probeAtom, refAtom) pairs) -> (P, Q), each mapping sorted by probe atom; probe
    atoms index ``n`` atoms and reference atoms ``n_ref`` (default ``n``). With ``order``, also the sort of the first
    mapping's pairs, and every mapping must list its probe atoms in that mapping's order (so that one weight per pair
    means one weight per probe atom)."""
    n_ref = n if n_ref is None else n_ref
    if mapping is None or len(mapping) == 0:
        raise ValueError(f"{what} must be a non-empty list of mappings")
    probe, refs, first = None, [], None
    for k, pairs in enumerate(mapping):
        arr = np.asarray(pairs)
        if arr.ndim != 2 or arr.shape[1] != 2 or len(arr) == 0 or not np.issubdtype(arr.dtype, np.integer):
            raise ValueError(f"{what}[{k}] must be a non-empty list of (probeAtom, refAtom) pairs")
        if order:
            if first is None:
                first = arr[:, 0].copy()
            elif not np.array_equal(arr[:, 0], first):
                raise ValueError(f"{what}[{k}] lists its probe atoms in another order than {what}[0], so its weights "
                                 "would fall on other atoms")
        sort = np.argsort(arr[:, 0], kind="stable")
        arr = arr[sort].astype(np.int64)
        p = _check_list(arr[:, 0], n, f"{what}[{k}] probe atoms")
        q = _check_list(arr[:, 1], n_ref, f"{what}[{k}] reference atoms")
        if probe is None:
            probe, perm = p, sort
        elif not np.array_equal(p, probe):
            raise ValueError(f"{what}[{k}] covers other probe atoms than {what}[0]")
        refs.append(q)
    return (probe, np.stack(refs), perm) if order else (probe, np.stack(refs))


def _self_match_lists(mol, maxMatches: int, symmetrize: bool, m: int):
    """(P, Q) of a molecule's matches onto itself: match ``t`` pairs probe atom q with reference atom ``t[q]``, as
    RDKit's ``GetBestRMS`` does (the probe is the query matched inside the reference), so P = 0 .. n-1 and Q = the
    matches themselves."""
    from nvmolkit_b200.rdkit_adapter import self_matches

    n = mol.GetNumAtoms()
    matches = np.array(self_matches(mol, maxMatches, symmetrize), np.int64)
    if matches.ndim != 2 or matches.shape[1] != n:
        raise ValueError(f"mol at index {m}: its matches onto itself must cover all {n} atoms")
    return np.arange(n, dtype=np.int64), matches


def _run(conf_counts: np.ndarray, atom_counts: np.ndarray, conf_order: Optional[torch.Tensor],
         conf_atom_start: torch.Tensor, xyz: torch.Tensor, prealigned: bool, stream,
         maps: Optional[MapTables] = None) -> List[AsyncGpuResult]:
    offsets = pair_offsets(conf_counts)
    mcs = np.concatenate([[0], np.cumsum(conf_counts)]).astype(np.int32)
    atoms = np.ascontiguousarray(atom_counts, np.int32)
    total = int(offsets[-1])
    out = torch.empty(total, dtype=torch.float64, device=xyz.device)
    args = (len(conf_counts), mcs.ctypes.data, atoms.ctypes.data,
            conf_order.data_ptr() if conf_order is not None else None, conf_atom_start.data_ptr(), xyz.data_ptr())
    tail = (1 if prealigned else 0, out.data_ptr() if total else None, stream_ptr(stream))
    if maps is None:
        _lib.call("b200mol_conformer_rmsd", *args, *tail)
    else:
        _lib.call("b200mol_conformer_rmsd_mapped", *args, maps.start.ctypes.data, maps.count.ctypes.data,
                  maps.length.ctypes.data, maps.atoms.ctypes.data, *tail)
    return [AsyncGpuResult(v) for v in torch.split(out, np.diff(offsets).tolist())]  # one call for all the views


def GetConformerRMSMatrixBatch(mols, prealigned: bool = False, stream: Optional[torch.cuda.Stream] = None, *,
                               coordinates: Optional[Device3DResult] = None, atomIds=None) -> List[AsyncGpuResult]:
    """Pairwise RMSD matrices of the conformers of every molecule, in one launch.

    Returns one :class:`AsyncGpuResult` per molecule, in the order of ``mols``: a float64 vector of C(C-1)/2 values
    for C conformers, pair (i, j), i > j, at ``i(i-1)/2 + j`` (RDKit's lower-triangle order), empty for fewer than two
    conformers. The results are views of one device buffer, computed asynchronously on ``stream`` (default: the
    current stream).

    ``coordinates``: a :class:`Device3DResult` whose molecule m pairs with ``mols[m]``; its conformers are read on the
    device, in ``conf_indices`` order (its index tables are copied to the host once to plan the call). Without it the
    molecules' RDKit conformers are used.

    ``atomIds``: one list of atom indices per molecule (None for all of its atoms): the RMSD over those atoms only.

    Raises ValueError for a ``None`` molecule, a molecule with conformers but no atoms or a bad ``atomIds`` (empty,
    repeated or out-of-range indices), TypeError for a ``stream`` that is not a ``torch.cuda.Stream`` or None; all
    before any device work.
    """
    _check_stream(stream)
    mols = _check_mols(mols)
    if atomIds is None:
        return _batch(mols, prealigned, stream, coordinates, None)
    atomIds = list(atomIds)
    if len(atomIds) != len(mols):
        raise ValueError(f"atomIds holds {len(atomIds)} lists, mols has {len(mols)}")
    lists = [_atom_ids_lists(ids, mol.GetNumAtoms(), f"atomIds[{m}]") for m, (mol, ids) in enumerate(zip(mols, atomIds))]
    return _batch(mols, prealigned, stream, coordinates, lists)


def _check_mols(mols) -> list:
    mols = list(mols)
    for i, mol in enumerate(mols):
        if mol is None:
            raise ValueError(f"mol at index {i} must not be None")
    return mols


def _batch(mols, prealigned, stream, coordinates, lists) -> List[AsyncGpuResult]:
    """The matrices of ``mols``; ``lists[m] = (P, Q)`` mapping tables, or None for all atoms by identity."""
    maps = MapTables(lists) if lists is not None else None
    atom_counts = np.array([mol.GetNumAtoms() for mol in mols], np.int64)
    if maps is not None and len(mols) and atom_counts.max() >= 32768:
        raise ValueError(f"mol at index {int(atom_counts.argmax())}: mapping tables take fewer than 32768 atoms")
    if coordinates is None:
        confs = [mol.GetConformers() for mol in mols]
        conf_counts = np.array([len(c) for c in confs], np.int64)
        _check_atoms(atom_counts, conf_counts)
        if not mols:
            return []
        blocks = []
        for m, cs in enumerate(confs):
            for c in cs:
                pos = np.asarray(c.GetPositions(), np.float64).reshape(-1, 3)
                if len(pos) != atom_counts[m]:
                    raise ValueError(f"mol at index {m} has a conformer of {len(pos)} atoms, the molecule has "
                                     f"{int(atom_counts[m])}")
                blocks.append(pos)
        cas = np.concatenate([[0], np.cumsum(np.repeat(atom_counts, conf_counts))]).astype(np.int32)
        host = np.concatenate(blocks) if blocks else np.zeros((0, 3))
        require_cuda()
        dev = torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev), stream_ctx(stream):
            xyz = torch.from_numpy(np.ascontiguousarray(host)).to(dev)
            d_cas = torch.from_numpy(cas).to(dev)
            return _run(conf_counts, atom_counts, None, d_cas, xyz, prealigned, stream, maps)

    if not isinstance(coordinates, Device3DResult):
        raise TypeError(f"coordinates must be a Device3DResult, got {type(coordinates).__name__}")
    if coordinates.n_mols != len(mols):
        raise ValueError(f"coordinates hold {coordinates.n_mols} molecules, mols has {len(mols)}")
    order, conf_counts, starts_t = device_conformer_order(coordinates, atom_counts)
    _check_atoms(atom_counts, conf_counts)
    if not mols:
        return []
    require_cuda()
    xyz = coordinates.values.torch()
    dev = xyz.device
    with torch.cuda.device(dev), stream_ctx(stream):
        d_order = torch.from_numpy(order).to(dev)
        d_cas = starts_t.to(device=dev, dtype=torch.int32).contiguous()
        return _run(conf_counts, atom_counts, d_order, d_cas, xyz.to(torch.float64).contiguous(), prealigned, stream,
                    maps)


def GetConformerRMSMatrix(mol, prealigned: bool = False, stream: Optional[torch.cuda.Stream] = None, *,
                          coordinates: Optional[Device3DResult] = None, atomIds=None) -> AsyncGpuResult:
    """The RMSD matrix of one molecule's conformers (:func:`GetConformerRMSMatrixBatch` of ``[mol]``); ``atomIds``: the
    atoms the RMSD runs over (None = all).

    Raises ValueError if ``mol`` is None, has conformers but no atoms or ``atomIds`` is bad, TypeError for a bad
    ``stream``."""
    _check_stream(stream)
    if mol is None:
        raise ValueError("mol must not be None")
    return GetConformerRMSMatrixBatch([mol], prealigned, stream, coordinates=coordinates,
                                      atomIds=None if atomIds is None else [atomIds])[0]


def GetAllConformerBestRMSBatch(mols, numThreads: int = 1, maxMatches: int = 1000000,
                                symmetrizeConjugatedTerminalGroups: bool = True, weights=None,
                                stream: Optional[torch.cuda.Stream] = None, *, maps=None,
                                coordinates: Optional[Device3DResult] = None,
                                prealigned: bool = False) -> List[AsyncGpuResult]:
    """Symmetry-aware RMSD matrices of the conformers of every molecule, in one launch (RDKit
    ``GetAllConformerBestRMS`` per molecule). Returns one :class:`AsyncGpuResult` per molecule, laid out as
    :func:`GetConformerRMSMatrixBatch`: pair (i, j), i > j, at ``i(i-1)/2 + j`` holds the minimum over the molecule's
    mappings of the RMSD between conformer i's probe atoms and conformer j's mapped atoms.

    ``maps``: one entry per molecule (None for the molecule's self matches), each in ``GetBestRMS``'s ``map`` form: a
    list of mappings, each a list of ``(probeAtom, refAtom)`` pairs; every mapping must cover the same probe atoms.
    Without it the mappings are :func:`nvmolkit_b200.rdkit_adapter.self_matches` ``(mol, maxMatches,
    symmetrizeConjugatedTerminalGroups)``: match ``t`` pairs probe atom ``q`` with reference atom ``t[q]``, as RDKit's
    ``GetBestRMS`` does. A molecule without atoms (and so without pairs) gets empty lists.
    ``numThreads`` is ignored. ``coordinates`` and ``stream`` as in :func:`GetConformerRMSMatrixBatch`.
    ``prealigned``: the minimum of the RMSDs on the coordinates as given (RDKit ``CalcRMS``).

    Raises ValueError for a ``None`` molecule, ``maxMatches < 1``, a non-empty ``weights``, a bad ``maps`` entry or a
    molecule with conformers but no atoms, TypeError for a bad ``stream``; all before any device work.
    """
    _check_stream(stream)
    mols = _check_mols(mols)
    if int(maxMatches) < 1:
        raise ValueError(f"maxMatches must be >= 1, got {maxMatches}")
    if weights is not None and len(weights):
        raise ValueError("weights are not supported: weighted RMSD is not computed")
    if maps is not None:
        maps = list(maps)
        if len(maps) != len(mols):
            raise ValueError(f"maps holds {len(maps)} entries, mols has {len(mols)}")
    lists = []
    for m, mol in enumerate(mols):
        n = mol.GetNumAtoms()
        if maps is not None and maps[m] is not None:
            lists.append(_map_lists(maps[m], n, f"maps[{m}]"))
        elif n == 0:
            lists.append(_atom_ids_lists(None, 0, f"mol at index {m}"))
        else:
            lists.append(_self_match_lists(mol, int(maxMatches), bool(symmetrizeConjugatedTerminalGroups), m))
    return _batch(mols, prealigned, stream, coordinates, lists)


def GetAllConformerBestRMS(mol, numThreads: int = 1, maxMatches: int = 1000000,
                           symmetrizeConjugatedTerminalGroups: bool = True, weights=None,
                           stream: Optional[torch.cuda.Stream] = None, *, map=None,
                           coordinates: Optional[Device3DResult] = None, prealigned: bool = False) -> AsyncGpuResult:
    """The symmetry-aware RMSD matrix of one molecule's conformers (:func:`GetAllConformerBestRMSBatch` of ``[mol]``,
    ``map`` as one entry of its ``maps``)."""
    _check_stream(stream)
    if mol is None:
        raise ValueError("mol must not be None")
    return GetAllConformerBestRMSBatch([mol], numThreads, maxMatches, symmetrizeConjugatedTerminalGroups, weights,
                                       stream, maps=[map], coordinates=coordinates, prealigned=prealigned)[0]
