"""Conformer alignment on the GPU (RDKit ``rdMolAlign.AlignMolConformers``, ``AlignMol`` and ``GetAlignmentTransform``;
and, over atom mappings, ``GetBestRMS``, ``GetBestAlignmentTransform`` and ``CalcRMS``).

Every call is one launch of ``b200mol_align`` (``csrc/align.cu``): one alignment job per probe conformer, the weighted
rigid superposition of its listed atoms onto a reference conformer's (Horn's quaternion method, as RDKit's
``AlignPoints``), its RMSD and, for the moving calls, the probe conformer rewritten in place (every atom, not only the
listed ones, as ``MolTransforms::transformConformer``).

Semantics, per job with pairs (p_i, r_i), weights w_i (default 1), L pairs and W = sum w:

* centroids p_bar = sum w p / W, r_bar = sum w r / W and covariance S = sum w (p - p_bar)(r - r_bar)^T; with ``reflect``
  every p is replaced by -p first (the probe's mirror image is aligned);
* lambda = the largest eigenvalue estimate of Horn's 4x4 matrix N(S) after at most ``maxIters`` cyclic Jacobi sweeps, q
  its unit eigenvector, R = R(q), t = r_bar - R p_bar; N = 0 (one pair, or coincident atoms) gives R = I, and when lambda
  is not a simple eigenvalue (collinear atoms) one of the equally good rotations is taken, deterministically;
* RMSD = sqrt(max(0, sum w |p - p_bar|^2 + sum w |r - r_bar|^2 - 2 lambda) / L): divided by the number of pairs, not by W;
* the transform is RDKit's ``Transform3D`` layout: row-major 4 x 4 acting on column vectors, [[+-R, t], [0 0 0 1]].

Differences from RDKit:

* Weights are checked: a weight that is negative or not finite, or weights that sum to 0, are refused (RDKit does not
  validate them).
* Batch forms (:func:`AlignMolConformersBatch`, :func:`AlignMolBatch`, :func:`GetAlignmentTransformBatch`) align many
  molecules in one launch and return :class:`AsyncGpuResult` values; ``AlignMolConformersBatch(coordinates=...)`` aligns
  the conformers of an on-device :class:`~nvmolkit_b200.types.Device3DResult` in place, without a host round trip.
* Sums are formed on coordinates shifted by each job's first pair, not as RDKit's raw sums, so molecules far from the
  origin keep their accuracy.
* Two points restate RDKit's ``MolAlign.cpp`` / ``AlignPoints.cpp`` from their source and are not checked against RDKit
  here: the RMSD divides by L also when weights are given, and ``reflect`` gives x' = -R (x - p_bar) + r_bar (RDKit
  negates the reference side and then applies ``Transform3D::Reflect``). ``tools/export_rdkit_fixtures.py`` writes
  ``tests/golden/rdkit_align.npz`` where RDKit exists, and the tests replay it when it is present.
* Argument errors (a ``None`` molecule, an unknown conformer id, empty, repeated or out-of-range atom indices, a weights
  length mismatch, bad weights, ``maxIters < 1``) raise ValueError, and a bad ``stream`` TypeError, before any device work.

:func:`GetBestRMS`, :func:`GetBestAlignmentTransform` and :func:`CalcRMS` (and their batch forms) compare a probe
conformer with a reference conformer of another molecule object over K atom mappings, in one launch of
``b200mol_best_align`` (``csrc/best_align.cu``). Semantics, restated from RDKit's ``MolAlign.cpp``:

* Mappings: ``ref.GetSubstructMatches(prb, uniquify=False, maxMatches=maxMatches, useChirality=False)``; match t pairs
  probe atom q with reference atom t[q]. With ``symmetrizeConjugatedTerminalGroups`` every match is followed by its
  compositions with the permutations of the probe's conjugated terminal groups (the order, duplicate removal and
  ``maxMatches`` cut of :func:`~nvmolkit_b200.rdkit_adapter.probe_ref_matches`). No match raises ValueError("No
  sub-structure match found between the reference and probe mol"). A user ``map`` (mappings of (probeAtom, refAtom)
  pairs) replaces the matches, and then ``maxMatches`` and the symmetrisation are ignored.
* ``GetBestRMS``: every mapping is aligned as ``AlignMol`` aligns (50 Jacobi sweeps); the result is the first mapping
  with the strictly smallest RMSD, and the probe conformer is moved by its transform, every atom.
  ``GetBestAlignmentTransform``: the same search with ``reflect`` and ``maxIters``; nothing moves; it returns (RMSD,
  transform, the mapping as ((probeAtom, refAtom), ...)). ``CalcRMS``: min over k of sqrt(sum w |p - r_k|^2 / L) on the
  coordinates as given; nothing moves.
* Weights are one per pair in the mapping's order (one per probe atom for the matches), checked as for ``AlignMol``.

Differences from RDKit for these three:

* RDKit symmetrises a copy of the query before matching, so a probe and a reference that draw a carboxylate or a nitro
  group with different bond orders match in RDKit; the restatement here finds no match for them and raises.
  ``tools/export_rdkit_fixtures.py`` writes ``tests/golden/rdkit_best_align.npz`` where RDKit exists, and
  ``tests/test_mol_align_best_rdkit.py`` replays it when it is present; until then the restatement and these semantics
  are not checked against RDKit.
* A user ``map`` is sorted by probe atom, and every mapping must cover the same probe atoms; with weights, every mapping
  must also list them in the same order. The match tuple of ``GetBestAlignmentTransform`` lists pairs by probe atom.
* ``numThreads`` is accepted and ignored. Mapping tables take molecules of fewer than 32768 atoms.
* A probe conformer that is its own pair's reference conformer (``GetBestRMS(mol, mol)`` with the default ids) is
  compared with a copy of itself taken before anything moves, so the RMSD is ~0, as in RDKit. A conformer moved as the
  probe of one pair may not be the reference of another pair of the same call, nor moved twice (ValueError).
* With ``coordinates=Device3DResult`` the call builds one temporary device buffer of the result's coordinates followed
  by the references, and with ``GetBestRMSBatch`` copies the result's part back: every conformer of the result makes
  that round trip (48 B per atom of device traffic and a second copy of ``values`` in device memory), not only the
  listed probes.
* Batch forms (:func:`GetBestRMSBatch`, :func:`CalcRMSBatch`, :func:`GetBestAlignmentTransformBatch`) take many probe
  conformers per molecule pair, find the pair's matches once, and can read and move the probes of a
  :class:`~nvmolkit_b200.types.Device3DResult` on the device.
"""

from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._hostutil import device_conformer_order
from nvmolkit_b200._interop import require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.conformerRmsd import _check_list, _check_mols, _check_stream
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult

__all__ = ["AlignMolConformers", "AlignMolConformersBatch", "AlignMol", "AlignMolBatch", "GetAlignmentTransform",
           "GetAlignmentTransformBatch", "GetBestRMS", "GetBestRMSBatch", "CalcRMS", "CalcRMSBatch",
           "GetBestAlignmentTransform", "GetBestAlignmentTransformBatch"]


def _check_iters(maxIters) -> int:
    if int(maxIters) < 1:
        raise ValueError(f"maxIters must be >= 1, got {maxIters}")
    return int(maxIters)


def _weights(weights, L: int, what: str) -> Optional[np.ndarray]:
    """float64 weights for L pairs, or None for all 1 (``None`` or empty, RDKit's default)."""
    if weights is None or len(weights) == 0:
        return None
    arr = np.asarray(weights, np.float64)
    if arr.ndim != 1 or len(arr) != L:
        raise ValueError(f"{what} holds {len(arr)} weights, {L} expected")
    if not np.all(np.isfinite(arr)) or np.any(arr < 0):
        raise ValueError(f"{what} must be finite and >= 0")
    if arr.sum() <= 0:
        raise ValueError(f"{what} sum to 0")
    return arr


def _per_mol(arg, n: int, what: str) -> list:
    if arg is None:
        return [None] * n
    arg = list(arg)
    if len(arg) != n:
        raise ValueError(f"{what} holds {len(arg)} entries, {n} expected")
    return arg


class PairLists:
    """The pair-list tables of ``b200mol_align``: list l holds ``pairs[start[l]:start[l + 1]]`` (probe atom, reference
    atom) with optional weights."""

    def __init__(self):
        self._pairs, self._weights, self._keys = [], [], {}

    def add(self, pairs: np.ndarray, weights: Optional[np.ndarray], key=None) -> int:
        """Index of the list; lists added again under the same ``key`` are stored once."""
        if key is not None and key in self._keys:
            return self._keys[key]
        self._pairs.append(np.asarray(pairs, np.int32).reshape(-1, 2))
        self._weights.append(weights)
        if key is not None:
            self._keys[key] = len(self._pairs) - 1
        return len(self._pairs) - 1

    def find(self, key) -> Optional[int]:
        return self._keys.get(key)

    def max_atoms(self, index: int) -> Tuple[int, int]:
        """The largest probe and reference atom index of list ``index``."""
        p = self._pairs[index]
        return int(p[:, 0].max()), int(p[:, 1].max())

    def tables(self):
        start = np.concatenate([[0], np.cumsum([len(p) for p in self._pairs])]).astype(np.int64)
        pairs = np.ascontiguousarray(np.concatenate(self._pairs) if self._pairs else np.zeros((0, 2)), np.int32)
        weights = None
        if any(w is not None for w in self._weights):
            weights = np.concatenate([np.ones(len(p)) if w is None else w for p, w in zip(self._pairs, self._weights)])
        return start, pairs, weights


def _run(probe, ref, lst, conf_atoms, d_cas: torch.Tensor, xyz: torch.Tensor, lists: PairLists, reflect: bool,
         maxIters: int, move: bool, transform: bool, stream) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """One ``b200mol_align`` launch on ``stream``: (RMSD [n], transforms [n, 4, 4] or None)."""
    probe, ref, lst = (np.ascontiguousarray(x, np.int32) for x in (probe, ref, lst))
    conf_atoms = np.ascontiguousarray(conf_atoms, np.int32)
    start, pairs, weights = lists.tables()
    n = len(probe)
    rmsd = torch.empty(n, dtype=torch.float64, device=xyz.device)
    trans = torch.empty((n, 4, 4), dtype=torch.float64, device=xyz.device) if transform else None
    _lib.call("b200mol_align", n, probe.ctypes.data, ref.ctypes.data, lst.ctypes.data, len(conf_atoms),
              conf_atoms.ctypes.data, d_cas.data_ptr(), xyz.data_ptr(), len(start) - 1, start.ctypes.data,
              pairs.ctypes.data, None if weights is None else weights.ctypes.data, 1 if reflect else 0, maxIters,
              1 if move else 0, rmsd.data_ptr() if n else None, trans.data_ptr() if transform and n else None,
              stream_ptr(stream))
    return rmsd, trans


# ---------------------------------------------------------------------------------------------- AlignMolConformers
def AlignMolConformersBatch(mols, atomIds=None, confIds=None, weights=None, reflect: bool = False, maxIters: int = 50, *,
                            coordinates: Optional[Device3DResult] = None,
                            stream: Optional[torch.cuda.Stream] = None) -> List[AsyncGpuResult]:
    """``AlignMolConformers`` for every molecule, in one launch.

    Per molecule, the reference is the first of its ``confIds`` (or its first conformer), and every other listed
    conformer (or every other conformer) is aligned onto it and moved; the reference and unlisted conformers are left
    as they are. Returns one :class:`AsyncGpuResult` per molecule: the float64 RMSDs of its aligned conformers, in
    order (C - 1 values for C listed conformers; empty for fewer than two).

    ``atomIds``, ``confIds``, ``weights``: one entry per molecule, each ``None`` or as in ``AlignMolConformers``
    (``weights``: one per atom of ``atomIds``, or per atom of the molecule).

    ``coordinates``: a :class:`Device3DResult` whose molecule m pairs with ``mols[m]``; its conformers are aligned in
    place on the device, asynchronously on ``stream``, taken in ``conf_indices`` order, and ``confIds`` name
    ``conf_indices`` values. Its ``values`` must be a contiguous float64 (n, 3) tensor; ``energies`` and ``converged``
    stay valid, since a rigid motion keeps them. Without it, the molecules' RDKit conformers are read, aligned and
    written back.
    """
    _check_stream(stream)
    mols = _check_mols(mols)
    maxIters = _check_iters(maxIters)
    nm = len(mols)
    atomIds, confIds, weights = (_per_mol(a, nm, w) for a, w in ((atomIds, "atomIds"), (confIds, "confIds"),
                                                               (weights, "weights")))
    atom_counts = np.array([mol.GetNumAtoms() for mol in mols], np.int64)
    sel = []
    for m in range(nm):
        n = int(atom_counts[m])
        ids = np.arange(n, dtype=np.int64) if atomIds[m] is None else _check_list(list(atomIds[m]), n, f"atomIds[{m}]")
        sel.append((ids, _weights(weights[m], len(ids), f"weights[{m}]")))

    if coordinates is None:
        confs = [mol.GetConformers() for mol in mols]
        conf_counts = np.array([len(c) for c in confs], np.int64)
        ids_of = [[c.GetId() for c in cs] for cs in confs]
        order = None
    else:
        if not isinstance(coordinates, Device3DResult):
            raise TypeError(f"coordinates must be a Device3DResult, got {type(coordinates).__name__}")
        if coordinates.n_mols != nm:
            raise ValueError(f"coordinates hold {coordinates.n_mols} molecules, mols has {nm}")
        values = coordinates.values.torch()
        if values.dtype != torch.float64 or values.ndim != 2 or values.shape[1] != 3 or not values.is_contiguous():
            raise ValueError("coordinates.values must be a contiguous float64 (n, 3) tensor to be aligned in place")
        order, conf_counts, starts_t = device_conformer_order(coordinates, atom_counts)
        if any(c is not None for c in confIds):
            conf_idx = coordinates.conf_indices.torch().cpu().numpy().astype(np.int64)[order]
        else:
            conf_idx = np.zeros(len(order), np.int64)
        first = np.concatenate([[0], np.cumsum(conf_counts)])
        ids_of = [conf_idx[first[m]:first[m + 1]].tolist() for m in range(nm)]

    # jobs: (probe, reference) positions in the molecule-by-molecule conformer order
    first = np.concatenate([[0], np.cumsum(conf_counts)]).astype(np.int64)
    lists = PairLists()
    probe, ref, lst, sizes = [], [], [], []
    for m in range(nm):
        if confIds[m] is None:
            pos = list(range(int(conf_counts[m])))
        else:
            where = {cid: k for k, cid in enumerate(ids_of[m])}
            pos = []
            for cid in confIds[m]:
                if int(cid) not in where:
                    raise ValueError(f"mol at index {m} has no conformer with id {cid}")
                pos.append(where[int(cid)])
            if len(set(pos)) != len(pos):
                raise ValueError(f"confIds[{m}] names a conformer twice")
        sizes.append(max(len(pos) - 1, 0))
        if len(pos) < 2:
            continue
        ids, w = sel[m]
        if len(ids) == 0:
            raise ValueError(f"mol at index {m} has conformers but no atoms")
        li = lists.add(np.stack([ids, ids], 1), w)
        probe += [first[m] + p for p in pos[1:]]
        ref += [first[m] + pos[0]] * (len(pos) - 1)
        lst += [li] * (len(pos) - 1)
    if not probe:
        return [AsyncGpuResult(torch.zeros(s, dtype=torch.float64)) for s in sizes]

    require_cuda()
    conf_atoms = np.repeat(atom_counts, conf_counts)
    if coordinates is None:
        host = np.concatenate([np.asarray(c.GetPositions(), np.float64).reshape(-1, 3) for cs in confs for c in cs])
        if len(host) != conf_atoms.sum():
            raise ValueError("a conformer's atom count differs from its molecule's")
        cas = np.concatenate([[0], np.cumsum(conf_atoms)]).astype(np.int32)
        dev = torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev), stream_ctx(stream):
            xyz = torch.from_numpy(np.ascontiguousarray(host)).to(dev)
            d_cas = torch.from_numpy(cas).to(dev)
            rmsd, _ = _run(probe, ref, lst, conf_atoms, d_cas, xyz, lists, reflect, maxIters, True, False, stream)
            out = xyz.cpu().numpy()
        from nvmolkit_b200.rdkit_adapter import write_back_conformers

        bounds = np.concatenate([[0], np.cumsum(conf_atoms)])
        k = 0
        per_mol = []
        for m in range(nm):
            per_mol.append([out[bounds[k + c]:bounds[k + c + 1]] for c in range(int(conf_counts[m]))])
            k += int(conf_counts[m])
        write_back_conformers(mols, per_mol)
    else:
        # conformer k of the order is conformer order[k] of the result
        probe, ref = order[np.asarray(probe)], order[np.asarray(ref)]
        atoms_of = np.empty(len(order), np.int64)
        atoms_of[order] = conf_atoms
        dev = values.device
        with torch.cuda.device(dev), stream_ctx(stream):
            d_cas = starts_t.to(device=dev, dtype=torch.int32).contiguous()
            rmsd, _ = _run(probe, ref, lst, atoms_of, d_cas, values, lists, reflect, maxIters, True, False, stream)
    return [AsyncGpuResult(v) for v in torch.split(rmsd, sizes)]


def AlignMolConformers(mol, atomIds=None, confIds=None, weights=None, reflect: bool = False, maxIters: int = 50,
                       RMSlist=None, *, stream: Optional[torch.cuda.Stream] = None) -> None:
    """Align the conformers of ``mol`` onto its first conformer (or the first of ``confIds``), in place (RDKit
    ``rdMolAlign.AlignMolConformers``). ``RMSlist``, if given, is extended with one RMSD per aligned conformer."""
    _check_stream(stream)
    if mol is None:
        raise ValueError("mol must not be None")
    res = AlignMolConformersBatch([mol], None if atomIds is None else [atomIds], None if confIds is None else [confIds],
                                  None if weights is None else [weights], reflect, maxIters, stream=stream)[0]
    if RMSlist is not None and res.torch().numel():
        RMSlist.extend(float(v) for v in res.numpy())


# ---------------------------------------------------------------------------------------------- AlignMol
def _conformer(mol, cid, what: str):
    confs = mol.GetConformers()
    if not confs:
        raise ValueError(f"{what} has no conformers")
    if int(cid) == -1:
        return confs[0]
    for c in confs:
        if c.GetId() == int(cid):
            return c
    raise ValueError(f"{what} has no conformer with id {cid}")


def _map_pairs(atomMap, n_prb: int, n_ref: int, what: str) -> np.ndarray:
    if atomMap is None or len(atomMap) == 0:
        if n_prb != n_ref:
            raise ValueError(f"{what} is empty: the identity needs equal atom counts, got {n_prb} and {n_ref}")
        if n_prb == 0:
            raise ValueError(f"{what}: the molecules have no atoms")
        ids = np.arange(n_prb, dtype=np.int64)
        return np.stack([ids, ids], 1)
    arr = np.asarray(atomMap)
    if arr.ndim != 2 or arr.shape[1] != 2 or not np.issubdtype(arr.dtype, np.integer):
        raise ValueError(f"{what} must be a list of (probeAtom, refAtom) pairs")
    return np.stack([_check_list(arr[:, 0], n_prb, f"{what} probe atoms"),
                     _check_list(arr[:, 1], n_ref, f"{what} reference atoms")], 1)


def _pairs_batch(prbMols, refMols, prbCids, refCids, atomMaps, weights, reflect, maxIters, stream, move: bool):
    _check_stream(stream)
    prbMols, refMols = _check_mols(prbMols), _check_mols(refMols)
    maxIters = _check_iters(maxIters)
    n = len(prbMols)
    if len(refMols) != n:
        raise ValueError(f"refMols holds {len(refMols)} molecules, prbMols {n}")
    prbCids = [-1] * n if prbCids is None else _per_mol(prbCids, n, "prbCids")
    refCids = [-1] * n if refCids is None else _per_mol(refCids, n, "refCids")
    atomMaps, weights = _per_mol(atomMaps, n, "atomMaps"), _per_mol(weights, n, "weights")
    lists = PairLists()
    slots, blocks, confs = {}, [], []

    def slot(mol, conf):
        key = (id(mol), conf.GetId())
        if key not in slots:
            slots[key] = len(blocks)
            blocks.append(np.asarray(conf.GetPositions(), np.float64).reshape(-1, 3))
            confs.append(conf)
        return slots[key]

    probe, ref, lst = [], [], []
    for i, (prb, refm) in enumerate(zip(prbMols, refMols)):
        rc = _conformer(refm, refCids[i], f"refMols[{i}]")
        amap, w = atomMaps[i], weights[i]
        np_, nr = prb.GetNumAtoms(), refm.GetNumAtoms()
        key = (("identity", np_, nr) if amap is None or len(amap) == 0 else id(amap), id(w) if w is not None else None)
        li = lists.find(key)
        if li is None:
            pairs = _map_pairs(amap, np_, nr, f"atomMaps[{i}]")
            li = lists.add(pairs, _weights(w, len(pairs), f"weights[{i}]"), key)
        elif lists.max_atoms(li)[0] >= np_ or lists.max_atoms(li)[1] >= nr:  # the same map object on other molecules
            raise ValueError(f"atomMaps[{i}] holds an atom index outside its molecules")
        lst.append(li)
        ref.append(slot(refm, rc))
    refs, moved = set(ref), set()
    for i, prb in enumerate(prbMols):
        pc = _conformer(prb, prbCids[i], f"prbMols[{i}]")
        s = slot(prb, pc)
        if move and (s in refs or s in moved):
            raise ValueError(f"prbMols[{i}] conformer {pc.GetId()} is moved twice or is also a reference")
        moved.add(s)
        probe.append(s)
    return probe, ref, lst, lists, blocks, confs, maxIters


def _launch(prbMols, refMols, prbCids, refCids, atomMaps, weights, reflect, maxIters, stream, move):
    probe, ref, lst, lists, blocks, confs, maxIters = _pairs_batch(prbMols, refMols, prbCids, refCids, atomMaps, weights,
                                                                   reflect, maxIters, stream, move)
    conf_atoms = np.array([len(b) for b in blocks], np.int64)
    require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev), stream_ctx(stream):
        xyz = torch.from_numpy(np.ascontiguousarray(np.concatenate(blocks) if blocks else np.zeros((0, 3)))).to(dev)
        d_cas = torch.from_numpy(np.concatenate([[0], np.cumsum(conf_atoms)]).astype(np.int32)).to(dev)
        rmsd, trans = _run(probe, ref, lst, conf_atoms, d_cas, xyz, lists, reflect, maxIters, move, not move, stream)
        if move:
            out = xyz.cpu().numpy()
    if move:
        from rdkit.Geometry import Point3D

        bounds = np.concatenate([[0], np.cumsum(conf_atoms)])
        for s in sorted(set(probe)):
            for a, (x, y, z) in enumerate(out[bounds[s]:bounds[s + 1]]):
                confs[s].SetAtomPosition(a, Point3D(float(x), float(y), float(z)))
    return rmsd, trans


def AlignMolBatch(prbMols, refMols, prbCids=None, refCids=None, atomMaps=None, weights=None, reflect: bool = False,
                  maxIters: int = 50, *, stream: Optional[torch.cuda.Stream] = None) -> AsyncGpuResult:
    """``AlignMol`` of every probe onto its reference in one launch; moves the probe conformers (RDKit conformers, written
    back) and returns the float64 RMSDs. ``prbCids`` / ``refCids``: conformer ids (-1: the first conformer);
    ``atomMaps[i]``: (probeAtom, refAtom) pairs, ``None`` or empty for the identity over all atoms (equal atom counts);
    ``weights[i]``: one per pair, or ``None``. A probe conformer may be moved once and may not be a reference."""
    rmsd, _ = _launch(prbMols, refMols, prbCids, refCids, atomMaps, weights, reflect, maxIters, stream, True)
    return AsyncGpuResult(rmsd)


def GetAlignmentTransformBatch(prbMols, refMols, prbCids=None, refCids=None, atomMaps=None, weights=None,
                               reflect: bool = False, maxIters: int = 50, *,
                               stream: Optional[torch.cuda.Stream] = None) -> Tuple[AsyncGpuResult, AsyncGpuResult]:
    """``GetAlignmentTransform`` of every probe onto its reference in one launch, asynchronously on ``stream``; nothing is
    moved. Returns (RMSDs [n], transforms [n, 4, 4]). A reference conformer shared by many probes (the same molecule
    object and conformer id) is uploaded once; so is an atom map passed as the same object (with the same weights
    object)."""
    rmsd, trans = _launch(prbMols, refMols, prbCids, refCids, atomMaps, weights, reflect, maxIters, stream, False)
    return AsyncGpuResult(rmsd), AsyncGpuResult(trans)


def AlignMol(prbMol, refMol, prbCid: int = -1, refCid: int = -1, atomMap=None, weights=None, reflect: bool = False,
             maxIters: int = 50, *, stream: Optional[torch.cuda.Stream] = None) -> float:
    """Align conformer ``prbCid`` of ``prbMol`` onto conformer ``refCid`` of ``refMol`` in place and return the RMSD
    (RDKit ``rdMolAlign.AlignMol``)."""
    _check_stream(stream)
    return float(AlignMolBatch([prbMol], [refMol], [prbCid], [refCid], [atomMap], [weights], reflect, maxIters,
                               stream=stream).numpy()[0])


def GetAlignmentTransform(prbMol, refMol, prbCid: int = -1, refCid: int = -1, atomMap=None, weights=None,
                          reflect: bool = False, maxIters: int = 50, *,
                          stream: Optional[torch.cuda.Stream] = None) -> Tuple[float, np.ndarray]:
    """(RMSD, 4 x 4 transform) of the best alignment of ``prbMol`` onto ``refMol``; nothing is moved (RDKit
    ``rdMolAlign.GetAlignmentTransform``)."""
    _check_stream(stream)
    rmsd, trans = GetAlignmentTransformBatch([prbMol], [refMol], [prbCid], [refCid], [atomMap], [weights], reflect,
                                             maxIters, stream=stream)
    return float(rmsd.numpy()[0]), trans.numpy()[0]


# ---------------------------------------------------------------------------------------------- GetBestRMS
_NO_MATCH = "No sub-structure match found between the reference and probe mol"


def _pair_lists(prb, ref, mapping, maxMatches: int, symmetrize: bool, weights, what: str):
    """(P, Q, weights in P's order or None) of one molecule pair: the user's ``map``, or the probe's matches inside the
    reference (:func:`~nvmolkit_b200.rdkit_adapter.probe_ref_matches`), P = every probe atom and Q = the matches."""
    from nvmolkit_b200.conformerRmsd import _map_lists

    n_p, n_r = prb.GetNumAtoms(), ref.GetNumAtoms()
    if max(n_p, n_r) >= 32768:
        raise ValueError(f"{what}: mapping tables take molecules of fewer than 32768 atoms")
    if mapping is not None and len(mapping):
        if weights is None or len(weights) == 0:
            P, Q = _map_lists(mapping, n_p, f"{what} map", n_r)
            return P, Q, None
        P, Q, perm = _map_lists(mapping, n_p, f"{what} map", n_r, order=True)
        return P, Q, _weights(weights, len(P), f"{what} weights")[perm]
    from nvmolkit_b200.rdkit_adapter import probe_ref_matches

    w = _weights(weights, n_p, f"{what} weights")
    matches = probe_ref_matches(prb, ref, maxMatches, symmetrize)
    if not matches:
        raise ValueError(_NO_MATCH)
    Q = np.array(matches, np.int64)
    if Q.ndim != 2 or Q.shape[1] != n_p:
        raise ValueError(f"{what}: every match must cover all {n_p} probe atoms")
    return np.arange(n_p, dtype=np.int64), Q, w


def _run_best(probe, ref, sets, conf_atoms, d_cas: torch.Tensor, xyz: torch.Tensor, lists, mode: int, reflect: bool,
              maxIters: int, move: bool, transform: bool, stream):
    """One ``b200mol_best_align`` launch on ``stream``: (RMSD [n], best mapping [n], transforms [n, 4, 4] or None).
    ``lists[s] = (P, Q, weights or None)``: mapping set s."""
    from nvmolkit_b200.conformerRmsd import MapTables

    probe, ref, sets = (np.ascontiguousarray(x, np.int32) for x in (probe, ref, sets))
    conf_atoms = np.ascontiguousarray(conf_atoms, np.int32)
    maps = MapTables([(p, q) for p, q, _ in lists])
    weights = None
    if any(w is not None for _, _, w in lists):
        weights = np.ascontiguousarray(np.concatenate([np.ones(len(p)) if w is None else w for p, _, w in lists]),
                                       np.float64)
    n = len(probe)
    rmsd = torch.empty(n, dtype=torch.float64, device=xyz.device)
    best = torch.empty(n, dtype=torch.int32, device=xyz.device)
    trans = torch.empty((n, 4, 4), dtype=torch.float64, device=xyz.device) if transform else None
    _lib.call("b200mol_best_align", n, probe.ctypes.data, ref.ctypes.data, sets.ctypes.data, len(conf_atoms),
              conf_atoms.ctypes.data, d_cas.data_ptr(), xyz.data_ptr(), len(lists), maps.start.ctypes.data,
              maps.count.ctypes.data, maps.length.ctypes.data, maps.atoms.ctypes.data,
              None if weights is None else weights.ctypes.data, mode, 1 if reflect else 0, maxIters, 1 if move else 0,
              rmsd.data_ptr() if n else None, best.data_ptr() if n else None,
              trans.data_ptr() if transform and n else None, stream_ptr(stream))
    return rmsd, best, trans


def _best_batch(prbMols, refMols, prbIds, refIds, maps, maxMatches, symmetrize, weights, reflect, maxIters, mode: int,
                move: bool, transform: bool, coordinates, stream):
    """The jobs of every molecule pair in one launch: (per-pair sizes, RMSD, best mapping, transforms or None, the
    mapping sets)."""
    _check_stream(stream)
    prbMols, refMols = _check_mols(prbMols), _check_mols(refMols)
    maxIters = _check_iters(maxIters)
    if int(maxMatches) < 1:
        raise ValueError(f"maxMatches must be >= 1, got {maxMatches}")
    n = len(prbMols)
    if len(refMols) != n:
        raise ValueError(f"refMols holds {len(refMols)} molecules, prbMols {n}")
    prbIds, maps, weights = (_per_mol(a, n, w) for a, w in ((prbIds, "prbIds"), (maps, "maps"), (weights, "weights")))
    refIds = [-1] * n if refIds is None else _per_mol(refIds, n, "refIds")

    if coordinates is not None:
        if not isinstance(coordinates, Device3DResult):
            raise TypeError(f"coordinates must be a Device3DResult, got {type(coordinates).__name__}")
        if coordinates.n_mols != n:
            raise ValueError(f"coordinates hold {coordinates.n_mols} molecules, prbMols has {n}")
        values = coordinates.values.torch()
        if values.dtype != torch.float64 or values.ndim != 2 or values.shape[1] != 3 or not values.is_contiguous():
            raise ValueError("coordinates.values must be a contiguous float64 (n, 3) tensor")
        atom_counts = np.array([m.GetNumAtoms() for m in prbMols], np.int64)
        order, dev_counts, starts_t = device_conformer_order(coordinates, atom_counts)
        conf_idx = coordinates.conf_indices.torch().cpu().numpy().astype(np.int64)[order]
        dev_first = np.concatenate([[0], np.cumsum(dev_counts)]).astype(np.int64)
        n_dev = len(order)
        dev_atoms = np.empty(n_dev, np.int64)
        dev_atoms[order] = np.repeat(atom_counts, dev_counts)
    else:
        n_dev = 0

    # RDKit conformers get slots n_dev, n_dev + 1, ...; device conformer c of the result is slot c
    slots, blocks, confs = {}, [], []

    def slot(mol, conf):
        key = (id(mol), conf.GetId())
        if key not in slots:
            slots[key] = n_dev + len(blocks)
            blocks.append(np.asarray(conf.GetPositions(), np.float64).reshape(-1, 3))
            confs.append(conf)
        return slots[key]

    cache, lists = {}, []
    probe, ref, sets, sizes = [], [], [], []
    for m, (prb, refm) in enumerate(zip(prbMols, refMols)):
        rc = _conformer(refm, refIds[m], f"refMols[{m}]")
        key = (id(prb), id(refm), id(maps[m]) if maps[m] is not None and len(maps[m]) else None,
               id(weights[m]) if weights[m] is not None and len(weights[m]) else None)
        if key not in cache:
            cache[key] = len(lists)
            lists.append(_pair_lists(prb, refm, maps[m], int(maxMatches), bool(symmetrize), weights[m],
                                     f"pair {m}"))
        s, r = cache[key], slot(refm, rc)
        if coordinates is None:
            if prbIds[m] is None:
                pcs = [c for c in prb.GetConformers() if not (prb is refm and c.GetId() == rc.GetId())]
            else:
                pcs = [_conformer(prb, cid, f"prbMols[{m}]") for cid in prbIds[m]]
            ps = [slot(prb, c) for c in pcs]
            if r in ps:  # the reference conformer is also this pair's probe: it is read from a copy taken beforehand
                blocks.append(blocks[r - n_dev].copy())
                confs.append(None)
                r = n_dev + len(blocks) - 1
        else:
            mine = order[dev_first[m]:dev_first[m + 1]]
            if prbIds[m] is None:
                ps = [int(c) for c in mine]
            else:
                where = {int(cid): int(c) for cid, c in zip(conf_idx[dev_first[m]:dev_first[m + 1]], mine)}
                ps = []
                for cid in prbIds[m]:
                    if int(cid) not in where:
                        raise ValueError(f"coordinates: molecule {m} has no conformer with id {cid}")
                    ps.append(where[int(cid)])
        probe += ps
        ref += [r] * len(ps)
        sets += [s] * len(ps)
        sizes.append(len(ps))
    if move:
        refs, moved = set(ref), set()
        for p in probe:
            if p in refs or p in moved:
                raise ValueError("a probe conformer is moved twice or is also a reference")
            moved.add(p)
    if not probe:
        empty = torch.zeros(0, dtype=torch.float64)
        return sizes, empty, torch.zeros(0, dtype=torch.int32), torch.zeros((0, 4, 4), dtype=torch.float64) if transform else None, lists

    require_cuda()
    host_atoms = np.array([len(b) for b in blocks], np.int64)
    if coordinates is None:
        dev = torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev), stream_ctx(stream):
            xyz = torch.from_numpy(np.ascontiguousarray(np.concatenate(blocks))).to(dev)
            d_cas = torch.from_numpy(np.concatenate([[0], np.cumsum(host_atoms)]).astype(np.int32)).to(dev)
            rmsd, best, trans = _run_best(probe, ref, sets, host_atoms, d_cas, xyz, lists, mode, reflect, maxIters,
                                          move, transform, stream)
            out = xyz.cpu().numpy() if move else None
        if move:
            from rdkit.Geometry import Point3D

            bounds = np.concatenate([[0], np.cumsum(host_atoms)])
            for p in sorted(set(probe)):
                for a, (x, y, z) in enumerate(out[bounds[p]:bounds[p + 1]]):
                    confs[p].SetAtomPosition(a, Point3D(float(x), float(y), float(z)))
    else:
        dev = values.device
        n_val = values.shape[0]
        with torch.cuda.device(dev), stream_ctx(stream):
            refs_host = np.concatenate(blocks)
            xyz = torch.cat([values, torch.from_numpy(np.ascontiguousarray(refs_host)).to(dev)])
            ref_starts = torch.from_numpy((n_val + np.concatenate([[0], np.cumsum(host_atoms)[:-1]])).astype(np.int32))
            d_cas = torch.cat([starts_t[:n_dev].to(device=dev, dtype=torch.int32), ref_starts.to(dev)]).contiguous()
            rmsd, best, trans = _run_best(probe, ref, sets, np.concatenate([dev_atoms, host_atoms]), d_cas, xyz, lists,
                                          mode, reflect, maxIters, move, transform, stream)
            if move:
                values.copy_(xyz[:n_val])
    return sizes, rmsd, best, trans, lists


def _split(t: Optional[torch.Tensor], sizes) -> List[AsyncGpuResult]:
    return [AsyncGpuResult(v) for v in torch.split(t, sizes)]


def GetBestRMSBatch(prbMols, refMols, prbIds=None, refIds=None, maps=None, maxMatches: int = 1000000,
                    symmetrizeConjugatedTerminalGroups: bool = True, weights=None, *,
                    coordinates: Optional[Device3DResult] = None,
                    stream: Optional[torch.cuda.Stream] = None) -> List[AsyncGpuResult]:
    """``GetBestRMS`` of many probe conformers per molecule pair, in one launch: every listed probe conformer of
    ``prbMols[m]`` is aligned onto conformer ``refIds[m]`` of ``refMols[m]`` by its best mapping and moved. Returns one
    :class:`AsyncGpuResult` per pair: the float64 RMSDs of its probes, in order.

    ``prbIds[m]``: probe conformer ids, ``None`` for every conformer except the reference conformer itself;
    ``refIds[m]``: one reference conformer id (-1: the first); ``maps[m]``: ``None`` for the probe's matches inside the
    reference, or mappings of (probeAtom, refAtom) pairs; ``weights[m]``: one per pair, or ``None``. The matches of a
    pair are found once, whatever its number of conformers.

    ``coordinates``: a :class:`Device3DResult` whose molecule m holds the probe conformers of pair m (``prbIds`` name
    its ``conf_indices`` values); they are moved in place on the device, asynchronously on ``stream``; the references
    still come from ``refMols``. Its ``values`` must be a contiguous float64 (n, 3) tensor. Without it the RDKit
    conformers are read, aligned and written back. A probe conformer may be moved once and may not be the reference of
    another pair; a probe that is its own pair's reference is aligned onto a copy of itself."""
    sizes, rmsd, _, _, _ = _best_batch(prbMols, refMols, prbIds, refIds, maps, maxMatches,
                                       symmetrizeConjugatedTerminalGroups, weights, False, 50, 0, True, False,
                                       coordinates, stream)
    return _split(rmsd, sizes)


def CalcRMSBatch(prbMols, refMols, prbIds=None, refIds=None, maps=None, maxMatches: int = 1000000,
                 symmetrizeConjugatedTerminalGroups: bool = True, weights=None, *,
                 coordinates: Optional[Device3DResult] = None,
                 stream: Optional[torch.cuda.Stream] = None) -> List[AsyncGpuResult]:
    """``CalcRMS`` as :func:`GetBestRMSBatch` lays it out: per probe the smallest RMSD over the mappings on the
    coordinates as given, without alignment. Nothing is moved."""
    sizes, rmsd, _, _, _ = _best_batch(prbMols, refMols, prbIds, refIds, maps, maxMatches,
                                       symmetrizeConjugatedTerminalGroups, weights, False, 50, 1, False, False,
                                       coordinates, stream)
    return _split(rmsd, sizes)


def GetBestAlignmentTransformBatch(prbMols, refMols, prbIds=None, refIds=None, maps=None, maxMatches: int = 1000000,
                                   symmetrizeConjugatedTerminalGroups: bool = True, weights=None,
                                   reflect: bool = False, maxIters: int = 50, *,
                                   coordinates: Optional[Device3DResult] = None,
                                   stream: Optional[torch.cuda.Stream] = None
                                   ) -> Tuple[List[AsyncGpuResult], List[AsyncGpuResult], List[AsyncGpuResult]]:
    """``GetBestAlignmentTransform`` as :func:`GetBestRMSBatch` lays it out; nothing is moved. Returns per pair (RMSDs,
    float64 transforms [n, 4, 4], int32 index of the best mapping: into ``maps[m]``, or into the pair's matches)."""
    sizes, rmsd, best, trans, _ = _best_batch(prbMols, refMols, prbIds, refIds, maps, maxMatches,
                                              symmetrizeConjugatedTerminalGroups, weights, reflect, maxIters, 0, False,
                                              True, coordinates, stream)
    return _split(rmsd, sizes), _split(trans, sizes), _split(best, sizes)


def _one(prbMol, refMol, prbId, refId, map, maxMatches, symmetrize, weights, reflect, maxIters, mode, move, transform,
         stream):
    _check_stream(stream)
    if prbMol is None or refMol is None:
        raise ValueError("prbMol and refMol must not be None")
    prbId = _conformer(prbMol, prbId, "prbMol").GetId()
    return _best_batch([prbMol], [refMol], [[prbId]], [refId], [map], maxMatches, symmetrize, [weights], reflect,
                       maxIters, mode, move, transform, None, stream)


def GetBestRMS(prbMol, refMol, prbId: int = -1, refId: int = -1, map=None, maxMatches: int = 1000000,
               symmetrizeConjugatedTerminalGroups: bool = True, weights=None, numThreads: int = 1, *,
               stream: Optional[torch.cuda.Stream] = None) -> float:
    """The RMSD of conformer ``prbId`` of ``prbMol`` aligned onto conformer ``refId`` of ``refMol`` by the best of their
    atom mappings, and the probe conformer moved by that alignment (RDKit ``rdMolAlign.GetBestRMS``)."""
    _, rmsd, _, _, _ = _one(prbMol, refMol, prbId, refId, map, maxMatches, symmetrizeConjugatedTerminalGroups, weights,
                            False, 50, 0, True, False, stream)
    return float(rmsd.cpu()[0])


def CalcRMS(prbMol, refMol, prbId: int = -1, refId: int = -1, map=None, maxMatches: int = 1000000,
            symmetrizeConjugatedTerminalGroups: bool = True, weights=None, *,
            stream: Optional[torch.cuda.Stream] = None) -> float:
    """The smallest RMSD over the atom mappings between two conformers as they are, without alignment (RDKit
    ``rdMolAlign.CalcRMS``); nothing is moved."""
    _, rmsd, _, _, _ = _one(prbMol, refMol, prbId, refId, map, maxMatches, symmetrizeConjugatedTerminalGroups, weights,
                            False, 50, 1, False, False, stream)
    return float(rmsd.cpu()[0])


def GetBestAlignmentTransform(prbMol, refMol, prbId: int = -1, refId: int = -1, map=None, maxMatches: int = 1000000,
                              symmetrizeConjugatedTerminalGroups: bool = True, weights=None, reflect: bool = False,
                              maxIters: int = 50, numThreads: int = 1, *, stream: Optional[torch.cuda.Stream] = None
                              ) -> Tuple[float, np.ndarray, Tuple[Tuple[int, int], ...]]:
    """(RMSD, 4 x 4 transform, the best mapping as ((probeAtom, refAtom), ...)) of the best alignment of ``prbMol`` onto
    ``refMol`` over their atom mappings; nothing is moved (RDKit ``rdMolAlign.GetBestAlignmentTransform``). The pairs
    are listed by probe atom."""
    _, rmsd, best, trans, lists = _one(prbMol, refMol, prbId, refId, map, maxMatches,
                                       symmetrizeConjugatedTerminalGroups, weights, reflect, maxIters, 0, False, True,
                                       stream)
    P, Q, _ = lists[0]
    k = int(best.cpu()[0])
    return float(rmsd.cpu()[0]), trans.cpu().numpy()[0], tuple((int(p), int(q)) for p, q in zip(P, Q[k]))
