"""Conformer RMSD matrices on the GPU (RDKit ``AllChem.GetConformerRMSMatrix``; reference:
``nvmolkit/conformerRmsd.py``).

:func:`GetConformerRMSMatrix` / :func:`GetConformerRMSMatrixBatch` keep the reference's names, arguments, return types
and errors. They compute with ``b200mol_conformer_rmsd`` (``csrc/conformer_rmsd.cu``): every pair's 3x3 covariance is a
block of one fp64 tensor-core Gram product per molecule, and the best superposition follows in closed form. Coordinates
come from the molecules' RDKit conformers or, with ``coordinates=``, from an on-device
:class:`~nvmolkit_b200.types.Device3DResult` (``EmbedMolecules(output=DEVICE)``), so conformers can stay on the GPU from
embedding through minimisation and this matrix to :func:`nvmolkit_b200.clustering.butina`.

Semantics:

* The RMSD uses every atom of the molecule (strip hydrogens first for a heavy-atom RMSD).
* ``prealigned=False``: the RMSD after the best proper rigid superposition (rotation and translation, no reflection),
  ``sqrt(max(0, Ga + Gb - 2 (s1 + s2 + sign(det H) s3)) / n)`` on centred coordinates. RDKit's own function first aligns
  every conformer to conformer 0 in place; here the input coordinates are never modified.
* ``prealigned=True``: ``sqrt(sum |a - b|^2 / n)`` on the coordinates as given.
* Per molecule with C conformers: a float64 vector of C(C-1)/2 values, pair (i, j), i > j, at ``i(i-1)/2 + j``; fewer
  than two conformers give an empty vector. Results are bitwise repeatable, and a molecule's matrix does not depend on
  the other molecules of the batch.
"""

from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._hostutil import device_conformer_order
from nvmolkit_b200._interop import require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult

__all__ = ["GetConformerRMSMatrix", "GetConformerRMSMatrixBatch"]


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


def _run(conf_counts: np.ndarray, atom_counts: np.ndarray, conf_order: Optional[torch.Tensor],
         conf_atom_start: torch.Tensor, xyz: torch.Tensor, prealigned: bool, stream) -> List[AsyncGpuResult]:
    offsets = pair_offsets(conf_counts)
    mcs = np.concatenate([[0], np.cumsum(conf_counts)]).astype(np.int32)
    atoms = np.ascontiguousarray(atom_counts, np.int32)
    total = int(offsets[-1])
    out = torch.empty(total, dtype=torch.float64, device=xyz.device)
    _lib.call("b200mol_conformer_rmsd", len(conf_counts), mcs.ctypes.data, atoms.ctypes.data,
              conf_order.data_ptr() if conf_order is not None else None, conf_atom_start.data_ptr(), xyz.data_ptr(),
              1 if prealigned else 0, out.data_ptr() if total else None, stream_ptr(stream))
    return [AsyncGpuResult(v) for v in torch.split(out, np.diff(offsets).tolist())]  # one call for all the views


def GetConformerRMSMatrixBatch(mols, prealigned: bool = False, stream: Optional[torch.cuda.Stream] = None, *,
                               coordinates: Optional[Device3DResult] = None) -> List[AsyncGpuResult]:
    """Pairwise RMSD matrices of the conformers of every molecule, in one launch.

    Returns one :class:`AsyncGpuResult` per molecule, in the order of ``mols``: a float64 vector of C(C-1)/2 values
    for C conformers, pair (i, j), i > j, at ``i(i-1)/2 + j`` (RDKit's lower-triangle order), empty for fewer than two
    conformers. The results are views of one device buffer, computed asynchronously on ``stream`` (default: the
    current stream).

    ``coordinates``: a :class:`Device3DResult` whose molecule m pairs with ``mols[m]``; its conformers are read on the
    device, in ``conf_indices`` order (its index tables are copied to the host once to plan the call). Without it the
    molecules' RDKit conformers are used.

    Raises ValueError for a ``None`` molecule or a molecule with conformers but no atoms, TypeError for a ``stream``
    that is not a ``torch.cuda.Stream`` or None; both before any device work.
    """
    _check_stream(stream)
    mols = list(mols)
    for i, mol in enumerate(mols):
        if mol is None:
            raise ValueError(f"mol at index {i} must not be None")
    atom_counts = np.array([mol.GetNumAtoms() for mol in mols], np.int64)
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
            return _run(conf_counts, atom_counts, None, d_cas, xyz, prealigned, stream)

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
        return _run(conf_counts, atom_counts, d_order, d_cas, xyz.to(torch.float64).contiguous(), prealigned, stream)


def GetConformerRMSMatrix(mol, prealigned: bool = False, stream: Optional[torch.cuda.Stream] = None, *,
                          coordinates: Optional[Device3DResult] = None) -> AsyncGpuResult:
    """The RMSD matrix of one molecule's conformers (:func:`GetConformerRMSMatrixBatch` of ``[mol]``).

    Raises ValueError if ``mol`` is None or has conformers but no atoms, TypeError for a bad ``stream``."""
    _check_stream(stream)
    if mol is None:
        raise ValueError("mol must not be None")
    return GetConformerRMSMatrixBatch([mol], prealigned, stream, coordinates=coordinates)[0]
