"""Morgan fingerprints on the GPU. API of ``nvmolkit/fingerprints.py`` (reference :25-108)."""

from __future__ import annotations

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._interop import require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.molgraph import MolGraphBatch, from_rdkit
from nvmolkit_b200.types import AsyncGpuResult

_VALID_FP_SIZES = (128, 256, 512, 1024, 2048)
_SIZE_CLASSES = (32, 64, 128, 256)  # atoms/bonds per molecule; larger molecules share one last class


def unpack_fingerprint(fp: torch.Tensor) -> torch.Tensor:
    """(n, fpSize/32) packed int32 -> (n, fpSize) bool."""
    if fp.dtype not in (torch.int32, torch.uint32):
        raise ValueError("Input tensor must have dtype int32 or uint32")
    n_fps, n_ints = fp.shape
    shifts = torch.arange(0, 32, device=fp.device, dtype=torch.int32)
    return ((fp.to(torch.int32).unsqueeze(2) >> shifts) & 1).bool().reshape(n_fps, n_ints * 32)


def pack_fingerprint(fp: torch.Tensor) -> torch.Tensor:
    """(n, fpSize) bool -> (n, ceil(fpSize/32)) packed int32, bit j -> word j//32, bit j%32."""
    n_fps, fp_size = fp.shape
    n_ints = (fp_size + 31) // 32
    if fp_size % 32 != 0:
        padded = torch.zeros((n_fps, n_ints * 32), dtype=torch.bool, device=fp.device)
        padded[:, :fp_size] = fp
        fp = padded
    powers = 1 << torch.arange(0, 32, device=fp.device, dtype=torch.int32)
    return (fp.reshape(n_fps, n_ints, 32) * powers.unsqueeze(0)).sum(dim=2, dtype=torch.int32)


class MorganFingerprintGenerator:
    """Morgan fingerprint generator (radius, fpSize in {128, 256, 512, 1024, 2048})."""

    def __init__(self, radius: int, fpSize: int):
        if fpSize not in _VALID_FP_SIZES:
            raise ValueError(f"fpSize must be one of {list(_VALID_FP_SIZES)}, got {fpSize}")
        if radius < 0:
            raise ValueError("radius must be non-negative")
        self.radius = int(radius)
        self.fpSize = int(fpSize)

    def GetFingerprints(self, mols, num_threads: int = 0, stream: torch.cuda.Stream | None = None) -> AsyncGpuResult:
        """``mols``: list of RDKit molecules, or a pre-flattened ``MolGraphBatch``. Returns int32 (n, fpSize/32)."""
        sptr = stream_ptr(stream)
        require_cuda()
        batch = mols if isinstance(mols, MolGraphBatch) else from_rdkit(list(mols))
        return AsyncGpuResult(self._run(batch, stream, sptr, "b200mol_morgan", self.fpSize // 32))

    def GetCountFingerprints(self, mols, num_threads: int = 0,
                             stream: torch.cuda.Stream | None = None) -> AsyncGpuResult:
        """Count twin of ``GetFingerprints``: int32 (n, fpSize), row i, bin j the number of accepted environments of
        molecule i whose code is j modulo fpSize (every atom at radius 0; an environment whose bond set an earlier one
        already had does not count). RDKit's ``GetCountFingerprintAsNumPy`` of ``GetMorganGenerator(radius, fpSize)``;
        ``pack_fingerprint(counts > 0)`` is ``GetFingerprints`` bit for bit. Same inputs, size classes and refusals."""
        sptr = stream_ptr(stream)
        require_cuda()
        batch = mols if isinstance(mols, MolGraphBatch) else from_rdkit(list(mols))
        return AsyncGpuResult(self._run(batch, stream, sptr, "b200mol_morgan_counts", self.fpSize))

    def _run(self, batch: MolGraphBatch, stream, sptr: int, entry: str, width: int) -> torch.Tensor:
        """(n, width) int32 from ``entry`` (b200mol_morgan or b200mol_morgan_counts), one call per size class"""
        n = len(batch)
        dev = torch.device("cuda", torch.cuda.current_device())
        with stream_ctx(stream):
            out = torch.empty((n, width), dtype=torch.int32, device=dev)
            if n == 0:
                return out
            size = np.maximum(batch.atoms_per_mol, batch.bonds_per_mol)
            cls = np.searchsorted(np.array(_SIZE_CLASSES), size, side="left")
            for c in np.unique(cls):
                idx = np.nonzero(cls == c)[0]
                sub = batch if len(idx) == n else batch.select(idx)
                t = [torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else
                                      (a.view(np.int16) if a.dtype == np.uint16 else a)).to(dev, non_blocking=True)
                     for a in (sub.atom_starts, sub.bond_starts, sub.atom_inv, sub.bond_inv, sub.bond_a, sub.bond_b)]
                dst = out if len(idx) == n else torch.empty((len(idx), width), dtype=torch.int32, device=dev)
                _lib.call(entry, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(),
                          t[4].data_ptr(), t[5].data_ptr(), len(idx), int(sub.atoms_per_mol.max(initial=0)),
                          int(sub.bonds_per_mol.max(initial=0)), self.radius, self.fpSize, dst.data_ptr(), sptr)
                if dst is not out:
                    out[torch.from_numpy(idx).to(dev)] = dst
        return out
