"""Result / option types of the hot path, mirroring ``nvmolkit/types.py`` of the reference (types.py:26-319)."""

from __future__ import annotations

from enum import Enum
from typing import Any, Iterable, List, NamedTuple, Optional

import torch


class HardwareOptions:
    """Batching knobs (reference: nvmolkit/types.py:26-122, src/hardware_options.h:26-35).

    This package runs one process per GPU and one persistent kernel per call, so ``batchSize`` /
    ``batchesPerGpu`` only bound how many conformers are resident at once; ``gpuIds`` selects the device
    (the first id) inside a single process. The fields, validation and (de)serialisation match the reference.
    """

    def __init__(self, preprocessingThreads: int = -1, batchSize: int = -1, batchesPerGpu: int = -1,
                 gpuIds: Iterable[int] | None = None) -> None:
        self.preprocessingThreads = int(preprocessingThreads)
        self.batchSize = int(batchSize)
        self._batchesPerGpu = -1
        self.batchesPerGpu = batchesPerGpu
        self.gpuIds = list(gpuIds) if gpuIds is not None else []

    @property
    def batchesPerGpu(self) -> int:
        return self._batchesPerGpu

    @batchesPerGpu.setter
    def batchesPerGpu(self, value: int) -> None:
        value = int(value)
        if value != -1 and value <= 0:
            raise ValueError("batchesPerGpu must be greater than 0 or -1 for automatic")
        self._batchesPerGpu = value

    def to_dict(self) -> dict[str, Any]:
        return {"preprocessingThreads": self.preprocessingThreads, "batchSize": self.batchSize,
                "batchesPerGpu": self.batchesPerGpu, "gpuIds": list(self.gpuIds)}

    @classmethod
    def from_dict(cls, data: dict[str, Any]) -> "HardwareOptions":
        known = {"preprocessingThreads", "batchSize", "batchesPerGpu", "gpuIds"}
        unknown = set(data) - known
        if unknown:
            raise KeyError(f"Unknown HardwareOptions keys: {sorted(unknown)}")
        return cls(**{key: data[key] for key in known if key in data})


class AsyncGpuResult:
    """Handle to a GPU result (reference: nvmolkit/types.py:125-162). Asynchronous: synchronise before reading."""

    def __init__(self, obj, gpu_id: Optional[int] = None):
        if isinstance(obj, torch.Tensor):
            self.arr = obj
            return
        if not hasattr(obj, "__cuda_array_interface__"):
            raise TypeError(f"Object {obj} does not have a __cuda_array_interface__ attribute")
        device = "cuda" if gpu_id is None else f"cuda:{int(gpu_id)}"
        self.arr = torch.as_tensor(obj, device=device)

    @property
    def __cuda_array_interface__(self):
        return self.arr.__cuda_array_interface__

    @property
    def device(self):
        return self.arr.device

    def torch(self):
        return self.arr

    def numpy(self):
        torch.cuda.synchronize()
        return self.arr.cpu().numpy()


class CoordinateOutput(Enum):
    RDKIT_CONFORMERS = "rdkit"
    DEVICE = "device"


class Dense3DResult(NamedTuple):
    values: "torch.Tensor"
    conf_mask: "torch.Tensor"
    atom_mask: "torch.Tensor"


class Device3DResult:
    """On-device CSR conformer result (reference: nvmolkit/types.py:196-319, src/conformer/device_coord_result.h:58-67)."""

    def __init__(self, values: AsyncGpuResult, atom_starts: AsyncGpuResult, mol_indices: AsyncGpuResult,
                 conf_indices: AsyncGpuResult, gpu_id: int, n_mols: int, energies: Optional[AsyncGpuResult] = None,
                 converged: Optional[AsyncGpuResult] = None) -> None:
        self.values = values
        self.atom_starts = atom_starts
        self.mol_indices = mol_indices
        self.conf_indices = conf_indices
        self.energies = energies
        self.converged = converged
        self.gpu_id = int(gpu_id)
        self.n_mols = int(n_mols)

    @property
    def num_conformers(self) -> int:
        return int(self.atom_starts.torch().numel()) - 1

    def per_molecule(self) -> List[List["torch.Tensor"]]:
        values = self.values.torch()
        atom_starts = self.atom_starts.torch().tolist()
        mol_indices = self.mol_indices.torch().tolist()
        result: List[List[torch.Tensor]] = [[] for _ in range(self.n_mols)]
        for conf_idx, mol_idx in enumerate(mol_indices):
            result[mol_idx].append(values[atom_starts[conf_idx]:atom_starts[conf_idx + 1]])
        return result

    def dense(self, pad_value: float = float("nan")) -> Dense3DResult:
        values = self.values.torch()
        atom_starts = self.atom_starts.torch().to(torch.int64)
        mol_indices = self.mol_indices.torch().to(torch.int64)
        conf_indices = self.conf_indices.torch().to(torch.int64)
        device, dtype = values.device, values.dtype
        if mol_indices.numel() == 0:
            return Dense3DResult(torch.full((self.n_mols, 0, 0, 3), pad_value, dtype=dtype, device=device),
                                 torch.zeros((self.n_mols, 0), dtype=torch.bool, device=device),
                                 torch.zeros((self.n_mols, 0, 0), dtype=torch.bool, device=device))
        sizes = atom_starts[1:] - atom_starts[:-1]
        max_confs = int(torch.bincount(mol_indices, minlength=self.n_mols).max().item())
        max_atoms = int(sizes.max().item())
        dense_vals = torch.full((self.n_mols, max_confs, max_atoms, 3), pad_value, dtype=dtype, device=device)
        conf_mask = torch.zeros((self.n_mols, max_confs), dtype=torch.bool, device=device)
        atom_mask = torch.zeros((self.n_mols, max_confs, max_atoms), dtype=torch.bool, device=device)
        conf_mask[mol_indices, conf_indices] = True
        mol_per_atom = mol_indices.repeat_interleave(sizes)
        conf_per_atom = conf_indices.repeat_interleave(sizes)
        within = torch.arange(values.shape[0], device=device, dtype=torch.int64) - atom_starts[:-1].repeat_interleave(sizes)
        dense_vals[mol_per_atom, conf_per_atom, within, :] = values
        atom_mask[mol_per_atom, conf_per_atom, within] = True
        return Dense3DResult(dense_vals, conf_mask, atom_mask)
