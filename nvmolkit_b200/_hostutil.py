"""Vectorised host-side index bookkeeping (no per-conformer Python loops: batches reach 1e6 conformers)."""

from __future__ import annotations

import numpy as np


def rows_of(starts: np.ndarray, order: np.ndarray) -> np.ndarray:
    """Concatenation of arange(starts[c], starts[c+1]) for c in `order` (CSR row gather), int64."""
    from nvmolkit_b200 import _lib

    mod = _lib.core()
    if mod is not None:
        return mod.rows_of(np.ascontiguousarray(starts, dtype=np.int64), np.ascontiguousarray(order, dtype=np.int64))
    starts = np.asarray(starts, dtype=np.int64)
    order = np.asarray(order, dtype=np.int64)
    sizes = starts[order + 1] - starts[order]
    total = int(sizes.sum())
    if total == 0:
        return np.zeros(0, dtype=np.int64)
    out_start = np.cumsum(sizes) - sizes
    return np.repeat(starts[order] - out_start, sizes) + np.arange(total, dtype=np.int64)


def device_conformer_order(coordinates, atom_counts):
    """Host plan of a :class:`~nvmolkit_b200.types.Device3DResult` whose molecule m pairs with the m-th entry of
    ``atom_counts``: ``(order, counts, atom_starts)``, where ``order`` (int32) lists the result's conformers molecule by
    molecule in ``conf_indices`` order, ``counts`` (int64) is the number of conformers per molecule and ``atom_starts``
    is the result's device tensor. Its index tables are copied to the host once. Raises ValueError for a molecule
    index outside ``atom_counts`` or a conformer whose atom count differs from its molecule's."""
    mol_idx = coordinates.mol_indices.torch().cpu().numpy().astype(np.int64)
    conf_idx = coordinates.conf_indices.torch().cpu().numpy().astype(np.int64)
    starts_t = coordinates.atom_starts.torch()
    sizes = np.diff(starts_t.cpu().numpy().astype(np.int64))
    if len(mol_idx) and (mol_idx.min() < 0 or mol_idx.max() >= len(atom_counts)):
        raise ValueError("coordinates: molecule index out of range")
    expect = np.asarray(atom_counts, np.int64)[mol_idx]
    if np.any(sizes != expect):
        bad = int(np.nonzero(sizes != expect)[0][0])
        raise ValueError(f"coordinates: conformer {bad} has {int(sizes[bad])} atoms, molecule {int(mol_idx[bad])} has "
                         f"{int(expect[bad])}")
    order = np.lexsort((conf_idx, mol_idx)).astype(np.int32)
    counts = np.bincount(mol_idx, minlength=len(atom_counts)).astype(np.int64)
    return order, counts, starts_t


def running_index(keys: np.ndarray) -> np.ndarray:
    """k-th occurrence number of each key, in order of appearance (conformer index within its molecule), int32."""
    from nvmolkit_b200 import _lib

    mod = _lib.core()
    if mod is not None:
        return mod.running_index(np.ascontiguousarray(keys, dtype=np.int64))
    keys = np.asarray(keys)
    n = len(keys)
    if n == 0:
        return np.zeros(0, dtype=np.int32)
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    first = np.concatenate([[True], sk[1:] != sk[:-1]])
    group_start = np.maximum.accumulate(np.where(first, np.arange(n), 0))
    out = np.empty(n, dtype=np.int32)
    out[order] = (np.arange(n) - group_start).astype(np.int32)
    return out
