"""ctypes front end of oracle_rmsd.c (conformer RMSD matrices in fp64) — TEST INFRASTRUCTURE ONLY, like the rest of
this package: the per-pair definition the GPU pass (nvmolkit_b200/csrc/conformer_rmsd.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import lib


def best_ssd(a, b) -> float:
    """Sum of squared deviations of point lists a, b ([n, 3]) after the best proper rigid superposition."""
    L = lib()
    L.oracle_best_ssd.restype = C.c_double
    L.oracle_best_ssd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    a = np.ascontiguousarray(a, np.float64).reshape(-1, 3)
    b = np.ascontiguousarray(b, np.float64).reshape(-1, 3)
    return float(L.oracle_best_ssd(a.ctypes.data, None, b.ctypes.data, None, len(a)))


def matrices(mol_conf_start, mol_atoms, conf_atom_start, xyz, prealigned=False, conf_order=None) -> list:
    """Per molecule the fp64 lower triangle (i > j, row-major) of the RMSD matrix, from the flat tables of
    b200mol_conformer_rmsd: conformer k of molecule m is conf_order[mol_conf_start[m] + k] (None = identity)."""
    L = lib()
    L.oracle_rms_matrix.restype = None
    L.oracle_rms_matrix.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    mcs = np.asarray(mol_conf_start, np.int64)
    order = np.arange(int(mcs[-1]), dtype=np.int32) if conf_order is None else np.ascontiguousarray(conf_order, np.int32)
    cas = np.ascontiguousarray(conf_atom_start, np.int32)
    xyz = np.ascontiguousarray(xyz, np.float64)
    out = []
    for m in range(len(mcs) - 1):
        n = int(mcs[m + 1] - mcs[m])
        res = np.zeros(max(n * (n - 1) // 2, 0), np.float64)
        confs = np.ascontiguousarray(order[mcs[m]:mcs[m + 1]])
        if n >= 2:
            L.oracle_rms_matrix(n, confs.ctypes.data, cas.ctypes.data, xyz.ctypes.data, int(mol_atoms[m]),
                                1 if prealigned else 0, res.ctypes.data)
        out.append(res)
    return out


def molecules(coords, prealigned=False) -> list:
    """``coords[m]``: the conformers of molecule m, [C, n, 3] (or a list of [n, 3]); the RMSD matrices per molecule."""
    blocks, cas, mcs, atoms = [], [0], [0], []
    for confs in coords:
        arr = [np.asarray(c, np.float64).reshape(-1, 3) for c in confs]
        atoms.append(len(arr[0]) if arr else 0)
        for a in arr:
            blocks.append(a)
            cas.append(cas[-1] + len(a))
        mcs.append(mcs[-1] + len(arr))
    xyz = np.concatenate(blocks) if blocks else np.zeros((0, 3))
    return matrices(mcs, atoms, cas, xyz, prealigned)

