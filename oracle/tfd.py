"""ctypes front end of oracle_tfd.c (torsion fingerprint deviation in fp64) — TEST INFRASTRUCTURE ONLY, like the rest
of this package: the per-pair definition the GPU pass (nvmolkit_b200/csrc/tfd.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import lib


def dihedral(p0, p1, p2, p3) -> float:
    """Signed dihedral in degrees, (-180, 180], 0 when a cross product is exactly zero."""
    L = lib()
    L.oracle_tfd_dihedral.restype = C.c_double
    L.oracle_tfd_dihedral.argtypes = [C.c_void_p] * 4
    p = [np.ascontiguousarray(x, np.float64) for x in (p0, p1, p2, p3)]
    return float(L.oracle_tfd_dihedral(*[x.ctypes.data for x in p]))


def matrices(mol_conf_start, conf_atom_start, xyz, tors_start, quartet_start, quartets, types, weight, maxdev,
             conf_order=None) -> list:
    """Per molecule the fp64 lower triangle (I > J, row-major) of the TFD matrix, from the flat tables of
    b200mol_tfd_matrices: conformer k of molecule m is conf_order[mol_conf_start[m] + k] (None = identity)."""
    L = lib()
    L.oracle_tfd_mol.restype = None
    L.oracle_tfd_mol.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 6
    mcs = np.asarray(mol_conf_start, np.int64)
    order = np.arange(int(mcs[-1]), dtype=np.int32) if conf_order is None else np.ascontiguousarray(conf_order, np.int32)
    cas = np.ascontiguousarray(conf_atom_start, np.int32)
    xyz = np.ascontiguousarray(xyz, np.float64)
    ts = np.asarray(tors_start, np.int64)
    qs = np.ascontiguousarray(quartet_start, np.int32)
    qa = np.ascontiguousarray(quartets, np.int16).reshape(-1, 4)
    ty = np.ascontiguousarray(types, np.uint8)
    w = np.ascontiguousarray(weight, np.float64)
    md = np.ascontiguousarray(maxdev, np.float64)
    out = []
    for m in range(len(mcs) - 1):
        n = int(mcs[m + 1] - mcs[m])
        res = np.zeros(max(n * (n - 1) // 2, 0), np.float64)
        confs = np.ascontiguousarray(order[mcs[m]:mcs[m + 1]])
        if n >= 2:
            L.oracle_tfd_mol(n, confs.ctypes.data, cas.ctypes.data, xyz.ctypes.data, int(ts[m]), int(ts[m + 1]),
                             qs.ctypes.data, qa.ctypes.data, ty.ctypes.data, w.ctypes.data, md.ctypes.data, res.ctypes.data)
        out.append(res)
    return out
