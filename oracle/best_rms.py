"""ctypes front end of oracle_best_rms.c (mapped conformer RMSD matrices in fp64) — TEST INFRASTRUCTURE ONLY, like the
rest of this package: the per-pair definition b200mol_conformer_rmsd_mapped (nvmolkit_b200/csrc/conformer_rmsd.cu) is
checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import lib


def molecules(coords, lists, prealigned=False) -> list:
    """``coords[m]``: the conformers of molecule m ([C, n, 3] or a list of [n, 3]); ``lists[m] = (P, Q)``: the probe list
    (L atoms) and the K x L reference lists. Per molecule the fp64 lower triangle of min_k RMSD(x_i[P], x_j[Q_k])."""
    L_ = lib()
    L_.oracle_rms_matrix_mapped.restype = None
    L_.oracle_rms_matrix_mapped.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                            C.c_int, C.c_void_p]
    out = []
    for confs, (p, q) in zip(coords, lists):
        arr = [np.asarray(c, np.float64).reshape(-1, 3) for c in confs]
        n = len(arr)
        res = np.zeros(max(n * (n - 1) // 2, 0), np.float64)
        if n >= 2:
            xyz = np.ascontiguousarray(np.concatenate(arr))
            cas = np.arange(0, len(xyz) + 1, len(arr[0]), dtype=np.int32)
            order = np.arange(n, dtype=np.int32)
            q = np.asarray(q, np.int64).reshape(-1, len(p))
            tab = np.ascontiguousarray(np.concatenate([np.asarray(p, np.int64), q.reshape(-1)]), np.int16)
            L_.oracle_rms_matrix_mapped(n, order.ctypes.data, cas.ctypes.data, xyz.ctypes.data, len(q), len(p),
                                        tab.ctypes.data, 1 if prealigned else 0, res.ctypes.data)
        out.append(res)
    return out
