"""ctypes front end of oracle_align.c (RDKit's AlignPoints restated in fp64) — TEST INFRASTRUCTURE ONLY, like the rest of
this package: the definition b200mol_align (nvmolkit_b200/csrc/align.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import lib


def _lib():
    L_ = lib()
    L_.oracle_align.restype = C.c_double
    L_.oracle_align.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L_.oracle_apply_transform.restype = None
    L_.oracle_apply_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    return L_


def align(prb, ref, pairs=None, weights=None, reflect=False, maxIters=50):
    """(RMSD, 4 x 4 transform) of probe conformer ``prb`` [A, 3] onto ``ref`` [B, 3] through ``pairs`` [L, 2] of
    (probe atom, reference atom) (None: the identity over all atoms); ``weights`` [L] or None."""
    prb = np.ascontiguousarray(prb, np.float64)
    ref = np.ascontiguousarray(ref, np.float64)
    if pairs is None:
        pairs = np.stack([np.arange(len(prb))] * 2, 1)
    pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    w = None if weights is None else np.ascontiguousarray(weights, np.float64)
    T = np.zeros((4, 4), np.float64)
    v = _lib().oracle_align(prb.ctypes.data, ref.ctypes.data, pairs.ctypes.data, None if w is None else w.ctypes.data,
                            len(pairs), 1 if reflect else 0, int(maxIters), T.ctypes.data)
    return float(v), T


def apply(T, xyz) -> np.ndarray:
    """A copy of ``xyz`` [n, 3] with the transform applied to every atom."""
    out = np.array(xyz, np.float64, order="C").reshape(-1, 3)
    _lib().oracle_apply_transform(np.ascontiguousarray(T, np.float64).ctypes.data, out.ctypes.data, len(out))
    return out
