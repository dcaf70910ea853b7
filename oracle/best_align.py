"""ctypes front end of oracle_best_align.c (the best of K atom mappings, aligned or in place, in fp64) — TEST
INFRASTRUCTURE ONLY, like the rest of this package: the per-job definition b200mol_best_align
(nvmolkit_b200/csrc/best_align.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import lib


def best_align(prb, ref, P, Q, weights=None, mode=0, reflect=False, maxIters=50):
    """Probe conformer ``prb`` [A, 3] against ``ref`` [B, 3] through mappings k pairing ``P[i]`` with ``Q[k][i]``
    (``Q``: K x L). ``mode`` 0 aligns (RDKit GetBestRMS), 1 compares in place (CalcRMS). Returns (RMSD, first best
    mapping, 4 x 4 transform (zeros in mode 1), every mapping's RMSD [K])."""
    L_ = lib()
    L_.oracle_best_align.restype = C.c_double
    L_.oracle_best_align.argtypes = [C.c_void_p] * 4 + [C.c_int] * 5 + [C.c_void_p] * 3
    prb = np.ascontiguousarray(prb, np.float64)
    ref = np.ascontiguousarray(ref, np.float64)
    P = np.asarray(P, np.int64)
    Q = np.asarray(Q, np.int64).reshape(-1, len(P))
    tab = np.ascontiguousarray(np.concatenate([P, Q.reshape(-1)]), np.int16)
    w = None if weights is None else np.ascontiguousarray(weights, np.float64)
    T = np.zeros((4, 4), np.float64)
    best = C.c_int(0)
    per = np.zeros(len(Q), np.float64)
    v = L_.oracle_best_align(prb.ctypes.data, ref.ctypes.data, tab.ctypes.data, None if w is None else w.ctypes.data,
                             len(Q), len(P), int(mode), 1 if reflect else 0, int(maxIters), T.ctypes.data,
                             C.addressof(best), per.ctypes.data)
    return float(v), best.value, T, per
