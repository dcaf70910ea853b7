"""ctypes front end of oracle_leader.c (Leader diversity picking on the CPU) — TEST INFRASTRUCTURE ONLY, like the rest
of this package: what the GPU picker (nvmolkit_b200/csrc/leader.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import METRIC, _fp, lib


def leader_pick(fp, pool_size: int, threshold: float, pick_size: int = 0, first_picks=(), metric: str = "tanimoto"):
    """int32 [nPicks]: RDKit's LeaderPicker list walk (OpenMP over each compaction); pick_size 0 = no limit."""
    L = lib()
    fn = L.oracle_leader_pick
    fn.restype = C.c_long
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_long, C.c_double, C.c_long, C.c_void_p, C.c_int, C.c_void_p]
    fp = _fp(fp)
    first = np.ascontiguousarray(first_picks, dtype=np.int32)
    cap = pool_size if pick_size == 0 else pick_size
    assert 1 <= cap <= pool_size <= fp.shape[0] and len(first) <= cap and 0.0 <= threshold <= 1.0
    assert len(set(first.tolist())) == len(first) and (first >= 0).all() and (first < pool_size).all()
    picks = np.empty(cap, dtype=np.int32)
    n = fn(fp.ctypes.data, fp.shape[1], METRIC[metric], int(pool_size), float(threshold), int(cap), first.ctypes.data,
           len(first), picks.ctypes.data)
    return picks[:n].copy()
