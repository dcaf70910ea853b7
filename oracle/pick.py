"""ctypes front end of oracle_pick.c (MaxMin diversity picking on the CPU) — TEST INFRASTRUCTURE ONLY, like the rest of
this package: what the GPU picker (nvmolkit_b200/csrc/maxmin.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import METRIC, _fp, lib


def _run(name, fp, pool_size, pick_size, first_picks, threshold, metric):
    L = lib()
    fn = getattr(L, name)
    fn.restype = C.c_double
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_long, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_void_p]
    fp = _fp(fp)
    first = np.ascontiguousarray(first_picks, dtype=np.int32)
    assert 1 <= len(first) and 1 <= pick_size <= pool_size <= fp.shape[0] and len(first) <= pick_size
    assert len(set(first.tolist())) == len(first) and (first >= 0).all() and (first < pool_size).all()
    picks = np.empty(pick_size, dtype=np.int32)
    thr = fn(fp.ctypes.data, fp.shape[1], METRIC[metric], int(pool_size), int(pick_size), first.ctypes.data, len(first),
             float(threshold), picks.ctypes.data)
    return picks, float(thr)


def maxmin_lazy(fp, pool_size: int, pick_size: int, first_picks, threshold: float = -1.0, metric: str = "tanimoto"):
    """(picks int32 [pick_size], -1 past a threshold stop; threshold) by RDKit's lazy list walk (serial)."""
    return _run("oracle_maxmin_lazy", fp, pool_size, pick_size, first_picks, threshold, metric)


def maxmin_dense(fp, pool_size: int, pick_size: int, first_picks, threshold: float = -1.0, metric: str = "tanimoto"):
    """The same by the plain definition: every pick updates every item (OpenMP over items)."""
    return _run("oracle_maxmin_dense", fp, pool_size, pick_size, first_picks, threshold, metric)
