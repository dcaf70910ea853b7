"""ctypes front end of oracle_threshold.c (threshold similarity search on the CPU) — TEST INFRASTRUCTURE ONLY, like the
rest of this package: what the GPU search (nvmolkit_b200/csrc/threshold.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import METRIC, _fp, lib


def threshold(q, library=None, t: float = 0.7, metric: str = "tanimoto"):
    """(indptr int64 [Q + 1], indices int32 [nnz], values fp64 [nnz]): per query, in ascending order, the columns whose
    entry of ``oracle.similarity_cross`` is ``>= t``, with those values, without the matrix. ``library=None`` searches the
    queries themselves."""
    L = lib()
    fn = L.oracle_threshold
    fn.restype = C.c_long
    fn.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p,
                   C.c_void_p]
    q = _fp(q)
    b = q if library is None else _fp(library)
    assert q.shape[1] == b.shape[1]
    indptr = np.empty(q.shape[0] + 1, dtype=np.int64)
    nnz = fn(q.ctypes.data, q.shape[0], b.ctypes.data, b.shape[0], q.shape[1], METRIC[metric], float(t),
             indptr.ctypes.data, None, None)
    indices = np.empty(nnz, dtype=np.int32)
    values = np.empty(nnz, dtype=np.float64)
    fn(q.ctypes.data, q.shape[0], b.ctypes.data, b.shape[0], q.shape[1], METRIC[metric], float(t), indptr.ctypes.data,
       indices.ctypes.data, values.ctypes.data)
    return indptr, indices, values
