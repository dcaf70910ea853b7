"""ctypes front end of oracle_topk.c (exact top-k similarity search on the CPU) — TEST INFRASTRUCTURE ONLY, like the rest
of this package: what the GPU search (nvmolkit_b200/csrc/topk.cu) is checked against."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import METRIC, _fp, lib


def topk(q, library=None, k: int = 10, metric: str = "tanimoto"):
    """(values [Q, k] fp64, indices [Q, k] int32): per query the first k columns of its row of
    ``oracle.similarity_cross`` ordered by (value descending, column ascending), without the matrix. ``library=None``
    searches the queries themselves."""
    L = lib()
    L.oracle_topk.restype = None
    L.oracle_topk.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    q = _fp(q)
    b = q if library is None else _fp(library)
    assert 1 <= k <= b.shape[0] and q.shape[1] == b.shape[1]
    values = np.empty((q.shape[0], k), dtype=np.float64)
    indices = np.empty((q.shape[0], k), dtype=np.int32)
    L.oracle_topk(q.ctypes.data, q.shape[0], b.ctypes.data, b.shape[0], q.shape[1], METRIC[metric], int(k),
                  values.ctypes.data, indices.ctypes.data)
    return values, indices
