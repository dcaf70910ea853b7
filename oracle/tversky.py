"""ctypes front end of oracle_tversky.c (Dice / Tversky similarity on the CPU) — TEST INFRASTRUCTURE ONLY, like the rest
of this package: what the GPU calls (b200mol_tversky_*) are checked against. ``alpha`` weights the bits only in the row
(group one) fingerprint; Dice is (0.5, 0.5)."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import _fp, lib

DICE = (0.5, 0.5)


def cross(a, b=None, alpha: float = 0.5, beta: float = 0.5) -> np.ndarray:
    """The (n, m) fp64 Tversky matrix; ``b=None``: ``a`` against itself."""
    L = lib()
    fn = L.oracle_tversky_cross
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_double, C.c_double, C.c_void_p]
    a = _fp(a)
    b = a if b is None else _fp(b)
    assert a.shape[1] == b.shape[1]
    out = np.empty((a.shape[0], b.shape[0]), dtype=np.float64)
    fn(a.ctypes.data, a.shape[0], b.ctypes.data, b.shape[0], a.shape[1], float(alpha), float(beta), out.ctypes.data)
    return out


def topk(q, library=None, k: int = 10, alpha: float = 0.5, beta: float = 0.5):
    """(values [Q, k] fp64, indices [Q, k] int32): per query the first k columns of its row of ``cross`` ordered by
    (value descending, column ascending), without the matrix."""
    L = lib()
    fn = L.oracle_tversky_topk
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_double, C.c_double, C.c_int, C.c_void_p,
                   C.c_void_p]
    q = _fp(q)
    b = q if library is None else _fp(library)
    assert 1 <= k <= b.shape[0] and q.shape[1] == b.shape[1]
    values = np.empty((q.shape[0], k), dtype=np.float64)
    indices = np.empty((q.shape[0], k), dtype=np.int32)
    fn(q.ctypes.data, q.shape[0], b.ctypes.data, b.shape[0], q.shape[1], float(alpha), float(beta), int(k),
       values.ctypes.data, indices.ctypes.data)
    return values, indices


def threshold(q, library=None, t: float = 0.7, alpha: float = 0.5, beta: float = 0.5):
    """(indptr int64 [Q + 1], indices int32 [nnz], values fp64 [nnz]): per query, ascending, the columns whose entry of
    ``cross`` is ``>= t``, with those values, without the matrix. ``library=None``: the queries against themselves."""
    L = lib()
    fn = L.oracle_tversky_threshold
    fn.restype = C.c_long
    fn.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p,
                   C.c_void_p, C.c_void_p]
    q = _fp(q)
    b = q if library is None else _fp(library)
    assert q.shape[1] == b.shape[1]
    args = (q.ctypes.data, q.shape[0], b.ctypes.data, b.shape[0], q.shape[1], float(alpha), float(beta), float(t))
    indptr = np.empty(q.shape[0] + 1, dtype=np.int64)
    nnz = fn(*args, indptr.ctypes.data, None, None)
    indices = np.empty(nnz, dtype=np.int32)
    values = np.empty(nnz, dtype=np.float64)
    fn(*args, indptr.ctypes.data, indices.ctypes.data, values.ctypes.data)
    return indptr, indices, values
