"""ctypes front end of oracle_count.c (Tanimoto, Dice and Tversky on count vectors, on the CPU) — TEST INFRASTRUCTURE
ONLY, like the rest of this package: what the GPU calls (b200mol_count_*) are checked against. Top-k and threshold are
derived from the matrix in NumPy (``lexsort``, ``nonzero``). ``alpha`` weights what only the row (group one) has."""

from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import lib

TANIMOTO = (1.0, 1.0)
DICE = (0.5, 0.5)


def _counts(x) -> np.ndarray:
    x = np.ascontiguousarray(x, dtype=np.int32)
    assert x.ndim == 2
    return x


def cross(a, b=None, alpha: float = 1.0, beta: float = 1.0) -> np.ndarray:
    """The (n, m) fp64 matrix; ``b=None``: ``a`` against itself."""
    fn = lib().oracle_count_cross
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_double, C.c_double, C.c_void_p]
    a = _counts(a)
    b = a if b is None else _counts(b)
    assert a.shape[1] == b.shape[1]
    out = np.empty((a.shape[0], b.shape[0]), dtype=np.float64)
    fn(a.ctypes.data, a.shape[0], b.ctypes.data, b.shape[0], a.shape[1], float(alpha), float(beta), out.ctypes.data)
    return out


def topk_of(m: np.ndarray, k: int):
    """(values [Q, k], indices [Q, k] int32): per row the first k columns by (value descending, column ascending)."""
    cols = np.arange(m.shape[1])
    order = np.array([np.lexsort((cols, -row))[:k] for row in m], dtype=np.int32).reshape(m.shape[0], k)
    return np.take_along_axis(m, order.astype(np.int64), 1), order


def threshold_of(m: np.ndarray, t: float):
    """(indptr int64, indices int32, values fp64): per row, ascending, the columns whose entry is >= t."""
    rows, cols = np.nonzero(m >= t)
    indptr = np.zeros(m.shape[0] + 1, dtype=np.int64)
    np.add.at(indptr, rows + 1, 1)
    return np.cumsum(indptr), cols.astype(np.int32), m[rows, cols]


def topk(q, library=None, k: int = 10, alpha: float = 1.0, beta: float = 1.0):
    return topk_of(cross(q, library, alpha, beta), k)


def threshold(q, library=None, t: float = 0.7, alpha: float = 1.0, beta: float = 1.0):
    return threshold_of(cross(q, library, alpha, beta), t)


def morgan_counts(atom_starts, bond_starts, atom_inv, bond_inv, bond_a, bond_b, radius: int, fp_bits: int) -> np.ndarray:
    """int32 (n, fp_bits): the unfolded codes of ``oracle.morgan_codes`` of each molecule, folded modulo fp_bits and
    counted (np.bincount)."""
    import oracle

    n = len(atom_starts) - 1
    out = np.zeros((n, fp_bits), dtype=np.int32)
    for i in range(n):
        a0, a1, b0, b1 = atom_starts[i], atom_starts[i + 1], bond_starts[i], bond_starts[i + 1]
        codes = oracle.morgan_codes(atom_inv[a0:a1], bond_inv[b0:b1], bond_a[b0:b1], bond_b[b0:b1], radius)
        out[i] = np.bincount(codes.astype(np.int64) % fp_bits, minlength=fp_bits)
    return out
