"""Butina on count vectors without a GPU: the refusals of b200mol_count_neighbor_edges and b200mol_count_butina_fused
that come before any device work, the argument errors of clustering.fused_butina_counts, and the soundness of the sum
band: in (sum, index) order, every neighbour pair of the count oracle lies inside the band of its first row's block.
``band_ends`` / ``band_pairs`` are the NumPy model the GPU tests hold the pass's pair count to."""

import ctypes as C

import numpy as np
import pytest
import torch

from nvmolkit_b200 import clustering
from oracle import count as oracle_count

WEIGHTS = {"tanimoto": (1.0, 1.0), "dice": (0.5, 0.5)}


def value(c, a, b, alpha, beta):
    """tverskyFromCounts in NumPy, one fp64 operation at a time in its order (0 where c = 0)."""
    c, a, b = (np.asarray(v, dtype=np.int64) for v in (c, a, b))
    d = (np.float64(alpha) * (a - c).astype(np.float64) + np.float64(beta) * (b - c).astype(np.float64)) + c
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(c == 0, 0.0, c / d)


def query_rows(bins: int) -> int:
    return 32 if bins <= 2048 else 16


def band_ends(sums_sorted, qb: int, cutoff: float, weights):
    """Per block of qb rows in sum order: the end of the columns its pass visits. The block's largest sum A bounds
    every pair of its rows with a later column j: 1 - value(A, A, sums[j]) <= cutoff holds on a prefix of the columns."""
    s = np.asarray(sums_sorted, dtype=np.int64)
    n = len(s)
    q0 = np.arange(0, n, qb)
    e = np.minimum(q0 + qb, n)
    big = s[e - 1]
    lo, hi = e.copy(), np.full(len(q0), n)
    while (lo < hi).any():
        act = lo < hi
        mid = (lo + hi) // 2
        ok = np.zeros(len(q0), bool)
        ok[act] = (1.0 - value(big[act], big[act], s[mid[act]], *weights)) <= cutoff
        lo = np.where(act & ok, mid + 1, lo)
        hi = np.where(act & ~ok, mid, hi)
    return q0, e, lo


def band_pairs(sums, bins: int, cutoff: float, weights) -> int:
    """The pairs (row, col > row) the pass compares: inside each block, and every block row against its band."""
    q0, e, end = band_ends(np.sort(np.asarray(sums, dtype=np.int64)), query_rows(bins), cutoff, weights)
    nq = (e - q0).astype(np.int64)
    return int((nq * (nq - 1) // 2 + nq * (end - e)).sum())


def clustered_counts(rng, n, bins, centres=20, changes=3, high=6):
    """Seeded centres, each member a copy of one with a few bins changed."""
    c = np.where(rng.random((centres, bins)) < 0.05, rng.integers(1, high, size=(centres, bins)), 0)
    x = c[rng.integers(0, centres, size=n)].copy()
    rows = np.repeat(np.arange(n), changes)
    x[rows, rng.integers(0, bins, size=n * changes)] = rng.integers(0, high, size=n * changes)
    return x.astype(np.int32)


@pytest.mark.parametrize("metric", ["tanimoto", "dice"])
@pytest.mark.parametrize("bins", [64, 3000])
def test_every_oracle_edge_lies_in_its_band(metric, bins):
    rng = np.random.default_rng(bins)
    x = np.concatenate([clustered_counts(rng, 300, bins),
                        np.where(rng.random((200, bins)) < 0.1, rng.integers(1, 400, size=(200, bins)), 0)]).astype(np.int32)
    x[:5] = 0
    order = np.argsort(x.sum(1), kind="stable")
    xs = x[order]
    sums = xs.sum(1)
    m = oracle_count.cross(xs, xs, *WEIGHTS[metric])
    qb = query_rows(bins)
    for cutoff in (0.0, 0.2, 0.3, 0.6, 1.0):
        i, j = np.nonzero(np.triu(1.0 - m <= cutoff, 1))
        _, _, end = band_ends(sums, qb, cutoff, WEIGHTS[metric])
        assert (j < end[i // qb]).all(), cutoff
        n = len(x)
        if cutoff == 1.0:
            assert band_pairs(sums, bins, cutoff, WEIGHTS[metric]) == n * (n - 1) // 2
        elif cutoff <= 0.3:
            assert band_pairs(sums, bins, cutoff, WEIGHTS[metric]) < n * (n - 1) // 2


def test_the_library_refuses_before_any_device_work(built_lib):
    L = built_lib
    ne = C.c_uint64(7)
    ncl = C.c_int32(7)
    for name in ("b200mol_count_neighbor_edges", "b200mol_count_butina_fused"):
        assert hasattr(L, name)

    def edges(x=16, n=4, bins=64, a=1.0, b=1.0, cutoff=0.3, counts=16, out=16, cap=4):
        return L.b200mol_count_neighbor_edges(x, n, bins, a, b, cutoff, counts, out, cap, C.byref(ne), None)

    def fused(x=16, n=4, bins=64, a=1.0, b=1.0, cutoff=0.3, ids=16):
        return L.b200mol_count_butina_fused(x, n, bins, a, b, cutoff, ids, 16, 16, C.byref(ncl), None)

    for call in (edges, fused):
        # weights: only Tanimoto (1, 1) and Dice (1/2, 1/2)
        for a, b in ((0.3, 0.7), (1.0, 0.0), (0.5, 1.0), (1.0, 0.5), (2.0, 2.0), (float("nan"), 1.0), (-1.0, 1.0)):
            assert call(a=a, b=b) == 1, (a, b)
            err = L.b200mol_last_error()
            assert b"Tanimoto (1, 1) or Dice (0.5, 0.5)" in err or b"Tversky weights" in err
        for cutoff in (-0.1, 1.0000000000000002, float("nan"), float("inf")):
            assert call(cutoff=cutoff) == 1 and b"cutoff" in L.b200mol_last_error()
        for bins in (0, -1, 4097):
            assert call(bins=bins) == 1 and b"bins" in L.b200mol_last_error()
        assert call(x=None) == 1 and b"null" in L.b200mol_last_error()
    assert edges(counts=None) == 1 and b"null" in L.b200mol_last_error()
    assert edges(out=None) == 1 and b"null" in L.b200mol_last_error()
    assert fused(ids=None) == 1 and b"null" in L.b200mol_last_error()
    # nothing to do: no device work, the totals are zero
    assert edges(x=None, n=0, counts=None, out=None) == 0 and ne.value == 0
    assert L.b200mol_count_butina_fused(None, 0, 64, 0.5, 0.5, 0.3, None, None, None, C.byref(ncl), None) == 0
    assert ncl.value == 0


def test_python_argument_errors():
    x = torch.zeros((4, 8), dtype=torch.int32)  # (these checks come before the input's)
    for metric in ("cosine", "tversky", "Tanimoto", None):
        with pytest.raises(ValueError, match="metric"):
            clustering.fused_butina_counts(x, 0.3, metric=metric)
    for cutoff in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="cutoff"):
            clustering.fused_butina_counts_device(x, cutoff)
    for stream in ("not a stream", 0, 1):
        with pytest.raises(TypeError):
            clustering.fused_butina_counts(x, 0.3, stream=stream)
