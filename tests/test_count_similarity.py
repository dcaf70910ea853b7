"""Tanimoto, Dice and Tversky on count vectors without a GPU: the count oracle against a NumPy restatement and against
RDKit's literal SparseIntVect expressions (compared with ==), its top-k and threshold against lexsort and nonzero, and
every refusal of the Python calls and the C-ABI. RDKit's own values are replayed when tests/golden/rdkit_fixtures.npz
holds them."""

import ctypes as C
import os

import numpy as np
import pytest

from nvmolkit_b200 import similarity as S
from oracle import count as oracle_count

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rdkit_fixtures.npz")
WEIGHTS = [(1.0, 1.0), (0.5, 0.5), (0.3, 0.7), (0.9, 0.1), (1.0, 0.0), (0.0, 1.0), (0.0, 0.0), (2.0, 2.0)]
BAD_WEIGHTS = [-0.1, 1000.5, float("nan"), float("inf"), True, "0.5", None]


def counts(rng, n, bins, density=0.05, high=5):
    return np.where(rng.random((n, bins)) < density, rng.integers(1, high, size=(n, bins)), 0).astype(np.int32)


def restated(x, y, alpha, beta):
    """The contract in NumPy, one fp64 operation at a time in its order."""
    c = np.minimum(x[:, None, :].astype(np.int64), y[None, :, :]).sum(-1)
    a, b = x.sum(1, dtype=np.int64)[:, None], y.sum(1, dtype=np.int64)[None, :]
    d = (np.float64(alpha) * (a - c).astype(np.float64) + np.float64(beta) * (b - c).astype(np.float64)) + c
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(c == 0, 0.0, c / d)


def _sets(rng, bins=97):
    q, lib = counts(rng, 40, bins), counts(rng, 130, bins, high=300)
    lib[10:20] = lib[3]  # duplicates
    lib[30:35] = 0       # empty rows
    lib[40] = q[0]       # identical to a query
    lib[41] = 65535      # full and at the count bound
    q[5] = 0
    return q, lib


@pytest.mark.parametrize("alpha,beta", WEIGHTS)
def test_oracle_matrix_is_the_numpy_restatement(alpha, beta):
    q, lib = _sets(np.random.default_rng(1))
    assert np.array_equal(oracle_count.cross(q, lib, alpha, beta), restated(q, lib, alpha, beta))
    assert np.array_equal(oracle_count.cross(q, None, alpha, beta), restated(q, q, alpha, beta))


def test_tanimoto_and_dice_are_rdkits_literal_expressions():
    """RDKit's SparseIntVect: TanimotoSimilarity = andSum / (v1Sum + v2Sum - andSum), DiceSimilarity =
    2 andSum / (v1Sum + v2Sum), 0 when the denominator is 0; Python floats, one rounding each."""
    q, lib = _sets(np.random.default_rng(2))
    tan, dice = oracle_count.cross(q, lib, 1.0, 1.0), oracle_count.cross(q, lib, 0.5, 0.5)
    for i in range(len(q)):
        for j in range(len(lib)):
            v1, v2 = int(q[i].sum()), int(lib[j].sum())
            andsum = int(np.minimum(q[i], lib[j]).sum())
            want_t = andsum / (v1 + v2 - andsum) if v1 + v2 - andsum else 0.0
            want_d = 2.0 * andsum / (v1 + v2) if v1 + v2 else 0.0
            assert tan[i, j] == want_t and dice[i, j] == want_d, (i, j)


@pytest.mark.parametrize("alpha,beta", [(1.0, 1.0), (0.5, 0.5), (0.3, 0.7)])
@pytest.mark.parametrize("k", [1, 7, 130])
def test_oracle_topk_and_threshold_are_lexsort_and_nonzero(alpha, beta, k):
    q, lib = _sets(np.random.default_rng(3))
    m = oracle_count.cross(q, lib, alpha, beta)
    v, i = oracle_count.topk(q, lib, k, alpha, beta)
    for r in range(len(q)):
        order = np.lexsort((np.arange(len(lib)), -m[r]))[:k]
        assert np.array_equal(i[r], order) and np.array_equal(v[r], m[r, order])
    indptr, idx, vals = oracle_count.threshold(q, lib, 0.3, alpha, beta)
    for r in range(len(q)):
        cols = np.nonzero(m[r] >= 0.3)[0]
        assert np.array_equal(idx[indptr[r]:indptr[r + 1]], cols) and np.array_equal(vals[indptr[r]:indptr[r + 1]], m[r, cols])


def test_sums_at_the_count_bound_are_exact():
    full = np.full((2, 4096), 65535, dtype=np.int32)
    full[1, 0] = 0
    m = oracle_count.cross(full, full, 1.0, 1.0)
    assert m[0, 0] == 1.0 and m[1, 1] == 1.0 and m[0, 1] == m[1, 0] == 4095 / 4096
    assert np.array_equal(oracle_count.cross(full, full, 0.3, 0.7), restated(full, full, 0.3, 0.7))


@pytest.mark.parametrize("bad", BAD_WEIGHTS)
def test_bad_weights_are_value_errors_before_any_device_work(bad):
    x = np.zeros((4, 8), np.int32)
    calls = [lambda **w: S.crossTverskyCountSimilarity(x, **w),
             lambda **w: S.topKTverskyCountSimilarity(x, k=2, **w),
             lambda **w: S.thresholdTverskyCountSimilarity(x, threshold=0.5, **w)]
    for call in calls:
        for w in ({"alpha": bad, "beta": 0.5}, {"alpha": 0.5, "beta": bad}):
            with pytest.raises(ValueError):
                call(**w)


def test_weights_are_keyword_only_and_stream_threshold_checks():
    x = np.zeros((4, 8), np.int32)
    with pytest.raises(TypeError):
        S.crossTverskyCountSimilarity(x, None, 0.5, 0.5)
    with pytest.raises(TypeError):
        S.topKTverskyCountSimilarity(x, None, 2, 0.5, 0.5)
    with pytest.raises(TypeError):
        S.thresholdTverskyCountSimilarity(x, None, 0.5, 0.5, 0.5)
    with pytest.raises(TypeError):
        S.crossTanimotoCountSimilarity(object(), stream="not a stream")
    with pytest.raises(TypeError):
        S.topKDiceCountSimilarity(object(), k=3, stream=0)
    with pytest.raises(TypeError):
        S.thresholdTanimotoCountSimilarity(object(), threshold=0.5, stream=1)  # (a valid threshold: the stream fails)
    for t in (0, -0.1, 1.5, float("nan"), True, "0.5"):
        with pytest.raises(ValueError):
            S.thresholdDiceCountSimilarity(x, threshold=t)


def test_count_threshold_checks_the_stream_before_the_threshold():
    """As the bit threshold calls do (test_threshold.py): both arguments bad is a TypeError."""
    with pytest.raises(TypeError):
        S.thresholdTanimotoCountSimilarity(object(), threshold=float("nan"), stream="not a stream")
    with pytest.raises(TypeError):
        S.thresholdTverskyCountSimilarity(object(), alpha=0.5, beta=0.5, threshold=2.0, stream=0)


def test_the_library_exports_the_entry_points_and_checks_their_arguments(built_lib):
    L = built_lib
    nnz = C.c_uint64(0)
    for name in ("b200mol_count_cross", "b200mol_count_topk", "b200mol_count_threshold"):
        assert hasattr(L, name)
    # bins
    for bins in (0, -1, 4097):
        assert L.b200mol_count_cross(16, 4, 16, 4, bins, 1.0, 1.0, 16, None) == 1
        assert b"bins" in L.b200mol_last_error()
        assert L.b200mol_count_topk(16, 4, 16, 100, bins, 1.0, 1.0, 5, 16, 16, None) == 1
        assert L.b200mol_count_threshold(16, 4, 16, 100, bins, 1.0, 1.0, 0.5, 16, 16, 16, 4, C.byref(nnz), None) == 1
    # null pointers
    assert L.b200mol_count_cross(None, 4, None, 0, 64, 1.0, 1.0, 16, None) == 1
    assert L.b200mol_count_cross(16, 4, None, 0, 64, 1.0, 1.0, None, None) == 1
    assert L.b200mol_count_topk(16, 4, None, 0, 64, 1.0, 1.0, 2, None, None, None) == 1
    assert L.b200mol_count_threshold(16, 4, None, 0, 64, 1.0, 1.0, 0.5, None, None, None, 0, C.byref(nnz), None) == 1
    assert L.b200mol_count_threshold(16, 4, None, 0, 64, 1.0, 1.0, 0.5, 16, None, None, 4, C.byref(nnz), None) == 1
    # weights
    for a, b in ((float("nan"), 0.5), (0.5, float("inf")), (-1e-300, 0.5), (0.5, 1000.0000001)):
        assert L.b200mol_count_cross(16, 4, 16, 4, 64, a, b, 16, None) == 1
        assert b"Tversky weights" in L.b200mol_last_error()
        assert L.b200mol_count_topk(16, 4, 16, 100, 64, a, b, 5, 16, 16, None) == 1
        assert L.b200mol_count_threshold(16, 4, 16, 100, 64, a, b, 0.5, 16, 16, 16, 4, C.byref(nnz), None) == 1
    # k and threshold
    for k, n in ((0, 100), (101, 100), (S.TOPK_MAX + 1, 1000)):
        assert L.b200mol_count_topk(16, 4, 16, n, 64, 1.0, 1.0, k, 16, 16, None) == 1
        assert b"k must be" in L.b200mol_last_error()
    for t in (0.0, -0.5, 1.0000001, float("nan")):
        assert L.b200mol_count_threshold(16, 4, 16, 100, 64, 0.5, 0.5, t, 16, 16, 16, 4, C.byref(nnz), None) == 1
        assert b"threshold" in L.b200mol_last_error()
    # nothing to do: no device work
    assert L.b200mol_count_cross(None, 0, None, 0, 64, 1.0, 1.0, None, None) == 0
    assert L.b200mol_count_topk(None, 0, 16, 5, 64, 1.0, 1.0, 2, None, None, None) == 0


@pytest.mark.skipif(not os.path.exists(FIXTURES), reason="no RDKit-exported fixtures (tools/export_rdkit_fixtures.py)")
def test_count_oracle_equals_rdkit():
    fx = np.load(FIXTURES, allow_pickle=False)
    if "count_tanimoto_r2" not in fx:
        pytest.skip("the fixtures predate the count fingerprints")
    x = fx["morgan_counts_r2"]
    assert np.array_equal(oracle_count.cross(x, None, 1.0, 1.0), fx["count_tanimoto_r2"])
    assert np.array_equal(oracle_count.cross(x, None, 0.5, 0.5), fx["count_dice_r2"])
