"""Dice and Tversky similarity without a GPU: the oracle against NumPy restatements, the Dice threshold table and
popcount band against the fp64 predicate, argument validation, and the exported symbols."""

import ctypes as C

import numpy as np
import pytest

import oracle
from nvmolkit_b200 import similarity
from oracle import topk as oracle_topk
from oracle import tversky as oracle_tversky

WEIGHTS = [(0.5, 0.5), (1.0, 1.0), (0.3, 0.7), (0.9, 0.1), (1.0, 0.0), (0.0, 1.0), (0.0, 0.0), (2.0, 2.0)]


def _fingerprints(rng, n, words, density=0.1):
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


def _counts(q, lib):
    unpack = lambda x: np.unpackbits(x.view(np.uint8), axis=1).astype(np.int64)  # noqa: E731
    a, b = unpack(q), unpack(lib)
    return a @ b.T, a.sum(1)[:, None], b.sum(1)[None, :]


def _tversky_np(c, a, b, alpha, beta):
    """The contract in NumPy, one fp64 operation at a time in its order (NumPy never fuses them)."""
    d = (np.float64(alpha) * (a - c).astype(np.float64) + np.float64(beta) * (b - c).astype(np.float64)) + c
    with np.errstate(invalid="ignore", divide="ignore"):
        v = c.astype(np.float64) / d
    return np.where(c == 0, 0.0, v)


def _sets(rng):
    lib = _fingerprints(rng, 170, 8)
    lib[40:60] = lib[3]   # duplicates
    lib[100:110] = 0      # empty fingerprints
    lib[120] = lib[4] | lib[5]  # a superset
    q = np.concatenate([_fingerprints(rng, 20, 8), lib[[3, 4, 105]], np.zeros((1, 8), np.uint32)])
    return q, lib


@pytest.mark.parametrize("alpha,beta", WEIGHTS)
def test_oracle_matrix_is_the_numpy_restatement(alpha, beta):
    q, lib = _sets(np.random.default_rng(1))
    c, a, b = _counts(q, lib)
    got = oracle_tversky.cross(q, lib, alpha, beta)
    assert (got == _tversky_np(c, a, b, alpha, beta)).all()
    assert ((got >= 0.0) & (got <= 1.0)).all()
    self_m = oracle_tversky.cross(lib, None, alpha, beta)
    nonempty = lib.any(1)
    assert (np.diag(self_m)[nonempty] == 1.0).all() and (np.diag(self_m)[~nonempty] == 0.0).all()
    # alpha weights the row's bits: the swapped call is the transpose
    assert (oracle_tversky.cross(lib, q, beta, alpha) == got.T).all()


def test_oracle_at_one_one_is_tanimoto_and_at_one_half_is_dice():
    q, lib = _sets(np.random.default_rng(2))
    assert (oracle_tversky.cross(q, lib, 1.0, 1.0) == oracle.similarity_cross(q, lib)).all()
    c, a, b = _counts(q, lib)
    with np.errstate(invalid="ignore"):
        dice = np.where(c == 0, 0.0, (2 * c).astype(np.float64) / (a + b))
    assert (oracle_tversky.cross(q, lib, 0.5, 0.5) == dice).all()
    with np.errstate(invalid="ignore"):
        half = np.where(c == 0, 0.0, 2.0 * (c / (a + b).astype(np.float64)))
    assert (dice == half).all()  # 2 RN(c / (a + b)) == RN(2c / (a + b))


def _lexsort_topk(sim, k):
    cols = np.arange(sim.shape[1])
    idx = np.stack([np.lexsort((cols, -row))[:k] for row in sim])
    return np.take_along_axis(sim, idx, axis=1), idx.astype(np.int32)


@pytest.mark.parametrize("alpha,beta", WEIGHTS)
@pytest.mark.parametrize("k", [1, 7, 150])
def test_oracle_topk_is_lexsort_of_the_matrix(alpha, beta, k):
    q, lib = _sets(np.random.default_rng(3))
    want_v, want_i = _lexsort_topk(oracle_tversky.cross(q, lib, alpha, beta), k)
    got_v, got_i = oracle_tversky.topk(q, lib, k, alpha, beta)
    assert (got_i == want_i).all() and (got_v == want_v).all()
    sv, si = oracle_tversky.topk(lib, None, k, alpha, beta)
    wv, wi = _lexsort_topk(oracle_tversky.cross(lib, None, alpha, beta), k)
    assert (si == wi).all() and (sv == wv).all()


def test_dice_topk_indices_are_tanimoto_topk_indices():
    q, lib = _sets(np.random.default_rng(4))
    for k in (1, 10, 170):
        assert (oracle_tversky.topk(q, lib, k, 0.5, 0.5)[1] == oracle_topk.topk(q, lib, k)[1]).all()


def test_tversky_one_zero_ties_supersets_of_the_query_at_one():
    q, lib = _sets(np.random.default_rng(5))
    v, i = oracle_tversky.topk(lib[4:5], lib, 3, 1.0, 0.0)
    assert v[0, 0] == 1.0 and v[0, 1] == 1.0 and i[0, 0] == 4 and 120 in i[0]


@pytest.mark.parametrize("alpha,beta", WEIGHTS)
@pytest.mark.parametrize("t", [1e-9, 0.3, 0.5, 2 / 3, 1.0])
def test_oracle_threshold_is_the_nonzero_entries_of_the_matrix(alpha, beta, t):
    q, lib = _sets(np.random.default_rng(6))
    for a, b in ((q, lib), (lib, None)):
        m = oracle_tversky.cross(a, b, alpha, beta)
        indptr, indices, values = oracle_tversky.threshold(a, b, t, alpha, beta)
        rows, cols = np.nonzero(m >= t)
        assert (indptr == np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=len(a)))])).all()
        assert (indices == cols).all() and (values == m[rows, cols]).all()


# ------------------------------------------------------------------ the Dice threshold table and the popcount band
def _dice_table(bits, t):
    """thresh[s] = the smallest c in [1, s / 2] with fp64 RN(2c / s) >= t (0xFFFF: none), by the kernel's bisection."""
    out = np.full(2 * bits + 1, 0xFFFF, np.int64)
    passes = lambda c, s: (2.0 * c) / s >= t  # noqa: E731  (2c exact: RN(2c / s))
    for s in range(2, 2 * bits + 1):
        lo, hi = 1, s // 2
        if passes(hi, s):
            while lo < hi:
                mid = (lo + hi) // 2
                lo, hi = (lo, mid) if passes(mid, s) else (mid + 1, hi)
            out[s] = lo
    return out


@pytest.mark.parametrize("t", [0.05, 1 / 3, 0.5, 0.7, 0.8, 0.95, 1.0])
def test_dice_table_equals_the_fp64_predicate_and_the_band_never_cuts_an_accepted_pair(t):
    bits = 4096
    thresh = _dice_table(bits, t)
    a = np.arange(bits + 1)[:, None]
    b = np.arange(bits + 1)[None, :]
    s = a + b
    m = np.minimum(a, b)
    # the table test c >= thresh[s] equals the fp64 predicate, for the largest c a pair can have and for one less
    for c in (m, np.maximum(m - 1, 0)):
        with np.errstate(invalid="ignore", divide="ignore"):
            pred = (c > 0) & (np.where(s > 0, (2.0 * c) / np.maximum(s, 1), 0.0) >= t)
        assert ((c >= thresh[s]) == pred).all()
    # the popcount band (tanimoto_tc.cu bandCuts): tmin = suffix minimum; cut iff tmin[A + b] > A
    tmin = np.minimum.accumulate(thresh[::-1])[::-1]
    cut = tmin[a + b] > a
    assert not (cut & (m >= thresh[s])).any()
    assert (cut[:, :-1] <= cut[:, 1:]).all() and (cut[1:, :] <= cut[:-1, :]).all()


# ------------------------------------------------------------------ the Python and C-ABI argument checks
BAD_WEIGHTS = [float("nan"), float("inf"), -float("inf"), -0.5, 1000.5, True, "1", None]


@pytest.mark.parametrize("bad", BAD_WEIGHTS)
def test_bad_weights_are_value_errors_before_any_device_work(bad):
    fp = np.zeros((4, 4), np.int32)
    calls = [lambda **w: similarity.crossTverskySimilarity(fp, **w),
             lambda **w: similarity.topKTverskySimilarity(fp, k=2, **w),
             lambda **w: similarity.thresholdTverskySimilarity(fp, threshold=0.5, **w),
             lambda **w: similarity.crossTverskySimilarityMemoryConstrained(fp, **w)]
    for call in calls:
        for w in ({"alpha": bad, "beta": 0.5}, {"alpha": 0.5, "beta": bad}):
            with pytest.raises(ValueError):
                call(**w)


def test_weights_at_the_range_ends_are_accepted():
    assert similarity._check_weights(0, 1000) == (0.0, 1000.0)
    assert similarity._check_weights(np.float32(0.5), np.int64(2)) == (0.5, 2.0)


def test_weights_are_keyword_only():
    fp = np.zeros((4, 4), np.int32)
    with pytest.raises(TypeError):
        similarity.crossTverskySimilarity(fp, None, 0.5, 0.5)
    with pytest.raises(TypeError):
        similarity.topKTverskySimilarity(fp, None, 2, 0.5, 0.5)
    with pytest.raises(TypeError):
        similarity.thresholdTverskySimilarity(fp, None, 0.5, 0.5, 0.5)
    with pytest.raises(TypeError):
        similarity.crossTverskySimilarityMemoryConstrained(fp, None, 0.5, 0.5)


def test_stream_k_and_threshold_checks():
    with pytest.raises(TypeError):
        similarity.crossDiceSimilarity(object(), stream="not a stream")
    with pytest.raises(TypeError):
        similarity.topKDiceSimilarity(object(), k=3, stream=0)
    with pytest.raises(TypeError):
        similarity.topKTverskySimilarity(object(), k=3, alpha=1, beta=0, stream="s")
    with pytest.raises(TypeError):
        similarity.thresholdTverskySimilarity(object(), alpha=1, beta=0, threshold=0.5, stream=1)
    for t in (0, -0.1, 1.5, float("nan"), True, "0.5"):  # (the check the Dice and Tversky searches share)
        with pytest.raises(ValueError):
            similarity._check_threshold(t)
    for k in (0, 11, similarity.TOPK_MAX + 1, 2.0, True):
        with pytest.raises(ValueError):
            similarity._check_k(k, 10)


def test_the_library_exports_the_entry_points_and_checks_their_arguments(built_lib):
    L = built_lib
    for name in ("b200mol_tversky_cross", "b200mol_tversky_cross_host", "b200mol_tversky_topk", "b200mol_tversky_threshold"):
        assert hasattr(L, name)
    nnz = C.c_uint64(0)
    # null pointers
    assert L.b200mol_tversky_cross(None, 4, None, 0, 64, 0.5, 0.5, None, None) != 0
    assert L.b200mol_tversky_cross_host(None, 4, 16, 3, 64, 0.5, 0.5, None, 0) != 0
    assert L.b200mol_tversky_topk(None, 4, None, 0, 64, 0.5, 0.5, 2, None, None, None) != 0
    assert L.b200mol_tversky_threshold(16, 4, None, 0, 64, 0.5, 0.5, 0.5, None, None, None, 0, C.byref(nnz), None) != 0
    # widths
    assert L.b200mol_tversky_topk(16, 4, 16, 100, 63, 0.3, 0.7, 5, 16, 16, None) != 0
    assert L.b200mol_tversky_threshold(16, 4, 16, 100, 63, 0.3, 0.7, 0.5, 16, 16, 16, 4, C.byref(nnz), None) != 0
    # weights out of range, on every entry point, Dice-adjacent values included
    for a, b in ((float("nan"), 0.5), (0.5, float("inf")), (-1e-300, 0.5), (0.5, 1000.0000001)):
        assert L.b200mol_tversky_cross(16, 4, 16, 4, 64, a, b, 16, None) != 0
        assert b"Tversky weights" in L.b200mol_last_error()
        assert L.b200mol_tversky_cross_host(16, 4, 16, 4, 64, a, b, 16, 0) != 0
        assert L.b200mol_tversky_topk(16, 4, 16, 100, 64, a, b, 5, 16, 16, None) != 0
        assert L.b200mol_tversky_threshold(16, 4, 16, 100, 64, a, b, 0.5, 16, 16, 16, 4, C.byref(nnz), None) != 0
        assert b"Tversky weights" in L.b200mol_last_error()
    # k out of range, threshold out of range
    assert L.b200mol_tversky_topk(16, 4, 16, 100, 64, 0.9, 0.1, 101, 16, 16, None) != 0
    assert L.b200mol_tversky_topk(16, 4, 16, 1000, 64, 0.5, 0.5, similarity.TOPK_MAX + 1, 16, 16, None) != 0
    assert b"k must be" in L.b200mol_last_error()
    assert L.b200mol_tversky_threshold(16, 4, 16, 100, 64, 0.9, 0.1, 0.0, 16, 16, 16, 4, C.byref(nnz), None) != 0
