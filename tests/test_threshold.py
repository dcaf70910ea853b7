"""Threshold similarity search without a GPU: the oracle against NumPy, argument validation, and the exported symbol."""

import ctypes as C

import numpy as np
import pytest

import oracle
from nvmolkit_b200 import similarity
from oracle import threshold as oracle_threshold


def _fingerprints(rng, n, words, density=0.1):
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


def _nonzero_csr(sim, t):
    rows, cols = np.nonzero(sim >= t)  # row-major: columns ascending within a row
    indptr = np.zeros(sim.shape[0] + 1, np.int64)
    np.add.at(indptr, rows + 1, 1)
    return np.cumsum(indptr), cols.astype(np.int32), sim[rows, cols]


def _check(q, lib, t, metric):
    want = _nonzero_csr(oracle.similarity_cross(q, q if lib is None else lib, metric), t)
    got = oracle_threshold.threshold(q, lib, t, metric)
    for g, w, dtype in zip(got, want, (np.int64, np.int32, np.float64)):
        assert g.dtype == dtype and g.shape == w.shape and (g == w).all()
    return got


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("t", [1e-3, 0.05, 0.1, 0.3, 1 / 3, 0.5, 0.7, 0.9, 1.0])
def test_oracle_is_nonzero_of_the_matrix(metric, t):
    rng = np.random.default_rng(31)
    lib = _fingerprints(rng, 170, 8)
    lib[40:60] = lib[3]  # duplicates: similarity 1 with each other
    lib[100:110] = 0  # similarity 0 with everything, themselves included
    q = np.concatenate([_fingerprints(rng, 20, 8), lib[[3, 45, 105]], np.zeros((2, 8), np.uint32)])
    _check(q, lib, t, metric)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_oracle_of_a_set_against_itself_keeps_the_self_matches_of_non_empty_fingerprints(metric):
    rng = np.random.default_rng(32)
    fp = _fingerprints(rng, 90, 4, density=0.3)
    fp[50] = fp[7]
    fp[60] = 0
    indptr, indices, values = _check(fp, None, 1.0, metric)
    row = lambda i: indices[indptr[i]:indptr[i + 1]].tolist()  # noqa: E731
    assert row(7) == [7, 50] and row(50) == [7, 50] and row(60) == [] and row(3) == [3]
    assert (values == 1.0).all()
    _check(fp, None, 1e-3, metric)


def test_oracle_of_empty_inputs():
    fp = _fingerprints(np.random.default_rng(33), 5, 4)
    indptr, indices, values = oracle_threshold.threshold(fp[:0], fp, 0.5)
    assert indptr.tolist() == [0] and len(indices) == len(values) == 0
    indptr, indices, values = oracle_threshold.threshold(fp, fp[:0], 0.5)
    assert indptr.tolist() == [0] * 6 and len(indices) == 0


def test_stream_argument_is_validated_first():
    with pytest.raises(TypeError):
        similarity.thresholdTanimotoSimilarity(object(), threshold=float("nan"), stream="not a stream")
    with pytest.raises(TypeError):
        similarity.thresholdCosineSimilarity(object(), threshold=2.0, stream=0)


@pytest.mark.parametrize("t", [0, 0.0, -0.5, 1.0000000000000002, 1.5, float("nan"), float("inf"), True, False, "0.5", None])
def test_threshold_outside_its_range_is_a_value_error(t):
    with pytest.raises(ValueError):
        similarity._check_threshold(t)


@pytest.mark.parametrize("t", [1, 1.0, 0.7, 5e-324, np.float32(0.5), np.float64(0.25)])
def test_thresholds_in_range_are_accepted(t):
    assert similarity._check_threshold(t) == float(t)


def test_the_library_exports_the_entry_point_and_checks_its_arguments(built_lib):
    assert hasattr(built_lib, "b200mol_similarity_threshold")
    call = built_lib.b200mol_similarity_threshold
    nnz = C.c_uint64(0)
    ok = (16, 100, 16, 200, 64, 0, 0.5, 16, 16, 16, 10, C.byref(nnz), None)  # a valid call, never made here

    def bad(**kw):
        args = list(ok)
        for k, v in kw.items():
            args[("q", "nq", "lib", "nlib", "words", "metric", "t", "indptr", "indices", "values", "cap", "nnz").index(k)] = v
        return call(*args)

    assert bad(metric=7) != 0 and b"metric" in built_lib.b200mol_last_error()
    for words in (63, 0, 132):
        assert bad(words=words) != 0 and b"width" in built_lib.b200mol_last_error()
    for t in (0.0, -0.1, 1.5, float("nan"), float("inf")):
        assert bad(t=t) != 0 and b"threshold" in built_lib.b200mol_last_error()
    assert bad(nq=1 << 31) != 0 and b"too many" in built_lib.b200mol_last_error()
    assert bad(nlib=1 << 31) != 0 and b"too many" in built_lib.b200mol_last_error()
    assert bad(q=None) != 0 and b"null" in built_lib.b200mol_last_error()
    assert bad(indptr=None) != 0 and b"null" in built_lib.b200mol_last_error()
    assert bad(nnz=None) != 0 and b"null" in built_lib.b200mol_last_error()
    assert bad(indices=None) != 0 and b"null" in built_lib.b200mol_last_error()
    assert bad(values=None) != 0 and b"null" in built_lib.b200mol_last_error()
    assert bad(q=20) != 0 and b"aligned" in built_lib.b200mol_last_error()
    assert bad(lib=24) != 0 and b"aligned" in built_lib.b200mol_last_error()
