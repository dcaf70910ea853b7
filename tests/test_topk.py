"""Top-k similarity search without a GPU: the oracle against NumPy, argument validation, and the exported symbol."""

import re

import numpy as np
import pytest

import oracle
from nvmolkit_b200 import similarity
from oracle import topk as oracle_topk


def _lexsort_topk(sim, k):
    cols = np.arange(sim.shape[1])
    idx = np.stack([np.lexsort((cols, -row))[:k] for row in sim])
    return np.take_along_axis(sim, idx, axis=1), idx.astype(np.int32)


def _fingerprints(rng, n, words, density=0.1):
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("k", [1, 7, 64, 150])
def test_oracle_topk_is_lexsort_of_the_matrix(metric, k):
    rng = np.random.default_rng(11)
    lib = _fingerprints(rng, 150, 8)
    lib[40:60] = lib[3]  # duplicates: every query ties over them
    lib[100:110] = 0  # similarity 0
    q = np.concatenate([_fingerprints(rng, 20, 8), lib[[3, 45, 105]]])
    want_v, want_i = _lexsort_topk(oracle.similarity_cross(q, lib, metric), k)
    got_v, got_i = oracle_topk.topk(q, lib, k, metric)
    assert (got_i == want_i).all() and (got_v == want_v).all()


def test_oracle_topk_of_a_set_against_itself_puts_the_self_match_before_later_duplicates():
    rng = np.random.default_rng(12)
    fp = _fingerprints(rng, 60, 4)
    fp[50] = fp[7]
    v, i = oracle_topk.topk(fp, None, 3)
    assert i[7, 0] == 7 and i[7, 1] == 50 and v[7, 0] == 1.0 and v[7, 1] == 1.0
    assert i[50, 0] == 7 and i[50, 1] == 50


def test_stream_argument_is_validated_first():
    with pytest.raises(TypeError):
        similarity.topKTanimotoSimilarity(object(), k=3, stream="not a stream")
    with pytest.raises(TypeError):
        similarity.topKCosineSimilarity(object(), k=3, stream=0)


@pytest.mark.parametrize("k", [0, -1, 11, similarity.TOPK_MAX + 1, 2.0, "3", True])
def test_k_outside_its_range_is_a_value_error(k):
    with pytest.raises(ValueError):
        similarity._check_k(k, 10 if k != similarity.TOPK_MAX + 1 else 10_000)


def test_k_limit_matches_the_header_and_the_library_exports_the_entry_point(built_lib):
    assert similarity._check_k(similarity.TOPK_MAX, 10_000) == similarity.TOPK_MAX
    import os

    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200mol.h")).read()
    assert int(re.search(r"#define\s+B200MOL_TOPK_MAX\s+(\d+)", header).group(1)) == similarity.TOPK_MAX >= 256
    assert hasattr(built_lib, "b200mol_similarity_topk")
    # the C-ABI checks its arguments before it touches the device
    assert built_lib.b200mol_similarity_topk(None, 4, None, 0, 64, 0, 5, None, None, None) != 0
    assert built_lib.b200mol_similarity_topk(16, 4, 16, 100, 64, 7, 5, 16, 16, None) != 0  # unknown metric
    assert built_lib.b200mol_similarity_topk(16, 4, 16, 100, 63, 0, 5, 16, 16, None) != 0  # width
    assert built_lib.b200mol_similarity_topk(16, 4, 16, 100, 64, 0, 101, 16, 16, None) != 0  # k > library
    assert built_lib.b200mol_similarity_topk(16, 4, 16, 1000, 64, 0, similarity.TOPK_MAX + 1, 16, 16, None) != 0
    assert b"k must be" in built_lib.b200mol_last_error()
