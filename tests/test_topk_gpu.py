"""Top-k similarity search on the GPU: values and indices equal (==) to the CPU oracle on both kernel paths."""

import contextlib

import numpy as np
import pytest
import torch

from nvmolkit_b200 import _lib, synthetic
from nvmolkit_b200.similarity import (TOPK_MAX, crossTanimotoSimilarity, topKCosineSimilarity, topKTanimotoSimilarity)
from nvmolkit_b200.types import AsyncGpuResult
from oracle import topk as oracle_topk

pytestmark = pytest.mark.gpu

SEARCH = {"tanimoto": topKTanimotoSimilarity, "cosine": topKCosineSimilarity}
SIMT, TENSOR = "simt", "tensor"


def _fingerprints(seed, n, words, density=0.08):
    rng = np.random.default_rng(seed)
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


@pytest.fixture
def path(cuda):
    """path(SIMT) / path(TENSOR, slab): force one kernel path (and the tensor path's slab size) until the test ends."""
    with contextlib.ExitStack() as scopes:
        def force(which, slab=256):
            scopes.enter_context(_lib.options(similarity_tensor_min_pairs=-1 if which == SIMT else 0, topk_slab_cols=slab))
        yield force


def _search(metric, q, lib, k, **kw):
    v, i = SEARCH[metric](_dev(q), None if lib is None else _dev(lib), k=k, **kw)
    return v.numpy(), i.numpy()


def _check(metric, q, lib, k, path, slab=256, slabs=None):
    want_v, want_i = oracle_topk.topk(q, lib, k, metric)
    for which in (SIMT, TENSOR):
        path(which, slab)
        got_v, got_i = _search(metric, q, lib, k)
        assert got_i.dtype == np.int32 and got_v.dtype == np.float64 and got_v.shape == (len(q), k)
        assert (got_i == want_i).all(), (which, np.argwhere(got_i != want_i)[:5])
        assert (got_v == want_v).all(), which
        if which == TENSOR and slabs is not None:
            assert _lib.get_option("topk_slabs_last") >= slabs


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("bits", [128, 256, 512, 1024, 2048])
def test_every_width_both_metrics_both_paths(path, metric, bits):
    lib = _fingerprints(bits, 1100, bits // 32)
    q = _fingerprints(bits + 1, 129, bits // 32)
    _check(metric, q, lib, 33, path, slabs=3)


@pytest.mark.parametrize("k", [1, 2, 31, 32, 33, 100, TOPK_MAX])
def test_k_values(path, k):
    lib = _fingerprints(20, 900, 16)
    _check("tanimoto", _fingerprints(21, 70, 16), lib, k, path, slabs=2)
    _check("cosine", _fingerprints(22, 5, 16), lib, k, path)


def test_k_equal_to_the_library_size(path):
    lib = _fingerprints(23, 200, 16)
    _check("tanimoto", _fingerprints(24, 40, 16), lib, 200, path)
    _check("cosine", _fingerprints(24, 40, 16), _fingerprints(25, 300, 16), 45, path, slab=64)


@pytest.mark.parametrize("nq", [1, 127, 128, 129, 1000])
def test_query_counts_around_the_tile(path, nq):
    _check("tanimoto", _fingerprints(30 + nq, nq, 32), _fingerprints(31, 1300, 32), 10, path, slabs=4)


@pytest.mark.parametrize("m", [257, 511, 512, 513, 767, 768, 769, 1024, 1025, 1281])
def test_library_sizes_around_tiles_and_slab_boundaries(path, m):
    _check("tanimoto", _fingerprints(40, 129, 32), _fingerprints(41 + m, m, 32), 20, path)
    _check("cosine", _fingerprints(40, 30, 32), _fingerprints(41 + m, m, 32), 20, path)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_library_of_identical_fingerprints_every_pair_ties_with_the_bar(path, metric):
    one = _fingerprints(50, 1, 64)
    lib = np.repeat(one, 1500, axis=0)
    q = np.concatenate([one, _fingerprints(51, 130, 64)])
    _check(metric, q, lib, 100, path)
    path(TENSOR)
    _, idx = _search(metric, q, lib, 100)
    assert (idx == np.arange(100)).all()  # ties go to the lowest index


def test_rows_whose_candidates_do_not_fit_are_redone_by_the_scan(path):
    """Slabs of 2,048 columns against 1,792 candidate slots per row. Cosine: in a library of identical fingerprints every
    pair ties with the bar, and the tile's float filter lets ties through. Tanimoto: every column is a superset of the
    query with one bit fewer than the column before it, so each one beats the bar."""
    one = _fingerprints(52, 1, 64)
    lib = np.repeat(one, 5000, axis=0)
    q = np.concatenate([one, _fingerprints(53, 140, 64)])
    _check("cosine", q, lib, 100, path, slab=2048, slabs=2)
    assert _lib.get_option("topk_rows_redone_last") > 0
    bits = np.zeros((4040, 4096), bool)
    bits[:, :50] = True
    for j in range(4040):
        bits[j, 50:50 + 4040 - j] = True
    lib = np.packbits(bits, axis=1, bitorder="little").view(np.uint32)
    q = np.concatenate([lib[-1:], _fingerprints(54, 10, 128)])
    _check("tanimoto", q, lib, 33, path, slab=2048, slabs=1)
    assert _lib.get_option("topk_rows_redone_last") > 0


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_planted_duplicates_empty_fingerprints_and_self_matches(path, metric):
    lib = _fingerprints(60, 2000, 64)
    rng = np.random.default_rng(61)
    lib[rng.choice(2000, 300, replace=False)] = lib[1234]  # duplicates at scattered indices
    lib[rng.choice(2000, 200, replace=False)] = 0          # similarity 0 with everything
    q = np.concatenate([lib[::97], np.zeros((3, 64), np.uint32), _fingerprints(62, 40, 64, density=0.01)])
    _check(metric, q, lib, 64, path)
    _check(metric, q, lib, TOPK_MAX, path)


def test_queries_against_themselves_self_match_first(path):
    fp = _fingerprints(70, 1500, 64)
    fp[900] = fp[10]
    want_v, want_i = oracle_topk.topk(fp, None, 5)
    for which in (SIMT, TENSOR):
        path(which)
        v, i = topKTanimotoSimilarity(_dev(fp), k=5)
        v, i = v.numpy(), i.numpy()
        assert (i == want_i).all() and (v == want_v).all()
        assert (v[:, 0] == 1.0).all() and i[10, 0] == 10 and i[10, 1] == 900 and i[900, 0] == 10 and i[900, 1] == 900


def test_inputs_streams_and_repeatability(path):
    lib, q = _fingerprints(80, 3000, 64), _fingerprints(81, 200, 64)
    want_v, want_i = oracle_topk.topk(q, lib, 12)
    path(TENSOR, 512)
    stream = torch.cuda.Stream()
    dq, dl = _dev(q), _dev(lib)
    torch.cuda.synchronize()
    v1, i1 = topKTanimotoSimilarity(AsyncGpuResult(dq), AsyncGpuResult(dl), k=12, stream=stream)
    v2, i2 = topKTanimotoSimilarity(dq, dl, k=12)
    assert isinstance(v1, AsyncGpuResult) and isinstance(i1, AsyncGpuResult)
    for v, i in ((v1, i1), (v2, i2)):
        assert (i.numpy() == want_i).all() and (v.numpy() == want_v).all()
    assert torch.equal(v1.torch(), v2.torch()) and torch.equal(i1.torch(), i2.torch())


def test_argument_validation(cuda):
    fp = _dev(_fingerprints(90, 50, 16))
    with pytest.raises(TypeError):
        topKTanimotoSimilarity(fp, k=3, stream=1)
    with pytest.raises(ValueError):
        topKTanimotoSimilarity(fp.to(torch.float32), k=3)
    with pytest.raises(ValueError):
        topKTanimotoSimilarity(fp[0], k=3)
    with pytest.raises(ValueError):
        topKTanimotoSimilarity(fp, fp[:, :8].contiguous(), k=3)
    for k in (0, 51, TOPK_MAX + 1):
        with pytest.raises(ValueError):
            topKCosineSimilarity(fp, k=k)


def test_values_agree_with_torch_topk_over_the_matrix(cuda):
    fps = synthetic.clustered_fingerprints(1440, 25, seed=5)
    q, lib = _dev(fps[:4096]), _dev(fps[4096:4096 + 32768])
    v, i = topKTanimotoSimilarity(q, lib, k=20)
    sim = crossTanimotoSimilarity(q, lib).torch()
    tv, _ = torch.topk(sim, 20, dim=1)
    assert torch.equal(v.torch(), tv)
    assert torch.equal(torch.gather(sim, 1, i.torch().long()), tv)  # indices may differ only inside a tie


def test_production_size_against_the_oracle(cuda):
    fps = synthetic.clustered_fingerprints(41_000, 25, seed=6)
    lib, q = fps[:1_000_000], fps[1_000_000:1_002_048]
    want_v, want_i = oracle_topk.topk(q, lib, 50)
    v, i = topKTanimotoSimilarity(_dev(q), _dev(lib), k=50)
    assert (i.numpy() == want_i).all() and (v.numpy() == want_v).all()
    assert _lib.get_option("topk_slabs_last") >= 3
