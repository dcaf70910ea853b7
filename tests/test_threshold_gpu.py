"""Threshold similarity search on the GPU: indptr, indices and values equal (==) to the CPU oracle on every path."""

import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from nvmolkit_b200 import _lib, synthetic
from nvmolkit_b200.similarity import thresholdCosineSimilarity, thresholdTanimotoSimilarity
from nvmolkit_b200.types import AsyncGpuResult
from oracle import threshold as oracle_threshold

pytestmark = pytest.mark.gpu

SEARCH = {"tanimoto": thresholdTanimotoSimilarity, "cosine": thresholdCosineSimilarity}
SIMT, TENSOR = "simt", "tensor"


def _fingerprints(seed, n, words, density=0.08):
    rng = np.random.default_rng(seed)
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


@pytest.fixture
def opts(cuda):
    """opts(key=value, ...): set library options until the test ends; opts(SIMT) / opts(TENSOR) forces a tile."""
    with contextlib.ExitStack() as scopes:
        def force(which=None, **kw):
            if which is not None:
                scopes.enter_context(_lib.options(similarity_tensor_min_pairs=-1 if which == SIMT else 0))
            scopes.enter_context(_lib.options(**kw))
        yield force


def _search(metric, q, lib, t, **kw):
    r = SEARCH[metric](_dev(q), None if lib is None else _dev(lib), threshold=t, **kw)
    return tuple(x.numpy() for x in r)


def _equal(got, want, what=""):
    for g, w, dtype in zip(got, want, (np.int64, np.int32, np.float64)):
        assert g.dtype == dtype and g.shape == w.shape, (what, g.shape, w.shape)
        assert (g == w).all(), (what, np.argwhere(g != w)[:5])


def _check(metric, q, lib, t, opts, paths=(SIMT, TENSOR)):
    want = oracle_threshold.threshold(q, lib, t, metric)
    for which in paths:
        opts(which)
        _equal(_search(metric, q, lib, t), want, (which, metric, t))
    return want


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("bits", list(range(128, 4097, 128)))
def test_every_width_both_metrics_both_tiles_cross_and_self(opts, metric, bits):
    fp = synthetic.clustered_fingerprints(12, 30, bits=bits, p=0.1, max_flips=max(2, bits // 256), seed=bits)
    fp[200:230] = fp[5]
    q, lib = fp[:70], fp[70:]
    t = 0.35
    _check(metric, q, lib, t, opts)
    _check(metric, fp, None, t, opts)


def _interval_fingerprints():
    """At 128 bits: queries [0, a) for a = 0..128, library every interval [s, e). A query and a library row realise
    every (|A|, |B|, c) with |A| + |B| - c <= 128 (B = [a - c, a - c + b))."""
    q = np.zeros((129, 128), bool)
    for a in range(129):
        q[a, :a] = True
    spans = [(s, e) for s in range(128) for e in range(s + 1, 129)]
    lib = np.zeros((len(spans), 128), bool)
    for k, (s, e) in enumerate(spans):
        lib[k, s:e] = True
    pack = lambda b: np.packbits(b, axis=1, bitorder="little").view(np.uint32)  # noqa: E731
    return pack(q), pack(lib)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_thresholds_on_a_pair_value_and_one_ulp_either_side_for_every_count_triple(opts, metric):
    q, lib = _interval_fingerprints()
    sims = np.unique(oracle_threshold.threshold(q, lib, 1e-9, metric)[2])
    picks = [sims[k] for k in np.linspace(0, len(sims) - 1, 9).astype(int)] + [0.7, 0.5, 1 / 3, 2 / 3]
    thresholds = sorted({x for s in picks for x in (np.nextafter(s, 0.0), s, np.nextafter(s, 2.0)) if 0.0 < x <= 1.0})
    for t in thresholds:
        want = oracle_threshold.threshold(q, lib, t, metric)
        tiles = [(SIMT, 1, 1), (TENSOR, 1, 1)] + ([(TENSOR, 4, 4), (TENSOR, 4, 1)] if metric == "tanimoto" else [])
        for which, s, c in tiles:
            opts(which, similarity_superpose=s, similarity_superpose_cols=c)
            _equal(_search(metric, q, lib, float(t)), want, (which, s, c, t))
            if which == TENSOR and metric == "tanimoto":
                assert _lib.get_option("similarity_superpose_last") == s * c


@pytest.mark.parametrize("self_search", [False, True])
def test_cross_graph_pass_superposition_band_and_clusters_give_identical_results(opts, self_search):
    fps = synthetic.clustered_fingerprints(400, 25, seed=40)
    q, lib = (fps, None) if self_search else (fps[:2500], fps[2500:])
    want = oracle_threshold.threshold(q, lib, 0.7)
    assert want[0][-1] > 10 * len(q)  # a real graph
    for s, c in ((4, 4), (4, 2), (4, 1), (1, 1)):
        for band in (0, 1):
            for cluster in (0, 1, 3):
                opts(TENSOR, similarity_superpose=s, similarity_superpose_cols=c, similarity_popcount_band=band,
                     similarity_tensor_cluster=cluster)
                _equal(_search("tanimoto", q, lib, 0.7), want, (s, c, band, cluster))
                assert _lib.get_option("similarity_superpose_last") == s * c


def test_a_loose_threshold_overflows_the_superposed_candidate_list_and_falls_back(opts):
    q, lib = _fingerprints(50, 4096, 32, density=0.1), _fingerprints(51, 65536, 32, density=0.1)
    lib[777] = q[5]
    want = oracle_threshold.threshold(q, lib, 0.7)
    assert 1 <= want[0][-1] < 1000
    opts(TENSOR)
    _equal(_search("tanimoto", q, lib, 0.7), want)
    assert _lib.get_option("similarity_superpose_last") < 16  # 4 x 4 overflowed; a narrower pass completed the search


def _abi(metric, q, lib, t, cap, stream=None):
    """b200mol_similarity_threshold with capacity `cap`: (nnz, indptr, indices[:cap], values[:cap]) on the device."""
    nq = q.shape[0]
    indptr = torch.full((nq + 1,), -7, dtype=torch.int64, device="cuda")
    indices = torch.full((max(cap, 1),), -7, dtype=torch.int32, device="cuda")
    values = torch.full((max(cap, 1),), -7.0, dtype=torch.float64, device="cuda")
    nnz = C.c_uint64(0)
    _lib.call("b200mol_similarity_threshold", q.data_ptr(), nq, None if lib is None else lib.data_ptr(),
              0 if lib is None else lib.shape[0], q.shape[1], _lib.METRIC[metric], t, indptr.data_ptr(),
              indices.data_ptr(), values.data_ptr(), cap, C.byref(nnz), 0 if stream is None else stream.cuda_stream)
    torch.cuda.synchronize()
    return int(nnz.value), indptr, indices, values


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_too_small_a_capacity_reports_the_total_and_writes_nothing(opts, metric):
    fps = synthetic.clustered_fingerprints(60, 25, seed=41)
    q, lib = _dev(fps[:500]), _dev(fps[500:])
    want = oracle_threshold.threshold(fps[:500], fps[500:], 0.6, metric)
    nnz = int(want[0][-1])
    assert nnz > 100
    for which in (SIMT, TENSOR):
        opts(which)
        for cap in (0, 1, nnz - 1):
            got, indptr, indices, values = _abi(metric, q, lib, 0.6, cap)
            assert got == nnz
            assert (indptr == -7).all() and (indices == -7).all() and (values == -7.0).all()
        got, indptr, indices, values = _abi(metric, q, lib, 0.6, nnz)
        assert got == nnz
        _equal((indptr.cpu().numpy(), indices.cpu().numpy(), values.cpu().numpy()), want)
        # a self search: the diagonal and the mirrored pairs count too
        want_self = oracle_threshold.threshold(fps, None, 0.6, metric)
        got, *_ = _abi(metric, _dev(fps), None, 0.6, 3)
        assert got == want_self[0][-1]


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_the_python_wrapper_retries_with_the_reported_size(opts, metric):
    """Every pair passes at 1e-3 among similar fingerprints: more than the first guess of max(2^20, 64 Q) entries."""
    fps = synthetic.clustered_fingerprints(1, 1100, seed=42)
    assert len(fps) * len(fps) > 1 << 20
    for which in (SIMT, TENSOR):
        opts(which)
        got = _search(metric, fps, None, 1e-3)
        _equal(got, oracle_threshold.threshold(fps, None, 1e-3, metric), which)
        assert got[0][-1] > 1 << 20


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_self_search_equals_the_set_passed_twice_with_empty_and_duplicate_fingerprints(opts, metric):
    fp = _fingerprints(60, 2000, 64)
    rng = np.random.default_rng(61)
    fp[rng.choice(2000, 300, replace=False)] = fp[1234]  # duplicates at scattered indices
    fp[rng.choice(2000, 100, replace=False)] = 0  # similarity 0 with everything, themselves included
    for t in (0.2, 1.0):
        want = _check(metric, fp, None, t, opts)
        _equal(_search(metric, fp, fp, t), want, "twice, tensor")
        opts(SIMT)
        _equal(_search(metric, fp, fp, t), want, "twice, simt")


@pytest.mark.parametrize("nq", [1, 127, 128, 129, 255, 256, 257])
@pytest.mark.parametrize("nlib", [1, 127, 129, 255, 256, 257])
def test_sizes_around_the_tile_edges(opts, nq, nlib):
    fps = synthetic.clustered_fingerprints(40, 15, seed=43)
    q, lib = fps[:nq], fps[600:600 + nlib]
    for metric in ("tanimoto", "cosine"):
        _check(metric, q, lib, 0.45, opts)
    if nlib == 1:
        _check("tanimoto", q, None, 0.45, opts)


def test_empty_inputs(opts):
    fp = _fingerprints(62, 10, 16)
    for which in (SIMT, TENSOR):
        opts(which)
        indptr, indices, values = _search("tanimoto", fp[:0], fp, 0.5)
        assert indptr.tolist() == [0] and len(indices) == len(values) == 0
        indptr, indices, values = _search("cosine", fp, fp[:0], 0.5)
        assert indptr.tolist() == [0] * 11 and len(indices) == 0


def test_side_stream_repeatability_and_inputs(opts):
    fps = synthetic.clustered_fingerprints(200, 25, seed=44)
    q, lib = fps[:1000], fps[1000:]
    want = oracle_threshold.threshold(q, lib, 0.65)
    opts(TENSOR)
    stream = torch.cuda.Stream()
    dq, dl = _dev(q), _dev(lib)
    torch.cuda.synchronize()
    one = thresholdTanimotoSimilarity(AsyncGpuResult(dq), AsyncGpuResult(dl), threshold=0.65, stream=stream)
    two = thresholdTanimotoSimilarity(dq, dl, threshold=0.65)
    assert all(isinstance(x, AsyncGpuResult) for x in one)
    _equal(tuple(x.numpy() for x in one), want)
    for a, b in zip(one, two):
        assert torch.equal(a.torch(), b.torch())
    indptr, indices, values = (x.torch() for x in two)
    m = torch.sparse_csr_tensor(indptr, indices, values, size=(len(q), len(lib)))
    assert torch.equal(m.to_dense().cpu(), torch.from_numpy(_dense(want, len(q), len(lib))))


def _dense(csr, n, m):
    out = np.zeros((n, m))
    indptr, indices, values = csr
    for i in range(n):
        out[i, indices[indptr[i]:indptr[i + 1]]] = values[indptr[i]:indptr[i + 1]]
    return out


def test_argument_validation(cuda):
    fp = _dev(_fingerprints(90, 50, 16))
    with pytest.raises(TypeError):
        thresholdTanimotoSimilarity(fp, threshold=float("nan"), stream=1)
    with pytest.raises(ValueError):
        thresholdTanimotoSimilarity(fp, threshold=0.0)
    with pytest.raises(ValueError):
        thresholdCosineSimilarity(fp, threshold=1.5)
    with pytest.raises(ValueError):
        thresholdTanimotoSimilarity(fp.to(torch.float32), threshold=0.5)
    with pytest.raises(ValueError):
        thresholdTanimotoSimilarity(fp, fp[:, :8].contiguous(), threshold=0.5)
    with pytest.raises(TypeError):
        thresholdTanimotoSimilarity(fp, 0.5)  # threshold is keyword-only


def test_production_size_against_the_oracle(cuda):
    fps = synthetic.clustered_fingerprints(41_000, 25, seed=6)
    lib, q = fps[:1_000_000], fps[1_000_000:1_002_048]
    want = oracle_threshold.threshold(q, lib, 0.7)
    assert want[0][-1] > 10 * len(q)
    _equal(_search("tanimoto", q, lib, 0.7), want, "tanimoto")
    q = q[:512]  # (the oracle's share of the test's time)
    _equal(_search("cosine", q, lib, 0.7), oracle_threshold.threshold(q, lib, 0.7, "cosine"), "cosine")
