"""Dice and Tversky on the GPU: matrices, top-k and threshold search equal (==) to the CPU oracle on the SIMT and the
tensor-core paths, at every width, for dyadic and non-dyadic weights."""

import contextlib

import numpy as np
import pytest
import torch

from nvmolkit_b200 import _lib, synthetic
from nvmolkit_b200 import similarity as S
from nvmolkit_b200.types import AsyncGpuResult
from oracle import tversky as O

pytestmark = pytest.mark.gpu

SIMT, TENSOR = "simt", "tensor"
DICE = (0.5, 0.5)
WEIGHTS = [DICE, (1.0, 1.0), (0.3, 0.7), (0.9, 0.1), (1.0, 0.0), (0.0, 1.0), (0.0, 0.0), (2.0, 2.0)]


def _fingerprints(seed, n, words, density=0.08):
    rng = np.random.default_rng(seed)
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


@pytest.fixture
def opts(cuda):
    """opts(SIMT) / opts(TENSOR, slab, key=value, ...): force a path (and library options) until the test ends."""
    with contextlib.ExitStack() as scopes:
        def force(which=None, slab=256, **kw):
            if which is not None:
                scopes.enter_context(_lib.options(similarity_tensor_min_pairs=-1 if which == SIMT else 0,
                                                  topk_slab_cols=slab))
            scopes.enter_context(_lib.options(**kw))
        yield force


def cross(q, lib, w):
    if w == DICE:
        return S.crossDiceSimilarity(_dev(q), _dev(lib)).numpy()
    return S.crossTverskySimilarity(_dev(q), _dev(lib), alpha=w[0], beta=w[1]).numpy()


def topk(q, lib, k, w):
    if w == DICE:
        v, i = S.topKDiceSimilarity(_dev(q), _dev(lib), k=k)
    else:
        v, i = S.topKTverskySimilarity(_dev(q), _dev(lib), k=k, alpha=w[0], beta=w[1])
    return v.numpy(), i.numpy()


def threshold(q, lib, t, w):
    if w == DICE:
        r = S.thresholdDiceSimilarity(_dev(q), _dev(lib), threshold=t)
    else:
        r = S.thresholdTverskySimilarity(_dev(q), _dev(lib), alpha=w[0], beta=w[1], threshold=t)
    return tuple(x.numpy() for x in r)


def _equal(got, want, what=""):
    for g, x in zip(got, want):
        assert g.dtype == x.dtype and g.shape == x.shape, (what, g.shape, x.shape)
        assert (g == x).all(), (what, np.argwhere(g != x)[:5])


def _check_all(q, lib, w, k, t, opts, paths=(SIMT, TENSOR)):
    want_m = O.cross(q, lib, *w)
    want_k = O.topk(q, lib, k, *w)
    want_t = O.threshold(q, lib, t, *w)
    for which in paths:
        opts(which)
        _equal((cross(q, lib, w),), (want_m,), (which, w, "cross"))
        _equal(topk(q, lib, k, w), want_k, (which, w, "topk"))
        _equal(threshold(q, lib, t, w), want_t, (which, w, "threshold"))


@pytest.mark.parametrize("w", WEIGHTS, ids=str)
@pytest.mark.parametrize("bits", list(range(128, 4097, 128)))
def test_every_width_every_weight_both_paths_cross_and_self(opts, bits, w):
    fp = synthetic.clustered_fingerprints(12, 30, bits=bits, p=0.1, max_flips=max(2, bits // 256), seed=bits)
    fp[200:230] = fp[5]
    fp[231:235] = 0
    q, lib = fp[:70], fp[70:]
    _check_all(q, lib, w, 17, 0.35, opts)
    _check_all(fp, None, w, 9, 0.35, opts)


@pytest.mark.parametrize("which", [SIMT, TENSOR])
def test_special_weights_equal_tanimoto_and_dice_and_dice_indices_equal_tanimoto(opts, which):
    fp = synthetic.clustered_fingerprints(40, 25, seed=3)
    q, lib = fp[:300], fp[300:]
    opts(which)
    dq, dl = _dev(q), _dev(lib)
    assert torch.equal(S.crossTverskySimilarity(dq, dl, alpha=1, beta=1).torch(), S.crossTanimotoSimilarity(dq, dl).torch())
    assert torch.equal(S.crossTverskySimilarity(dq, dl, alpha=0.5, beta=0.5).torch(), S.crossDiceSimilarity(dq, dl).torch())
    tv, ti = S.topKTanimotoSimilarity(dq, dl, k=40)
    v1, i1 = S.topKTverskySimilarity(dq, dl, k=40, alpha=1, beta=1)
    dv, di = S.topKDiceSimilarity(dq, dl, k=40)
    assert torch.equal(v1.torch(), tv.torch()) and torch.equal(i1.torch(), ti.torch())
    assert torch.equal(di.torch(), ti.torch())
    for a, b in zip(S.thresholdTverskySimilarity(dq, dl, alpha=1, beta=1, threshold=0.6),
                    S.thresholdTanimotoSimilarity(dq, dl, threshold=0.6)):
        assert torch.equal(a.torch(), b.torch())
    for a, b in zip(S.thresholdTverskySimilarity(dq, None, alpha=0.5, beta=0.5, threshold=0.6),
                    S.thresholdDiceSimilarity(dq, None, threshold=0.6)):
        assert torch.equal(a.torch(), b.torch())
    host = S.crossTverskySimilarityMemoryConstrained(q, lib, alpha=0.9, beta=0.1)
    assert (host == O.cross(q, lib, 0.9, 0.1)).all()
    assert (S.crossDiceSimilarityMemoryConstrained(q, None) == O.cross(q, None, 0.5, 0.5)).all()


@pytest.mark.parametrize("which", [SIMT, TENSOR])
def test_asymmetry_transpose_and_self_search_equals_the_set_passed_twice(opts, which):
    fp = synthetic.clustered_fingerprints(20, 25, seed=4)
    q, lib = fp[:150], fp[150:]
    opts(which)
    for a, b in ((0.9, 0.1), (1.0, 0.0), (0.3, 0.7)):
        assert (cross(q, lib, (a, b)) == cross(lib, q, (b, a)).T).all()
        _equal(threshold(fp, None, 0.5, (a, b)), threshold(fp, fp, 0.5, (a, b)), (which, a, b))
        _equal(threshold(fp, None, 0.5, (a, b)), O.threshold(fp, None, 0.5, a, b))


def _interval_fingerprints():
    """At 128 bits: queries [0, a), library every interval [s, e): every (|A|, |B|, c) with |A| + |B| - c <= 128."""
    q = np.zeros((129, 128), bool)
    for a in range(129):
        q[a, :a] = True
    spans = [(s, e) for s in range(128) for e in range(s + 1, 129)]
    lib = np.zeros((len(spans), 128), bool)
    for k, (s, e) in enumerate(spans):
        lib[k, s:e] = True
    pack = lambda b: np.packbits(b, axis=1, bitorder="little").view(np.uint32)  # noqa: E731
    return pack(q), pack(lib)


@pytest.mark.parametrize("w", [DICE, (0.3, 0.7), (0.9, 0.1)], ids=str)
def test_thresholds_on_a_pair_value_and_one_ulp_either_side_for_every_count_triple(opts, w):
    q, lib = _interval_fingerprints()
    vals = np.unique(O.threshold(q, lib, 1e-9, *w)[2])
    picks = [vals[k] for k in np.linspace(0, len(vals) - 1, 7).astype(int)] + [0.7, 0.5, 1 / 3, 2 / 3]
    ts = sorted({x for s in picks for x in (np.nextafter(s, 0.0), s, np.nextafter(s, 2.0)) if 0.0 < x <= 1.0})
    for t in ts:
        want = O.threshold(q, lib, t, *w)
        tiles = [(SIMT, 1, 1), (TENSOR, 1, 1)] + ([(TENSOR, 4, 4), (TENSOR, 4, 1)] if w == DICE else [])
        for which, s, c in tiles:
            opts(which, similarity_superpose=s, similarity_superpose_cols=c)
            _equal(threshold(q, lib, float(t), w), want, (which, s, c, t))


@pytest.mark.parametrize("self_search", [False, True])
def test_dice_graph_pass_superposition_band_and_clusters_give_identical_results(opts, self_search):
    fps = synthetic.clustered_fingerprints(400, 25, seed=40)
    q, lib = (fps, None) if self_search else (fps[:2500], fps[2500:])
    want = O.threshold(q, lib, 0.8, *DICE)
    assert want[0][-1] > 10 * len(q)
    for s, c in ((4, 4), (4, 2), (4, 1), (1, 1)):
        for band in (0, 1):
            for cluster in (0, 1, 3):
                opts(TENSOR, similarity_superpose=s, similarity_superpose_cols=c, similarity_popcount_band=band,
                     similarity_tensor_cluster=cluster)
                _equal(threshold(q, lib, 0.8, DICE), want, (s, c, band, cluster))
                assert _lib.get_option("similarity_superpose_last") == s * c


def test_a_loose_dice_threshold_overflows_the_superposed_candidate_list_and_falls_back(opts):
    q, lib = _fingerprints(50, 4096, 32, density=0.1), _fingerprints(51, 65536, 32, density=0.1)
    lib[777] = q[5]
    want = O.threshold(q, lib, 0.82, *DICE)
    assert 1 <= want[0][-1] < 1000
    opts(TENSOR)
    _equal(threshold(q, lib, 0.82, DICE), want)
    assert _lib.get_option("similarity_superpose_last") < 16


@pytest.mark.parametrize("w", [DICE, (0.9, 0.1), (1.0, 0.0)], ids=str)
def test_topk_ties_identical_library_and_supersets(opts, w):
    one = _fingerprints(50, 1, 64)
    lib = np.repeat(one, 1500, axis=0)
    q = np.concatenate([one, _fingerprints(51, 130, 64)])
    for which in (SIMT, TENSOR):
        opts(which)
        _equal(topk(q, lib, 100, w), O.topk(q, lib, 100, *w), (which, w))
    assert (topk(q, lib, 100, w)[1][0] == np.arange(100)).all()
    # Tversky(1, 0): every superset of a query scores 1.0; the ties go to the lowest index, before the self-match
    base = _fingerprints(52, 1, 32, density=0.05)
    lib = _fingerprints(53, 2000, 32)
    sup = np.random.default_rng(54).choice(2000, 300, replace=False)
    lib[sup] |= base
    lib[1500] = base[0]
    for which in (SIMT, TENSOR):
        opts(which)
        v, i = topk(lib, None, 50, (1.0, 0.0))
        wv, wi = O.topk(lib, None, 50, 1.0, 0.0)
        assert (v == wv).all() and (i == wi).all()
        assert (v[1500] == 1.0).all() and (i[1500] == np.unique(np.append(sup, 1500))[:50]).all()


def test_rows_whose_candidates_do_not_fit_are_redone_by_the_scan(opts):
    one = _fingerprints(52, 1, 64)
    lib = np.repeat(one, 5000, axis=0)
    q = np.concatenate([one, _fingerprints(53, 140, 64)])
    for w in ((0.9, 0.1), DICE):
        opts(TENSOR, 2048)
        _equal(topk(q, lib, 100, w), O.topk(q, lib, 100, *w), w)
    bits = np.zeros((4040, 4096), bool)
    bits[:, :50] = True
    for j in range(4040):
        bits[j, 50:50 + 4040 - j] = True
    lib = np.packbits(bits, axis=1, bitorder="little").view(np.uint32)
    q = np.concatenate([lib[-1:], _fingerprints(54, 10, 128)])
    opts(TENSOR, 2048)
    _equal(topk(q, lib, 33, DICE), O.topk(q, lib, 33, *DICE))
    assert _lib.get_option("topk_rows_redone_last") > 0
    _equal(topk(q, lib, 33, (0.0, 1.0)), O.topk(q, lib, 33, 0.0, 1.0))
    assert _lib.get_option("topk_rows_redone_last") > 0


@pytest.mark.parametrize("n", [1, 127, 128, 129, 257])
def test_tile_edges_empty_inputs_and_empty_fingerprints(opts, n):
    fp = _fingerprints(60 + n, n, 32)
    fp[::7] = 0
    lib = _fingerprints(61, 300, 32)
    lib[::11] = 0
    for w in (DICE, (0.9, 0.1)):
        _check_all(fp, lib, w, 1, 0.3, opts)
        _check_all(fp, None, w, 1, 0.3, opts)
    empty = np.zeros((0, 32), np.uint32)
    opts(TENSOR)
    assert cross(empty, lib, (0.9, 0.1)).shape == (0, 300)
    ip, ix, v = threshold(empty, lib, 0.5, (0.9, 0.1))
    assert ip.tolist() == [0] and len(ix) == 0 and len(v) == 0


def test_side_stream_repeatability_and_threshold_capacity_retry(opts):
    fps = synthetic.clustered_fingerprints(300, 25, seed=7)
    q, lib = fps[:500], fps[500:]
    opts(TENSOR, 512)
    stream = torch.cuda.Stream()
    dq, dl = _dev(q), _dev(lib)
    torch.cuda.synchronize()
    v1, i1 = S.topKTverskySimilarity(AsyncGpuResult(dq), AsyncGpuResult(dl), k=12, alpha=0.9, beta=0.1, stream=stream)
    m1 = S.crossTverskySimilarity(dq, dl, alpha=0.3, beta=0.7, stream=stream)
    stream.synchronize()
    v2, i2 = S.topKTverskySimilarity(dq, dl, k=12, alpha=0.9, beta=0.1)
    assert torch.equal(v1.torch(), v2.torch()) and torch.equal(i1.torch(), i2.torch())
    assert (m1.numpy() == O.cross(q, lib, 0.3, 0.7)).all()
    # a dense result (over the first-guess capacity of 2^20 entries) is fetched with a second call
    fp = np.repeat(_fingerprints(8, 3, 16, density=0.3), 700, axis=0)
    want = O.threshold(fp, None, 0.2, 0.9, 0.1)
    assert want[0][-1] > (1 << 20)
    _equal(threshold(fp, None, 0.2, (0.9, 0.1)), want)
    want = O.threshold(fp, None, 0.2, *DICE)
    _equal(threshold(fp, None, 0.2, DICE), want)


def test_production_size_against_the_oracle(cuda):
    fps = synthetic.clustered_fingerprints(41_000, 25, seed=6)
    lib, q = fps[:1_000_000], fps[1_000_000:1_002_048]
    want_v, want_i = O.topk(q, lib, 50, 0.9, 0.1)
    v, i = topk(q, lib, 50, (0.9, 0.1))
    assert (i == want_i).all() and (v == want_v).all()
    assert _lib.get_option("topk_slabs_last") >= 3
    _equal(threshold(q, lib, 0.8, DICE), O.threshold(q, lib, 0.8, *DICE))  # (the superposed graph pass)
