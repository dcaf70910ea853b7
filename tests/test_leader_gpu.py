"""Leader diversity picking on the GPU: picks equal (==) to the CPU oracle, with the bulk pass on the SIMT tile and on
the tensor-core tile, and with windows forced small so that windows and resolver blocks cut through the picks."""

import contextlib

import numpy as np
import pytest
import torch

from nvmolkit_b200 import _lib, synthetic
from nvmolkit_b200.diversity import LeaderPicker
from nvmolkit_b200.similarity import crossCosineSimilarity, crossTanimotoSimilarity
from nvmolkit_b200.types import AsyncGpuResult
from oracle import leader as oracle_leader

pytestmark = pytest.mark.gpu

BLOCK = 1024  # survivors per resolver block (leader.cu kBlock)
SIMT, TENSOR = -1, 0  # values of similarity_tensor_min_pairs
# (bulk tile, leader_window_rows): automatic windows, and windows that cut through resolver blocks and picks
PATHS = [(SIMT, 0), (TENSOR, 0), (SIMT, 300), (TENSOR, 2500)]


def _fingerprints(seed, n, words, density=0.08):
    rng = np.random.default_rng(seed)
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


def _clustered(seed, n, words, centres=12, flips=10):
    rng = np.random.default_rng(seed)
    base = _fingerprints(seed + 1, centres, words, 0.1)
    out = base[rng.integers(0, centres, n)].copy()
    pos = rng.integers(0, words * 32, (n, flips))
    keep = rng.integers(0, flips + 1, n)
    for k in range(flips):
        rows = np.nonzero(keep > k)[0]
        out[rows, pos[rows, k] >> 5] ^= np.uint32(1) << (pos[rows, k] & 31).astype(np.uint32)
    return out


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


@pytest.fixture
def path(cuda):
    """path(min_pairs, window_rows): force the bulk pass's tile and the window size until the test ends."""
    with contextlib.ExitStack() as scopes:
        def force(min_pairs, window):
            scopes.enter_context(_lib.options(similarity_tensor_min_pairs=min_pairs, leader_window_rows=window))
        yield force


def _pick(fp, pool, threshold, pick=0, first=(), metric="tanimoto", **kw):
    return LeaderPicker().LazyBitVectorPick(fp, pool, threshold, pick, first, metric=metric, **kw).numpy()


def _check(path, fp, pool, threshold, pick=0, first=(), metric="tanimoto", paths=PATHS):
    want = oracle_leader.leader_pick(fp, pool, threshold, pick, first, metric)
    d = _dev(fp)
    for min_pairs, window in paths:
        path(min_pairs, window)
        got = _pick(d, pool, threshold, pick, first, metric)
        assert got.dtype == np.int32 and got.shape == want.shape, (min_pairs, window, got.shape, want.shape)
        assert (got == want).all(), (min_pairs, window, np.argwhere(got != want)[:5].ravel(), got[:10], want[:10])
    return want


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("bits", list(range(128, 4097, 128)))
def test_every_width_both_metrics_both_bulk_tiles(path, metric, bits):
    fp = _clustered(bits, 1500, bits // 32, centres=40, flips=bits // 64)
    want = _check(path, fp, 1500, 0.35, 0, [7], metric=metric)
    assert 40 <= len(want) < 1500


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_windows_and_blocks_cut_through_many_picks(path, metric):
    fp = _clustered(2, 12_000, 16, centres=3000, flips=6)
    want = _check(path, fp, 12_000, 0.3, metric=metric, paths=PATHS + [(SIMT, 7), (TENSOR, BLOCK + 1)])
    assert len(want) > 2 * BLOCK  # the resolver runs several blocks in one window
    path(SIMT, 300)
    _pick(_dev(fp), 12_000, 0.3, metric=metric)
    assert _lib.get_option("leader_windows_last") == 40
    assert _lib.get_option("leader_bulk_pairs_last") > 0 and _lib.get_option("leader_block_pairs_last") > 0


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_threshold_on_a_pair_distance_and_one_ulp_either_side(path, metric):
    fp = _clustered(3, 600, 32, centres=20)
    cross = crossTanimotoSimilarity if metric == "tanimoto" else crossCosineSimilarity
    sim = cross(_dev(fp)).numpy()
    rng = np.random.default_rng(3)
    for i, j in rng.integers(0, 600, (6, 2)):
        if i == j:
            continue
        d = 1.0 - sim[i, j]
        pair = fp[[min(i, j), max(i, j)]]
        for thr, covered in ((d, True), (np.nextafter(d, -1.0), False), (np.nextafter(d, 2.0), True)):
            if not 0.0 <= thr <= 1.0:
                continue
            got = _check(path, pair, 2, thr, metric=metric)
            assert got.tolist() == ([0] if covered else [0, 1]), (i, j, thr, d)
            _check(path, fp, 600, thr, 0, [int(i)], metric=metric)


def test_degenerate_thresholds(path):
    fp = _fingerprints(4, 3000, 16)
    assert _check(path, fp, 3000, 0.0).tolist() == list(range(3000))  # distinct: every item is a pick
    assert _check(path, fp, 3000, 1.0).tolist() == [0]  # only the first pick
    assert _check(path, fp, 3000, 1.0, 0, [2999]).tolist() == [2999]
    assert _check(path, fp, 3000, 1.0, 0, [5, 1, 1700]).tolist() == [5, 1, 1700]  # first picks that leave nothing


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_duplicates_and_empty_fingerprints(path, metric):
    dup = np.repeat(_fingerprints(5, 700, 8), 3, axis=0)  # distance 0 within each run of three
    assert _check(path, dup, 2100, 0.0, metric=metric).tolist() == list(range(0, 2100, 3))
    fp = _clustered(6, 2500, 32, centres=30)
    rng = np.random.default_rng(6)
    empty = rng.choice(2500, 300, replace=False)
    fp[empty] = 0
    for thr in (0.0, 0.5, 0.99):
        got = _check(path, fp, 2500, thr, metric=metric)
        assert set(empty.tolist()) <= set(got.tolist()) and len(set(got.tolist())) == len(got)  # each picked once
    got = _check(path, fp, 2500, 1.0, 0, [int(empty[0])], metric=metric)
    assert got.tolist() == [int(empty[0])]  # threshold 1 covers even empty fingerprints
    assert _check(path, np.zeros((1500, 8), np.uint32), 1500, 0.7, metric=metric).tolist() == list(range(1500))


@pytest.mark.parametrize("n", [1, BLOCK - 1, BLOCK, BLOCK + 1])
def test_pool_sizes_at_the_block_edges(path, n):
    fp = _fingerprints(n, n + 40, 16)
    assert _check(path, fp, n, 0.0).tolist() == list(range(n))  # every item survives: blocks of exactly BLOCK
    _check(path, _clustered(n, n + 40, 16, centres=200), n, 0.4, 0, [n // 2])


def test_pool_shorter_than_the_matrix(path):
    fp = _clustered(7, 5000, 16, centres=400)
    full = _check(path, fp, 5000, 0.3)
    short = _check(path, fp, 3100, 0.3)
    assert short.tolist() == full[full < 3100].tolist()  # an item's fate depends only on the items before it


def test_pick_size_reached_exactly_at_a_window_end(path):
    fp = _fingerprints(8, 4000, 8)
    for window in (500, BLOCK, 1300):
        for pick in (window, 2 * window, window + 1, 1):
            _check(path, fp, 4000, 0.0, pick, paths=[(SIMT, window), (TENSOR, window)])
    fp = _clustered(9, 6000, 16, centres=800)
    full = _check(path, fp, 6000, 0.3)
    for pick in (1, 2, 300, len(full) - 1, len(full), len(full) + 1):
        got = _check(path, fp, 6000, 0.3, pick)
        assert got.tolist() == full[:pick].tolist()
    _check(path, fp, 6000, 0.3, 40, list(range(0, 6000, 150)))  # first picks fill pickSize


def test_first_picks_that_cover_each_other_and_items_below_them(path):
    fp = _clustered(10, 8000, 32, centres=100)
    sim = crossTanimotoSimilarity(_dev(fp[:200]), _dev(fp)).numpy()
    near = np.nonzero(1.0 - sim[0] <= 0.3)[0]
    first = [int(near[-1]), 0, 7999, int(near[len(near) // 2])]
    got = _check(path, fp, 8000, 0.3, 0, list(dict.fromkeys(first)))
    assert (np.diff(got[len(set(first)):]) > 0).all()


def test_side_stream_repeatability_and_morgan_input(path):
    fp = _clustered(11, 30_000, 64, centres=600)
    want = oracle_leader.leader_pick(fp, 30_000, 0.4, 0, [77])
    d = _dev(fp)
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    p1 = LeaderPicker().LazyBitVectorPick(AsyncGpuResult(d), 30_000, 0.4, 0, [77], 4, stream=stream)
    assert isinstance(p1, AsyncGpuResult) and (p1.numpy() == want).all()
    runs = [LeaderPicker().LazyBitVectorPick(d, 30_000, 0.4, firstPicks=[77]) for _ in range(3)]
    for p in runs:
        assert torch.equal(p.torch(), runs[0].torch()) and (p.numpy() == want).all()
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    graphs = synthetic.random_molgraphs(700, seed=12)
    morgan = MorganFingerprintGenerator(2, 1024).GetFingerprints(graphs)
    for thr in (0.3, 0.7):
        want = oracle_leader.leader_pick(morgan.numpy(), 700, thr)
        assert (LeaderPicker().LazyBitVectorPick(morgan, 700, thr).numpy() == want).all()


def test_one_million_2048_bit_clustered_against_the_oracle(path):
    fp = synthetic.clustered_fingerprints(20_000, 50, seed=31)
    want = oracle_leader.leader_pick(fp, len(fp), 0.65, 2000)  # (capped: about 30 s on 8 CPU threads)
    d = _dev(fp)
    for min_pairs in (1 << 24, SIMT):
        path(min_pairs, 0)
        got = LeaderPicker().LazyBitVectorPick(d, len(fp), 0.65, 2000).numpy()
        assert (got == want).all(), min_pairs
