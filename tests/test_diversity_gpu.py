"""MaxMin diversity picking on the GPU: picks equal (==) to the CPU oracles and the threshold bit-equal, in both modes,
with the pool resident in shared memory and streamed."""

import contextlib

import numpy as np
import pytest
import torch

from nvmolkit_b200 import _lib, synthetic
from nvmolkit_b200.diversity import MaxMinPicker, seeded_first_pick
from nvmolkit_b200.similarity import crossCosineSimilarity, crossTanimotoSimilarity
from nvmolkit_b200.types import AsyncGpuResult
from oracle import pick as oracle_pick

pytestmark = pytest.mark.gpu

DENSE, DEFERRED = 0, 1
STREAMED, RESIDENT = 0, -1  # values of maxmin_resident_rows
PATHS = [(m, r) for m in (DENSE, DEFERRED) for r in (RESIDENT, STREAMED)]


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
    """path(mode, resident_rows): force a mode and a fingerprint placement until the test ends."""
    with contextlib.ExitStack() as scopes:
        def force(mode, resident):
            scopes.enter_context(_lib.options(maxmin_mode=mode, maxmin_resident_rows=resident))
        yield force


def _pick(fp, pool, pick, first=(), threshold=None, metric="tanimoto", **kw):
    picker = MaxMinPicker()
    if threshold is None:
        return picker.LazyBitVectorPick(fp, pool, pick, firstPicks=first, metric=metric, **kw).numpy(), None
    p, t = picker.LazyBitVectorPickWithThreshold(fp, pool, pick, threshold, firstPicks=first, metric=metric, **kw)
    return p.numpy(), float(t.numpy()[0])


def _check(path, fp, pool, pick, first, threshold=None, metric="tanimoto", paths=PATHS, oracle=oracle_pick.maxmin_lazy):
    want_p, want_t = oracle(fp, pool, pick, first, -1.0 if threshold is None else threshold, metric)
    d = _dev(fp)
    for mode, resident in paths:
        path(mode, resident)
        got_p, got_t = _pick(d, pool, pick, first, threshold, metric)
        assert got_p.dtype == np.int32 and got_p.shape == (pick,)
        assert (got_p == want_p).all(), (mode, resident, np.argwhere(got_p != want_p)[:5].ravel(), got_p[:10], want_p[:10])
        if threshold is not None:
            assert got_t == want_t, (mode, resident, got_t, want_t)  # bit-equal fp64
        assert _lib.get_option("maxmin_resident_last") == (1 if resident else 0)
    return want_p, want_t


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("bits", [128, 256, 384, 512, 1024, 2048, 4096])
def test_every_width_both_metrics_both_modes_both_placements(path, metric, bits):
    fp = _clustered(bits, 1001, bits // 32)
    _check(path, fp, 1001, 90, [5], threshold=-1.0, metric=metric)


@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 1000, 1001, 5003, 17_000])
def test_pool_sizes_and_uneven_slices(path, n):
    fp = _clustered(n, n + 7, 16)
    _check(path, fp, n, min(n, 40), [n // 2])


def test_pick_size_equal_to_the_pool_and_a_pool_shorter_than_the_matrix(path):
    fp = _clustered(1, 700, 16)
    _check(path, fp, 300, 300, [0])
    _check(path, fp, 650, 650, [649], metric="cosine")
    _check(path, fp, 1, 1, [0], threshold=0.0)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_all_duplicate_pool_ties_at_distance_zero_go_to_the_lowest_index(path, metric):
    fp = np.repeat(_fingerprints(2, 1, 64), 900, axis=0)
    want, _ = _check(path, fp, 900, 50, [400], metric=metric)
    assert want.tolist() == [400] + list(range(49))
    _check(path, fp, 900, 50, [400], threshold=0.0, metric=metric)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_empty_fingerprints(path, metric):
    fp = _clustered(3, 1500, 32)
    rng = np.random.default_rng(4)
    fp[rng.choice(1500, 200, replace=False)] = 0
    _check(path, fp, 1500, 120, [int(np.nonzero(fp.any(axis=1))[0][0])], threshold=-1.0, metric=metric)
    _check(path, fp, 1500, 120, [int(np.nonzero(~fp.any(axis=1))[0][0])], threshold=-1.0, metric=metric)
    _check(path, np.zeros((300, 8), np.uint32), 300, 30, [3], threshold=-1.0, metric=metric)


def test_one_and_many_first_picks(path):
    fp = _clustered(5, 3000, 64, centres=30)
    _check(path, fp, 3000, 100, [2999])
    _check(path, fp, 3000, 100, list(range(0, 3000, 97)), threshold=-1.0)
    _check(path, fp, 3000, 31, list(range(0, 3000, 97)), threshold=0.1)  # the first picks fill pickSize: -1


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_threshold_on_and_between_max_min_values(path, metric):
    fp = _clustered(6, 2500, 64, centres=25)
    full, _ = oracle_pick.maxmin_lazy(fp, 2500, 80, [9], -1.0, metric)
    sim = (crossTanimotoSimilarity if metric == "tanimoto" else crossCosineSimilarity)(_dev(fp[full])).numpy()
    mins = [float((1.0 - sim[k, :k]).min()) for k in range(1, 80)]
    for k in (1, 20, 60):
        for thr in (mins[k], (mins[k] + mins[k - 1]) / 2, np.nextafter(mins[k], 2.0)):
            _, got = _check(path, fp, 2500, 80, [9], threshold=thr, metric=metric)
            assert got == mins[k - 1] or got in mins  # the max-min of the last pick added
    _, got = _check(path, fp, 2500, 80, [9], threshold=1.0, metric=metric)  # stops before the first loop pick
    assert got == -1.0


def test_seeded_first_pick_is_the_python_restatement(path):
    fp = _clustered(7, 4000, 64)
    for seed in (0, 42, 12345):
        first = seeded_first_pick(4000, seed)
        want, _ = oracle_pick.maxmin_lazy(fp, 4000, 25, [first])
        got = MaxMinPicker().LazyBitVectorPick(_dev(fp), 4000, 25, seed=seed).numpy()
        assert (got == want).all()
    got = MaxMinPicker().LazyBitVectorPick(_dev(fp), 4000, 25).numpy()  # seed -1: a random start, still a valid pick set
    assert len(set(got.tolist())) == 25 and (got >= 0).all() and (got < 4000).all()


def test_side_stream_repeatability_and_morgan_input(path):
    fp = _clustered(8, 20_000, 64, centres=200)
    want, _ = oracle_pick.maxmin_lazy(fp, 20_000, 150, [77])
    d = _dev(fp)
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    p1, t1 = MaxMinPicker().LazyBitVectorPickWithThreshold(AsyncGpuResult(d), 20_000, 150, -1.0, [77], stream=stream)
    p2 = MaxMinPicker().LazyBitVectorPick(d, 20_000, 150, [77])
    assert isinstance(p1, AsyncGpuResult) and isinstance(t1, AsyncGpuResult)
    assert (p1.numpy() == want).all() and (p2.numpy() == want).all()
    runs = [MaxMinPicker().LazyBitVectorPickWithThreshold(d, 20_000, 150, 0.05, [77]) for _ in range(3)]
    for p, t in runs[1:]:
        assert torch.equal(p.torch(), runs[0][0].torch()) and torch.equal(t.torch(), runs[0][1].torch())
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    graphs = synthetic.random_molgraphs(500, seed=9)
    morgan = MorganFingerprintGenerator(2, 1024).GetFingerprints(graphs)
    want, _ = oracle_pick.maxmin_lazy(morgan.numpy(), 500, 60, [0])
    assert (MaxMinPicker().LazyBitVectorPick(morgan, 500, 60, [0]).numpy() == want).all()


def test_deferred_mode_evaluates_fewer_distances_on_clustered_data(path):
    fp = synthetic.clustered_fingerprints(2000, 25, seed=11)
    d = _dev(fp)
    counts = {}
    picks = {}
    for mode in (DENSE, DEFERRED):
        path(mode, RESIDENT)
        picks[mode] = MaxMinPicker().LazyBitVectorPick(d, len(fp), 500, [0]).numpy()
        counts[mode] = _lib.get_option("maxmin_distances_last")
    assert (picks[DENSE] == picks[DEFERRED]).all()
    assert 0 < counts[DEFERRED] < counts[DENSE], counts


def _torch_loop(d, pool, pick, first):
    """What a user could build from the public calls: a one-row similarity, torch.minimum, torch.argmax per pick."""
    picks = list(first)
    mn = torch.full((pool,), float("inf"), dtype=torch.float64, device=d.device)
    for p in picks:
        mn = torch.minimum(mn, 1.0 - crossTanimotoSimilarity(d[p:p + 1], d[:pool]).torch()[0])
    taken = torch.zeros(pool, dtype=torch.bool, device=d.device)
    taken[picks] = True
    while len(picks) < pick:
        w = int(torch.argmax(torch.where(taken, -1.0, mn)))  # first maximum: the lowest index
        picks.append(w)
        taken[w] = True
        mn = torch.minimum(mn, 1.0 - crossTanimotoSimilarity(d[w:w + 1], d[:pool]).torch()[0])
    return np.array(picks, np.int32)


@pytest.mark.parametrize("mode", [DENSE, DEFERRED])
def test_host_driven_torch_loop_at_50k(path, mode):
    fp = synthetic.clustered_fingerprints(2000, 25, seed=12)
    d = _dev(fp)
    want = _torch_loop(d, 50_000, 300, [123])
    path(mode, -1)
    assert (MaxMinPicker().LazyBitVectorPick(d, 50_000, 300, [123]).numpy() == want).all()


def test_one_million_2048_bit_clustered_against_the_dense_oracle(path):
    fp = synthetic.clustered_fingerprints(40_000, 25, seed=13)
    want, want_t = oracle_pick.maxmin_dense(fp, len(fp), 200, [0], 0.0)
    d = _dev(fp)
    for mode in (DENSE, DEFERRED):
        path(mode, -1)
        p, t = MaxMinPicker().LazyBitVectorPickWithThreshold(d, len(fp), 200, 0.0, [0])
        assert (p.numpy() == want).all() and float(t.numpy()[0]) == want_t, mode
        assert _lib.get_option("maxmin_resident_last") == 0


def test_state_in_global_memory_above_two_million_items(path):
    fp = _clustered(14, 2_100_000, 4, centres=5000, flips=3)
    want, _ = oracle_pick.maxmin_dense(fp, len(fp), 60, [1])
    d = _dev(fp)
    for mode in (DENSE, DEFERRED):
        path(mode, -1)
        assert (MaxMinPicker().LazyBitVectorPick(d, len(fp), 60, [1]).numpy() == want).all(), mode
