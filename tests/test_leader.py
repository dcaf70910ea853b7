"""Leader diversity picking without a GPU: the CPU oracle against a NumPy definition, and argument validation in Python
and through the C-ABI."""

import numpy as np
import pytest

import oracle
from nvmolkit_b200 import diversity
from oracle import leader as oracle_leader


def _fingerprints(rng, n, words, density=0.1):
    bits = rng.random((n, words * 32)) < density
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32)


def _clustered(rng, n, words, centres=6, flips=6):
    base = _fingerprints(rng, centres, words)
    out = base[rng.integers(0, centres, n)].copy()
    for row in out:
        for b in rng.integers(0, words * 32, rng.integers(0, flips + 1)):
            row[b >> 5] ^= np.uint32(1) << np.uint32(b & 31)
    return out


def _numpy_leader(fp, pool, threshold, pick=0, first=(), metric="tanimoto"):
    """The definition: first picks, then every item in index order that no earlier pick covers (1 - s <= threshold)."""
    dist = 1.0 - oracle.similarity_cross(fp[:pool], fp[:pool], metric)
    cap = pool if pick == 0 else pick
    picks = list(first)
    for i in range(pool):
        if len(picks) >= cap:
            break
        if i in picks or any(dist[p, i] <= threshold for p in first):
            continue
        if not any(dist[p, i] <= threshold for p in picks[len(first):]):
            picks.append(i)
    return np.array(picks[:cap], np.int32)


def _pools():
    rng = np.random.default_rng(21)
    empty = _fingerprints(rng, 90, 8)
    empty[rng.choice(90, 25, replace=False)] = 0
    yield "random", _fingerprints(rng, 150, 8)
    yield "clustered", _clustered(rng, 200, 16)
    yield "identical", np.repeat(_fingerprints(rng, 1, 8), 40, axis=0)
    yield "empty_rows", empty


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("threshold", [0.0, 0.35, 0.65, 0.9, 1.0])
def test_oracle_is_the_numpy_definition(metric, threshold):
    for name, fp in _pools():
        pool = len(fp) - 3
        for pick in (0, 1, 7):
            for first in ((), (17,), (30, 3, 5)):
                want = _numpy_leader(fp, pool, threshold, pick, first, metric)
                if pick and len(first) > pick:
                    continue
                got = oracle_leader.leader_pick(fp, pool, threshold, pick, first, metric)
                assert got.dtype == np.int32 and (got.tolist() == want.tolist()), (name, pick, first, got, want)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_first_picks_that_cover_each_other_and_items_below_them(metric):
    rng = np.random.default_rng(22)
    fp = _clustered(rng, 300, 16, centres=4, flips=3)
    dist = 1.0 - oracle.similarity_cross(fp, fp, metric)
    # two first picks in one cluster (each covers the other) and a third far above index 0 of its cluster
    a = int(np.nonzero(dist[0, 1:] <= 0.2)[0][-1]) + 1
    first = [a, 0, 250]
    for thr in (0.2, 0.5):
        assert dist[a, 0] <= thr
        want = _numpy_leader(fp, 300, thr, 0, first, metric)
        got = oracle_leader.leader_pick(fp, 300, thr, 0, first, metric)
        assert got.tolist() == want.tolist()
        assert got[:3].tolist() == first and (np.diff(got[3:]) > 0).all()
        # nothing after the first picks lies within the threshold of a first pick
        assert (dist[np.ix_(first, got[3:])] > thr).all()
    # first picks that leave nothing: threshold 1 covers every item
    assert oracle_leader.leader_pick(fp, 300, 1.0, 0, [9, 4], metric).tolist() == [9, 4]


def test_degenerate_thresholds():
    rng = np.random.default_rng(23)
    fp = _fingerprints(rng, 120, 8)
    assert oracle_leader.leader_pick(fp, 120, 0.0).tolist() == list(range(120))  # distinct: every item is a pick
    assert oracle_leader.leader_pick(fp, 120, 1.0).tolist() == [0]
    assert oracle_leader.leader_pick(fp, 120, 1.0, 0, [57]).tolist() == [57]
    dup = np.repeat(fp[:3], 5, axis=0)  # distance 0 within each run of five
    assert oracle_leader.leader_pick(dup, 15, 0.0).tolist() == [0, 5, 10]
    zero = np.zeros((6, 4), np.uint32)  # empty fingerprints: distance 1 to everything, each picked once
    assert oracle_leader.leader_pick(zero, 6, 0.99).tolist() == list(range(6))
    assert oracle_leader.leader_pick(zero, 6, 1.0).tolist() == [0]


def test_pick_size_caps_a_run_and_zero_means_no_limit():
    rng = np.random.default_rng(24)
    fp = _clustered(rng, 400, 8, centres=30)
    full = oracle_leader.leader_pick(fp, 400, 0.3)
    assert len(full) > 10
    for cap in (1, 5, len(full), len(full) + 3):
        assert oracle_leader.leader_pick(fp, 400, 0.3, cap).tolist() == full[:cap].tolist()
    assert oracle_leader.leader_pick(fp, 380, 0.3).tolist() == _numpy_leader(fp, 380, 0.3).tolist()  # pool < rows


def test_oracle_threads_do_not_change_the_picks():
    rng = np.random.default_rng(25)
    fp = _clustered(rng, 3000, 32, centres=60)
    before = oracle.set_threads(0)
    try:
        oracle.set_threads(1)
        one = oracle_leader.leader_pick(fp, 3000, 0.4, 0, [77])
        oracle.set_threads(max(2, before))
        many = oracle_leader.leader_pick(fp, 3000, 0.4, 0, [77])
    finally:
        oracle.set_threads(before)
    assert one.tolist() == many.tolist() == _numpy_leader(fp, 3000, 0.4, 0, [77]).tolist()


@pytest.mark.parametrize("kw", [
    dict(poolSize=0), dict(poolSize=101), dict(pickSize=-1), dict(pickSize=51), dict(poolSize=50, pickSize=51),
    dict(firstPicks=[1, 2, 3], pickSize=2), dict(firstPicks=[50]), dict(firstPicks=[-1]), dict(firstPicks=[4, 4]),
    dict(metric="dice"), dict(words=6), dict(words=132), dict(words=0), dict(poolSize=5.0), dict(pickSize=True),
    dict(threshold=float("nan")), dict(threshold=-1e-300), dict(threshold=1.0000000000000002), dict(threshold="x"),
    dict(threshold=None), dict(pickSize=False),
])
def test_argument_errors(kw):
    args = dict(n=100, words=64, poolSize=50, threshold=0.5, pickSize=10, firstPicks=(), metric="tanimoto")
    args.update(kw)
    with pytest.raises(ValueError):
        diversity._leader_args(**args)


def test_valid_arguments_and_stream_checked_first():
    assert diversity._leader_args(100, 4, 100, 0.0, 0, np.array([3, 99]), "cosine") == (100, 0.0, [3, 99])
    assert diversity._leader_args(100, 128, 1, 1, 1, (), "tanimoto") == (1, 1.0, [])
    assert diversity._leader_args(100, 8, 60, 0.65, 0, (), "tanimoto")[0] == 60  # pickSize 0: no limit
    with pytest.raises(TypeError):
        diversity.LeaderPicker().LazyBitVectorPick(object(), 10, 0.5, stream="not a stream")


def test_c_abi_checks_its_arguments_before_device_work(built_lib):
    first = (np.ctypeslib.as_ctypes_type(np.int32) * 2)(3, 3)
    one = (np.ctypeslib.as_ctypes_type(np.int32) * 1)(3)
    call = built_lib.b200mol_leader_pick
    assert call(16, 100, 64, 7, 0.5, one, 1, 10, 16, 16, None) != 0  # metric
    assert b"metric" in built_lib.b200mol_last_error()
    assert call(16, 100, 63, 0, 0.5, one, 1, 10, 16, 16, None) != 0  # width
    assert call(16, 100, 132, 0, 0.5, one, 1, 10, 16, 16, None) != 0  # width
    for thr in (float("nan"), -0.1, 1.5):
        assert call(16, 100, 64, 0, thr, one, 1, 10, 16, 16, None) != 0
        assert b"threshold" in built_lib.b200mol_last_error()
    assert call(16, 100, 64, 0, 0.5, one, 1, 101, 16, 16, None) != 0  # pickSize > pool
    assert call(16, 100, 64, 0, 0.5, one, 1, 0, 16, 16, None) != 0  # pickSize 0 (the Python layer maps it)
    assert call(16, 0, 64, 0, 0.5, one, 1, 1, 16, 16, None) != 0  # empty pool
    assert call(16, 100, 64, 0, 0.5, first, 2, 1, 16, 16, None) != 0  # more first picks than pickSize
    assert call(16, 100, 64, 0, 0.5, first, 2, 10, 16, 16, None) != 0  # repeated
    assert b"repeated" in built_lib.b200mol_last_error()
    assert call(16, 3, 64, 0, 0.5, one, 1, 2, 16, 16, None) != 0  # outside the pool
    assert b"outside the pool" in built_lib.b200mol_last_error()
    assert call(None, 100, 64, 0, 0.5, one, 1, 10, 16, 16, None) != 0  # null fingerprints
    assert call(16, 100, 64, 0, 0.5, one, 1, 10, None, 16, None) != 0  # null picks
    assert call(16, 100, 64, 0, 0.5, one, 1, 10, 16, None, None) != 0  # null pick count
    assert call(16, 100, 64, 0, 0.5, None, 1, 10, 16, 16, None) != 0  # null first picks with nFirst = 1
    assert b"null pointer" in built_lib.b200mol_last_error()
    assert call(20, 100, 64, 0, 0.5, one, 1, 10, 16, 16, None) != 0  # misaligned
    assert b"aligned" in built_lib.b200mol_last_error()
