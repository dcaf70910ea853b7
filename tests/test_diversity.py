"""MaxMin diversity picking without a GPU: both CPU oracles against the NumPy definition, the first-pick generator, and
argument validation."""

import numpy as np
import pytest

import oracle
from nvmolkit_b200 import diversity
from oracle import pick as oracle_pick


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


def _numpy_maxmin(fp, pool, pick, first, threshold=-1.0, metric="tanimoto"):
    """The definition: argmax over the running min of 1 - similarity_cross, ties to the lowest index."""
    dist = 1.0 - oracle.similarity_cross(fp[:pool], fp[:pool], metric)
    picks = list(first)
    mn = np.full(pool, np.inf)
    for p in picks:
        mn = np.minimum(mn, dist[:, p])
    last = -1.0
    while len(picks) < pick:
        cand = mn.copy()
        cand[picks] = -np.inf
        w = int(np.argmax(cand))  # first occurrence: the lowest index
        if threshold >= 0.0 and cand[w] <= threshold:
            break
        picks.append(w)
        last = float(cand[w])
        mn = np.minimum(mn, dist[:, w])
    return np.array(picks + [-1] * (pick - len(picks)), np.int32), last


def _pools():
    rng = np.random.default_rng(3)
    empty = _fingerprints(rng, 90, 8)
    empty[rng.choice(90, 25, replace=False)] = 0
    yield "random", _fingerprints(rng, 150, 8)
    yield "clustered", _clustered(rng, 200, 16)
    yield "identical", np.repeat(_fingerprints(rng, 1, 8), 40, axis=0)
    yield "empty_rows", empty


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("first", [[0], [17], [5, 3, 30]])
def test_lazy_oracle_is_the_numpy_definition(metric, first):
    for name, fp in _pools():
        pool = len(fp) - 3
        for pick in (1 + len(first), 12, pool):
            if pick < len(first):
                continue
            want = _numpy_maxmin(fp, pool, pick, first, metric=metric)
            got = oracle_pick.maxmin_lazy(fp, pool, pick, first, metric=metric)
            assert (got[0] == want[0]).all(), (name, pick, got[0], want[0])
            assert got[1] == want[1], name


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_threshold_stops_exactly_on_and_between_max_min_values(metric):
    rng = np.random.default_rng(4)
    fp = _clustered(rng, 180, 8)
    full, _ = _numpy_maxmin(fp, 180, 40, [7], metric=metric)
    dist = 1.0 - oracle.similarity_cross(fp, fp, metric)
    mins = [dist[full[k], full[:k]].min() for k in range(1, 40)]  # the max-min value of each loop pick
    for k in (3, 10, 25):
        for thr in (mins[k], np.nextafter(mins[k], 1.0), (mins[k] + mins[k - 1]) / 2):
            want = _numpy_maxmin(fp, 180, 40, [7], thr, metric)
            for run in (oracle_pick.maxmin_lazy, oracle_pick.maxmin_dense):
                got = run(fp, 180, 40, [7], thr, metric)
                assert (got[0] == want[0]).all() and got[1] == want[1], (run.__name__, k, thr)
                assert (got[0] == -1).sum() > 0 or thr < min(mins)
    # a stop before the first loop pick, and first picks that fill pickSize: threshold -1 in both cases
    assert oracle_pick.maxmin_lazy(fp, 180, 5, [7], 2.0, metric)[1] == -1.0
    p, t = oracle_pick.maxmin_lazy(fp, 180, 2, [7, 8], -1.0, metric)
    assert p.tolist() == [7, 8] and t == -1.0


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
def test_dense_oracle_is_the_lazy_oracle(metric):
    for name, fp in _pools():
        for first in ([0], [len(fp) // 2, 1]):
            want = oracle_pick.maxmin_lazy(fp, len(fp), len(fp), first, metric=metric)
            got = oracle_pick.maxmin_dense(fp, len(fp), len(fp), first, metric=metric)
            assert (got[0] == want[0]).all() and got[1] == want[1], name
    rng = np.random.default_rng(5)
    fp = _clustered(rng, 3000, 64, centres=40)
    want = oracle_pick.maxmin_lazy(fp, 2900, 150, [11], metric=metric)
    got = oracle_pick.maxmin_dense(fp, 2900, 150, [11], metric=metric)
    assert (got[0] == want[0]).all() and got[1] == want[1]


def test_mt19937_ten_thousandth_output_is_the_standard_value():
    g = diversity.MT19937(5489)
    for _ in range(9999):
        g()
    assert g() == 4123659995


@pytest.mark.parametrize("seed", [0, 1, 42, 5489, 2**31 - 1, 2**32 - 1])
def test_mt19937_equals_numpy_legacy_seeding(seed):
    bg = np.random.MT19937()
    bg._legacy_seeding(seed)
    want = bg.random_raw(1300)  # past one twist of the 624-word state
    g = diversity.MT19937(seed)
    assert [g() for _ in range(1300)] == want.tolist()


def test_uniform_int_buckets_by_hand():
    def words(*ws):
        it = iter(ws)
        return lambda: next(it)

    # one item: no word is drawn
    assert diversity.uniform_int(words(), 1) == 0
    # a power of two: buckets of 2^32 / 2^k, never a rejection (0xFFFFFFFF % 8 == 7 adds one to 0xFFFFFFFF // 8)
    assert [diversity.uniform_int(words(w), 8) for w in (0, 0x1FFFFFFF, 0x20000000, 0xFFFFFFFF)] == [0, 0, 1, 7]
    # 2^31 + 1 items: buckets of one value; words >= 2^31 + 1 are drawn again
    n = 2**31 + 1
    assert diversity.uniform_int(words(0xFFFFFFFF, 0x80000001, 0x80000000), n) == 0x80000000
    # 3 items: 0xFFFFFFFF % 3 == 0, buckets of 0x55555555; only 0xFFFFFFFF falls past the last one
    assert diversity.uniform_int(words(0xFFFFFFFF, 0x55555555), 3) == 1
    assert diversity.uniform_int(words(0x55555554), 3) == 0


def test_seeded_first_pick_is_deterministic_and_in_the_pool():
    picks = [diversity.seeded_first_pick(1000, s) for s in range(50)]
    assert picks == [diversity.seeded_first_pick(1000, s) for s in range(50)]
    assert all(0 <= p < 1000 for p in picks) and len(set(picks)) > 30
    g = diversity.MT19937(42)
    assert diversity.seeded_first_pick(1000, 42) == g() // (0xFFFFFFFF // 1000)
    assert 0 <= diversity.seeded_first_pick(7, -1) < 7


@pytest.mark.parametrize("kw", [
    dict(poolSize=0), dict(poolSize=101), dict(pickSize=0), dict(pickSize=51), dict(poolSize=50, pickSize=51),
    dict(firstPicks=[1, 2, 3], pickSize=2), dict(firstPicks=[50]), dict(firstPicks=[-1]), dict(firstPicks=[4, 4]),
    dict(metric="dice"), dict(words=6), dict(words=132), dict(words=0), dict(poolSize=5.0), dict(pickSize=True),
])
def test_argument_errors(kw):
    args = dict(n=100, words=64, poolSize=50, pickSize=10, firstPicks=(), metric="tanimoto")
    args.update(kw)
    with pytest.raises(ValueError):
        diversity._check_args(**args)


def test_valid_arguments_and_stream_checked_first():
    assert diversity._check_args(100, 4, 100, 100, np.array([3, 99]), "cosine") == [3, 99]
    assert diversity._check_args(100, 128, 1, 1, (), "tanimoto") == []
    with pytest.raises(TypeError):
        diversity.MaxMinPicker().LazyBitVectorPick(object(), 10, 5, stream="not a stream")
    with pytest.raises(TypeError):
        diversity.MaxMinPicker().LazyBitVectorPickWithThreshold(object(), 10, 5, 0.5, stream=0)


def test_c_abi_checks_its_arguments_before_device_work(built_lib):
    first = (np.ctypeslib.as_ctypes_type(np.int32) * 2)(3, 3)
    one = (np.ctypeslib.as_ctypes_type(np.int32) * 1)(3)
    call = built_lib.b200mol_maxmin_pick
    assert call(16, 100, 64, 7, one, 1, 10, -1.0, 16, 16, None) != 0  # metric
    assert call(16, 100, 63, 0, one, 1, 10, -1.0, 16, 16, None) != 0  # width
    assert call(16, 100, 64, 0, one, 1, 101, -1.0, 16, 16, None) != 0  # pickSize > pool
    assert call(16, 0, 64, 0, one, 1, 1, -1.0, 16, 16, None) != 0  # empty pool
    assert call(16, 100, 64, 0, one, 0, 10, -1.0, 16, 16, None) != 0  # no first pick
    assert call(16, 100, 64, 0, first, 2, 10, -1.0, 16, 16, None) != 0  # repeated
    assert b"repeated" in built_lib.b200mol_last_error()
    assert call(16, 3, 64, 0, one, 1, 2, -1.0, 16, 16, None) != 0  # outside the pool
    assert b"outside the pool" in built_lib.b200mol_last_error()
