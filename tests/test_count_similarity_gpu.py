"""Tanimoto, Dice and Tversky on count vectors on the GPU, compared with == against the count oracle: every measure,
cross and self, at 1, 127, 2048 and 4096 bins (both query-block shapes), count and row edges, top-k ties, sizes and the
slab protocol with its redo, threshold boundaries and the capacity retry, streams and repeatability."""

import ctypes as C

import numpy as np
import pytest
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200 import similarity as S
from oracle import count as oracle_count

pytestmark = pytest.mark.gpu
MEASURES = [((1.0, 1.0), "Tanimoto"), ((0.5, 0.5), "Dice"), ((0.3, 0.7), "Tversky"), ((0.9, 0.1), "Tversky"),
            ((1.0, 0.0), "Tversky"), ((2.0, 0.25), "Tversky")]


def calls(name):
    return (getattr(S, f"cross{name}CountSimilarity"), getattr(S, f"topK{name}CountSimilarity"),
            getattr(S, f"threshold{name}CountSimilarity"))


def kw(weights, name):
    return {"alpha": weights[0], "beta": weights[1]} if name == "Tversky" else {}


def counts(rng, n, bins, density=0.05, high=5):
    return np.where(rng.random((n, bins)) < density, rng.integers(1, high, size=(n, bins)), 0).astype(np.int32)


def dev(x, dtype=torch.int32):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dtype).cuda()


def edge_rows(rng, bins):
    q, lib = counts(rng, 70, bins, 0.3, 4), counts(rng, 300, bins, 0.1, 300)
    lib[[0, 1]] = 0
    lib[2] = 65535              # fully dense at the bound
    lib[3] = q[0]               # identical
    lib[4] = q[0]               # a tie of the identical one
    lib[5] = np.where(q[1] > 0, 65535, 0)
    lib[6, :] = rng.choice([0, 1, 255, 256, 65535], size=bins)
    lib[10:20] = lib[7]         # duplicates: ties
    q[2] = 0
    q[3] = lib[6]
    return q, lib


@pytest.mark.parametrize("bins", [1, 127, 2048, 4096])
@pytest.mark.parametrize("weights,name", MEASURES)
def test_matrix_cross_and_self(cuda, bins, weights, name):
    rng = np.random.default_rng(bins)
    q, lib = edge_rows(rng, bins)
    cross = calls(name)[0]
    got = cross(dev(q), dev(lib), **kw(weights, name)).numpy()
    assert np.array_equal(got, oracle_count.cross(q, lib, *weights))
    got = cross(dev(lib), **kw(weights, name)).numpy()
    assert np.array_equal(got, oracle_count.cross(lib, lib, *weights))
    if name == "Tanimoto":
        assert (np.diag(got)[lib.sum(1) > 0] == 1.0).all() and (got[[0, 1]] == 0).all()


def test_input_dtypes_and_the_count_range(cuda):
    rng = np.random.default_rng(5)
    q, lib = counts(rng, 40, 300, 0.2, 255), counts(rng, 50, 300, 0.2, 255)
    want = oracle_count.cross(q, lib)
    for dtype in (torch.uint8, torch.int16, torch.int32):
        assert np.array_equal(S.crossTanimotoCountSimilarity(dev(q, dtype), dev(lib, dtype)).numpy(), want)
    ok = np.array([[0, 1, 255, 256, 65535]], np.int32)
    assert S.crossTanimotoCountSimilarity(dev(ok)).numpy()[0, 0] == 1.0
    out = torch.full((1, 1), 7.0, dtype=torch.float64, device="cuda")
    for bad, dtype in (([[0, 65536]], torch.int32), ([[-1, 3]], torch.int32), ([[-1, 3]], torch.int16)):
        b = dev(np.array(bad), dtype)
        for call in (lambda: S.crossDiceCountSimilarity(b), lambda: S.topKTanimotoCountSimilarity(b, k=1),
                     lambda: S.thresholdTverskyCountSimilarity(b, alpha=0.3, beta=0.7, threshold=0.5)):
            with pytest.raises(ValueError, match="outside 0 .. 65535"):
                call()
        with pytest.raises(ValueError):
            _lib.call("b200mol_count_cross", b.to(torch.int32).data_ptr(), 1, None, 1, 2, 1.0, 1.0, out.data_ptr(), None)
        assert out.item() == 7.0  # nothing written
    for bad in (np.zeros((3, 4097), np.int32), np.zeros((3, 0), np.int32)):
        with pytest.raises(ValueError, match="bins"):
            S.crossTanimotoCountSimilarity(dev(bad))
    with pytest.raises(ValueError, match="dtype"):
        S.crossTanimotoCountSimilarity(dev(q, torch.int64))
    with pytest.raises(ValueError, match="2D"):
        S.crossTanimotoCountSimilarity(dev(q[0]))
    with pytest.raises(ValueError, match="widths"):
        S.crossTanimotoCountSimilarity(dev(q), dev(lib[:, :299]))
    with pytest.raises(ValueError, match="k must"):
        S.topKTanimotoCountSimilarity(dev(q), dev(lib), k=51)


@pytest.mark.parametrize("bins", [127, 2048, 4096])
@pytest.mark.parametrize("weights,name", MEASURES)
def test_topk_and_threshold(cuda, bins, weights, name):
    rng = np.random.default_rng(bins + 1)
    q, lib = edge_rows(rng, bins)
    _, topk, thresh = calls(name)
    m = oracle_count.cross(q, lib, *weights)
    for k in (1, 5, 256, len(lib)) if len(lib) <= 256 else (1, 5, 256):
        v, i = (r.numpy() for r in topk(dev(q), dev(lib), k=k, **kw(weights, name)))
        wv, wi = oracle_count.topk_of(m, k)
        assert np.array_equal(i, wi) and np.array_equal(v, wv), k
    v, i = (r.numpy() for r in topk(dev(lib[:200]), k=200, **kw(weights, name)))  # self search, k = the library size
    wv, wi = oracle_count.topk_of(oracle_count.cross(lib[:200], None, *weights), 200)
    assert np.array_equal(i, wi) and np.array_equal(v, wv)
    # thresholds at attained values and one ulp above them
    vals = np.unique(m[m > 0])
    for t in (vals[len(vals) // 2], vals[-1], np.nextafter(vals[len(vals) // 2], 2.0), 1.0, 0.05):
        if not 0 < t <= 1:
            continue
        got = [r.numpy() for r in thresh(dev(q), dev(lib), threshold=float(t), **kw(weights, name))]
        want = oracle_count.threshold_of(m, t)
        assert all(g.shape == w.shape and np.array_equal(g, w) for g, w in zip(got, want)), t
    got = [r.numpy() for r in thresh(dev(lib), threshold=0.3, **kw(weights, name))]
    want = oracle_count.threshold_of(oracle_count.cross(lib, None, *weights), 0.3)
    assert all(g.shape == w.shape and np.array_equal(g, w) for g, w in zip(got, want))


def test_topk_multi_slab_and_the_redo(cuda):
    """Strictly increasing values along the library: every column of a later slab beats the bar, more than the slots
    hold, so those slabs are redone by the scan. Then a random library, more than 4,096 queries (fewer slots)."""
    lib = np.zeros((6000, 3), np.int32)
    lib[:, 0] = np.arange(1, 6001)
    lib[:, 1] = np.arange(6000) % 7
    q = np.array([[65535, 3, 0], [6000, 0, 2], [1, 1, 1]], np.int32)
    for weights in ((1.0, 1.0), (0.3, 0.7)):
        m = oracle_count.cross(q, lib, *weights)
        for k in (1, 100, 256):
            v, i = (r.numpy() for r in S.topKTverskyCountSimilarity(dev(q), dev(lib), k=k, alpha=weights[0], beta=weights[1]))
            wv, wi = oracle_count.topk_of(m, k)
            assert np.array_equal(i, wi) and np.array_equal(v, wv)
    rng = np.random.default_rng(9)
    q, lib = counts(rng, 4200, 64, 0.2), counts(rng, 3000, 64, 0.2)
    lib[2000:2100] = lib[5]
    m = oracle_count.cross(q, lib, 0.5, 0.5)
    for k in (10, 256):
        v, i = (r.numpy() for r in S.topKDiceCountSimilarity(dev(q), dev(lib), k=k))
        wv, wi = oracle_count.topk_of(m, k)
        assert np.array_equal(i, wi) and np.array_equal(v, wv)


def test_threshold_capacity_retry_and_empty_inputs(cuda):
    x = np.zeros((1100, 16), np.int32)
    x[:, 3] = 2
    indptr, idx, vals = (r.numpy() for r in S.thresholdTanimotoCountSimilarity(dev(x), threshold=1.0))
    assert len(idx) == 1100 * 1100 and (vals == 1.0).all() and np.array_equal(indptr, np.arange(1101) * 1100)
    assert np.array_equal(idx, np.tile(np.arange(1100), 1100))
    # the C-ABI reports the size when the caller's room is short, and writes nothing
    d = dev(x[:10])
    nnz = C.c_uint64(0)
    indptr_t = torch.full((11,), -5, dtype=torch.int64, device="cuda")
    _lib.call("b200mol_count_threshold", d.data_ptr(), 10, None, 10, 16, 1.0, 1.0, 1.0, indptr_t.data_ptr(), 0, 0, 0,
              C.byref(nnz), None)
    assert nnz.value == 100 and (indptr_t == -5).all()
    e = torch.zeros((0, 16), dtype=torch.int32, device="cuda")
    indptr, idx, vals = (r.numpy() for r in S.thresholdDiceCountSimilarity(e, d, threshold=0.5))
    assert indptr.tolist() == [0] and len(idx) == 0
    assert S.crossTanimotoCountSimilarity(e, d).numpy().shape == (0, 10)


def test_streams_repeats_and_morgan_counts_at_size(cuda):
    from nvmolkit_b200 import synthetic
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    g = synthetic.random_molgraphs(3000, seed=11)
    x = MorganFingerprintGenerator(2, 2048).GetCountFingerprints(g)
    xs = x.numpy()
    q, lib = x.torch()[:400], x.torch()
    side = torch.cuda.Stream()
    m = S.crossTanimotoCountSimilarity(q, lib).numpy()
    assert np.array_equal(m, oracle_count.cross(xs[:400], xs))
    assert np.array_equal(S.crossTanimotoCountSimilarity(q, lib, stream=side).numpy(), m)
    v1, i1 = (r.numpy() for r in S.topKTanimotoCountSimilarity(q, lib, k=100))
    v2, i2 = (r.numpy() for r in S.topKTanimotoCountSimilarity(q, lib, k=100, stream=side))
    wv, wi = oracle_count.topk_of(m, 100)
    assert np.array_equal(i1, wi) and np.array_equal(v1, wv) and np.array_equal(i2, i1) and np.array_equal(v2, v1)
    t1 = [r.numpy() for r in S.thresholdTanimotoCountSimilarity(q, lib, threshold=0.5)]
    t2 = [r.numpy() for r in S.thresholdTanimotoCountSimilarity(q, lib, threshold=0.5, stream=side)]
    want = oracle_count.threshold_of(m, 0.5)
    assert all(np.array_equal(a, w) and np.array_equal(b, w) for a, b, w in zip(t1, t2, want))
