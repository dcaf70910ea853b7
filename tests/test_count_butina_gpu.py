"""Butina on count vectors on the GPU, compared exactly (==): the neighbour edges and degrees of
b200mol_count_neighbor_edges against the count oracle's matrix, at 1, 127, 2048 and 4096 bins, Tanimoto and Dice, on
the fp64 boundary and over rows that stress the sum order and band; clusters against the CPU oracle's dense Butina and
the GPU dense route; edges at about 150k rows against the threshold search; the pair count against the NumPy band model;
and the call protocol (the edge-cap rerun, n = 0 and 1, input dtypes, Morgan counts, streams, repeats, refusals)."""

import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import test_count_butina as CB
from nvmolkit_b200 import _lib
from nvmolkit_b200 import similarity as S
from nvmolkit_b200.clustering import butina, fused_butina_counts, fused_butina_counts_device
from oracle import count as oracle_count

pytestmark = pytest.mark.gpu
WEIGHTS = CB.WEIGHTS
BOUNDARY = 0.30000000000000004  # 1 - 0.7 in fp64


def dev(x, dtype=torch.int32):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dtype).cuda()


def gpu_edges(x, cutoff, metric, cap=None):
    """(degrees [n], edges (i, j) sorted) from the C-ABI, retrying once with the reported size."""
    d = x if isinstance(x, torch.Tensor) else dev(x)
    n, bins = d.shape
    cap = max(1, 64 * n) if cap is None else cap
    for _ in range(2):
        counts = torch.zeros(n, dtype=torch.int32, device="cuda")
        edges = torch.empty((max(cap, 1), 2), dtype=torch.int32, device="cuda")
        ne = C.c_uint64(0)
        _lib.call("b200mol_count_neighbor_edges", d.data_ptr(), n, bins, *WEIGHTS[metric], float(cutoff), counts.data_ptr(),
                  edges.data_ptr(), cap, C.byref(ne), None)
        if ne.value <= cap:
            break
        cap = ne.value
    e = edges[: ne.value].cpu().numpy()
    return counts.cpu().numpy(), e[np.lexsort((e[:, 1], e[:, 0]))]


def oracle_edges(x, cutoff, metric):
    m = oracle_count.cross(x, x, *WEIGHTS[metric])
    i, j = np.nonzero(np.triu(1.0 - m <= cutoff, 1))
    deg = np.bincount(i, minlength=len(x)) + np.bincount(j, minlength=len(x))
    return deg.astype(np.int32), np.stack([i, j], 1).astype(np.int32)


def row_mix(rng, bins):
    """The boundary rows first, then zero rows, duplicates, rows at 65535, many equal sums and a wide spread of sums."""
    if bins == 1:
        head = np.array([[7], [10], [7], [13], [0], [0], [65535], [65535]], np.int32)  # 7/10 Tanimoto, 14/20 Dice
        return np.concatenate([head, rng.integers(0, 30, size=(150, 1)), rng.integers(0, 65536, size=(20, 1))]).astype(np.int32)
    n = 300 if bins <= 2048 else 200
    x = np.where(rng.random((n, bins)) < 0.05, rng.integers(1, 6, size=(n, bins)), 0)
    x[:3] = 0
    x[0, :2] = (7, 3)                      # Tanimoto [7, 3] / [7, 0]: 0.7
    x[1, 0] = 7
    if bins >= 3:
        x[2, [0, 2]] = (7, 3)              # Dice [7, 3, 0] / [7, 0, 3]: 0.7
    x[3:6] = 0
    x[6] = 65535
    x[7] = np.where(rng.random(bins) < 0.5, 65535, 0)
    x[10:25] = x[30]                       # duplicates
    k = np.arange(60)
    x[40:100] = 0
    x[40 + k, (k * 7) % bins] = 5          # equal sums: ties in the sort
    x[100:110] = np.where(rng.random((10, bins)) < 0.5, rng.integers(1000, 3000, size=(10, bins)), 0)  # a long band
    return x.astype(np.int32)


@pytest.mark.parametrize("bins", [1, 127, 2048, 4096])
@pytest.mark.parametrize("metric", ["tanimoto", "dice"])
def test_edges_and_degrees_equal_the_oracle(cuda, bins, metric):
    rng = np.random.default_rng(bins + (metric == "dice"))
    x = row_mix(rng, bins)
    for cutoff in (0.0, 0.3, BOUNDARY, 0.5, 1.0):
        deg, e = gpu_edges(x, cutoff, metric)
        wdeg, we = oracle_edges(x, cutoff, metric)
        assert np.array_equal(e, we) and np.array_equal(deg, wdeg), cutoff
        assert _lib.get_option("count_neighbor_pairs_last") == CB.band_pairs(x.sum(1), bins, cutoff, WEIGHTS[metric])
    # the boundary pair: 1 - 0.7 = 0.30000000000000004 > 0.3
    pair = (0, 1) if (metric == "tanimoto" or bins == 1) else (0, 2)
    if bins == 1 and metric == "dice":
        pair = (0, 3)
    for cutoff, inside in ((0.3, False), (BOUNDARY, True)):
        _, e = gpu_edges(x, cutoff, metric)
        assert (tuple(pair) in set(map(tuple, e.tolist()))) == inside, (cutoff, pair)


def test_empty_rows_are_neighbours_only_at_cutoff_one(cuda):
    x = np.zeros((5, 16), np.int32)
    x[2:, 3] = 4
    for metric in WEIGHTS:
        deg, e = gpu_edges(x, np.nextafter(1.0, 0.0), metric)
        assert e.tolist() == [[2, 3], [2, 4], [3, 4]]
        deg, e = gpu_edges(x, 1.0, metric)
        assert len(e) == 10 and (deg == 4).all()


@pytest.mark.parametrize("bins,n", [(2048, 2000), (127, 4000), (4096, 1500)])
@pytest.mark.parametrize("metric", ["tanimoto", "dice"])
def test_clusters_equal_the_oracle_dense_butina(cuda, bins, n, metric):
    rng = np.random.default_rng(n + bins)
    x = CB.clustered_counts(rng, n, bins, centres=n // 40)
    x[: n // 20] = np.where(rng.random((n // 20, bins)) < 0.05, rng.integers(1, 50, size=(n // 20, bins)), 0)
    m = oracle_count.cross(x, x, *WEIGHTS[metric])
    for cutoff in (0.2, 0.35, BOUNDARY):
        want_ids, want_cen = oracle.butina_dense(1.0 - m, cutoff)
        ids, cen = fused_butina_counts_device(dev(x), cutoff, metric=metric)
        assert np.array_equal(ids.cpu().numpy(), want_ids) and np.array_equal(cen.cpu().numpy(), want_cen), cutoff
        clusters, sizes, cents = fused_butina_counts(dev(x), cutoff, return_centroids=True, metric=metric)
        assert cents == want_cen.tolist() and sizes[-1] == n and [c[0] for c in clusters] == cents
    assert len(want_cen) < n  # (not all singletons)


@pytest.mark.parametrize("metric", ["tanimoto", "dice"])
def test_clusters_equal_the_gpu_dense_route_at_20k(cuda, metric):
    rng = np.random.default_rng(20)
    x = dev(CB.clustered_counts(rng, 20000, 512, centres=400, changes=4))
    cross = S.crossTanimotoCountSimilarity if metric == "tanimoto" else S.crossDiceCountSimilarity
    for cutoff in (0.25, 0.4):
        want_ids, want_cen = butina(1.0 - cross(x).torch(), cutoff, return_centroids=True)
        ids, cen = fused_butina_counts_device(x, cutoff, metric=metric)
        assert torch.equal(ids, want_ids.torch()) and torch.equal(cen, want_cen.torch())
        n = 20000
        pairs = _lib.get_option("count_neighbor_pairs_last")
        assert pairs == CB.band_pairs(x.sum(1).cpu().numpy(), 512, cutoff, WEIGHTS[metric]) < n * (n - 1) // 2


@pytest.fixture(scope="module")
def morgan_150k(cuda):
    from nvmolkit_b200 import synthetic
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    return MorganFingerprintGenerator(2, 2048).GetCountFingerprints(synthetic.random_molgraphs(150000, seed=5)).torch()


@pytest.mark.parametrize("metric", ["tanimoto", "dice"])
def test_edges_at_150k_equal_the_threshold_search(morgan_150k, metric):
    """More units than a grid dimension holds; the reference is the threshold self search just below 1 - cutoff,
    filtered by the exact predicate on its values."""
    x = morgan_150k
    n, cutoff = x.shape[0], {"tanimoto": 0.6, "dice": 0.5}[metric]  # (the same pairs: Dice 0.5 is Tanimoto 1/3)
    deg, e = gpu_edges(x, cutoff, metric)
    search = S.thresholdTanimotoCountSimilarity if metric == "tanimoto" else S.thresholdDiceCountSimilarity
    indptr, idx, vals = (r.numpy() for r in search(x, threshold=(1.0 - cutoff) - 1e-9))
    rows = np.repeat(np.arange(n), np.diff(indptr))
    keep = (rows < idx) & (1.0 - vals <= cutoff)
    want = np.stack([rows[keep], idx[keep]], 1).astype(np.int32)
    assert np.array_equal(e, want)
    assert np.array_equal(deg, (np.bincount(want[:, 0], minlength=n) + np.bincount(want[:, 1], minlength=n)).astype(np.int32))
    sums = x.sum(1).cpu().numpy()
    units = sum(-(-(end - q0) // 4096) for q0, _, end in zip(*CB.band_ends(np.sort(sums), 32, cutoff, WEIGHTS[metric])))
    assert units > 65535
    pairs = _lib.get_option("count_neighbor_pairs_last")
    assert pairs == CB.band_pairs(sums, 2048, cutoff, WEIGHTS[metric]) < n * (n - 1) // 2


def test_band_pair_count_at_cutoff_one_is_every_pair(cuda):
    rng = np.random.default_rng(3)
    x = CB.clustered_counts(rng, 1000, 300)
    for metric in WEIGHTS:
        gpu_edges(x, 1.0, metric)
        assert _lib.get_option("count_neighbor_pairs_last") == 1000 * 999 // 2
        gpu_edges(x, 0.2, metric)
        assert _lib.get_option("count_neighbor_pairs_last") == CB.band_pairs(x.sum(1), 300, 0.2, WEIGHTS[metric]) < 1000 * 999 // 2


def test_the_edge_cap_rerun_and_small_inputs(cuda):
    rng = np.random.default_rng(4)
    x = CB.clustered_counts(rng, 3000, 64)
    ids, cen = fused_butina_counts_device(dev(x), 1.0)  # 4.5M edges: more than 64 per point, one rerun
    assert (ids.cpu().numpy() == 0).all() and cen.cpu().numpy().tolist() == [2999]
    deg, e = gpu_edges(x[:100], 1.0, "tanimoto", cap=10)  # the C-ABI reports the total past the cap
    assert len(e) == 4950 and (deg == 99).all()
    for n in (0, 1):
        ids, cen = fused_butina_counts_device(dev(x[:n]), 0.3)
        assert ids.cpu().numpy().tolist() == list(range(n)) and cen.cpu().numpy().tolist() == list(range(n))
        clusters, sizes = fused_butina_counts(dev(x[:n]), 0.3)
        assert clusters == [(0,)] * n and sizes == list(range(n + 1))


def test_dtypes_morgan_counts_streams_and_repeats(cuda):
    from nvmolkit_b200 import synthetic
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    rng = np.random.default_rng(6)
    x = CB.clustered_counts(rng, 1500, 300, high=200)
    want = oracle.butina_dense(1.0 - oracle_count.cross(x, x, 1.0, 1.0), 0.3)
    for dtype in (torch.uint8, torch.int16, torch.int32):
        ids, cen = fused_butina_counts_device(dev(x, dtype), 0.3)
        assert np.array_equal(ids.cpu().numpy(), want[0]) and np.array_equal(cen.cpu().numpy(), want[1])
    fp = MorganFingerprintGenerator(2, 2048).GetCountFingerprints(synthetic.random_molgraphs(2000, seed=8))
    xs = fp.numpy()
    want = oracle.butina_dense(1.0 - oracle_count.cross(xs, xs, 0.5, 0.5), 0.35)
    side = torch.cuda.Stream()
    runs = [fused_butina_counts_device(fp, 0.35, metric="dice"),
            fused_butina_counts_device(fp, 0.35, metric="dice", stream=side),
            fused_butina_counts_device(fp, 0.35, metric="dice")]
    for ids, cen in runs:
        assert np.array_equal(ids.cpu().numpy(), want[0]) and np.array_equal(cen.cpu().numpy(), want[1])


def test_refusals_leave_the_outputs_untouched(cuda):
    bad = dev(np.array([[0, 65536], [1, 2], [3, 4]], np.int32))
    counts = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    edges = torch.full((8, 2), -7, dtype=torch.int32, device="cuda")
    ne = C.c_uint64(5)
    with pytest.raises(ValueError, match="outside 0 .. 65535"):
        _lib.call("b200mol_count_neighbor_edges", bad.data_ptr(), 3, 2, 1.0, 1.0, 1.0, counts.data_ptr(), edges.data_ptr(), 8,
                  C.byref(ne), None)
    assert (counts == -7).all() and (edges == -7).all()
    ids = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    cen = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="outside 0 .. 65535"):
        _lib.call("b200mol_count_butina_fused", bad.data_ptr(), 3, 2, 0.5, 0.5, 0.3, ids.data_ptr(), cen.data_ptr(), None,
                  None, None)
    assert (ids == -7).all() and (cen == -7).all()
    with pytest.raises(ValueError, match="outside 0 .. 65535"):
        fused_butina_counts(dev(np.array([[-1, 3]]), torch.int16), 0.3)
    ok = dev(np.ones((4, 8), np.int32))
    with pytest.raises(ValueError, match="dtype"):
        fused_butina_counts(ok.to(torch.int64), 0.3)
    with pytest.raises(ValueError, match="2D"):
        fused_butina_counts(ok[0], 0.3)
    with pytest.raises(ValueError, match="bins"):
        fused_butina_counts(torch.zeros((3, 4097), dtype=torch.int32, device="cuda"), 0.3)
    with pytest.raises(ValueError, match="CUDA"):
        fused_butina_counts(torch.ones((3, 4), dtype=torch.int32), 0.3)
