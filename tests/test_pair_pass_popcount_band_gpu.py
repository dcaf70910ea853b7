"""The popcount band of the ordered neighbour pass: per row group of 8,192 fingerprints in popcount order, the tile
columns whose popcounts no row of the group can reach a neighbour with are skipped (popcountBandKernel, UnitWalk).

- CPU, exhaustive: the cut against the fp64 definition for every popcount pair up to 4096 bits, and its monotonicity.
- CPU model: tools/pilot_model.band_ends against a per-group scan, with partial last groups.
- GPU, boundary: a group whose largest popcount A and a column's popcount sit exactly on the cut, the cut on, one column
  inside and one column past a tile-column boundary; every tile variant and superposition, band on and off, against the
  fp64 graph; the units the kernel walked equal the host's count and the NumPy model's.
- GPU, wide spread: popcounts 20 to 200, where the band skips over 30 % of the units: clusters, centroids and the sharded
  pass equal the pass with the band off.
"""

import numpy as np
import pytest
import torch

import oracle
import test_pair_pass_boundary as B
import test_pair_pass_popcount_order_gpu as P
import test_path_a_gpu as A
from nvmolkit_b200 import synthetic as S
from tools import pilot_model as M


# ------------------------------------------------------------------ CPU: the cut against the fp64 definition
@pytest.mark.parametrize("cutoff", B.CUTOFFS)
def test_band_cut_never_excludes_an_accepted_pair_and_is_monotone(cutoff):
    bits = 4096
    t = M.thresh_table(bits, cutoff)
    assert (t == B.thresh_table(bits, cutoff)).all()
    a = np.arange(bits + 1)[:, None]
    b = np.arange(bits + 1)[None, :]
    cut = M.band_cuts(M.band_table(t), a, b)
    # the largest intersection a pair of popcounts (a, b) can have is min(a, b): if even that one fails, all fail
    assert not (cut & M.is_neighbour(np.minimum(a, b), a, b, cutoff)).any()
    assert (cut[:, :-1] <= cut[:, 1:]).all()  # cut at b => cut at b + 1
    assert (cut[1:, :] <= cut[:-1, :]).all()  # cut at A => cut at A - 1 (every smaller row of the group)
    if cutoff >= 1.0:
        assert not cut.any()


@pytest.mark.parametrize("n", [1, 100, 8192, 8193, 20_000, 40_960])
def test_band_ends_model_equals_a_scan_per_group(n):
    rng = np.random.default_rng(n)
    pop = np.sort(np.concatenate([rng.integers(0, 4, 3), rng.integers(20, 200, n)]))[:n]
    for cutoff in (0.0, 0.3, 0.65, 1.0):
        t = M.thresh_table(2048, cutoff)
        tmin = M.band_table(t)
        for col_span in (256, 512, 1024):
            ends = M.band_ends(pop, pop, t, col_span)
            tiles_n = -(-n // col_span)
            assert len(ends) == -(-n // 8192)
            for g, e in enumerate(ends):
                a = pop[min(n, (g + 1) * 8192) - 1]
                keep = np.flatnonzero(~M.band_cuts(tmin, a, pop))  # every column the cut keeps
                j_cut = keep[-1] + 1 if len(keep) else 0
                assert e == min(tiles_n, -(-j_cut // col_span)), (n, cutoff, col_span, g)


# ------------------------------------------------------------------ GPU: the cut at a group / tile-column boundary
@pytest.fixture(params=[(1, 4, 4), (1, 4, 1), (1, 1, 1), (0, 4, 4), (0, 4, 1), (3, 4, 4), (3, 4, 1)],
                ids=["pair-4x4", "pair-4x1", "pair-plain", "single-4x4", "single-4x1", "stationary-4x4", "stationary-4x1"])
def variant(cuda, request):
    from nvmolkit_b200 import _lib

    cl, s, c = request.param
    with _lib.options(similarity_tensor_min_pairs=0, similarity_tensor_cluster=cl, similarity_superpose=s,
                      similarity_superpose_cols=c):
        yield request.param


def _boundary_set(bits, cutoff, delta, seed):
    """8,192 rows (popcounts <= A, three of them empty, row R = 8191 of popcount A: the group's largest) and columns of
    popcount bOk (the largest the cut keeps for A) and bOk + 1, 1024 + delta of them at bOk, given in the pass's order: in the pass's order the cut
    falls on a tile-column boundary (delta 0), one column inside (-1) or past it (+1). The last bOk column holds R
    (c = A, a neighbour of R), so does the first bOk + 1 column (c = A, not one). Returns (fp, A, bOk)."""
    rng = np.random.default_rng(seed)
    t = M.thresh_table(bits, cutoff)
    A_ = bits // 32
    b_ok = max(b for b in range(A_, bits - A_) if not M.band_cuts(M.band_table(t), A_, b))
    assert M.is_neighbour(A_, A_, b_ok, cutoff) and not M.is_neighbour(A_, A_, b_ok + 1, cutoff)

    def rows(k, pops):
        m = np.zeros((k, bits), dtype=bool)
        for r, p in enumerate(pops):
            m[r, rng.choice(bits, p, replace=False)] = True
        return m

    low = rows(8192, np.concatenate([[0, 0, 0], rng.integers(A_ - 3, A_ + 1, 8188), [A_]]))
    r_bits = np.flatnonzero(low[-1])
    n_ok = 1024 + delta
    ok = rows(n_ok, [b_ok] * n_ok)
    cut = rows(1100, [b_ok + 1] * 1100)  # (at least one whole tile column past the cut)
    for m, at, p in ((ok, n_ok - 1, b_ok), (cut, 0, b_ok + 1)):
        rest = rng.choice(np.setdiff1d(np.arange(bits), r_bits), p - A_, replace=False)
        m[at] = False
        m[at, r_bits] = True
        m[at, rest] = True
    fp = S.pack_bits(np.concatenate([low, ok, cut]))
    fp = np.ascontiguousarray(fp[P._stable_order(fp)])  # in the pass's order: R stays row 8191, the two columns 8192 + n_ok - 1, + n_ok
    return fp, A_, b_ok


def _units_model(fp, cutoff, cl, s, c, band):
    pop = np.sort(P._popcounts(fp))
    ends = M.band_ends(pop, pop, M.thresh_table(32 * fp.shape[1], cutoff), 256 * c) if band else None
    return int(M.group_units(len(fp), s, c, ends, pair=cl != 0, run=16 if cl == 3 else 1).sum())


def _pass(fp, cutoff, cuda, band):
    from nvmolkit_b200 import _lib

    with _lib.options(similarity_popcount_band=band):
        deg, edges = P._neighbor_edges(fp, cutoff, cuda)
    return deg, edges, _lib.get_option("similarity_units_last"), _lib.get_option("similarity_units_planned_last")


_SETS = {}


def _boundary_case(bits, cutoff, delta, cuda):
    """_boundary_set and its fp64 graph, built once per (bits, cutoff, delta) for all variants."""
    key = (bits, cutoff, delta)
    if key not in _SETS:
        fp, a, b_ok = _boundary_set(bits, cutoff, delta, seed=bits + delta)
        _SETS[key] = (fp, *P._reference_graph(fp, cutoff, cuda))
    return _SETS[key]


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [1024, 2048, 4096])
def test_band_cut_on_a_tile_column_boundary(cuda, variant, bits):
    from nvmolkit_b200 import _lib

    cl, s, c = variant
    if cl == 3 and bits > 1024:
        pytest.skip("the row-stationary tile serves fingerprints up to 1024 bits")
    ordered = s * c > 1  # (1 x 1 runs in the caller's order, without the band)
    for cutoff in (0.3, 0.0):
        for delta in (-1, 0, 1):
            fp, want_deg, want_key = _boundary_case(bits, cutoff, delta, cuda)
            r, p1, p2 = 8191, 8192 + 1024 + delta - 1, 8192 + 1024 + delta
            key = set(want_key.tolist())
            assert r * len(fp) + p1 in key and r * len(fp) + p2 not in key
            what = (bits, cutoff, delta, variant)
            deg, edges, units, planned = _pass(fp, cutoff, cuda, 1)
            tiles = _lib.get_option("similarity_tiles_last")
            P._assert_graph(deg, edges, want_deg, want_key, len(fp), what)
            assert units == planned == _units_model(fp, cutoff, cl, s, c, ordered), what
            deg0, edges0, units0, planned0 = _pass(fp, cutoff, cuda, 0)
            tiles0 = _lib.get_option("similarity_tiles_last")
            P._assert_graph(deg0, edges0, want_deg, want_key, len(fp), what)
            assert units0 == planned0 == _units_model(fp, cutoff, cl, s, c, False), what
            # the band skips at least one tile column of group 0 (a unit of the row-stationary tile spans 16 of them)
            assert tiles < tiles0 if ordered else tiles == tiles0, what


@pytest.mark.gpu
def test_band_cuts_nothing_at_cutoff_one_and_keeps_empty_fingerprints(cuda, variant):
    """Cutoff 1.0: every pair is a neighbour, the band must cut nothing. Empty rows and an all-empty set."""
    cl, s, c = variant
    rng = np.random.default_rng(5)
    m = rng.random((700, 1024)) < 0.05
    m[:20] = False
    fp = S.pack_bits(m)
    for cutoff in (1.0, 0.3):
        want_deg, want_key = P._reference_graph(fp, cutoff, cuda)
        deg, edges, units, planned = _pass(fp, cutoff, cuda, 1)
        P._assert_graph(deg, edges, want_deg, want_key, len(fp), (cutoff, variant))
        assert units == planned
        if cutoff == 1.0:
            assert units == _units_model(fp, cutoff, cl, s, c, False)
    empty = S.pack_bits(np.zeros((300, 1024), dtype=bool))
    for cutoff in (0.3, 1.0):
        want_deg, want_key = P._reference_graph(empty, cutoff, cuda)
        deg, edges, units, planned = _pass(empty, cutoff, cuda, 1)
        P._assert_graph(deg, edges, want_deg, want_key, len(empty), (cutoff, "empty", variant))


# ------------------------------------------------------------------ GPU: wide popcount spread
def _wide(n, seed):
    """Clustered fingerprints at bit densities from 1 % to 10 % of 2048 bits (popcounts about 20 to 200), shuffled."""
    parts = [S.clustered_fingerprints(n // (10 * 20) + 1, 20, bits=2048, p=p, seed=seed + k)
             for k, p in enumerate(np.linspace(0.01, 0.1, 10))]
    fp = np.concatenate(parts)
    return np.ascontiguousarray(fp[np.random.default_rng(seed).permutation(len(fp))[:n]])


@pytest.mark.gpu
def test_wide_popcount_spread_clusters_equal_the_pass_without_band(cuda):
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    fp = _wide(40_000, seed=11)
    pop = P._popcounts(fp)
    assert pop.min() < 40 and pop.max() > 150
    dev = A._dev(fp, cuda)
    out = {}
    for band in (1, 0):
        with _lib.options(similarity_tensor_min_pairs=0, similarity_popcount_band=band):
            deg, edges = P._neighbor_edges(fp, 0.3, cuda)
            units = _lib.get_option("similarity_units_last")
            assert units == _lib.get_option("similarity_units_planned_last")
            ids, cen = fused_butina_device(dev, 0.3)
        out[band] = (deg, np.sort(edges[:, 0] * len(fp) + edges[:, 1]), ids.cpu().numpy(), cen.cpu().numpy(), units)
    (deg, key, ids, cen, units), (deg0, key0, ids0, cen0, units0) = out[1], out[0]
    assert units < 0.7 * units0, (units, units0)  # the band skips over 30 % of the triangle's units
    assert (deg == deg0).all() and len(key) == len(key0) and (key == key0).all()
    assert (ids == ids0).all() and (cen == cen0).all()
    ids_cpu, cen_cpu = oracle.butina_fp(fp[:4000], 0.3)
    ids4, cen4 = fused_butina_device(A._dev(fp[:4000], cuda), 0.3)
    assert (ids4.cpu().numpy() == ids_cpu).all() and (cen4.cpu().numpy() == cen_cpu).all()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_wide_popcount_spread_sharded_pass_equals_one_pass(cuda, world):
    from nvmolkit_b200 import _lib

    fp = _wide(40_000, seed=world)
    with _lib.options(similarity_tensor_min_pairs=0):
        ids, cen, edges, deg, per_rank = A._sharded_butina_one_gpu(fp, 0.3, world, cuda)
        ids1, cen1, edges1, deg1, _ = A._sharded_butina_one_gpu(fp, 0.3, 1, cuda)
    assert (deg == deg1).all() and (ids == ids1).all() and (cen == cen1).all()
    key = np.sort(edges[:, 0].astype(np.int64) * len(fp) + edges[:, 1])
    key1 = np.sort(edges1[:, 0].astype(np.int64) * len(fp) + edges1[:, 1])
    assert (edges[:, 0] < edges[:, 1]).all() and len(key) == len(key1) and (key == key1).all()


@pytest.mark.gpu
def test_superposed_pass_lists_the_candidates_the_banded_model_predicts(cuda):
    """The pilot is a superposed pass over a sample: at the pilot's size and factors the candidate count of the pass
    equals tools/pilot_model.candidates with the band."""
    from nvmolkit_b200 import _lib

    fp = S.clustered_fingerprints(400, 50, seed=S.SEED)[:16384]
    fp = np.ascontiguousarray(fp[P._stable_order(fp)])
    for c in (4, 2, 1):
        with _lib.options(similarity_tensor_min_pairs=0, similarity_superpose_auto=0, similarity_superpose_cols=c):
            P._neighbor_edges(fp, 0.3, cuda)
            assert _lib.get_option("similarity_superpose_last") == 4 * c
            assert _lib.get_option("similarity_candidates_last") == M.candidates(fp, 0.3, 4, c, band=True), c
