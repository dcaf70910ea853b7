"""The superposed neighbour pass runs on the fingerprints ordered by popcount (ascending, ties by index) and maps every
pair back to the caller's indices.

- Boundary pairs in groups that are tight AFTER the ordering: the group holding A and B sums exactly c and its smallest
  popcounts are |A| and |B|, so the pre-filter is pinned at its margin.
- Inputs whose popcount order is far from their index order: counts, edge set, i < j and clusters.
- The sharded pass (ranks own row groups of the ordered set) equals the plain pass.
- An unsuperposed fallback, of a pipeline chunk or of one rank, covers the same row groups as the pass it completes.
- The pilot on the bench generator picks what the CPU model (tools/pilot_model.py) predicts for the same data.
"""

import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import test_pair_pass_boundary as B
import test_path_a_gpu as A
from nvmolkit_b200 import synthetic as S
from tools import pilot_model

pytestmark = pytest.mark.gpu


def _popcounts(fp):
    return np.unpackbits(np.ascontiguousarray(fp).view(np.uint8), axis=1).sum(1)


def _stable_order(fp):
    """The pass's order: ascending popcount, ties by index."""
    return np.argsort(_popcounts(fp), kind="stable")


@pytest.fixture(params=[(4, 4), (4, 2), (4, 1), (2, 1)], ids=["super4x4", "super4x2", "super4x1", "super2x1"])
def superposition(cuda, request):
    """The tensor-core neighbour pass at rows x columns superposition, no pilot."""
    from nvmolkit_b200 import _lib

    _lib.set_option("similarity_tensor_min_pairs", 0)
    _lib.set_option("similarity_superpose", request.param[0])
    _lib.set_option("similarity_superpose_cols", request.param[1])
    yield request.param
    _lib.set_option("similarity_superpose", 4)
    _lib.set_option("similarity_superpose_cols", 4)
    _lib.set_option("similarity_tensor_min_pairs", 1 << 24)


def _neighbor_edges(fp, cutoff, cuda, group_offset=0, group_stride=1):
    """b200mol_neighbor_edges: (degrees, edges [k][2] int64)."""
    from nvmolkit_b200 import _lib

    n = len(fp)
    d = A._dev(fp, cuda)
    cap = 1 << 16
    while True:
        counts = torch.zeros(n, dtype=torch.int32, device=cuda)
        edges = torch.empty((cap, 2), dtype=torch.int32, device=cuda)
        found = C.c_uint64(0)
        _lib.call("b200mol_neighbor_edges", d.data_ptr(), n, fp.shape[1], 0, float(cutoff), group_offset, group_stride,
                  counts.data_ptr(), edges.data_ptr(), cap, C.byref(found), torch.cuda.current_stream().cuda_stream)
        if found.value <= cap:
            return counts.cpu().numpy(), edges[: found.value].cpu().numpy().astype(np.int64)
        cap = int(found.value)


def _reference_graph(fp, cutoff, cuda):
    """(degrees, sorted i < j edge keys i n + j) from exact counts (float64 matmul of the 0/1 expansions on the device)
    and the fp64 predicate; no self pairs."""
    e = torch.from_numpy(B._expand(fp)).to(cuda)
    c = (e @ e.T).cpu().numpy()
    pop = _popcounts(fp)
    ref = B.is_neighbour(c, pop[:, None], pop[None, :], cutoff)
    np.fill_diagonal(ref, False)
    wi, wj = np.nonzero(np.triu(ref))
    return ref.sum(1).astype(np.int32), np.sort(wi.astype(np.int64) * len(fp) + wj)


def _assert_graph(deg, edges, want_deg, want_key, n, what):
    assert (deg == want_deg).all(), what
    assert (edges[:, 0] < edges[:, 1]).all(), what
    key = np.sort(edges[:, 0] * n + edges[:, 1])
    assert len(key) == len(want_key) and (key == want_key).all(), what


# ------------------------------------------------------------------ boundary pairs, tight after the ordering
def _tight_block(rng, bits, a, b, c):
    """Eight fingerprints whose popcount order D is [A, three row fillers, B, three column fillers] with |A| = a <= b = |B|,
    |A & B| = c, fillers of a (row) and b (column) bits, all supports disjoint except A & B. In D, the rows' group of
    S <= 4 holding A and the columns' group of C <= 4 holding B then sum exactly c, with smallest popcounts a and b.
    The caller gets D in DESCENDING popcount order (ties by position in D), which the stable ascending sort turns back
    into D. Returns (fingerprints in the caller's order, caller index of A, of B)."""
    perm = rng.permutation(bits)
    d = np.zeros((8, bits), dtype=bool)
    d[0, perm[:a]] = True
    d[4, perm[a - c:a - c + b]] = True
    at = a + b - c
    for r, k in ((1, a), (2, a), (3, a), (5, b), (6, b), (7, b)):
        d[r, perm[at:at + k]] = True
        at += k
    assert at <= bits
    pop = d.sum(1)
    caller = np.lexsort((np.arange(8), -pop))  # caller row k = D row caller[k]
    fp = S.pack_bits(d[caller])
    assert (S.pack_bits(d) == fp[_stable_order(fp)]).all()  # the pass sees D
    where = np.argsort(caller)  # D row r sits at caller index where[r]
    return fp, int(where[0]), int(where[4])


@pytest.mark.parametrize("bits", [2048, 4096])
def test_neighbor_edges_on_the_boundary_in_popcount_order(cuda, superposition, bits):
    """Each smallest-margin boundary pair (c = thresh and c = thresh - 1) and each sim = 7/10 pair in a block that is
    tight in the pass's order: a strict pre-filter or a pre-filter term rounded up drops a true neighbour here. Degrees
    and edge set must equal the fp64 definition's."""
    from nvmolkit_b200 import _lib

    sup_s, sup_c = superposition
    rng = np.random.default_rng(bits + 7)
    for cutoff in B.CUTOFFS:
        for a, b, c in B._cases(bits, cutoff, fit_block=True):
            a, b = min(a, b), max(a, b)
            fp, ia, ib = _tight_block(rng, bits, a, b, c)
            # the group the pass forms around the pair: rows [A, fillers][:S], columns [B, fillers][:C] of D
            d = fp[_stable_order(fp)]
            e = B._expand(d)
            assert (e[:sup_s].sum(0) @ e[4:4 + sup_c].sum(0)) == c
            assert e[:sup_s].sum(1).min() == a and e[4:4 + sup_c].sum(1).min() == b
            ref = B._reference(fp, fp, cutoff)
            assert ref[ia, ib] == B.is_neighbour(c, a, b, cutoff)
            want_deg, want_key = _reference_graph(fp, cutoff, cuda)
            deg, edges = _neighbor_edges(fp, cutoff, cuda)
            assert _lib.get_option("similarity_superpose_last") == sup_s * sup_c
            _assert_graph(deg, edges, want_deg, want_key, len(fp), (cutoff, a, b, c))


# ------------------------------------------------------------------ mapping back to the caller's order
def _descending(n, bits, seed):
    """Clustered fingerprints at three bit densities, rows in DESCENDING popcount order: the pass's order reverses
    the caller's."""
    parts = [S.clustered_fingerprints(n // 60 + 1, 20, bits=bits, p=p, seed=seed + k) for k, p in enumerate((0.01, 0.03, 0.08))]
    fp = np.concatenate(parts)
    fp = fp[np.random.default_rng(seed).permutation(len(fp))[:n]]
    return np.ascontiguousarray(fp[np.argsort(-_popcounts(fp), kind="stable")])


@pytest.mark.parametrize("bits", [640, 4096])
@pytest.mark.parametrize("n", [2, 5, 127, 1023, 9000])
def test_superposed_pass_maps_back_to_the_callers_order(cuda, superposition, n, bits):
    from nvmolkit_b200.clustering import fused_butina_device

    fp = _descending(n, bits, seed=n + bits)
    pop = _popcounts(fp)
    assert n < 3 or (pop[:-1] >= pop[1:]).all() and pop[0] > pop[-1]
    for cutoff in (0.3, 0.62):
        want_deg, want_key = _reference_graph(fp, cutoff, cuda)
        deg, edges = _neighbor_edges(fp, cutoff, cuda)
        _assert_graph(deg, edges, want_deg, want_key, n, (n, bits, cutoff))
        ids, cen = fused_butina_device(A._dev(fp, cuda), cutoff)
        ids_cpu, cen_cpu = oracle.butina_fp(fp, cutoff)
        assert (ids.cpu().numpy() == ids_cpu).all() and (cen.cpu().numpy() == cen_cpu).all(), (n, bits, cutoff)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_pass_in_popcount_order_equals_the_plain_pass(cuda, world):
    """40,000 points (five row groups) in descending popcount order over 2 and 3 "ranks": the ranks own row groups of
    the ORDERED set, and together they must list every unordered pair once. Degrees, edge set and clusters equal those
    of one unsuperposed pass."""
    from nvmolkit_b200 import _lib

    fp = _descending(40_000, 2048, seed=world)
    _lib.set_option("similarity_tensor_min_pairs", 0)
    try:
        ids, cen, edges, deg, per_rank = A._sharded_butina_one_gpu(fp, 0.3, world, cuda)
        assert all(c > 0 for c in per_rank)
        _lib.set_option("similarity_superpose", 1)
        _lib.set_option("similarity_superpose_cols", 1)
        ids1, cen1, edges1, deg1, _ = A._sharded_butina_one_gpu(fp, 0.3, 1, cuda)
    finally:
        _lib.set_option("similarity_superpose", 4)
        _lib.set_option("similarity_superpose_cols", 4)
        _lib.set_option("similarity_tensor_min_pairs", 1 << 24)
    assert (deg == deg1).all() and (ids == ids1).all() and (cen == cen1).all()
    key = np.sort(edges[:, 0].astype(np.int64) * len(fp) + edges[:, 1])
    key1 = np.sort(edges1[:, 0].astype(np.int64) * len(fp) + edges1[:, 1])
    assert (edges[:, 0] < edges[:, 1]).all() and len(key) == len(key1) and (key == key1).all()


# ------------------------------------------------------------------ unsuperposed fallbacks stay in popcount order
def _band(n, bits, seed):
    """n fingerprints of popcount 100: a shared core of 75 bits plus 25 bits of their own. Every pair has c ~ 75 and
    similarity ~ 0.6, so none is a neighbour at cutoff 0.3, but every superposed group of them sums far above the
    pre-filter's bound: they fill the candidate list without adding edges."""
    rng = np.random.default_rng(seed)
    pos = rng.permutation(bits)
    core, rest = pos[:75], pos[75:]
    own = rest[np.argpartition(rng.random((n, len(rest)), dtype=np.float32), 25, axis=1)[:, :25]]
    m = np.zeros((n, bits), dtype=bool)
    m[:, core] = True
    m[np.arange(n)[:, None], own] = True
    return S.pack_bits(m)


def _with_band(n_clustered, n_band, seed):
    """Bench-like clustered fingerprints (popcounts ~51) and a band of popcount-100 rows, shuffled together: in the
    pass's order the band is the last n_band rows."""
    fp = np.concatenate([S.clustered_fingerprints(n_clustered // 50 + 1, 50, seed=seed)[:n_clustered], _band(n_band, 2048, seed)])
    fp = np.ascontiguousarray(fp[np.random.default_rng(seed).permutation(len(fp))])
    pop = _popcounts(fp)
    assert (pop == 100).sum() == n_band and (pop[pop != 100] < 100).all()
    return fp


def _plain_graph(fp, cuda):
    """Degrees, edge keys and clusters of one unsuperposed, unpipelined pass (the path the small tests pin to the
    oracle)."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    _lib.set_option("similarity_superpose", 1)
    _lib.set_option("similarity_superpose_cols", 1)
    _lib.set_option("similarity_pipeline_chunks", 1)
    try:
        deg, edges = _neighbor_edges(fp, 0.3, cuda)
        ids, cen = fused_butina_device(A._dev(fp, cuda), 0.3)
    finally:
        _lib.set_option("similarity_superpose", 4)
        _lib.set_option("similarity_superpose_cols", 4)
        _lib.set_option("similarity_pipeline_chunks", 4)
    return deg, np.sort(edges[:, 0] * len(fp) + edges[:, 1]), ids.cpu().numpy(), cen.cpu().numpy()


def test_pipeline_chunk_that_overflows_twice_reruns_unsuperposed_in_popcount_order(cuda):
    """140,000 points (18 row groups: a pipeline of 4 chunks), the last 20,000 of the pass's order a band that fills
    the candidate lists. The chunk owning the band's second row group overflows at 4 x 4 and again at 4 x 1, and is
    redone unsuperposed: that pass must cover the same (popcount-order) row groups as the chunk, or pairs are counted
    twice and others never. Degrees, edge set and clusters equal those of one unsuperposed pass."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    fp = _with_band(120_000, 20_000, seed=140)
    _lib.set_option("similarity_tensor_min_pairs", 0)
    _lib.set_option("similarity_superpose_auto", 0)
    try:
        deg, edges = _neighbor_edges(fp, 0.3, cuda)
        ids, cen = fused_butina_device(A._dev(fp, cuda), 0.3)
        assert _lib.get_option("similarity_superpose_last") == 16
        deg1, key1, ids1, cen1 = _plain_graph(fp, cuda)
    finally:
        _lib.set_option("similarity_superpose_auto", 1)
        _lib.set_option("similarity_tensor_min_pairs", 1 << 24)
    assert len(key1) > 0
    _assert_graph(deg, edges, deg1, key1, len(fp), "pipelined fallback")
    assert (ids.cpu().numpy() == ids1).all() and (cen.cpu().numpy() == cen1).all()


def test_sharded_pass_where_one_rank_falls_back_to_the_plain_pass(cuda):
    """40,960 points over two "ranks", the band = row groups 3 and 4 of the pass's order, both owned by rank 0. Rank 0
    overflows at 4 x 4 and 4 x 1 and runs unsuperposed; rank 1 stays at 4 x 4. Their row groups must still partition
    ONE order: degrees, edge set and clusters equal those of one unsuperposed pass."""
    from nvmolkit_b200 import _lib

    fp = _with_band(24_576, 16_384, seed=2)
    n = len(fp)
    sptr = torch.cuda.current_stream().cuda_stream
    _lib.set_option("similarity_tensor_min_pairs", 0)
    try:
        total = np.zeros(n, dtype=np.int64)
        parts, ran = [], []
        for r in range(2):
            deg_r, edges_r = _neighbor_edges(fp, 0.3, cuda, group_offset=r, group_stride=2)
            ran.append(_lib.get_option("similarity_superpose_last"))
            total += deg_r
            parts.append(edges_r)
        assert ran == [1, 16], ran
        all_edges = np.concatenate(parts)
        deg1, key1, ids1, cen1 = _plain_graph(fp, cuda)
        de = torch.from_numpy(all_edges.astype(np.int32)).to(cuda).contiguous()
        counts = torch.from_numpy(total.astype(np.int32)).to(cuda)
        ids = torch.empty(n, dtype=torch.int32, device=cuda)
        cen = torch.empty(n, dtype=torch.int32, device=cuda)
        ncl = torch.zeros(1, dtype=torch.int32, device=cuda)
        _lib.call("b200mol_butina_from_edges", n, counts.data_ptr(), de.data_ptr(), de.shape[0], ids.data_ptr(), cen.data_ptr(),
                  ncl.data_ptr(), None, sptr)
        k = int(ncl.item())
    finally:
        _lib.set_option("similarity_tensor_min_pairs", 1 << 24)
    assert len(key1) > 0
    _assert_graph(total.astype(np.int32), all_edges, deg1, key1, n, "sharded fallback")
    assert (ids.cpu().numpy() == ids1).all() and (cen[:k].cpu().numpy() == cen1).all()


# ------------------------------------------------------------------ the pilot against its CPU model
def test_pilot_on_the_bench_generator_picks_what_the_model_predicts(cuda):
    """The bench generator at 2,000 centres (100,000 points, enough for the pilot): the factor the pass runs equals the
    CPU model's choice for the same data, and ids and centroids equal those of the unsuperposed pass."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    fp = S.clustered_fingerprints(2000, 50, seed=S.SEED)
    model = pilot_model.pilot(fp, 0.3)
    dev = A._dev(fp, cuda)
    ids, cen = fused_butina_device(dev, 0.3)
    chosen = _lib.get_option("similarity_superpose_last")
    try:
        _lib.set_option("similarity_superpose", 1)
        _lib.set_option("similarity_superpose_cols", 1)
        ids1, cen1 = fused_butina_device(dev, 0.3)
    finally:
        _lib.set_option("similarity_superpose", 4)
        _lib.set_option("similarity_superpose_cols", 4)
    assert chosen == model["chosen"][0] * model["chosen"][1], (chosen, model)
    assert torch.equal(ids, ids1) and torch.equal(cen, cen1)
