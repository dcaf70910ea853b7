"""GPU parity of path A (through the Python surface, which calls the C-ABI): bit-exact vs the CPU oracle."""

import numpy as np
import pytest
import torch

import oracle
from nvmolkit_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _dev(fp, cuda):
    return torch.from_numpy(np.ascontiguousarray(fp).view(np.int32)).to(cuda)


def _with_every_density(fp, seed):
    """fp with rows 1, 2, ... (as many as there are) replaced by an empty row, an all-ones row and rows of bit density
    0.02, 0.5 and 0.97, each followed by a near duplicate (1 to 8 flipped bits). Intersections and unions then reach the
    full width, and similarities span [0, 1]."""
    n, words = fp.shape
    bits = 32 * words
    rng = np.random.default_rng(seed)
    rows = []
    for p in (0.0, 1.0, 0.02, 0.5, 0.97):
        r = rng.random(bits) < p
        d = r.copy()
        d[rng.choice(bits, size=rng.integers(1, 9), replace=False)] ^= True
        rows += [r, d]
    out = fp.copy()
    k = min(len(rows), n - 1)
    if k > 0:
        out[1:1 + k] = S.pack_bits(np.array(rows[:k]))
    return out


# Fingerprint widths the C-ABI accepts (multiples of 128 bits up to 4096) beyond the powers of two. On the SIMT tile:
# a row narrower than 128 bytes that is no power of two of words (384 - 896 bits), a partial last K chunk (1152, 3072
# bits), more K chunks than stages (3072, 4096 bits). On the tensor tile: odd K-chunk counts (384, 640, 896 bits: 3, 5,
# 7) for the row-stationary variant, 9 chunks (1152) just past its limit, 24 and 32 chunks.
SIMT_WIDTHS = [384, 640, 768, 896, 1152, 3072, 4096]
TENSOR_WIDTHS = [384, 640, 896, 1152, 3072, 4096]


# ------------------------------------------------------------------ similarity
@pytest.mark.parametrize("bits", [128, 256, 512, 1024, 2048] + SIMT_WIDTHS)
@pytest.mark.parametrize("n,m", [(1, 1), (1, 300), (127, 129), (128, 128), (257, 513)])
def test_cross_tanimoto_bit_exact(cuda, bits, n, m):
    from nvmolkit_b200.similarity import crossCosineSimilarity, crossTanimotoSimilarity

    a = _with_every_density(S.random_fingerprints(n, bits=bits, p=0.05, seed=n * 7 + bits, near_dups=n // 4), bits)
    b = _with_every_density(S.random_fingerprints(m, bits=bits, p=0.05, seed=m * 11 + bits + 1, near_dups=m // 4), bits + 1)
    b[: min(n, m) // 2] = a[: min(n, m) // 2]
    da, db = _dev(a, cuda), _dev(b, cuda)
    got = crossTanimotoSimilarity(da, db).numpy()
    assert got.dtype == np.float64 and got.shape == (n, m)
    assert (got == oracle.similarity_cross(a, b)).all()
    assert (crossCosineSimilarity(da, db).numpy() == oracle.similarity_cross(a, b, metric="cosine")).all()


def test_cross_tanimoto_config1_1k_x_1k(cuda):
    # BASELINE config 1 stand-in: u32[1000][64] x2, Bernoulli(0.025) bits + planted near duplicates, seed 20260924
    from nvmolkit_b200.similarity import crossTanimotoSimilarity

    a = S.random_fingerprints(1000, seed=S.SEED, near_dups=100)
    b = S.random_fingerprints(1000, seed=S.SEED + 1, near_dups=100)
    b[:50] = a[:50]
    got = crossTanimotoSimilarity(_dev(a, cuda), _dev(b, cuda)).numpy()
    want = oracle.similarity_cross(a, b)
    assert (got == want).all()
    assert got.max() == 1.0 and got.min() == 0.0


def test_self_similarity_and_empty_rows(cuda):
    from nvmolkit_b200.similarity import crossCosineSimilarity, crossTanimotoSimilarity

    a = S.random_fingerprints(200, seed=5, near_dups=40)
    a[3] = 0  # empty fingerprint: similarity 0 to everything, itself included (src/load_store.cuh:264-269)
    d = _dev(a, cuda)
    t = crossTanimotoSimilarity(d).numpy()
    assert (t == oracle.similarity_cross(a)).all()
    assert t[3].max() == 0.0 and np.allclose(np.delete(np.diag(t), 3), 1.0)
    c = crossCosineSimilarity(d).numpy()
    assert (c == oracle.similarity_cross(a, metric="cosine")).all()


def test_zero_rows_and_errors(cuda):
    from nvmolkit_b200.similarity import crossTanimotoSimilarity

    a = _dev(S.random_fingerprints(5), cuda)
    assert crossTanimotoSimilarity(a[:0], a).numpy().shape == (0, 5)
    with pytest.raises(TypeError):
        crossTanimotoSimilarity(a, a, stream="not a stream")
    with pytest.raises(ValueError):
        crossTanimotoSimilarity(a, a[:, :32].contiguous())
    with pytest.raises(ValueError):
        crossTanimotoSimilarity(a.to(torch.float32))


def test_non_default_stream(cuda):
    from nvmolkit_b200.similarity import crossTanimotoSimilarity

    a = S.random_fingerprints(300, seed=9, near_dups=50)
    d = _dev(a, cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    res = crossTanimotoSimilarity(d, stream=s)
    s.synchronize()
    assert (res.torch().cpu().numpy() == oracle.similarity_cross(a)).all()


def test_memory_constrained_host_variant(cuda):
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.similarity import crossCosineSimilarityMemoryConstrained, crossTanimotoSimilarityMemoryConstrained

    a = S.random_fingerprints(700, seed=21, near_dups=100)
    b = S.random_fingerprints(333, seed=22, near_dups=50)
    assert (crossTanimotoSimilarityMemoryConstrained(a.view(np.int32), b.view(np.int32)) == oracle.similarity_cross(a, b)).all()
    assert (crossCosineSimilarityMemoryConstrained(torch.from_numpy(a.view(np.int32))) ==
            oracle.similarity_cross(a, metric="cosine")).all()
    # force several row blocks through the two device buffers
    out = np.empty((700, 333))
    _lib.call("b200mol_similarity_cross_host", a.ctypes.data, 700, b.ctypes.data, 333, 64, 0, out.ctypes.data,
              2 * 128 * 333 * 8)
    assert (out == oracle.similarity_cross(a, b)).all()
    # 4096 bits, every density class, both metrics, several row blocks
    a = _with_every_density(S.random_fingerprints(700, bits=4096, seed=23, near_dups=100), 23)
    b = _with_every_density(S.random_fingerprints(333, bits=4096, seed=24, near_dups=50), 24)
    b[:20] = a[:20]
    for metric in ("tanimoto", "cosine"):
        out = np.empty((700, 333))
        _lib.call("b200mol_similarity_cross_host", a.ctypes.data, 700, b.ctypes.data, 333, 128, _lib.METRIC[metric],
                  out.ctypes.data, 2 * 128 * 333 * 8)
        assert (out == oracle.similarity_cross(a, b, metric=metric)).all(), metric


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("cutoff", [0.0, 0.3, 0.35, 0.65, 1.0])
def test_count_ge_exact(cuda, metric, cutoff):
    """SIMT tile, at every width class and with rows of every density, both signs."""
    from nvmolkit_b200 import _lib

    for bits, dense in [(2048, False), (2048, True)] + [(bits, True) for bits in SIMT_WIDTHS]:
        x = S.clustered_fingerprints(12, 25, bits=bits, seed=31)
        y = S.clustered_fingerprints(12, 11, bits=bits, seed=31)  # same centres, other members
        if dense:
            x, y = _with_every_density(x, bits), _with_every_density(y, bits + 1)
        dx, dy = _dev(x, cuda), _dev(y, cuda)
        for sign in (-1, 1):
            counts = torch.full((x.shape[0],), 1000, dtype=torch.int32, device=cuda)
            _lib.call("b200mol_tanimoto_count_ge", dx.data_ptr(), x.shape[0], dy.data_ptr(), y.shape[0], bits // 32,
                      _lib.METRIC[metric], cutoff, sign, counts.data_ptr(), torch.cuda.current_stream().cuda_stream)
            want = oracle.count_ge(x, y, cutoff, metric=metric, sign=sign, counts=np.full(x.shape[0], 1000, dtype=np.int32))
            assert (counts.cpu().numpy() == want).all(), (bits, sign)


def test_threshold_boundary_is_fp64_exact(cuda):
    """Pairs whose 1 - c/u sits exactly on / next to the cutoff: integer table must agree with the fp64 predicate."""
    from nvmolkit_b200 import _lib

    rng = np.random.default_rng(0)
    rows = []
    for u, c in [(10, 7), (20, 14), (100, 70), (1000, 700), (10, 6), (3, 2), (7, 5)]:
        bits_a = np.zeros(2048, dtype=bool)
        bits_b = np.zeros(2048, dtype=bool)
        perm = rng.permutation(2048)
        bits_a[perm[:u]] = True  # |A| = u, B subset of A with |B| = c  -> sim = c/u
        bits_b[perm[:c]] = True
        rows.append((S.pack_bits(bits_a[None])[0], S.pack_bits(bits_b[None])[0]))
    x = np.stack([r[0] for r in rows])
    y = np.stack([r[1] for r in rows])
    dx, dy = _dev(x, cuda), _dev(y, cuda)  # keep the device buffers alive across the asynchronous calls
    for cutoff in (0.3, 1.0 - 0.7, 0.30000000000000004, 0.29999999999999993, 1 / 3, 0.4):
        counts = torch.zeros(len(x), dtype=torch.int32, device=cuda)
        _lib.call("b200mol_tanimoto_count_ge", dx.data_ptr(), len(x), dy.data_ptr(), len(y), 64,
                  0, cutoff, 1, counts.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert (counts.cpu().numpy() == oracle.count_ge(x, y, cutoff)).all(), cutoff


# ------------------------------------------------------------------ butina
def _assert_same_clustering(ids, cen, ids_cpu, cen_cpu):
    assert (ids == ids_cpu).all()
    assert (cen == cen_cpu).all()


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("centres,members,cutoff", [(1, 1, 0.3), (3, 1, 0.3), (40, 25, 0.3), (25, 40, 0.2), (60, 17, 0.5)])
def test_fused_butina_equals_rdkit_definition(cuda, metric, centres, members, cutoff):
    from nvmolkit_b200.clustering import fused_butina_device

    fp = S.clustered_fingerprints(centres, members, seed=centres * 100 + members)
    ids, cen = fused_butina_device(_dev(fp, cuda), cutoff, metric=metric)
    ids_cpu, cen_cpu = oracle.butina_fp(fp, cutoff, metric=metric)
    _assert_same_clustering(ids.cpu().numpy(), cen.cpu().numpy(), ids_cpu, cen_cpu)


def test_fused_butina_5k(cuda):
    from nvmolkit_b200.clustering import fused_butina_device

    fp = S.clustered_fingerprints(100, 50, seed=S.SEED)
    ids, cen = fused_butina_device(_dev(fp, cuda), 0.3)
    ids_cpu, cen_cpu = oracle.butina_fp(fp, 0.3)
    _assert_same_clustering(ids.cpu().numpy(), cen.cpu().numpy(), ids_cpu, cen_cpu)
    sizes = np.bincount(ids.cpu().numpy())
    assert (np.diff(sizes) <= 0).all()  # cluster 0 is the largest, sizes non-increasing


def test_fused_butina_python_return_shape(cuda):
    from nvmolkit_b200.clustering import fused_butina

    fp = S.clustered_fingerprints(10, 9, seed=3)
    clusters, sizes, centroids = fused_butina(_dev(fp, cuda), 0.3, return_centroids=True)
    assert sizes[0] == 0 and sizes[-1] == 90 and len(sizes) == len(clusters) + 1
    assert sorted(m for c in clusters for m in c) == list(range(90))
    for c, cen in zip(clusters, centroids):
        assert c[0] == cen
    with pytest.raises(ValueError):
        fused_butina(_dev(fp, cuda), 1.5)
    with pytest.raises(ValueError):
        fused_butina(_dev(fp, cuda), 0.3, metric="dice")


def test_fused_butina_identical_and_all_distinct(cuda):
    # nvmolkit/tests/test_clustering.py:154-295: all-identical -> one cluster; random -> all singletons
    from nvmolkit_b200.clustering import fused_butina_device

    one = np.repeat(S.random_fingerprints(1, seed=1), 300, axis=0)  # dense graph: exercises the edge-buffer regrow
    ids, cen = fused_butina_device(_dev(one, cuda), 0.3)
    assert (ids.cpu().numpy() == 0).all() and cen.cpu().numpy().tolist() == [299]
    rnd = S.random_fingerprints(500, seed=2)
    ids, cen = fused_butina_device(_dev(rnd, cuda), 0.3)
    assert sorted(ids.cpu().numpy().tolist()) == list(range(500))
    assert cen.cpu().numpy().tolist() == list(range(499, -1, -1))


def test_dense_butina_known_answer_and_oracle(cuda):
    from nvmolkit_b200.clustering import butina

    d = np.ones((10, 10))
    np.fill_diagonal(d, 0.0)
    for j in (1, 2, 3):
        d[0, j] = d[j, 0] = 0.05
    for j in (5, 6):
        d[4, j] = d[j, 4] = 0.05
    ids, cen = butina(torch.from_numpy(d).to(cuda), 0.1, return_centroids=True)
    ids, cen = ids.numpy(), cen.numpy()
    assert sorted(np.nonzero(ids == 0)[0].tolist()) == [0, 1, 2, 3] and cen[0] == 0  # tests/test_butina.cpp:241-273
    assert sorted(np.nonzero(ids == 1)[0].tolist()) == [4, 5, 6] and cen[1] == 4
    assert len(cen) == 5

    fp = S.clustered_fingerprints(30, 30, seed=77)
    dist = 1.0 - oracle.similarity_cross(fp)
    for cutoff in (0.1, 0.3, 0.6):
        ids, cen = butina(torch.from_numpy(dist).to(cuda), cutoff, return_centroids=True)
        ids_cpu, cen_cpu = oracle.butina_dense(dist, cutoff)
        _assert_same_clustering(ids.numpy(), cen.numpy(), ids_cpu, cen_cpu)
    with pytest.raises(ValueError):
        butina(torch.from_numpy(dist).to(cuda), 0.3, neighborlist_max_size=17)


# ------------------------------------------------------------------ morgan
@pytest.mark.parametrize("radius", [0, 1, 2, 3, 5])
@pytest.mark.parametrize("fp_size", [128, 1024, 2048])
def test_morgan_bit_exact(cuda, radius, fp_size):
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    g = S.random_molgraphs(400, min_atoms=1, max_atoms=70, seed=radius * 10 + fp_size)
    got = MorganFingerprintGenerator(radius, fp_size).GetFingerprints(g).numpy().view(np.uint32)
    want = oracle.morgan(g.atom_starts, g.bond_starts, g.atom_inv, g.bond_inv, g.bond_a, g.bond_b, radius, fp_size)
    assert got.shape == want.shape and (got == want).all()
    assert (got != 0).any(axis=1).all()  # regression test_gh_issue_84: never empty


def test_morgan_large_molecules_on_gpu(cuda):
    # the reference sends >=128-atom molecules to a CPU twin (src/morgan_fingerprint_gpu.cpp:181-198); here they stay on the GPU
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    g = S.random_molgraphs(40, min_atoms=120, max_atoms=300, seed=5)
    got = MorganFingerprintGenerator(3, 2048).GetFingerprints(g).numpy().view(np.uint32)
    want = oracle.morgan(g.atom_starts, g.bond_starts, g.atom_inv, g.bond_inv, g.bond_a, g.bond_b, 3, 2048)
    assert (got == want).all()


def test_morgan_known_answer_bits(cuda):
    """Bits of pentane at radius 2 = the 7 distinct codes of the golden test, folded."""
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator, unpack_fingerprint
    from nvmolkit_b200.molgraph import MolGraphBatch, atom_invariant

    t, m = atom_invariant(6, 4, 3, 0, 0, False), atom_invariant(6, 4, 2, 0, 0, False)
    g = MolGraphBatch([0, 5], [0, 4], [t, m, m, m, t], [1, 1, 1, 1], [0, 1, 2, 3], [1, 2, 3, 4])
    fp = MorganFingerprintGenerator(2, 2048).GetFingerprints(g)
    bits = unpack_fingerprint(fp.torch()).cpu().numpy()[0]
    codes = oracle.morgan_codes([t, m, m, m, t], [1, 1, 1, 1], [0, 1, 2, 3], [1, 2, 3, 4], 2)
    assert set(np.nonzero(bits)[0].tolist()) == {int(c) % 2048 for c in codes}
    assert len(set(codes.tolist())) == 7


def test_pack_unpack_roundtrip(cuda):
    from nvmolkit_b200.fingerprints import pack_fingerprint, unpack_fingerprint

    fp = torch.from_numpy(S.random_fingerprints(9, bits=256).view(np.int32)).to(cuda)
    assert (pack_fingerprint(unpack_fingerprint(fp)) == fp).all()


@pytest.mark.parametrize("min_commits", [0, 32, 10 ** 9])  # rounds to exhaustion | default hybrid | stepwise loop only
@pytest.mark.parametrize("n,degree", [(60, 3), (400, 10), (1500, 40)])
def test_butina_parallel_rounds_keep_the_greedy_order(cuda, min_commits, n, degree):
    """Overlapping neighbourhoods (a random graph, no cluster structure): many rounds whose commits depend on each
    other. Every mode must reproduce the sequential greedy result - members, centroids AND ids (creation order)."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import butina

    rng = np.random.default_rng(n * 7 + degree)
    d = rng.random((n, n))
    d = np.minimum(d, d.T)
    np.fill_diagonal(d, 0.0)
    cutoff = 1.0 - (1.0 - degree / n) ** 0.5  # P(min(u, v) <= c) = degree / n
    with _lib.options(butina_min_round_commits=min_commits):
        ids, cen = butina(torch.from_numpy(d).to(cuda), cutoff, return_centroids=True)
    ids_cpu, cen_cpu = oracle.butina_dense(d, cutoff)
    assert (ids.numpy() == ids_cpu).all() and (cen.numpy() == cen_cpu).all()


# ------------------------------------------------------------------ tensor-core (wgmma u8) path of the count pass
@pytest.fixture(params=[(1, 4, 4), (0, 4, 4), (2, 4, 4), (3, 4, 4), (1, 1, 1), (3, 1, 1), (0, 2, 1), (1, 4, 1), (1, 1, 4),
                        (0, 2, 4)],
                ids=["multicast_pair-super4x4", "single_cta-super4x4", "pair_mma-super4x4", "row_stationary-super4x4",
                     "multicast_pair-plain", "row_stationary-plain", "single_cta-super2x1", "multicast_pair-super4x1",
                     "multicast_pair-super1x4", "single_cta-super2x4"])
def force_tensor_path(cuda, request):
    """Every test that takes this fixture runs on all values of similarity_tensor_cluster: 1 (CTA pair, multicast column
    operand), 0 (one CTA per tile), 2 (accepted for callers of the CTA-pair MMA that Hopper lacks: runs as 1),
    3 (CTA pair, multicast column operand, row operand stationary for fingerprints up to 1024 bits) - crossed with the
    row x column superposition of the Butina neighbour pass (4 x 4 = default ... 1 x 1 = off)."""
    from nvmolkit_b200 import _lib

    with _lib.options(similarity_tensor_min_pairs=0, similarity_tensor_cluster=request.param[0],
                      similarity_superpose=request.param[1], similarity_superpose_cols=request.param[2]):
        yield request.param


@pytest.mark.parametrize("bits", [128, 512, 2048] + TENSOR_WIDTHS)
@pytest.mark.parametrize("nx,ny", [(1, 1), (127, 255), (128, 256), (129, 257), (700, 333)])
def test_tensor_count_ge_exact(cuda, force_tensor_path, bits, nx, ny):
    from nvmolkit_b200 import _lib

    x = _with_every_density(S.clustered_fingerprints(max(1, nx // 25 + 1), 25, bits=bits, seed=41)[:nx], bits)
    y = _with_every_density(S.clustered_fingerprints(max(1, ny // 11 + 1), 11, bits=bits, seed=41)[:ny], bits + 1)
    dx, dy = _dev(x, cuda), _dev(y, cuda)
    for cutoff in (0.3, 0.65):
        for sign in (1, -1):
            counts = torch.full((nx,), 7, dtype=torch.int32, device=cuda)
            _lib.call("b200mol_tanimoto_count_ge", dx.data_ptr(), nx, dy.data_ptr(), ny, bits // 32, 0, cutoff, sign,
                      counts.data_ptr(), torch.cuda.current_stream().cuda_stream)
            want = oracle.count_ge(x, y, cutoff, sign=sign, counts=np.full(nx, 7, dtype=np.int32))
            assert (counts.cpu().numpy() == want).all(), (bits, nx, ny, cutoff, sign)


@pytest.mark.parametrize("centres,members,cutoff", [(1, 1, 0.3), (7, 40, 0.3), (40, 25, 0.3), (60, 17, 0.5), (100, 50, 0.3)])
def test_tensor_fused_butina_equals_rdkit_definition(cuda, force_tensor_path, centres, members, cutoff):
    from nvmolkit_b200.clustering import fused_butina_device

    fp = S.clustered_fingerprints(centres, members, seed=centres * 100 + members)
    ids, cen = fused_butina_device(_dev(fp, cuda), cutoff)
    ids_cpu, cen_cpu = oracle.butina_fp(fp, cutoff)
    assert (ids.cpu().numpy() == ids_cpu).all() and (cen.cpu().numpy() == cen_cpu).all()


@pytest.mark.parametrize("n", [2, 3, 5, 127, 129, 897, 1023])
def test_tensor_fused_butina_on_ragged_sizes(cuda, force_tensor_path, n):
    """Sizes that are no multiple of the superposition factors, the tile rows (128) or the tile columns (256): the
    last super row / super column sums fewer fingerprints, the last tile is clipped."""
    from nvmolkit_b200.clustering import fused_butina_device

    fp = S.clustered_fingerprints(26, 40, seed=n)[:n].copy()
    for cutoff in (0.3, 0.62):
        ids, cen = fused_butina_device(_dev(fp, cuda), cutoff)
        ids_cpu, cen_cpu = oracle.butina_fp(fp, cutoff)
        assert (ids.cpu().numpy() == ids_cpu).all() and (cen.cpu().numpy() == cen_cpu).all(), (n, cutoff)


@pytest.mark.parametrize("bits", [640, 4096])
def test_tensor_fused_butina_at_wide_and_odd_widths(cuda, force_tensor_path, bits):
    """Fused Butina on 4096-bit fingerprints (32 K chunks) and on 640-bit ones (no power of two: 5 K chunks), with rows
    of every density among the clustered ones."""
    from nvmolkit_b200.clustering import fused_butina_device

    fp = _with_every_density(S.clustered_fingerprints(40, 25, bits=bits, seed=bits), bits)
    for cutoff in (0.3, 0.62):
        ids, cen = fused_butina_device(_dev(fp, cuda), cutoff)
        ids_cpu, cen_cpu = oracle.butina_fp(fp, cutoff)
        assert (ids.cpu().numpy() == ids_cpu).all() and (cen.cpu().numpy() == cen_cpu).all(), (bits, cutoff)


@pytest.mark.parametrize("metric", ["tanimoto", "cosine"])
@pytest.mark.parametrize("bits", [640, 4096])
def test_fused_butina_at_wide_and_odd_widths(cuda, metric, bits):
    """The same on the SIMT tile, for both metrics."""
    from nvmolkit_b200.clustering import fused_butina_device

    fp = _with_every_density(S.clustered_fingerprints(40, 25, bits=bits, seed=bits), bits)
    for cutoff in (0.3, 0.62):
        ids, cen = fused_butina_device(_dev(fp, cuda), cutoff, metric=metric)
        ids_cpu, cen_cpu = oracle.butina_fp(fp, cutoff, metric=metric)
        assert (ids.cpu().numpy() == ids_cpu).all() and (cen.cpu().numpy() == cen_cpu).all(), (bits, cutoff)


def test_tensor_neighbor_counts_on_a_many_tile_problem(cuda, force_tensor_path):
    """9,000 points = 71 tile rows x 36 tile columns: several row groups, and for the CTA pairs an odd number of tile
    rows (the last pair's lower tile lies past the end)."""
    from nvmolkit_b200.clustering import fused_butina_device

    fp = S.clustered_fingerprints(180, 50, seed=99)
    ids, cen = fused_butina_device(_dev(fp, cuda), 0.3)
    ids_cpu, cen_cpu = oracle.butina_fp(fp, 0.3)
    assert (ids.cpu().numpy() == ids_cpu).all() and (cen.cpu().numpy() == cen_cpu).all()


@pytest.mark.parametrize("superpose", [1, 4])
def test_row_stationary_tile_reloads_its_row_operand(cuda, superpose):
    """1024-bit fingerprints keep the row tile of the row-stationary variant in shared memory: 9,000 points are several
    runs of 16 tile columns per tile row with a row-operand reload between them (and, superposed, several row groups)."""
    from nvmolkit_b200 import _lib

    fp = S.clustered_fingerprints(180, 50, bits=1024, seed=98)
    counts = torch.zeros(len(fp), dtype=torch.int32, device=cuda)
    dfp = _dev(fp, cuda)
    with _lib.options(similarity_tensor_min_pairs=0, similarity_tensor_cluster=3, similarity_superpose=superpose,
                      similarity_superpose_cols=superpose):
        _lib.call("b200mol_tanimoto_count_ge", dfp.data_ptr(), len(fp), dfp.data_ptr(), len(fp), 32, 0, 0.3, 1,
                  counts.data_ptr(), torch.cuda.current_stream().cuda_stream)
        from nvmolkit_b200.clustering import fused_butina_device

        ids, cen = fused_butina_device(dfp, 0.3)
    assert (counts.cpu().numpy() == oracle.count_ge(fp, fp, 0.3)).all()
    ids_cpu, cen_cpu = oracle.butina_fp(fp, 0.3)
    assert (ids.cpu().numpy() == ids_cpu).all() and (cen.cpu().numpy() == cen_cpu).all()


def test_pilot_chosen_superposition_gives_the_unsuperposed_answer(cuda):
    """70,000 points: the neighbour pass first runs its pilot over a prefix sample per column factor, picks a factor,
    then runs; cluster ids and centroids must equal those of the unsuperposed pass (which the smaller tests pin
    to the oracle). Dense (p = 0.08) and sparse (p = 0.012) fingerprints make the pilot choose differently."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    with _lib.options(similarity_tensor_min_pairs=0, similarity_superpose=4, similarity_superpose_cols=4):
        chosen = []
        for dens in (0.08, 0.012):
            fp = S.random_fingerprints(70_000, p=dens, seed=5, near_dups=30_000)
            dev = _dev(fp, cuda)
            ids, cen = fused_butina_device(dev, 0.35)
            chosen.append(_lib.get_option("similarity_superpose_last"))
            with _lib.options(similarity_superpose=1, similarity_superpose_cols=1):
                ids1, cen1 = fused_butina_device(dev, 0.35)
            assert torch.equal(ids, ids1) and torch.equal(cen, cen1)
        assert chosen == [4, 16], chosen  # sparse rows carry 4 x 4 sums, dense ones only rows


def test_pipelined_verification_gives_the_same_graph(cuda):
    """From 16 row groups up the superposed pass runs as a pipeline of 4 chunks (the verification of one chunk overlaps
    the tensor pass of the next, on a second stream). Same cluster ids and centroids as the one-chunk pass - also when
    every chunk's candidate list overflows (clusters of 400: ~27 M edges) and each chunk is redone with fewer pairs per
    accumulator after the others."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    for centres, members, auto in ((2700, 50, 1), (338, 400, 0)):
        dev = _dev(S.clustered_fingerprints(centres, members, seed=centres), cuda)
        with _lib.options(similarity_tensor_min_pairs=0, similarity_superpose_auto=auto, similarity_pipeline_chunks=4):
            ids, cen = fused_butina_device(dev, 0.3)
            listed = _lib.get_option("similarity_candidates_last")
            with _lib.options(similarity_pipeline_chunks=1):
                ids1, cen1 = fused_butina_device(dev, 0.3)
        assert torch.equal(ids, ids1) and torch.equal(cen, cen1), (centres, members)
        assert listed > 0


def test_superposed_pass_falls_back_when_its_candidate_list_overflows(cuda):
    """12,000 identical fingerprints: every pair is an edge, so the 4 x 4 superposed pass lists ~4.5 M candidates and its
    4 x 1 rerun ~18 M, both more than the list holds; nothing may have been counted when they notice, and the unsuperposed
    rerun must give the exact answer."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    one = np.repeat(S.random_fingerprints(1, seed=3), 12000, axis=0)
    with _lib.options(similarity_tensor_min_pairs=0):
        ids, cen = fused_butina_device(_dev(one, cuda), 0.3)
        assert _lib.get_option("similarity_superpose_last") == 1
    assert (ids.cpu().numpy() == 0).all() and cen.cpu().numpy().tolist() == [11999]


def test_tensor_and_simt_paths_agree_on_identical_rows(cuda, force_tensor_path):
    from nvmolkit_b200.clustering import fused_butina_device

    one = np.repeat(S.random_fingerprints(1, seed=1), 600, axis=0)  # dense graph: every pair is an edge, buffer regrows
    ids, cen = fused_butina_device(_dev(one, cuda), 0.3)
    assert (ids.cpu().numpy() == 0).all() and cen.cpu().numpy().tolist() == [599]


@pytest.mark.parametrize("bits", [128, 1024, 2048] + TENSOR_WIDTHS)
@pytest.mark.parametrize("n,m", [(1, 1), (127, 300), (129, 256), (640, 513)])
def test_tensor_cross_similarity_bit_exact(cuda, force_tensor_path, bits, n, m):
    from nvmolkit_b200.similarity import crossCosineSimilarity, crossTanimotoSimilarity

    a = _with_every_density(S.random_fingerprints(n, bits=bits, p=0.05, seed=n * 7 + bits, near_dups=n // 4), bits)
    b = _with_every_density(S.random_fingerprints(m, bits=bits, p=0.05, seed=m * 11 + bits + 1, near_dups=m // 4), bits + 1)
    b[: min(n, m) // 2] = a[: min(n, m) // 2]
    a[0] = 0  # empty fingerprint row
    da, db = _dev(a, cuda), _dev(b, cuda)
    assert (crossTanimotoSimilarity(da, db).numpy() == oracle.similarity_cross(a, b)).all()
    assert (crossCosineSimilarity(da, db).numpy() == oracle.similarity_cross(a, b, metric="cosine")).all()
    assert (crossTanimotoSimilarity(da).numpy() == oracle.similarity_cross(a)).all()


# ------------------------------------------------------------------ sharded pair pass (the multi-GPU path, on ONE GPU)
def _sharded_butina_one_gpu(fp, cutoff, world, cuda):
    """What fused_butina_sharded does over `world` ranks, replayed on one device: every "rank" runs
    b200mol_neighbor_edges with (group_offset, group_stride) = (r, world); counts are summed (the all-reduce), edge
    lists concatenated (the all-gather-v), then b200mol_butina_from_edges clusters the full graph."""
    import ctypes as C

    from nvmolkit_b200 import _lib

    d = _dev(fp, cuda)
    n, words = d.shape
    sptr = torch.cuda.current_stream().cuda_stream
    total = torch.zeros(n, dtype=torch.int32, device=cuda)
    parts, per_rank = [], []
    for r in range(world):
        cap = 1 << 20
        while True:
            counts = torch.zeros(n, dtype=torch.int32, device=cuda)
            edges = torch.empty((cap, 2), dtype=torch.int32, device=cuda)
            found = C.c_uint64(0)
            _lib.call("b200mol_neighbor_edges", d.data_ptr(), n, words, 0, float(cutoff), r, world, counts.data_ptr(),
                      edges.data_ptr(), cap, C.byref(found), sptr)
            if found.value <= cap:
                break
            cap = int(found.value)
        total += counts
        parts.append(edges[: found.value])
        per_rank.append(int(found.value))
    all_edges = torch.cat(parts).contiguous()
    ids = torch.empty(n, dtype=torch.int32, device=cuda)
    cen = torch.empty(max(n, 1), dtype=torch.int32, device=cuda)
    ncl = torch.zeros(1, dtype=torch.int32, device=cuda)
    deg = total.clone()
    _lib.call("b200mol_butina_from_edges", n, total.data_ptr(), all_edges.data_ptr(), all_edges.shape[0], ids.data_ptr(),
              cen.data_ptr(), ncl.data_ptr(), None, sptr)
    k = int(ncl.item())
    return ids.cpu().numpy(), cen[:k].cpu().numpy(), all_edges.cpu().numpy(), deg.cpu().numpy(), per_rank


def test_sharded_pipelined_pass_equals_the_plain_pass(cuda):
    """270,000 points over two "ranks": each owns 17 row groups, enough for its superposed pass to run as a pipeline of
    four chunks (group stride 2 x 4). Degrees, edge set and clusters must equal those of ONE unsuperposed, unpipelined
    pass over everything (the path the small tests pin to the oracle)."""
    from nvmolkit_b200 import _lib

    fp = S.clustered_fingerprints(5400, 50, seed=11)
    with _lib.options(similarity_tensor_min_pairs=0):
        ids, cen, edges, deg, per_rank = _sharded_butina_one_gpu(fp, 0.3, 2, cuda)
        assert all(c > 0 for c in per_rank)
        with _lib.options(similarity_pipeline_chunks=1, similarity_superpose=1, similarity_superpose_cols=1):
            ids1, cen1, edges1, deg1, _ = _sharded_butina_one_gpu(fp, 0.3, 1, cuda)
    assert (deg == deg1).all() and (ids == ids1).all() and (cen == cen1).all()
    key = np.sort(edges[:, 0].astype(np.int64) * len(fp) + edges[:, 1])
    key1 = np.sort(edges1[:, 0].astype(np.int64) * len(fp) + edges1[:, 1])
    assert (edges[:, 0] < edges[:, 1]).all() and len(key) == len(key1) and (key == key1).all()


@pytest.mark.parametrize("tensor", [0, 1, 3], ids=["simt_tile", "tensor_tile", "tensor_row_stationary"])
@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("centres,members", [(30, 20), (130, 50)])  # 600 and 6500 points: 5 and 51 tile rows
def test_sharded_neighbor_pass_equals_oracle(cuda, world, centres, members, tensor):
    """Parity of the multi-GPU fused Butina path (VERDICT r01 weak 9): the union of the ranks' tiles must be every
    unordered pair exactly once - same edge set, same degrees, same clusters as the single-pass CPU definition."""
    from nvmolkit_b200 import _lib

    fp = S.clustered_fingerprints(centres, members, seed=centres + world)
    with _lib.options(similarity_tensor_min_pairs=0 if tensor else -1, similarity_tensor_cluster=tensor if tensor else 1):
        ids, cen, edges, deg, per_rank = _sharded_butina_one_gpu(fp, 0.3, world, cuda)
    ids_cpu, cen_cpu = oracle.butina_fp(fp, 0.3)
    want_deg = oracle.count_ge(fp, fp, 0.3) - 1  # neighbours other than the point itself
    assert (deg == want_deg).all()
    assert (edges[:, 0] < edges[:, 1]).all()
    key = edges[:, 0].astype(np.int64) * len(fp) + edges[:, 1]
    assert len(np.unique(key)) == len(key) == int(want_deg.sum()) // 2  # every neighbour pair exactly once
    assert (ids == ids_cpu).all() and (cen == cen_cpu).all()
    rows_per_group = 8192 if tensor else 4096  # row group of the tensor tiles (any variant / superposition) | of the SIMT tile
    if -(-len(fp) // rows_per_group) >= world and centres * members >= 1000:  # every rank owns a group -> finds edges
        assert all(c > 0 for c in per_rank), per_rank
