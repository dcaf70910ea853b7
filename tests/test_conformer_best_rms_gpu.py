"""Symmetry-aware conformer RMSD matrices on the GPU (b200mol_conformer_rmsd_mapped, conformerRmsd.GetAllConformerBestRMS
and atomIds) against the fp64 oracle (oracle_best_rms.c) at the tolerances of test_conformer_rmsd_gpu.py: the identity
table equals the plain call bit for bit, mapped matrices at conformer counts around the 32-tile, list lengths around the
16-atom chunks (with 1-3 atoms and collinear sets), K from 1 to 1,296 and forced chunk sizes, orientation independence,
repeatability, batching, streams, the Device3DResult path, and agreement with RMS pruning on the same tables."""
import itertools

import numpy as np
import pytest
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200 import conformerRmsd as cr
from nvmolkit_b200.pruning import rms_prune
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult
from oracle import best_rms as oracle_best

pytestmark = pytest.mark.gpu

R = 32  # pair-pass tile side (csrc/conformer_rmsd.cu)


class StandIn:
    """A molecule with conformers and a fixed list of self matches (the RDKit surface the module uses)."""

    def __init__(self, coords, n, matches):
        self.coords = [np.asarray(c, np.float64) for c in coords]
        self.n = n
        self.matches = matches

    def GetNumAtoms(self):
        return self.n

    def GetConformers(self):
        return [_Conf(c) for c in self.coords]

    def GetAtoms(self):
        return []

    def GetSubstructMatches(self, query, uniquify=True, maxMatches=1000, useChirality=False):
        return self.matches[:maxMatches]


class _Conf:
    def __init__(self, xyz):
        self.xyz = xyz

    def GetPositions(self):
        return self.xyz


def assert_close(got, want, what=""):
    assert got.dtype == np.float64 and got.shape == want.shape, what
    if len(want):
        err = np.abs(got - want)
        assert err.max() <= 1e-5, (what, float(err.max()))
        far = want >= 0.05
        if far.any():
            assert err[far].max() <= 1e-8, (what, float(err[far].max()))


def rotation(rng):
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1.0
    return q


def conformers(rng, c, n, spread=0.6):
    base = rng.normal(size=(n, 3)) * 1.5
    return [base @ rotation(rng) + rng.normal(size=3) * 3.0 + rng.normal(size=(n, 3)) * spread for _ in range(c)]


def device_inputs(coords, atoms):
    counts = np.array([len(c) for c in coords], np.int64)
    atoms = np.asarray(atoms, np.int64)
    blocks = [np.asarray(x, np.float64) for c in coords for x in c]
    xyz = torch.from_numpy(np.concatenate(blocks) if blocks else np.zeros((0, 3))).cuda()
    cas = torch.from_numpy(np.concatenate([[0], np.cumsum(np.repeat(atoms, counts))]).astype(np.int32)).cuda()
    return counts, atoms, xyz, cas


def atom_counts(coords, lists):
    return [len(c[0]) if len(c) else int(max(np.max(p), np.max(q))) + 1 for c, (p, q) in zip(coords, lists)]


def mapped(coords, lists, prealigned=False, stream=None):
    counts, atoms, xyz, cas = device_inputs(coords, atom_counts(coords, lists))
    res = cr._run(counts, atoms, None, cas, xyz, prealigned, stream, cr.MapTables(lists))
    torch.cuda.synchronize()
    return [r.torch().cpu().numpy() for r in res]


def check(coords, lists, prealigned=False):
    got = mapped(coords, lists, prealigned)
    want = oracle_best.molecules(coords, lists, prealigned)
    for m, (g, w) in enumerate(zip(got, want)):
        assert_close(g, w, (m, prealigned))
    return got


def random_lists(rng, n, L, K, identity_first=True):
    p = rng.choice(n, L, replace=False)
    qs = [p] if identity_first else []
    while len(qs) < K:
        qs.append(rng.choice(n, L, replace=False))
    return p, np.stack(qs)


@pytest.mark.parametrize("prealigned", [False, True])
def test_identity_table_equals_the_plain_call_bitwise(cuda, prealigned):
    rng = np.random.default_rng(1)
    shapes = [(0, 12), (1, 12), (2, 12), (R - 1, 12), (R, 12), (R + 1, 12), (2 * R + 1, 12), (37, 1), (37, 2), (37, 3),
              (37, 15), (37, 16), (37, 17), (37, 33), (37, 48), (37, 49), (20, 1000)]
    coords = [conformers(rng, c, n) for c, n in shapes]
    counts, atoms, xyz, cas = device_inputs(coords, [n for _, n in shapes])
    plain = cr._run(counts, atoms, None, cas, xyz, prealigned, None)
    ident = cr._run(counts, atoms, None, cas, xyz, prealigned, None,
                    cr.MapTables([(np.arange(n), np.arange(n)[None]) for n in atoms]))
    torch.cuda.synchronize()
    for m, (a, b) in enumerate(zip(plain, ident)):
        assert torch.equal(a.torch().view(torch.int64), b.torch().view(torch.int64)), m


@pytest.mark.parametrize("prealigned", [False, True])
def test_conformer_counts_around_the_tile(cuda, prealigned):
    rng = np.random.default_rng(2)
    counts = [0, 1, 2, R - 1, R, R + 1, 2 * R - 1, 2 * R + 1, 5]
    coords = [conformers(rng, c, 12) for c in counts]
    check(coords, [random_lists(rng, 12, 9, 3) for _ in counts], prealigned)


@pytest.mark.parametrize("prealigned", [False, True])
def test_list_lengths_around_the_chunks(cuda, prealigned):
    rng = np.random.default_rng(3)
    cases = [(1, 4), (2, 4), (3, 5), (15, 20), (16, 20), (17, 20), (31, 40), (32, 40), (33, 40), (47, 50), (48, 50),
             (49, 60)]
    coords = [conformers(rng, 35, n) for _, n in cases]
    check(coords, [random_lists(rng, n, L, 2) for L, n in cases], prealigned)


def test_collinear_and_tiny_selections(cuda):
    """Rank-deficient covariances: selections on a line, and one-, two- and three-atom selections of rigid motions."""
    rng = np.random.default_rng(4)
    line = np.outer(rng.normal(size=9), [0.3, -0.8, 0.5])
    moves = lambda a, k: [a @ rotation(rng) + rng.normal(size=3) * 4.0 for _ in range(k)]  # noqa: E731
    coords = [moves(line, 6) + [line * 1.3], moves(rng.normal(size=(5, 3)), 6), moves(rng.normal(size=(5, 3)), 6)]
    lists = [(np.arange(9), np.stack([np.arange(9), np.arange(9)[::-1]])),
             (np.array([2]), np.array([[2], [4]])), (np.array([0, 3, 1]), np.array([[0, 3, 1], [3, 0, 1]]))]
    got = check(coords, lists)
    for m, k in enumerate([6, 6, 6]):
        assert max(got[m][i * (i - 1) // 2 + j] for i in range(k) for j in range(i)) <= 1e-5, m


@pytest.mark.parametrize("K", [1, 2, 7, 48])
def test_mapping_counts(cuda, K):
    rng = np.random.default_rng(10 + K)
    coords = [conformers(rng, c, n) for c, n in [(40, 20), (R + 3, 33), (3, 8)]]
    lists = [random_lists(rng, 20, 20, K), random_lists(rng, 33, 30, K), random_lists(rng, 8, 5, K)]
    for prealigned in (False, True):
        check(coords, lists, prealigned)


def methyl_mappings(n_methyl=4):
    """A core of 4 atoms and n methyls (C + 3 H): every rotation of each methyl's hydrogens (3^n), times the first 16
    permutations of the methyls among themselves (all of them for n <= 2): 81 x 16 = 1,296 mappings for n = 4."""
    n = 4 + 4 * n_methyl
    rots = list(itertools.product(range(3), repeat=n_methyl))  # 81
    perms = [p for p in itertools.permutations(range(n_methyl))][:16]  # 16
    qs = []
    for perm in perms:
        for rot in rots:
            q = list(range(4))
            for i in range(n_methyl):
                src = perm[i]
                base = 4 + 4 * src
                q += [base] + [base + 1 + (h + rot[i]) % 3 for h in range(3)]
            qs.append(q)
    return np.arange(n), np.array(qs)


def test_1296_mappings_next_to_one_and_to_short_molecules(cuda):
    rng = np.random.default_rng(20)
    p, q = methyl_mappings()
    assert len(q) == 1296 and len({tuple(x) for x in q}) == 1296
    n = len(p)
    coords = [conformers(rng, 45, n), conformers(rng, 33, 7), conformers(rng, 1, n), conformers(rng, 0, n),
              conformers(rng, 5, n)]
    lists = [(p, q), (np.arange(7), np.arange(7)[None]), (p, q[:3]), (p, q[:2]), (p, q[::100])]
    for prealigned in (False, True):
        check(coords, lists, prealigned)


@pytest.mark.parametrize("chunk", [1, 3, 5, 46])
def test_forced_chunks_split_K_unevenly(cuda, chunk):
    rng = np.random.default_rng(30)
    coords = [conformers(rng, c, n) for c, n in [(R + 5, 14), (9, 10), (40, 20)]]
    lists = [random_lists(rng, 14, 12, 11), random_lists(rng, 10, 10, 1), random_lists(rng, 20, 17, 47)]
    want = [check(coords, lists, pre) for pre in (False, True)]
    with _lib.options(rmsd_match_chunk=chunk):
        for pre, w in zip((False, True), want):
            got = mapped(coords, lists, pre)
            assert _lib.get_option("rmsd_match_chunks_last") == -(-47 // chunk)
            assert all(np.array_equal(g.view(np.int64), x.view(np.int64)) for g, x in zip(got, w)), (chunk, pre)


def test_orientation_independence_for_inverse_closed_lists(cuda):
    """A permutation group of mappings: swapping probe and reference (the transposed matrix) gives the same values."""
    rng = np.random.default_rng(40)
    p, q = methyl_mappings(2)
    group = {tuple(x) for x in q}
    assert all(tuple(np.argsort(x)) in group for x in q)  # closed under inversion
    c = 30
    coords = [conformers(rng, c, len(p))]
    fwd = mapped(coords, [(p, q)])[0]
    rev = mapped([coords[0][::-1]], [(p, q)])[0]  # conformer order reversed: every pair's roles swap
    sq_f, sq_r = np.zeros((c, c)), np.zeros((c, c))
    sq_f[np.tril_indices(c, -1)] = fwd
    sq_r[np.tril_indices(c, -1)] = rev
    sq_r = sq_r[::-1, ::-1].T
    assert np.abs(sq_f - sq_r)[np.tril_indices(c, -1)].max() <= 1e-10


def test_rigid_permuted_copy_is_zero_only_under_its_mapping(cuda):
    rng = np.random.default_rng(41)
    n = 10
    a = rng.normal(size=(n, 3)) * 1.5
    perm = rng.permutation(n)
    b = np.empty_like(a)
    b[perm] = a @ rotation(rng) + rng.normal(size=3) * 5.0  # atom k of a sits at perm[k] of b
    # conformer 1 = a (probe), conformer 0 = b (reference): mapping q[k] = perm[k]
    got = mapped([[b, a]], [(np.arange(n), np.stack([np.arange(n), perm]))])[0]
    plain = mapped([[b, a]], [(np.arange(n), np.arange(n)[None])])[0]
    assert got[0] <= 1e-6 and plain[0] > 0.1


def test_repeatable_batch_independent_and_on_any_stream(cuda):
    rng = np.random.default_rng(50)
    shapes = [(40, 20, 7), (70, 33, 48), (3, 5, 2), (65, 60, 3)]
    coords = [conformers(rng, c, n) for c, n, _ in shapes]
    lists = [random_lists(rng, n, n - 1, k) for _, n, k in shapes]
    a = mapped(coords, lists)
    b = mapped(coords, lists)
    s = torch.cuda.Stream()
    c = mapped(coords, lists, stream=s)
    for m in range(len(coords)):
        single = mapped([coords[m]], [lists[m]])[0]
        for x in (b[m], c[m], single):
            assert np.array_equal(a[m].view(np.int64), x.view(np.int64)), m


def test_public_functions_and_device_coordinates(cuda):
    """GetAllConformerBestRMS from self matches, from ``map`` and through a shuffled Device3DResult; atomIds."""
    rng = np.random.default_rng(60)
    n = 8
    coords = [conformers(rng, c, n) for c in (5, 0, 40, 1, 33)]
    # a 3-cycle without its inverse (as a maxMatches cut can leave): match t pairs probe atom q with reference atom t[q]
    matches = [tuple(range(n)), (1, 2, 0, 3, 4, 5, 7, 6), (0, 1, 2, 3, 4, 5, 7, 6), (1, 0, 2, 3, 4, 5, 6, 7)]
    mols = [StandIn(c, n, matches) for c in coords]
    want = oracle_best.molecules(coords, [(np.arange(n), np.array(matches))] * len(coords))
    host = cr.GetAllConformerBestRMSBatch(mols)
    for g, w in zip(host, want):
        assert_close(g.torch().cpu().numpy(), w)
    one = cr.GetAllConformerBestRMS(mols[2], map=[[(q, int(r)) for q, r in enumerate(m)] for m in matches])
    assert torch.equal(one.torch(), host[2].torch())
    entries = [(m, k, c) for m, confs in enumerate(coords) for k, c in enumerate(confs)]
    entries = [entries[i] for i in rng.permutation(len(entries))]
    t = lambda a: AsyncGpuResult(torch.as_tensor(np.asarray(a)).cuda())  # noqa: E731
    starts = np.concatenate([[0], np.cumsum([len(e[2]) for e in entries])]).astype(np.int32)
    res = Device3DResult(t(np.concatenate([e[2] for e in entries])), t(starts),
                         t(np.array([e[0] for e in entries], np.int32)), t(np.array([e[1] for e in entries], np.int32)),
                         0, len(mols))
    xyz_before = res.values.torch().clone()
    dev = cr.GetAllConformerBestRMSBatch(mols, coordinates=res)
    assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(host, dev))
    assert torch.equal(res.values.torch(), xyz_before)  # coordinates are not modified
    ids = [0, 2, 5, 7]
    sub = cr.GetConformerRMSMatrix(mols[2], atomIds=ids).torch().cpu().numpy()
    assert_close(sub, oracle_best.molecules([coords[2]], [(np.array(ids), np.array([ids]))])[0])
    batch = cr.GetConformerRMSMatrixBatch(mols, atomIds=[ids] * len(mols), coordinates=res)
    assert torch.equal(batch[2].torch(), cr.GetConformerRMSMatrix(mols[2], atomIds=ids).torch())
    for pre in (False, True):
        allat = cr.GetConformerRMSMatrixBatch(mols, pre, atomIds=[None] * len(mols))
        plain = cr.GetConformerRMSMatrixBatch(mols, pre)
        assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(allat, plain))


def test_matrix_agrees_with_rms_pruning(cuda):
    """Pruning keeps a conformer whose minimum RMSD over the lists to every kept earlier one is >= the threshold: a
    greedy walk over the mapped matrix, with P as pruning's list 0 and its lists as the Q_k (Q_1 = P)."""
    rng = np.random.default_rng(70)
    n, c = 12, 60
    coords = [conformers(rng, c, n, spread=0.5) for _ in range(3)]
    lists = [random_lists(rng, n, L, k) for L, k in [(12, 4), (9, 1), (10, 6)]]
    mats = mapped(coords, lists)
    vals = np.sort(np.concatenate(mats))
    gaps = [(a + b) / 2 for a, b in zip(vals[:-1], vals[1:]) if b - a > 2e-6]
    thresh = min(gaps, key=lambda t: abs(t - np.median(vals)))
    counts, atoms, xyz, cas = device_inputs(coords, [n] * len(coords))
    mcs = np.concatenate([[0], np.cumsum(counts)])
    keep = rms_prune(xyz, cas.cpu().numpy(), mcs, thresh, [np.asarray(q) for _, q in lists], atoms).cpu().numpy()
    for m in range(3):
        kept = []
        for i in range(c):
            if all(mats[m][i * (i - 1) // 2 + j] >= thresh for j in kept):
                kept.append(i)
        assert np.nonzero(keep[mcs[m]:mcs[m + 1]])[0].tolist() == kept, m


def test_a_molecule_without_atoms_or_conformers_next_to_one_with_pairs(cuda):
    """An empty molecule (no atoms, no conformers) in a batch with pairs: the plain, atomIds and best-RMS calls give it an
    empty result and the other molecule its oracle matrix."""
    from oracle import rmsd as oracle_rmsd

    rng = np.random.default_rng(80)
    n = 7
    coords = conformers(rng, 37, n)
    matches = [tuple(range(n)), (1, 0, 2, 3, 4, 5, 6)]
    mols = [StandIn(coords, n, matches), StandIn([], 0, [()]), StandIn(coords[:3], n, matches)]
    for pre in (False, True):
        plain = cr.GetConformerRMSMatrixBatch(mols, pre)
        ids = cr.GetConformerRMSMatrixBatch(mols, pre, atomIds=[[0, 2, 5], None, None])
        best = cr.GetAllConformerBestRMSBatch(mols, prealigned=pre)
        assert [r.torch().numel() for r in plain] == [666, 0, 3] == [r.torch().numel() for r in best]
        assert [r.torch().numel() for r in ids] == [666, 0, 3]
        assert_close(plain[0].torch().cpu().numpy(), oracle_rmsd.molecules([coords], pre)[0])
        assert_close(ids[0].torch().cpu().numpy(),
                     oracle_best.molecules([coords], [(np.array([0, 2, 5]), np.array([[0, 2, 5]]))], pre)[0])
        assert_close(best[0].torch().cpu().numpy(),
                     oracle_best.molecules([coords], [(np.arange(n), np.array(matches))], pre)[0])
        assert torch.equal(plain[2].torch(), cr.GetConformerRMSMatrix(mols[2], pre).torch())
