"""Pins the CPU oracle against the known answers the reference's own tests hold for path A (SURVEY.md §8c)."""

import numpy as np

import oracle
from nvmolkit_b200 import synthetic as S
from nvmolkit_b200.molgraph import atom_invariant

SINGLE, DOUBLE = 1, 2


def _sizes(atom_inv, bonds, types):
    ba = [b[0] for b in bonds]
    bb = [b[1] for b in bonds]
    return [len(set(oracle.morgan_codes(atom_inv, types, ba, bb, r).tolist())) for r in range(4)]


def test_morgan_sparse_sizes_pentane():
    # tests/test_morgan_fingerprint_ref.cpp:46-56 ("CCCCC" -> {2, 5, 7, 7}), values from RDKit's testMorganFP()
    t, m = atom_invariant(6, 4, 3, 0, 0, False), atom_invariant(6, 4, 2, 0, 0, False)
    assert _sizes([t, m, m, m, t], [(0, 1), (1, 2), (2, 3), (3, 4)], [SINGLE] * 4) == [2, 5, 7, 7]


def _cyclopropyl_acetic(order):
    # O=C(O)CC1CC1 : atoms 0 O=, 1 C, 2 OH, 3 CH2, 4 CH(ring), 5 CH2(ring), 6 CH2(ring)
    inv = [atom_invariant(8, 1, 0, 0, 0, False), atom_invariant(6, 3, 0, 0, 0, False),
           atom_invariant(8, 2, 1, 0, 0, False), atom_invariant(6, 4, 2, 0, 0, False),
           atom_invariant(6, 4, 1, 0, 0, True), atom_invariant(6, 4, 2, 0, 0, True),
           atom_invariant(6, 4, 2, 0, 0, True)]
    bonds = [(0, 1, DOUBLE), (1, 2, SINGLE), (1, 3, SINGLE), (3, 4, SINGLE), (4, 5, SINGLE), (5, 6, SINGLE),
             (6, 4, SINGLE)]
    pos = {a: i for i, a in enumerate(order)}
    inv2 = [inv[a] for a in order]
    b2 = [(pos[u], pos[v]) for u, v, _ in bonds]
    return inv2, b2, [t for _, _, t in bonds]


def test_morgan_sparse_sizes_cyclopropylacetic_and_atom_order_invariance():
    # tests/test_morgan_fingerprint_ref.cpp:46-56: "O=C(O)CC1CC1" and "OC(=O)CC1CC1" -> {6, 12, 16, 17}
    for order in ([0, 1, 2, 3, 4, 5, 6], [2, 1, 0, 3, 4, 5, 6]):
        inv, bonds, types = _cyclopropyl_acetic(order)
        assert _sizes(inv, bonds, types) == [6, 12, 16, 17]


def test_morgan_symmetry_butanediol():
    # tests/test_morgan_fingerprint_ref.cpp:58-67: "OCCCCO" radius 2 -> 7 distinct codes, each count in {2, 4}
    o, c = atom_invariant(8, 2, 1, 0, 0, False), atom_invariant(6, 4, 2, 0, 0, False)
    codes = oracle.morgan_codes([o, c, c, c, c, o], [SINGLE] * 5, [0, 1, 2, 3, 4], [1, 2, 3, 4, 5], 2)
    vals, counts = np.unique(codes, return_counts=True)
    assert len(vals) == 7
    assert set(counts.tolist()) <= {2, 4}


def test_python_atom_invariant_equals_c():
    for args in [(6, 4, 3, 0, 0, False), (7, 3, 1, 1, 0, True), (8, 1, 0, -1, 2, False), (35, 1, 0, 0, -1, True)]:
        assert atom_invariant(*args) == oracle.morgan_atom_invariant(*args)


def test_butina_known_answer_centroids():
    # tests/test_butina.cpp:241-273: 10 points, cutoff 0.1 -> {0,1,2,3} c0, {4,5,6} c4, three singletons
    d = np.ones((10, 10))
    np.fill_diagonal(d, 0.0)
    for j in (1, 2, 3):
        d[0, j] = d[j, 0] = 0.05
    for j in (5, 6):
        d[4, j] = d[j, 4] = 0.05
    ids, cen = oracle.butina_dense(d, 0.1)
    assert len(cen) == 5
    assert sorted(np.nonzero(ids == 0)[0].tolist()) == [0, 1, 2, 3] and cen[0] == 0
    assert sorted(np.nonzero(ids == 1)[0].tolist()) == [4, 5, 6] and cen[1] == 4
    for c in range(2, 5):
        members = np.nonzero(ids == c)[0]
        assert len(members) == 1 and cen[c] == members[0]
    # singletons in descending index order (RDKit sorts (count, idx) tuples in reverse)
    assert cen[2:].tolist() == [9, 8, 7]


def test_butina_all_far_gives_singletons():
    # tests/test_butina.cpp:219-237
    d = np.ones((17, 17))
    np.fill_diagonal(d, 0.0)
    ids, cen = oracle.butina_dense(d, 0.1)
    assert sorted(ids.tolist()) == list(range(17)) and len(cen) == 17


def _greedy_check(ids, cen, adj):
    """nvmolkit/tests/test_clustering.py:23-51: each cluster's size equals the max available neighbour count."""
    n = len(ids)
    free = np.ones(n, dtype=bool)
    for c, centre in enumerate(cen):
        members = np.nonzero(ids == c)[0]
        counts = (adj & free[None, :]).sum(1)
        counts[~free] = -1
        assert counts[centre] == counts.max()
        assert len(members) == counts[centre] + 1
        assert adj[centre, members[members != centre]].all()
        free[members] = False
    assert not free.any()


def test_butina_fp_structural_and_greedy():
    fp = S.clustered_fingerprints(30, 20, seed=7)
    sim = oracle.similarity_cross(fp)
    adj = (1.0 - sim) <= 0.3
    np.fill_diagonal(adj, False)
    ids, cen = oracle.butina_fp(fp, 0.3)
    _greedy_check(ids, cen, adj)
    sizes = np.bincount(ids)
    assert (np.diff(sizes) <= 0).all()
    ids2, cen2 = oracle.butina_dense(1.0 - sim, 0.3)
    assert (ids == ids2).all() and (cen == cen2).all()


def test_tanimoto_definition():
    a = np.array([[0b1011, 0], [0, 0]], dtype=np.uint32)
    b = np.array([[0b0011, 1], [0, 0], [0b0100, 0]], dtype=np.uint32)
    s = oracle.similarity_cross(a, b)
    assert s[0, 0] == 2 / 4 and s[0, 1] == 0.0 and s[0, 2] == 0.0 and s[1, 1] == 0.0
    c = oracle.similarity_cross(a, b, metric="cosine")
    assert c[0, 0] == 2 / np.sqrt(3 * 3)


def test_count_ge_matches_matrix():
    x = S.random_fingerprints(97, seed=3, near_dups=20)
    y = S.random_fingerprints(55, seed=4, near_dups=10)
    y[:10] = x[:10]
    for metric in ("tanimoto", "cosine"):
        sim = oracle.similarity_cross(x, y, metric=metric)
        want = ((1.0 - sim) <= 0.35).sum(1)
        assert (oracle.count_ge(x, y, 0.35, metric=metric) == want).all()


def test_reciprocal_newton_quotient_is_correctly_rounded():
    """The tensor tile's fp64 epilogue computes c/u as fma(fma(-q0,u,c), r, q0) with r = RN(1/u), q0 = RN(c*r).
    The oracle runs that formula in C (libm fma) on every pair 1 <= c <= u <= 8192, the range of 4096-bit fingerprints,
    and counts where it differs from the correctly rounded c / u: never. Without the Newton step the same check finds
    mismatches, so it is able to see one. A Python restatement pins the C loop on a sample."""
    from fractions import Fraction

    assert oracle.recip_quotient_mismatches(8192) == 0
    assert oracle.recip_quotient_mismatches(8192, newton=False) > 0

    rng = np.random.default_rng(0)
    us = np.concatenate([np.arange(1, 300), rng.integers(300, 8193, size=700)])
    for u in us.tolist():
        r = 1.0 / u
        for c in (1, u // 3 + 1, u // 2 + 1, u - 1 if u > 1 else 1, u):
            q = c * r
            rem = float(Fraction(c) - Fraction(q) * u)  # exactly representable (|rem| tiny, fma semantics)
            q1 = float(Fraction(q) + Fraction(rem) * Fraction(r))  # round-to-nearest of the exact sum = fma result
            assert q1 == c / u, (c, u)
