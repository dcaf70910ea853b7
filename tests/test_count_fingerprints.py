"""Morgan count fingerprints without a GPU: the count oracle (oracle.morgan_codes folded with bincount) against the
restatement of RDKit's environment walk in test_morgan.py on its graph families, against the bit oracle, on RDKit's
known answers, and every refusal of the generator and the C-ABI. RDKit's own counts are replayed when
tests/golden/rdkit_fixtures.npz holds them."""

import collections
import ctypes as C
import os

import numpy as np
import pytest

import oracle
import test_morgan as M
from oracle import count as oracle_count
from nvmolkit_b200.molgraph import atom_invariant

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rdkit_fixtures.npz")
SINGLE = 1


def counts_of(g, radius, bits):
    return oracle_count.morgan_counts(g.atom_starts, g.bond_starts, g.atom_inv, g.bond_inv, g.bond_a, g.bond_b, radius,
                                      bits)


def _restated(mols, radius, bits):
    out = np.zeros((len(mols), bits), dtype=np.int32)
    for i, m in enumerate(mols):
        for code, n in collections.Counter(c % bits for c in M.morgan_codes_py(m, radius)).items():
            out[i, code] = n
    return out


@pytest.mark.parametrize("family", sorted(M.FAMILIES))
@pytest.mark.parametrize("radius", [0, 1, 2, 4])
def test_count_oracle_equals_the_restatement_and_its_bits_the_bit_oracle(family, radius):
    mols = M.FAMILIES[family]()
    g = M.batch(mols)
    for bits in (128, 2048):
        got = counts_of(g, radius, bits)
        assert np.array_equal(got, _restated(mols, radius, bits))
        packed = np.packbits(got > 0, axis=1, bitorder="little").view(np.uint32)
        assert np.array_equal(packed, M.want(g, radius, bits))


def test_every_atom_counts_at_radius_zero():
    g = M.batch(M.fragment_family())
    got = counts_of(g, 0, 2048)
    assert np.array_equal(got.sum(axis=1), g.atoms_per_mol)


def test_known_answers():
    # "OCCCCO" at radius 2: 7 distinct codes, each counted 2 or 4 times (RDKit's testMorganFP)
    o, c = atom_invariant(8, 2, 1, 0, 0, False), atom_invariant(6, 4, 2, 0, 0, False)
    mol = M.Mol(6, [(i, i + 1) for i in range(5)], [o, c, c, c, c, o], [SINGLE] * 5)
    got = counts_of(M.batch([mol]), 2, 2048)[0]
    assert np.count_nonzero(got) == 7 and set(got[got > 0].tolist()) <= {2, 4}
    # "CCCCC": 2, 5, 7 and 7 environments at radius 0, 1, 2 and 3
    t, m = atom_invariant(6, 4, 3, 0, 0, False), atom_invariant(6, 4, 2, 0, 0, False)
    mol = M.Mol(5, [(i, i + 1) for i in range(4)], [t, m, m, m, t], [SINGLE] * 4)
    sizes = [np.count_nonzero(counts_of(M.batch([mol]), r, 2048)[0]) for r in range(4)]
    assert sizes == [2, 5, 7, 7]
    assert counts_of(M.batch([mol]), 0, 2048)[0].sum() == 5


def test_generator_refuses_widths_and_radius_before_device_work():
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    for bits in (0, 64, 4096, 3000):
        with pytest.raises(ValueError):
            MorganFingerprintGenerator(2, bits)
    with pytest.raises(ValueError):
        MorganFingerprintGenerator(-1, 2048)


def test_the_library_refuses_counts_arguments(built_lib):
    L = built_lib
    L.b200mol_morgan_counts.restype = C.c_int
    args = lambda radius, bits, out=16: (16, 16, 16, 16, 16, 16, 3, 10, 10, radius, bits, out, None)  # noqa: E731
    for radius, bits, msg in ((2, 0, b"fpBits"), (2, 48, b"fpBits"), (-1, 2048, b"radius"), (17, 2048, b"radius")):
        assert L.b200mol_morgan_counts(*args(radius, bits)) == 1
        assert msg in L.b200mol_last_error()
    assert L.b200mol_morgan_counts(*args(2, 2048, None)) == 1 and b"null" in L.b200mol_last_error()
    assert L.b200mol_morgan_counts(16, 16, 16, 16, 16, 16, 3, 65536, 10, 2, 2048, 16, None) == 1
    assert L.b200mol_morgan_counts(None, None, None, None, None, None, 0, 10, 10, 2, 2048, None, None) == 0  # nothing to do


@pytest.mark.skipif(not os.path.exists(FIXTURES), reason="no RDKit-exported fixtures (tools/export_rdkit_fixtures.py)")
def test_count_oracle_equals_rdkit():
    fx = np.load(FIXTURES, allow_pickle=False)
    if "morgan_counts_r0" not in fx:
        pytest.skip("the fixtures predate the count fingerprints")
    g = [fx[f"graph_{k}"] for k in ("atom_starts", "bond_starts", "atom_inv", "bond_inv", "bond_a", "bond_b")]
    for r in range(4):
        assert np.array_equal(oracle_count.morgan_counts(*g, r, 2048), fx[f"morgan_counts_r{r}"]), f"radius {r}"
