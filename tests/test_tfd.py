"""TFD torsion tables and the fp64 oracle on the CPU (fake RDKit): the reference's known answers replayed on hand-built
heavy-atom graphs, the option switches, the error contract of GetTFDMatrices, and the oracle's per-pair contract.

Known answers: nvMolKit v0.5.0 tests/test_tfd_cpu.cpp:52-167 (torsion lists), :173-205 (weights), :278-331 (butane).
Atoms and bonds follow RDKit's SMILES parse order; hydrogens are implicit, as in a molecule from SMILES."""
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import tfd as oracle_tfd
from nvmolkit_b200 import synthetic as S
from nvmolkit_b200 import tfd
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult

FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rdkit_tfd.npz")


@pytest.fixture
def Chem(monkeypatch):
    monkeypatch.syspath_prepend(FAKE)
    for name in [m for m in sys.modules if m in ("rdkit", "tfd_molecules") or m.startswith("rdkit.")]:
        monkeypatch.delitem(sys.modules, name)
    import rdkit
    import tfd_molecules
    from rdkit import Chem as chem

    assert rdkit.__file__.startswith(FAKE)
    yield types.SimpleNamespace(Mol=tfd_molecules.Mol, BondType=chem.BondType)
    for name in [m for m in sys.modules if m in ("rdkit", "tfd_molecules") or m.startswith("rdkit.")]:
        sys.modules.pop(name, None)


@pytest.fixture
def legacy_rdkit(Chem, monkeypatch):
    """The fake announcing an RDKit older than 2026.03.1 (the _calculateBeta rule of the reference's known answers)."""
    import rdkit

    monkeypatch.setattr(rdkit, "__version__", "2025.09.3", raising=False)
    return Chem


_VALENCE = {6: 4, 7: 3, 8: 2}


def make_mol(Chem, z, bonds, rings=(), orders=None, conformers=()):
    """Heavy-atom graph; `orders` maps bond index -> 2 / 3 / 1.5; hydrogens implicit (valence minus bond orders)."""
    n = len(z)
    nbrs = [[] for _ in range(n)]
    for i, j in bonds:
        nbrs[i].append(j)
        nbrs[j].append(i)
    orders = orders or {}
    kind = {1: Chem.BondType.SINGLE, 2: Chem.BondType.DOUBLE, 3: Chem.BondType.TRIPLE, 1.5: Chem.BondType.AROMATIC}
    types = [kind[orders.get(k, 1)] for k in range(len(bonds))]
    used = [0.0] * n
    for k, (i, j) in enumerate(bonds):
        used[i] += orders.get(k, 1)
        used[j] += orders.get(k, 1)
    hs = [max(0, int(round(_VALENCE[int(a)] - u))) for a, u in zip(z, used)]
    d = {"z": np.array(z), "bonds": list(bonds), "nbrs": nbrs, "topo": S._topological_distances(n, nbrs), "implicit_hs": hs}
    return Chem.Mol(d, conformers=conformers, rings=rings, bond_types=types)


def chain(Chem, n, **kw):
    return make_mol(Chem, [6] * n, [(i, i + 1) for i in range(n - 1)], **kw)


def benzene(Chem, **kw):
    return make_mol(Chem, [6] * 6, [(0, 1), (1, 2), (2, 3), (3, 4), (4, 5), (0, 5)], rings=[(0, 5, 4, 3, 2, 1)],
                    orders={k: 1.5 for k in range(6)}, **kw)


def cyclohexyl(Chem):  # CC(=O)[C@H]1CCCC[C@@H]1CN
    bonds = [(0, 1), (1, 2), (1, 3), (3, 4), (4, 5), (5, 6), (6, 7), (7, 8), (3, 8), (8, 9), (9, 10)]
    return make_mol(Chem, [6, 6, 8, 6, 6, 6, 6, 6, 6, 6, 7], bonds, rings=[(3, 8, 7, 6, 5, 4)], orders={1: 2})


def cyclopropyl(Chem):  # C[C@@H](CN(C)C(=O)C#CCN)C1CC1
    bonds = [(0, 1), (1, 2), (2, 3), (3, 4), (3, 5), (5, 6), (5, 7), (7, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13),
             (11, 13)]
    return make_mol(Chem, [6, 6, 6, 7, 6, 6, 8, 6, 6, 6, 7, 6, 6, 6], bonds, rings=[(11, 12, 13)], orders={5: 2, 7: 3})


def quartets(tors, m=0):
    return [t[0] for t in tors.molecule(m)]


# ----------------------------------------------------------------------------------------------- torsion lists
def test_chain_torsion_lists(Chem):
    """tests/test_tfd_cpu.cpp:56-101: CCCC, CCCCC, CCCCCC."""
    for n, want in ((4, [[(0, 1, 2, 3)]]), (5, [[(0, 1, 2, 3)], [(1, 2, 3, 4)]]),
                    (6, [[(0, 1, 2, 3)], [(1, 2, 3, 4)], [(2, 3, 4, 5)]])):
        t = tfd.tfd_torsions([chain(Chem, n)])
        assert quartets(t) == want
        assert all(x[1] == tfd.SINGLE and x[3] == 180.0 for x in t.molecule(0))


def test_benzene_is_one_ring_torsion(Chem):
    """:103-126: one ring torsion of 6 quartets in ring order, maxDev 180 exp(-0.025 * 64) = 36.34."""
    t = tfd.tfd_torsions([benzene(Chem)])
    (q, typ, _w, md), = t.molecule(0)
    assert typ == tfd.RING and abs(md - 36.34) < 0.01
    assert q == [(0, 5, 4, 3), (5, 4, 3, 2), (4, 3, 2, 1), (3, 2, 1, 0), (2, 1, 0, 5), (1, 0, 5, 4)]


def test_cyclohexyl_torsions(Chem):
    """:128-145: two non-ring torsions {0,1,3,4}, {3,8,9,10} (both by the smallest-invariant fallback on one side) and
    the ring {3,8,7,6} ... {4,3,8,7}, maxDev 36.34. The fallback picks depend on the invariants' hash values; these
    are the repository's Morgan restatement's, and they reproduce the reference's picks."""
    t = tfd.tfd_torsions([cyclohexyl(Chem)])
    mol = t.molecule(0)
    assert [x[0] for x in mol[:2]] == [[(0, 1, 3, 4)], [(3, 8, 9, 10)]]
    ring = mol[2]
    assert ring[1] == tfd.RING and len(ring[0]) == 6 and abs(ring[3] - 36.34) < 0.01
    assert ring[0][0] == (3, 8, 7, 6) and ring[0][5] == (4, 3, 8, 7)


def test_cyclopropyl_torsions_and_colinear_skip(Chem):
    """:147-166: {0,1,2,3}, {1,2,3,4}, {4,3,5,7}, the symmetric pair {0,1,11,12} / {0,1,11,13}; the bonds at C#C carry no
    torsion; the 3-ring has maxDev 180 exp(-0.025 * 121) = 8.74."""
    t = tfd.tfd_torsions([cyclopropyl(Chem)])
    mol = t.molecule(0)
    assert [x[0] for x in mol[:3]] == [[(0, 1, 2, 3)], [(1, 2, 3, 4)], [(4, 3, 5, 7)]]
    assert mol[3][0] == [(0, 1, 11, 12), (0, 1, 11, 13)] and mol[3][1] == tfd.SYMMETRIC
    assert mol[4][1] == tfd.RING and len(mol[4][0]) == 3 and abs(mol[4][3] - 8.74) < 0.01
    assert len(mol) == 5


def test_symmetry_radius_zero_uses_degree(Chem):
    t = tfd.tfd_torsions([cyclopropyl(Chem)], symmRadius=0)
    assert t.molecule(0)[3][0] == [(0, 1, 11, 12), (0, 1, 11, 13)]  # 12 and 13 both have degree 2


# ---------------------------------------------------------------------------------------------------- weights
WEIGHTS = [  # tests/test_tfd_cpu.cpp:183-189
    (lambda C: chain(C, 4), [1.0]),
    (lambda C: chain(C, 5), [1.0, 0.1]),
    (lambda C: chain(C, 6), [0.1, 1.0, 0.1]),
    (cyclohexyl, [0.3593813664, 0.3593813664, 0.1748047999]),
    (cyclopropyl, [0.5623413252, 1.0, 0.5623413252, 0.1, 0.0025021508]),
]


@pytest.mark.parametrize("case", range(len(WEIGHTS)))
def test_weights_known_answers_with_the_older_beta_rule(legacy_rdkit, case):
    build, want = WEIGHTS[case]
    w = tfd.tfd_torsions([build(legacy_rdkit)]).weight
    assert np.abs(w - np.array(want)).max() < 5e-4, w


def test_newer_beta_rule_counts_only_bonds_of_two_non_terminal_atoms(Chem):
    """RDKit 2026.03.1 tests both ends: for CCCCC dmax = 1 (not 2), beta = 4 ln 10, the end torsion weighs 1e-4."""
    assert tfd._legacy_beta_rule() is False
    w = tfd.tfd_torsions([chain(Chem, 5)]).weight
    assert abs(w[0] - 1.0) < 1e-12 and abs(w[1] - 1e-4) < 1e-12


def test_unweighted_tables_have_unit_weights(legacy_rdkit):
    t = tfd.tfd_torsions([cyclopropyl(legacy_rdkit)], useWeights=False)
    assert (t.weight == 1.0).all()


# ---------------------------------------------------------------------------------------------------- options
def test_spec_and_equal(Chem):
    """Ring-only molecules: identical tables; CC(C)CC: the symmetric torsion's maxDev becomes 90 (one side is a single
    neighbour, the other two symmetric ones)."""
    a, b = tfd.tfd_torsions([benzene(Chem)], maxDev="equal"), tfd.tfd_torsions([benzene(Chem)], maxDev="spec")
    assert a.molecule(0) == b.molecule(0)
    iso = lambda: make_mol(Chem, [6] * 5, [(0, 1), (1, 2), (1, 3), (3, 4)])  # noqa: E731
    e, s = tfd.tfd_torsions([iso()], maxDev="equal"), tfd.tfd_torsions([iso()], maxDev="spec")
    assert quartets(e) == [[(0, 1, 3, 4), (2, 1, 3, 4)]] and e.type[0] == tfd.SYMMETRIC
    assert e.maxdev[0] == 180.0 and s.maxdev[0] == 90.0


def test_colinear_bonds_walk_the_chain(Chem):
    """CCCC#CCC: with ignoreColinearBonds=True only 1-2 carries a torsion (the bonds at the C#C ends do not); with False
    the bond 2-3 walks across the triple bond to the middle atoms 2 and 5, which adds the torsion (1, 2, 5, 6)."""
    mk = lambda: make_mol(Chem, [6] * 7, [(i, i + 1) for i in range(6)], orders={3: 3})  # noqa: E731
    on, off = tfd.tfd_torsions([mk()]), tfd.tfd_torsions([mk()], ignoreColinearBonds=False)
    assert quartets(on) == [[(0, 1, 2, 3)]]
    assert len(off.type) >= len(on.type)
    assert quartets(off) == [[(0, 1, 2, 3)], [(1, 2, 5, 6)]]


# ---------------------------------------------------------------------------------------------------- errors
def test_error_contract(Chem):
    butane = chain(Chem, 4, conformers=[np.zeros((4, 3))] * 2)
    with pytest.raises(ValueError):
        tfd.GetTFDMatrices([butane], maxDev="max")
    with pytest.raises(ValueError):
        tfd.GetTFDMatrices([butane], return_type="dict")
    with pytest.raises(ValueError):
        tfd.GetTFDMatrices([chain(Chem, 4)])  # no conformers
    with pytest.raises(ValueError):
        tfd.GetTFDMatrices([None])
    class Big:  # only the atom count is read before the refusal
        def GetNumAtoms(self):
            return 32768

    with pytest.raises(ValueError):
        tfd.tfd_torsions([Big()])
    with pytest.raises(ValueError):
        tfd.GetTFDMatrices([Big()])
    t = lambda a: AsyncGpuResult(torch.as_tensor(a))  # noqa: E731  (host tensors: validation happens before the device)
    two = Device3DResult(t(np.zeros((8, 3))), t(np.array([0, 4, 8], np.int32)), t(np.array([0, 0], np.int32)),
                         t(np.array([0, 1], np.int32)), 0, 2)
    with pytest.raises(ValueError):  # molecule count
        tfd.GetTFDMatrices([butane], coordinates=two)
    wrong = Device3DResult(t(np.zeros((10, 3))), t(np.array([0, 5, 10], np.int32)), t(np.array([0, 0], np.int32)),
                           t(np.array([0, 1], np.int32)), 0, 1)
    with pytest.raises(ValueError):  # atom count
        tfd.GetTFDMatrices([butane], coordinates=wrong)
    tors = tfd.TFDTorsions.from_lists([[([(0, 1, 2, 9)], tfd.SINGLE, 1.0, 180.0)]])
    flat = tfd.FlatTFDMolecules.from_coordinates(tors, [[np.zeros((4, 3))] * 2])
    with pytest.raises(ValueError):  # quartet outside the molecule
        tfd.GetTFDMatrices(flat)
    with pytest.raises(ValueError):
        tfd.TFDTorsions(np.array([0, 1]), np.array([0, 1]), np.zeros((1, 4)), np.array([0]), np.array([1.0]), np.array([]))


# ---------------------------------------------------------------------------------------------------- oracle pins
def oracle_one(torsions, confs):
    flat = tfd.FlatTFDMolecules.from_coordinates(torsions, [confs])
    t = flat.torsions
    return oracle_tfd.matrices(flat.mol_conf_start, flat.conf_atom_start, flat.xyz, t.tors_start, t.quartet_start,
                               t.quartets, t.type, t.weight, t.maxdev)[0]


def butane(phi_deg, r=1.5):
    """C0 at +x from C1, C1-C2 along +y, C3 rotated by phi about the bond (phi = 0: C0 and C3 on the same side)."""
    p = math.radians(phi_deg)
    return np.array([[1.0, 0, 0], [0, 0, 0], [0, r, 0], [math.cos(p), r, -math.sin(p)]])


def test_oracle_butane_known_answer(Chem):
    """tests/test_tfd_cpu.cpp:278-331: the two hand-set butane conformers differ by 120 degrees -> TFD 0.667."""
    t = tfd.tfd_torsions([chain(Chem, 4)], useWeights=False)
    c0 = np.array([[1.0, 0, 0], [0, 0, 0], [0, 1.5, 0], [1.0, 1.5, 0]])
    c1 = np.array([[1.0, 0, 0], [0, 0, 0], [0, 1.5, 0], [-0.5, 1.5, 0.866]])
    out = oracle_one(t, [c0, c1])
    assert out.shape == (1,) and abs(out[0] - 0.667) < 0.05 and abs(out[0] - 120.0 / 180.0) < 1e-4


def test_oracle_dihedral_convention():
    assert abs(oracle_tfd.dihedral(*butane(60.0)) - 60.0) < 1e-9
    assert abs(oracle_tfd.dihedral(*butane(-60.0)) + 60.0) < 1e-9
    assert oracle_tfd.dihedral(*butane(180.0)) == 180.0 or abs(oracle_tfd.dihedral(*butane(180.0)) - 180.0) < 1e-9
    collinear = np.array([[0.0, 0, 0], [1.0, 0, 0], [2.0, 0, 0], [2.0, 1.0, 0]])
    assert oracle_tfd.dihedral(*collinear) == 0.0  # exactly zero cross product


SINGLE_T = tfd.TFDTorsions.from_lists([[([(0, 1, 2, 3)], tfd.SINGLE, 1.0, 180.0)]])


def test_oracle_identical_and_mirror_conformers():
    out = oracle_one(SINGLE_T, [butane(37.0), butane(37.0), butane(-37.0), butane(179.0), butane(-179.0)])
    assert out[0] == 0.0  # (1, 0) identical
    assert abs(out[1] - 74.0 / 180) < 1e-12 and abs(out[2] - 74.0 / 180) < 1e-12  # (2, 0), (2, 1): phi against -phi
    assert abs(out[9] - 2.0 / 180) < 1e-12  # (4, 3): 179 against -179 across the wrap


def test_oracle_ring_average_and_symmetric_minimum_and_scaling():
    # ring over the two quartets (0,1,2,3) and (3,2,1,0): mean |phi| only
    ring = tfd.TFDTorsions.from_lists([[([(0, 1, 2, 3), (3, 2, 1, 0)], tfd.RING, 1.0, 36.0)]])
    out = oracle_one(ring, [butane(50.0), butane(-80.0)])
    assert abs(out[0] - 30.0 / 36.0) < 1e-12  # |50 - 80| / 36, the sign does not count
    # symmetric: quartets (0,1,2,3) and (0,1,2,4); conformer 1 swaps atoms 3 and 4 -> minimum 0
    a = np.vstack([butane(60.0), butane(-60.0)[3:]])
    b = np.vstack([butane(-60.0), butane(60.0)[3:]])
    sym = tfd.TFDTorsions.from_lists([[([(0, 1, 2, 3), (0, 1, 2, 4)], tfd.SYMMETRIC, 1.0, 90.0)]])
    assert oracle_one(sym, [a, b])[0] == 0.0
    c = np.vstack([butane(90.0), butane(-150.0)[3:]])
    assert abs(oracle_one(sym, [a, c])[0] - 30.0 / 90.0) < 1e-12  # min over the four pairs: |60 - 90|
    # maxDev scaling and the weighted mean
    two = tfd.TFDTorsions.from_lists([[([(0, 1, 2, 3)], tfd.SINGLE, 3.0, 180.0), ([(3, 2, 1, 0)], tfd.SINGLE, 1.0, 60.0)]])
    out = oracle_one(two, [butane(10.0), butane(40.0)])
    assert abs(out[0] - (3.0 * 30 / 180 + 1.0 * 30 / 60) / 4.0) < 1e-12


def test_oracle_zero_weights_and_no_torsions_give_zero():
    zero = tfd.TFDTorsions.from_lists([[([(0, 1, 2, 3)], tfd.SINGLE, 0.0, 180.0)]])
    assert (oracle_one(zero, [butane(0.0), butane(90.0)]) == 0.0).all()
    none = tfd.TFDTorsions.from_lists([[]])
    assert (oracle_one(none, [butane(0.0), butane(90.0), butane(30.0)]) == 0.0).all()


# ---------------------------------------------------------------------------------------------------- RDKit parity
@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="tests/golden/rdkit_tfd.npz not exported (tools/export_rdkit_fixtures.py)")
def test_oracle_equals_rdkit_tfd_matrices():
    """RDKit's own torsion lists, weights and GetTFDMatrix on ETKDG conformers: the exported tables through the oracle
    reproduce the matrices."""
    fx = np.load(GOLDEN)
    out = oracle_tfd.matrices(fx["mol_conf_start"], fx["conf_atom_start"], fx["xyz"], fx["tors_start"],
                              fx["quartet_start"], fx["quartets"], fx["type"], fx["weight"], fx["maxdev"])
    want = np.split(fx["tfd"], np.cumsum(fx["tfd_sizes"])[:-1])
    for m, (got, ref) in enumerate(zip(out, want)):
        assert np.abs(got - ref).max(initial=0.0) < 1e-4, m


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="tests/golden/rdkit_tfd.npz not exported (tools/export_rdkit_fixtures.py)")
def test_adapter_tables_equal_rdkit_torsion_lists():
    """tfd_torsions run against the exporting RDKit builds RDKit's own torsion lists, maxDevs and weights."""
    fx = np.load(GOLDEN)
    for k in ("tors_start", "quartet_start", "quartets", "type"):
        assert np.array_equal(fx[f"adapter_{k}"], fx[k]), k
    assert np.abs(fx["adapter_maxdev"] - fx["maxdev"]).max(initial=0.0) < 1e-6
    assert np.abs(fx["adapter_weight"] - fx["weight"]).max(initial=0.0) < 1e-6
