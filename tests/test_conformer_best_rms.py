"""Symmetry-aware conformer RMSD matrices on the CPU: the mapped fp64 oracle (oracle_best_rms.c) against a NumPy SVD
Kabsch minimum over the mappings, the mapping tables built from ``map``, ``atomIds`` and a molecule's self matches
(``maxMatches`` and the conjugated-terminal-group restatement), every argument refusal before device work, the C-ABI's
table checks without a device, and the "rmsd_match_chunk" option."""
import os
import re

import numpy as np
import pytest

from nvmolkit_b200 import _lib
from nvmolkit_b200 import conformerRmsd as cr
from nvmolkit_b200.rdkit_adapter import self_matches
from oracle import best_rms as oracle_best

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def kabsch_rmsd(p, q):
    p = p - p.mean(0)
    q = q - q.mean(0)
    u, s, vt = np.linalg.svd(p.T @ q)
    d = np.sign(np.linalg.det(p.T @ q))
    s[-1] *= d if d != 0.0 else 1.0
    return np.sqrt(max(((p * p).sum() + (q * q).sum() - 2.0 * s.sum()) / len(p), 0.0))


def rotation(rng):
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1.0
    return q


# ------------------------------------------------------------------ stand-in molecules
class Atom:
    def __init__(self, mol, i):
        self.mol, self.i = mol, i

    def GetIdx(self):
        return self.i

    def GetAtomicNum(self):
        return self.mol.z[self.i]

    def GetDegree(self):
        return sum(self.i in b[:2] for b in self.mol.bonds)

    def GetBonds(self):
        return [Bond(self.mol, b) for b in self.mol.bonds if self.i in b[:2]]


class Bond:
    def __init__(self, mol, b):
        self.b = b

    def GetOtherAtomIdx(self, i):
        return self.b[1] if self.b[0] == i else self.b[0]

    def GetIsConjugated(self):
        return self.b[2]


class StandIn:
    """Atoms, bonds (a, b, conjugated), conformers and the list of self matches its GetSubstructMatches returns."""

    def __init__(self, z, bonds, matches, coords=()):
        self.z, self.bonds, self.matches, self.coords = list(z), list(bonds), list(matches), list(coords)
        self.calls = []

    def GetNumAtoms(self):
        return len(self.z)

    def GetAtoms(self):
        return [Atom(self, i) for i in range(len(self.z))]

    def GetAtomWithIdx(self, i):
        return Atom(self, i)

    def GetConformers(self):
        raise AssertionError("conformers read before the arguments were checked")

    def GetSubstructMatches(self, query, uniquify=True, maxMatches=1000, useChirality=True):
        self.calls.append((query is self, uniquify, maxMatches, useChirality))
        return self.matches[:maxMatches]


def acetate():
    """CH3-C(=O)O-: atoms C0 (methyl), C1, O2, O3; the two C-O bonds conjugated; the query's own match only."""
    return StandIn([6, 6, 8, 8], [(0, 1, False), (1, 2, True), (1, 3, True)], [(0, 1, 2, 3)])


def nitro_ester():
    """A nitro group N1(O2)(O3) on C0, and an ester-like O4 on C0 with a conjugated bond: O4 is alone on C0."""
    return StandIn([6, 7, 8, 8, 8], [(0, 1, False), (1, 2, True), (1, 3, True), (0, 4, True)], [(0, 1, 2, 3, 4)])


# ------------------------------------------------------------------ oracle
@pytest.mark.parametrize("L,K", [(1, 3), (3, 2), (8, 5), (30, 4)])
def test_oracle_is_the_kabsch_minimum_over_the_mappings(L, K):
    rng = np.random.default_rng(L * 10 + K)
    n = max(L, 4) + 2
    confs = [rng.normal(size=(n, 3)) * 2.0 + rng.normal(size=3) * 20.0 for _ in range(9)]
    p = rng.choice(n, L, replace=False)
    q = np.stack([rng.choice(n, L, replace=False) for _ in range(K)])
    got = oracle_best.molecules([confs], [(p, q)])[0]
    want = np.array([min(kabsch_rmsd(confs[i][p], confs[j][qk]) for qk in q) for i in range(9) for j in range(i)])
    assert np.abs(got - want).max() <= 1e-10
    pre = oracle_best.molecules([confs], [(p, q)], prealigned=True)[0]
    want = np.array([min(np.sqrt(((confs[i][p] - confs[j][qk]) ** 2).sum() / L) for qk in q)
                     for i in range(9) for j in range(i)])
    assert np.abs(pre - want).max() <= 1e-12


def test_rigid_permuted_copy_is_zero_under_its_mapping_only():
    rng = np.random.default_rng(1)
    n = 9
    a = rng.normal(size=(n, 3)) * 1.5
    perm = rng.permutation(n)
    b = np.empty_like(a)
    b[perm] = a @ rotation(rng) + rng.normal(size=3) * 5.0
    lists = [(np.arange(n), np.stack([np.arange(n), perm]))]
    assert oracle_best.molecules([[b, a]], lists)[0][0] <= 1e-6
    assert oracle_best.molecules([[b, a]], [(np.arange(n), np.arange(n)[None])])[0][0] > 0.1


# ------------------------------------------------------------------ table building
def test_map_tables_layout():
    t = cr.MapTables([(np.array([0, 2]), np.array([[0, 2], [2, 0], [1, 0]])), (np.arange(3), np.arange(3)[None])])
    assert t.count.tolist() == [3, 1] and t.length.tolist() == [2, 3] and t.start.tolist() == [0, 8, 14]
    assert t.atoms.dtype == np.int16 and t.atoms.tolist() == [0, 2, 0, 2, 2, 0, 1, 0, 0, 1, 2, 0, 1, 2]


def test_map_form_is_sorted_by_probe_atom():
    p, q = cr._map_lists([[(2, 0), (0, 1)], [(0, 0), (2, 1)]], 3, "map")
    assert p.tolist() == [0, 2] and q.tolist() == [[1, 0], [0, 1]]


@pytest.mark.parametrize("bad,msg", [
    ([], "non-empty list of mappings"),
    ([[]], r"map\[0\] must be a non-empty list"),
    ([[(0, 1, 2)]], r"map\[0\] must be a non-empty list"),
    ([[(0.5, 1)]], r"map\[0\] must be a non-empty list"),
    ([[(0, 3)]], "outside"),
    ([[(-1, 0)]], "outside"),
    ([[(0, 1), (0, 2)]], "twice"),
    ([[(0, 1), (1, 1)]], "twice"),
    ([[(0, 1)], [(1, 0)]], "other probe atoms"),
])
def test_bad_maps_are_refused(bad, msg):
    with pytest.raises(ValueError, match=msg):
        cr._map_lists(bad, 3, "map")


def test_self_matches_ask_for_every_match_without_chirality():
    mol = StandIn([6, 6], [(0, 1, False)], [(0, 1), (1, 0)])
    assert self_matches(mol, 7) == [(0, 1), (1, 0)]
    assert mol.calls == [(True, False, 7, False)]
    assert self_matches(mol, 1) == [(0, 1)]


def test_symmetrize_restatement_on_carboxylate_and_nitro():
    assert self_matches(acetate(), 100, False) == [(0, 1, 2, 3)]
    assert self_matches(acetate(), 100, True) == [(0, 1, 2, 3), (0, 1, 3, 2)]
    assert self_matches(acetate(), 1, True) == [(0, 1, 2, 3)]  # the maxMatches cut applies after the expansion
    got = self_matches(nitro_ester(), 100, True)  # O4 has no partner on C0; the nitro oxygens swap
    assert got == [(0, 1, 2, 3, 4), (0, 1, 3, 2, 4)]
    # a match composed with the swap, from a molecule whose query already matches two ways
    mol = StandIn([6, 6, 8, 8], [(0, 1, False), (1, 2, True), (1, 3, True)], [(0, 1, 2, 3), (1, 0, 2, 3)])
    assert self_matches(mol, 100, True) == [(0, 1, 2, 3), (0, 1, 3, 2), (1, 0, 2, 3), (1, 0, 3, 2)]
    # unconjugated or terminal atoms of different elements are not made equivalent
    mol = StandIn([6, 8, 8, 7], [(0, 1, False), (0, 2, True), (0, 3, True)], [(0, 1, 2, 3)])
    assert self_matches(mol, 100, True) == [(0, 1, 2, 3)]


def test_self_matches_are_the_reference_lists():
    """A match t pairs probe atom q (the query) with reference atom t[q], as RDKit's GetBestRMS: Q = t itself. A list cut
    by maxMatches need not be closed under inversion, so the inverse would differ here: (1, 2, 0) is kept, its inverse
    (2, 0, 1) is cut."""
    mol = StandIn([6, 6, 6], [(0, 1, False), (1, 2, False), (0, 2, False)], [(0, 1, 2), (1, 2, 0), (2, 0, 1)])
    p, q = cr._self_match_lists(mol, 2, True, 0)
    assert p.tolist() == [0, 1, 2] and q.tolist() == [[0, 1, 2], [1, 2, 0]]
    # the same mapping through GetBestRMS's map form: pairs (probe q, reference t[q])
    p2, q2 = cr._map_lists([[(k, t[k]) for k in range(3)] for t in ((0, 1, 2), (1, 2, 0))], 3, "map")
    assert np.array_equal(p, p2) and np.array_equal(q, q2)


def test_a_molecule_without_atoms_gets_empty_lists():
    p, q = cr._atom_ids_lists(None, 0, "mol")
    assert p.shape == (0,) and q.shape == (1, 0)
    t = cr.MapTables([(p, q), (np.arange(2), np.arange(2)[None])])
    assert t.count.tolist() == [1, 1] and t.length.tolist() == [0, 2] and t.start.tolist() == [0, 0, 4]


# ------------------------------------------------------------------ refusals before device work
def test_refusals_come_before_any_device_work():
    mol = acetate()  # reading its conformers would raise AssertionError
    for kw, err in [({"maxMatches": 0}, ValueError), ({"weights": [1.0] * 4}, ValueError),
                    ({"map": [[(0, 9)]]}, ValueError), ({"stream": 0}, TypeError)]:
        with pytest.raises(err):
            cr.GetAllConformerBestRMS(mol, **kw)
    with pytest.raises(ValueError, match="must not be None"):
        cr.GetAllConformerBestRMS(None)
    with pytest.raises(ValueError, match="must not be None"):
        cr.GetAllConformerBestRMSBatch([mol, None])
    with pytest.raises(ValueError, match="maps holds 1"):
        cr.GetAllConformerBestRMSBatch([mol, mol], maps=[None])
    for ids, msg in [([], "non-empty"), ([0, 0], "twice"), ([4], "outside"), ([-1], "outside"), ([0.5], "non-empty")]:
        with pytest.raises(ValueError, match=msg):
            cr.GetConformerRMSMatrix(mol, atomIds=ids)
    with pytest.raises(ValueError, match="atomIds holds 1"):
        cr.GetConformerRMSMatrixBatch([mol, mol], atomIds=[[0]])
    with pytest.raises(TypeError):
        cr.GetConformerRMSMatrix(mol, stream=0, atomIds=[0])


def test_existing_positional_order_is_kept():
    import inspect

    params = list(inspect.signature(cr.GetConformerRMSMatrix).parameters.values())
    assert [p.name for p in params[:3]] == ["mol", "prealigned", "stream"]
    assert params[-1].name == "atomIds" and params[-1].kind is inspect.Parameter.KEYWORD_ONLY
    params = list(inspect.signature(cr.GetAllConformerBestRMS).parameters.values())
    assert [p.name for p in params[:6]] == ["mol", "numThreads", "maxMatches", "symmetrizeConjugatedTerminalGroups",
                                             "weights", "stream"]


# ------------------------------------------------------------------ C-ABI checks without a device
def call_mapped(counts, atoms, start, count, length, table):
    mcs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    atoms = np.asarray(atoms, np.int32)
    start, count, length = (np.asarray(x, t) for x, t in ((start, np.int64), (count, np.int32), (length, np.int32)))
    table = np.asarray(table, np.int16)
    return _lib.call("b200mol_conformer_rmsd_mapped", len(counts), mcs.ctypes.data, atoms.ctypes.data, None, None, None,
                     start.ctypes.data, count.ctypes.data, length.ctypes.data, table.ctypes.data, 0, None, None)


@pytest.mark.parametrize("start,count,length,table,msg", [
    ([0, 6], [0], [3], [0, 1, 2, 0, 1, 2], "mapping count 0 must be >= 1"),
    ([0, 0], [1], [0], [], "mapping length 0 must be in"),
    ([0, 10], [1], [5], list(range(10)), "mapping length 5 must be in"),
    ([0, 6], [1], [3], [0, 1, 4, 0, 1, 2], "holds atom 4, outside"),
    ([0, 6], [1], [3], [0, 1, 2, 0, -1, 2], "holds atom -1, outside"),
    ([0, 6], [1], [3], [0, 1, 2, 0, 2, 2], "list 1 holds atom 2 twice"),
    ([0, 7], [1], [3], [0, 1, 2, 0, 1, 2, 0], "(K + 1) L"),
    ([-1, 5], [1], [3], [0, 1, 2, 0, 1, 2], "must not start below 0"),
])
def test_c_abi_refuses_bad_tables(built_lib, start, count, length, table, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        call_mapped([3], [4], start, count, length, table)


def test_c_abi_refuses_null_tables_and_huge_molecules(built_lib):
    mcs, atoms = np.array([0, 2], np.int32), np.array([4], np.int32)
    with pytest.raises(ValueError, match="null mapping table"):
        _lib.call("b200mol_conformer_rmsd_mapped", 1, mcs.ctypes.data, atoms.ctypes.data, None, None, None, None, None,
                  None, None, 0, None, None)
    with pytest.raises(ValueError, match="fewer than 32768"):
        call_mapped([2], [40000], [0, 2], [1], [1], [0, 0])
    # a valid table for molecules without pairs needs no device and writes nothing
    call_mapped([1, 0], [4, 4], [0, 2, 4], [1, 1], [1, 1], [0, 0, 3, 3])
    # a molecule without atoms takes empty lists, and only those
    call_mapped([0, 1], [0, 4], [0, 0, 2], [1, 1], [0, 1], [0, 0])
    with pytest.raises(ValueError, match=re.escape("molecule 0 has no atoms: its mapping length 1 must be 0")):
        call_mapped([0], [0], [0, 2], [1], [1], [0, 0])


# ------------------------------------------------------------------ option
def test_match_chunk_option(built_lib):
    assert _lib.get_option("rmsd_match_chunk") == 0
    with _lib.options(rmsd_match_chunk=5):
        assert _lib.get_option("rmsd_match_chunk") == 5
    assert _lib.get_option("rmsd_match_chunk") == 0
    for bad in (-1, 1 << 31):
        with pytest.raises(ValueError, match=re.escape("rmsd_match_chunk must be in [0, 2^31)")):
            _lib.set_option("rmsd_match_chunk", bad)
    with pytest.raises(ValueError, match="read-only"):
        _lib.set_option("rmsd_match_chunks_last", 1)
    assert _lib.get_option("rmsd_match_chunks_last") >= 0
    text = open(os.path.join(ROOT, "include", "b200mol.h")).read()
    doc = text[text.index("Tuning knobs"):text.index("int b200mol_get_option(")]
    assert '"rmsd_match_chunk"' in doc and '"rmsd_match_chunks_last"' in doc
