"""Replays tests/golden/rdkit_best_align.npz (written by tools/export_rdkit_fixtures.py where RDKit exists): RDKit's
GetBestRMS, CalcRMS and GetBestAlignmentTransform against the matching restatement
(``rdkit_adapter.probe_ref_matches``) and the oracle on the CPU, and against nvmolkit_b200.molAlign on the GPU. This
pins what the best alignment restates from RDKit's source: the match direction, the terminal groups taken from the
probe, the cut after the expansion, CalcRMS's division by L with weights, the first strict minimum and the match tuple.
Skipped while the file is absent."""
import os
import sys

import numpy as np
import pytest

from nvmolkit_b200.rdkit_adapter import probe_ref_matches
from oracle import align as oa
from oracle import best_align as ob

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rdkit_best_align.npz")
FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")
pytestmark = pytest.mark.skipif(not os.path.exists(PATH),
                                reason="tests/golden/rdkit_best_align.npz has not been exported")


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(PATH))


class _Atom:
    def __init__(self, mol, i):
        self.mol, self.i = mol, i

    def GetIdx(self):
        return self.i

    def GetAtomicNum(self):
        return int(self.mol.z[self.i])

    def GetDegree(self):
        return sum(self.i in b[:2] for b in self.mol.bonds)

    def GetBonds(self):
        return [_Bond(b) for b in self.mol.bonds if self.i in b[:2]]


class _Bond:
    def __init__(self, b):
        self.b = b

    def GetOtherAtomIdx(self, i):
        return self.b[1] if self.b[0] == i else self.b[0]

    def GetIsConjugated(self):
        return bool(self.b[2])


class Recorded:
    """A molecule as exported: atoms, bonds with their conjugation, and RDKit's raw matches of it onto itself."""

    def __init__(self, fx, i):
        self.z, self.raw = fx[f"bam{i}_z"], [tuple(int(a) for a in t) for t in fx[f"bam{i}_raw"]]
        self.bonds = [tuple(int(x) for x in b) for b in fx[f"bam{i}_bonds"]]

    def GetNumAtoms(self):
        return len(self.z)

    def GetAtoms(self):
        return [_Atom(self, i) for i in range(len(self.z))]

    def GetAtomWithIdx(self, i):
        return _Atom(self, i)

    def GetSubstructMatches(self, query, uniquify=True, maxMatches=1000, useChirality=False):
        assert not uniquify and not useChirality
        return self.raw[:maxMatches]


def cases(fx):
    mols = [Recorded(fx, i) for i in range(int(fx["n_bam"]))]
    for j in range(int(fx["n_ba"])):
        i, c = int(fx[f"ba{j}_mol"]), int(fx[f"ba{j}_conf"])
        w = fx[f"ba{j}_weights"]
        xyz = fx[f"bam{i}_xyz"]
        matches = probe_ref_matches(mols[i], mols[i], int(fx["max_matches"]), bool(fx[f"ba{j}_sym"]))
        yield j, xyz[c], xyz[0], np.array(matches, np.int64), (w if len(w) else None)


def rdkit_mapping(fx, j, Q):
    """The index in Q of RDKit's best match (pairs (probe atom, reference atom))."""
    match = dict((int(p), int(r)) for p, r in fx[f"ba{j}_match"])
    row = [match[q] for q in range(Q.shape[1])]
    hits = [k for k in range(len(Q)) if Q[k].tolist() == row]
    assert hits, (j, "RDKit's match is not among the restated matches")
    return hits[0]


def check_pick(fx, j, prb, ref, Q, w, k, rmsd, T):
    """RMSDs as RDKit's; the mapping RDKit chose, with its transform, or one whose RMSD ties with it. True when the
    mapping is RDKit's."""
    assert abs(rmsd - float(fx[f"ba{j}_trmsd"])) <= 1e-8, j
    kr = rdkit_mapping(fx, j, Q)
    if k == kr:
        assert np.abs(T - fx[f"ba{j}_transform"]).max() <= 1e-6, j
        return True
    other = ob.best_align(prb, ref, np.arange(Q.shape[1]), Q[kr:kr + 1], w)[0]
    assert abs(other - rmsd) <= 1e-8, (j, k, kr)
    return False


def test_oracle_and_matches_replay_rdkit(fx):
    for j, prb, ref, Q, w in cases(fx):
        P = np.arange(Q.shape[1])
        rmsd, k, T, _ = ob.best_align(prb, ref, P, Q, w)
        same = check_pick(fx, j, prb, ref, Q, w, k, rmsd, T)
        assert abs(rmsd - float(fx[f"ba{j}_rmsd"])) <= 1e-8, j
        assert not same or np.abs(oa.apply(T, prb) - fx[f"ba{j}_moved"]).max() <= 1e-6, j
        assert abs(ob.best_align(prb, ref, P, Q, w, 1)[0] - float(fx[f"ba{j}_calc"])) <= 1e-8, j


@pytest.mark.gpu
def test_library_replays_rdkit(fx, cuda, monkeypatch):
    monkeypatch.syspath_prepend(FAKE)
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        monkeypatch.delitem(sys.modules, name)
    from rdkit import Chem

    from nvmolkit_b200 import molAlign as ma

    mk = lambda xyz: Chem.Mol({"z": [6] * len(xyz), "bonds": [], "nbrs": [[] for _ in xyz]},  # noqa: E731
                              conformers=[xyz])
    for j, prb, ref, Q, w in cases(fx):
        maps = [[(q, int(t[q])) for q in range(Q.shape[1])] for t in Q]
        rmsd, T, match = ma.GetBestAlignmentTransform(mk(prb), mk(ref), map=maps, weights=w)
        k = next(i for i, t in enumerate(Q) if [r for _, r in match] == t.tolist())
        same = check_pick(fx, j, prb, ref, Q, w, k, rmsd, T)
        assert abs(ma.CalcRMS(mk(prb), mk(ref), map=maps, weights=w) - float(fx[f"ba{j}_calc"])) <= 1e-8, j
        moved = mk(prb)
        assert abs(ma.GetBestRMS(moved, mk(ref), map=maps, weights=w) - float(fx[f"ba{j}_rmsd"])) <= 1e-8, j
        assert not same or np.abs(moved.GetConformers()[0].GetPositions() - fx[f"ba{j}_moved"]).max() <= 1e-6, j
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        sys.modules.pop(name, None)
