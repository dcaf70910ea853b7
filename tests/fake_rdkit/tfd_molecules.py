"""Fake-RDKit molecules with the ring and bond accessors the TFD torsion builder (nvmolkit_b200.tfd.tfd_torsions) reads
- TEST INFRASTRUCTURE ONLY. Subclasses of the stand-in's Mol / Bond / RingInfo (rdkit.Chem of this directory) that add
Bond.GetIdx and RingInfo.AtomRings / BondRings / NumBondRings as RDKit lists them: atoms in ring order, and the bonds
between consecutive ring atoms in the same order."""
from rdkit import Chem


class Bond(Chem.Bond):
    def GetIdx(self):
        return self._k


class RingInfo(Chem.RingInfo):
    def __init__(self, rings, n, bonds):
        super().__init__(rings, n)
        self._bonds = [tuple(b) for b in bonds]

    def AtomRings(self):
        return tuple(tuple(r) for r in self._r)

    def BondRings(self):
        index = {frozenset(b): k for k, b in enumerate(self._bonds)}
        return tuple(tuple(index[frozenset((r[i], r[(i + 1) % len(r)]))] for i in range(len(r))) for r in self._r)

    def NumBondRings(self, k):
        return sum(1 for r in self.BondRings() if k in r)


class Mol(Chem.Mol):
    def GetBonds(self):
        return [Bond(self, k) for k in range(len(self.d["bonds"]))]

    def GetBondBetweenAtoms(self, i, j):
        b = super().GetBondBetweenAtoms(i, j)
        return None if b is None else Bond(self, b._k)

    def GetRingInfo(self):
        return RingInfo(self.rings, self.GetNumAtoms(), self.d["bonds"])
