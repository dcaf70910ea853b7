"""Flattened molecular graphs — the data format at the seam below RDKit (SURVEY.md §8b, Appendix B).

``MolGraphBatch`` is what the C-ABI consumes for Morgan fingerprints: CSR atom/bond arrays with RDKit-derived
invariants. ``from_rdkit`` builds it from RDKit ``Mol`` objects when RDKit is importable (it performs exactly the
per-atom feature extraction of the reference's MorganInvariantsGenerator, src/morgan_fingerprint_common.cpp:43-124);
everything downstream of this record runs on the GPU.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def _hash_combine(seed: int, v: int) -> int:
    return (seed ^ ((v + 0x9E3779B9 + ((seed << 6) & 0xFFFFFFFF) + (seed >> 2)) & 0xFFFFFFFF)) & 0xFFFFFFFF


def atom_invariant(z: int, total_degree: int, total_hs: int, charge: int, delta_mass: int, in_ring: bool) -> int:
    """gboost::hash<vector<uint32>> of {Z, degree+Hs, Hs, charge, deltaMass[, 1 if in ring]} in uint32."""
    seed = 0
    for v in (z, total_degree, total_hs, charge & 0xFFFFFFFF, delta_mass & 0xFFFFFFFF):
        seed = _hash_combine(seed, v & 0xFFFFFFFF)
    if in_ring:
        seed = _hash_combine(seed, 1)
    return seed


@dataclass
class MolGraphBatch:
    atom_starts: np.ndarray  # int32 [nMols+1]
    bond_starts: np.ndarray  # int32 [nMols+1]
    atom_inv: np.ndarray  # uint32 [totalAtoms]
    bond_inv: np.ndarray  # uint32 [totalBonds]  (RDKit bond type as integer)
    bond_a: np.ndarray  # uint16 [totalBonds]  molecule-local begin atom
    bond_b: np.ndarray  # uint16 [totalBonds]  molecule-local end atom

    def __post_init__(self):
        self.atom_starts = np.ascontiguousarray(self.atom_starts, dtype=np.int32)
        self.bond_starts = np.ascontiguousarray(self.bond_starts, dtype=np.int32)
        self.atom_inv = np.ascontiguousarray(self.atom_inv, dtype=np.uint32)
        self.bond_inv = np.ascontiguousarray(self.bond_inv, dtype=np.uint32)
        self.bond_a = np.ascontiguousarray(self.bond_a, dtype=np.uint16)
        self.bond_b = np.ascontiguousarray(self.bond_b, dtype=np.uint16)
        if len(self.atom_starts) != len(self.bond_starts) or len(self.atom_starts) < 1:
            raise ValueError("atom_starts and bond_starts must both have nMols+1 entries")
        # The kernel trusts these: an endpoint past its molecule would index outside the molecule's working memory, and
        # a self-loop would be counted twice there but once by RDKit.
        for name, starts, n in (("atom", self.atom_starts, len(self.atom_inv)),
                                ("bond", self.bond_starts, len(self.bond_inv))):
            if starts[0] != 0 or (np.diff(starts) < 0).any() or starts[-1] != n:
                raise ValueError(f"{name}_starts must start at 0, not decrease and end at the number of {name}s ({n})")
        if len(self.bond_a) != len(self.bond_inv) or len(self.bond_b) != len(self.bond_inv):
            raise ValueError("bond_a, bond_b and bond_inv must have one entry per bond")
        n_atoms = np.repeat(np.diff(self.atom_starts), np.diff(self.bond_starts))
        if (self.bond_a >= n_atoms).any() or (self.bond_b >= n_atoms).any():
            raise ValueError("a bond endpoint is not an atom of its molecule")
        if (self.bond_a == self.bond_b).any():
            raise ValueError("a bond joins an atom to itself")

    def __len__(self) -> int:
        return len(self.atom_starts) - 1

    @property
    def atoms_per_mol(self) -> np.ndarray:
        return np.diff(self.atom_starts)

    @property
    def bonds_per_mol(self) -> np.ndarray:
        return np.diff(self.bond_starts)

    def select(self, idx: np.ndarray) -> "MolGraphBatch":
        """Sub-batch of the given molecule indices (in that order)."""
        idx = np.asarray(idx, dtype=np.int64)
        na, nb = self.atoms_per_mol[idx], self.bonds_per_mol[idx]
        a_starts = np.concatenate([[0], np.cumsum(na)]).astype(np.int32)
        b_starts = np.concatenate([[0], np.cumsum(nb)]).astype(np.int32)

        def gather(starts, lens, arr):
            if len(idx) == 0:
                return arr[:0]
            pos = np.repeat(starts[idx].astype(np.int64) - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
            return arr[pos + np.arange(int(lens.sum()))]

        return MolGraphBatch(a_starts, b_starts, gather(self.atom_starts, na, self.atom_inv),
                             gather(self.bond_starts, nb, self.bond_inv), gather(self.bond_starts, nb, self.bond_a),
                             gather(self.bond_starts, nb, self.bond_b))


def from_rdkit(mols) -> MolGraphBatch:
    """RDKit Mol list -> MolGraphBatch (needs RDKit; mirrors src/morgan_fingerprint_common.cpp:43-124)."""
    from rdkit import Chem  # noqa: F401  (hard requirement of this adapter only)

    table = Chem.GetPeriodicTable()
    a_starts, b_starts, ainv, binv, ba, bb = [0], [0], [], [], [], []
    for mol in mols:
        if mol is None:
            raise ValueError("molecule is None")
        ring = mol.GetRingInfo()
        for atom in mol.GetAtoms():
            nbr_hs = sum(1 for n in atom.GetNeighbors() if n.GetAtomicNum() == 1)
            hs = atom.GetNumExplicitHs() + atom.GetNumImplicitHs()
            delta = int(atom.GetMass() - table.GetAtomicWeight(atom.GetAtomicNum()))
            ainv.append(atom_invariant(atom.GetAtomicNum(), hs + atom.GetDegree(), hs + nbr_hs,
                                       atom.GetFormalCharge(), delta, ring.NumAtomRings(atom.GetIdx()) > 0))
        for bond in mol.GetBonds():
            binv.append(int(bond.GetBondType()))
            ba.append(bond.GetBeginAtomIdx())
            bb.append(bond.GetEndAtomIdx())
        a_starts.append(len(ainv))
        b_starts.append(len(binv))
    return MolGraphBatch(np.array(a_starts), np.array(b_starts), np.array(ainv, dtype=np.uint32),
                         np.array(binv, dtype=np.uint32), np.array(ba, dtype=np.uint16), np.array(bb, dtype=np.uint16))
