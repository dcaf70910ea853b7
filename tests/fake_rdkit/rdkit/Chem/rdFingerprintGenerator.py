"""Stand-in for RDKit's Morgan generator as far as the TFD torsion builder uses it: the per-atom environment codes of
each radius in the bit-info map (includeRedundantEnvironments=True, so every atom with a neighbour has one per radius).
Atom invariants are the repository's restatement of RDKit's (molgraph.atom_invariant), the environment hash the one
oracle_fp.c restates (src/morgan_fingerprint_cpu.cpp): the codes pin the algorithm, not RDKit's own hash values."""
from nvmolkit_b200.molgraph import _hash_combine, atom_invariant


class AdditionalOutput:
    def __init__(self):
        self._map = None

    def AllocateBitInfoMap(self):
        self._map = {}

    def GetBitInfoMap(self):
        return self._map


class _MorganGenerator:
    def __init__(self, radius):
        self.radius = radius

    def GetSparseCountFingerprint(self, mol, additionalOutput=None):
        n = mol.GetNumAtoms()
        cur = []
        for a in mol.GetAtoms():
            hs = a.GetNumExplicitHs() + a.GetNumImplicitHs()
            nbr_hs = sum(1 for x in a.GetNeighbors() if x.GetAtomicNum() == 1)
            cur.append(atom_invariant(a.GetAtomicNum(), hs + a.GetDegree(), hs + nbr_hs, a.GetFormalCharge(), 0,
                                      mol.GetRingInfo().NumAtomRings(a.GetIdx()) > 0))
        codes = {}
        for a in range(n):
            codes.setdefault(cur[a], []).append((a, 0))
        bonds = [(b.GetBeginAtomIdx(), b.GetEndAtomIdx(), int(b.GetBondType())) for b in mol.GetBonds()]
        for layer in range(self.radius):
            nxt = list(cur)
            for a in range(n):
                pairs = sorted((bt, cur[j if i == a else i]) for i, j, bt in bonds if a in (i, j))
                if not pairs:
                    continue
                inv = _hash_combine(layer, cur[a])
                for bt, c in pairs:
                    inv = _hash_combine(inv, _hash_combine(_hash_combine(0, bt), c))
                nxt[a] = inv
                codes.setdefault(inv, []).append((a, layer + 1))
            cur = nxt
        if additionalOutput is not None and additionalOutput._map is not None:
            additionalOutput._map.update({k: tuple(v) for k, v in codes.items()})
        return codes


def GetMorganGenerator(radius=2, **_options):
    return _MorganGenerator(radius)
