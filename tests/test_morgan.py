"""Morgan fingerprints on the CPU: the oracle against an independent restatement of RDKit's getEnvironments, on the
graph families the GPU tests use; a mirror of the kernel's slab layout and launch rule, pinned to its limits; and the
checks ``MolGraphBatch`` makes before a graph can reach the device."""

import numpy as np
import pytest

import oracle
from nvmolkit_b200.molgraph import MolGraphBatch, atom_invariant

# ------------------------------------------------------------------ mirror of nvmolkit_b200/csrc/morgan.cu
SHARED_BUDGET = 200 * 1024  # kSharedBudget: bytes of shared memory one CTA's slabs may take
GLOBAL_SLAB_CAP = 256 << 20  # kGlobalSlabCap: the largest slab, and the global scratch of one call


def _r16(x):
    return (x + 15) & ~15


def slab_bytes(max_atoms, max_bonds, radius, fp_bits):
    """morganLayout(...).total: bytes of one molecule's working memory."""
    a, b = max(max_atoms, 1), max(max_bonds, 1)
    w, r = (b + 31) // 32, max(radius, 1)
    return (2 * _r16(4 * a) + 2 * _r16(4 * a * w) + _r16(4 * r * a * w) + _r16(4 * (a + 1)) + 2 * _r16(4 * b)
            + 2 * _r16(a) + _r16(fp_bits // 8))


def shared_warps(max_atoms, max_bonds, radius, fp_bits):
    """Warps per CTA of the shared-memory launch (budget / 2 / slab, clamped to 1-8); None when the slab goes to global
    memory, and 0 when the call is refused."""
    s = slab_bytes(max_atoms, max_bonds, radius, fp_bits)
    if s > GLOBAL_SLAB_CAP:
        return 0
    if s > SHARED_BUDGET:
        return None
    return min(8, max(1, SHARED_BUDGET // 2 // s))


def largest_square(radius, fp_bits, limit):
    """Largest n such that a molecule of n atoms and n bonds has a slab of at most `limit` bytes."""
    lo, hi = 1, 65535
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if slab_bytes(mid, mid, radius, fp_bits) <= limit else (lo, mid - 1)
    return lo


def size_for_warps(w, radius=2, fp_bits=2048):
    """Largest n (atoms = bonds) whose shared-memory launch puts w warps in a CTA."""
    return max(n for n in range(1, 2000) if shared_warps(n, n, radius, fp_bits) == w)


# ------------------------------------------------------------------ graphs
C_INV = atom_invariant(6, 4, 0, 0, 0, False)  # one invariant for every atom of the symmetric families


class Mol:
    """One molecule: atom invariants, and bonds as (a, b, type)."""

    def __init__(self, n, edges, inv=None, btype=1):
        self.n = n
        self.edges = [(int(e[0]), int(e[1])) for e in edges]
        self.inv = np.full(n, C_INV, dtype=np.uint32) if inv is None else np.asarray(inv, dtype=np.uint64).astype(np.uint32)
        self.btype = (np.full(len(edges), btype, dtype=np.uint64) if np.isscalar(btype)
                      else np.asarray(btype, dtype=np.uint64)).astype(np.uint32)

    def arrays(self):
        e = np.array(self.edges, dtype=np.int64).reshape(-1, 2)
        return self.inv, self.btype, e[:, 0].astype(np.uint16), e[:, 1].astype(np.uint16)

    def diameter(self):
        adj = [[] for _ in range(self.n)]
        for u, v in self.edges:
            adj[u].append(v)
            adj[v].append(u)
        best = 0
        for s in range(self.n):
            dist, front = {s: 0}, [s]
            while front:
                nxt = []
                for x in front:
                    for y in adj[x]:
                        if y not in dist:
                            dist[y] = dist[x] + 1
                            nxt.append(y)
                front = nxt
            best = max(best, max(dist.values()))
        return best


def batch(mols):
    a_starts, b_starts = np.cumsum([0] + [m.n for m in mols]), np.cumsum([0] + [len(m.edges) for m in mols])
    parts = [m.arrays() for m in mols]
    cat = [np.concatenate([p[i] for p in parts]) if parts else np.zeros(0) for i in range(4)]
    return MolGraphBatch(a_starts, b_starts, cat[0], cat[1], cat[2], cat[3])


def want(g, radius, fp_bits):
    return oracle.morgan(g.atom_starts, g.bond_starts, g.atom_inv, g.bond_inv, g.bond_a, g.bond_b, radius, fp_bits)


def complete(n):
    return Mol(n, [(i, j) for i in range(n) for j in range(i + 1, n)])


def star(k):
    return Mol(k + 1, [(0, i) for i in range(1, k + 1)])


def cycle(n):
    return Mol(n, [(i, (i + 1) % n) for i in range(n)])


def prism(n):  # two n-cycles joined rung by rung: 3-regular
    return Mol(2 * n, [(i, (i + 1) % n) for i in range(n)] + [(n + i, n + (i + 1) % n) for i in range(n)]
               + [(i, n + i) for i in range(n)])


def hypercube(d):  # d-regular on 2^d atoms (d = 3: the cube)
    return Mol(1 << d, [(i, i ^ (1 << k)) for i in range(1 << d) for k in range(d) if i < i ^ (1 << k)])


def benzene():
    return Mol(6, cycle(6).edges, [atom_invariant(6, 3, 1, 0, 0, True)] * 6, 12)


def cubane():
    return Mol(8, hypercube(3).edges, [atom_invariant(6, 4, 1, 0, 0, True)] * 8)


def neopentane():
    return Mol(5, star(4).edges, [atom_invariant(6, 4, 0, 0, 0, False)] + [atom_invariant(6, 4, 3, 0, 0, False)] * 4)


def adamantane():
    # CH atoms 0-3, CH2 atoms 4-9; every CH2 bridges two CH
    bridges = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    edges = [e for k, (u, v) in enumerate(bridges) for e in ((u, 4 + k), (v, 4 + k))]
    ch, ch2 = atom_invariant(6, 4, 1, 0, 0, True), atom_invariant(6, 4, 2, 0, 0, True)
    return Mol(10, edges, [ch] * 4 + [ch2] * 6)


def symmetric_family():
    mols = [complete(n) for n in range(2, 18)] + [star(15), star(16)] + [cycle(n) for n in range(3, 71)]
    mols += [prism(n) for n in range(3, 9)] + [hypercube(3), hypercube(4)]
    mols += [Mol(2, [(0, 1)]), benzene(), cubane(), neopentane(), adamantane()]
    return mols


def random_graph(n_atoms, n_bonds, rng, max_deg=4, n_inv=6, btypes=(1, 2, 12)):
    """Connected when n_bonds >= n_atoms - 1 (a random tree plus ring closures), otherwise a forest. No self-loop and
    no atom above max_deg."""
    assert n_bonds <= n_atoms * max_deg // 2 - n_atoms // 2 and (n_bonds < n_atoms or n_atoms > 4), "too many bonds"
    deg = np.zeros(n_atoms, dtype=np.int64)
    edges, have = [], set()
    for a in range(1, min(n_atoms, n_bonds + 1)):
        choices = np.nonzero(deg[:a] < max_deg)[0]
        q = int(choices[rng.integers(0, len(choices))])
        edges.append((q, a))
        have.add((q, a))
        deg[q] += 1
        deg[a] += 1
    while len(edges) < n_bonds:
        u, v = (int(x) for x in rng.integers(0, n_atoms, size=2))
        u, v = min(u, v), max(u, v)
        if u == v or (u, v) in have or deg[u] >= max_deg or deg[v] >= max_deg:
            continue
        edges.append((u, v))
        have.add((u, v))
        deg[u] += 1
        deg[v] += 1
    perm = rng.permutation(len(edges))  # bond order is not the tree order
    edges = [edges[i] for i in perm]
    inv = rng.integers(0, 1 << 32, size=n_inv, dtype=np.uint64)[rng.integers(0, n_inv, size=n_atoms)]
    return Mol(n_atoms, edges, inv, np.array(btypes)[rng.integers(0, len(btypes), size=len(edges))])


def copies(frag, k):
    """k disjoint copies of one fragment in one molecule."""
    edges = [(u + i * frag.n, v + i * frag.n) for i in range(k) for u, v in frag.edges]
    return Mol(frag.n * k, edges, np.tile(frag.inv, k), np.tile(frag.btype, k))


def with_isolated(frags, positions, n_total, iso_inv=None):
    """The fragments' atoms spread over n_total local indices, leaving the given ones as isolated atoms."""
    rest = [i for i in range(n_total) if i not in set(positions)]
    inv = np.full(n_total, C_INV if iso_inv is None else iso_inv, dtype=np.uint32)
    edges, types, at = [], [], 0
    for f in frags:
        idx = rest[at:at + f.n]
        inv[idx] = f.inv
        edges += [(idx[u], idx[v]) for u, v in f.edges]
        types += list(f.btype)
        at += f.n
    assert at == len(rest), "fragments must fill every index that is not isolated"
    return Mol(n_total, edges, inv, np.array(types, dtype=np.uint64))


def fragment_family():
    rng = np.random.default_rng(11)
    mols = [copies(benzene(), k) for k in (1, 2, 3, 5)] + [copies(cycle(4), 8), copies(Mol(2, [(0, 1)]), 20)]
    mols += [copies(random_graph(7, 7, rng), 4), copies(adamantane(), 3)]
    frags = [benzene(), cycle(5), random_graph(9, 8, rng), random_graph(13, 14, rng)]  # 33 atoms
    mols += [with_isolated(frags, [0, 31, 32, 36], 37), with_isolated(frags, [0, 31, 32, 36], 37, iso_inv=7)]
    mols += [Mol(40, []), Mol(40, [], rng.integers(0, 4, size=40)), Mol(1, []), Mol(0, [])]
    return mols


def value_edge_family():
    big = [1, 1 << 31, 0xFFFFFFFF, 5, (1 << 31) + 7, 0x80000001, 2]
    mols = [Mol(8, star(7).edges, [C_INV] * 8, big), Mol(8, star(7).edges, [0] + [0xFFFFFFFF] * 7, big)]
    mols += [Mol(7, cycle(7).edges, [0, 0xFFFFFFFF, 0, 0xFFFFFFFF, 1, 0xFFFFFFFE, 0], [0xFFFFFFFF, 1] * 3 + [0])]
    # invariants congruent modulo 128, 2048 and 65536: they share bits, but not environments
    mols += [Mol(6, cycle(6).edges, [3 + k * 65536 for k in range(6)], [1 << 31] * 6)]
    mols += [Mol(9, [(i, i + 1) for i in range(8)], [77 + 2048 * k for k in range(9)], [12, 12, 1, 1 << 31] * 2)]
    return mols


# ------------------------------------------------------------------ RDKit's getEnvironments, restated
def _hc(seed, v):
    return (seed ^ ((v + 0x9E3779B9 + (seed << 6) + (seed >> 2)) & 0xFFFFFFFF)) & 0xFFFFFFFF


def morgan_codes_py(m, radius):
    """Codes in emission order: round 0 every atom; each later round sorts (bitset, invariant, atom) and keeps a tuple
    only when its bitset was not emitted before (this round or earlier); a tuple that loses kills its atom."""
    adj = [[] for _ in range(m.n)]
    for b, (u, v) in enumerate(m.edges):
        adj[u].append((b, v))
        adj[v].append((b, u))
    inv = [int(x) for x in m.inv]
    nbhd, dead, emitted = [0] * m.n, [False] * m.n, set()
    codes = list(inv)
    for layer in range(radius):
        nxt, new_nbhd, tuples = [0] * m.n, list(nbhd), []
        for a in range(m.n):
            if dead[a]:
                continue
            if not adj[a]:
                dead[a] = True
                continue
            env, pairs = nbhd[a], []
            for b, o in adj[a]:
                env |= (1 << b) | nbhd[o]
                t = int(m.btype[b])
                pairs.append((t - (1 << 32) if t >= 1 << 31 else t, inv[o]))  # RDKit keeps the bond type as int32
            invar = _hc(layer, inv[a])
            for t, s in sorted(pairs):
                invar = _hc(invar, _hc(_hc(0, t & 0xFFFFFFFF), s))
            nxt[a], new_nbhd[a] = invar, env
            tuples.append((env, invar, a))
        for env, invar, a in sorted(tuples):
            if env in emitted:
                dead[a] = True
            else:
                emitted.add(env)
                codes.append(invar)
        inv, nbhd = nxt, new_nbhd
    return codes


def _fold(codes, fp_bits):
    fp = np.zeros(fp_bits // 32, dtype=np.uint32)
    for c in codes:
        fp[(c % fp_bits) >> 5] |= np.uint32(1 << ((c % fp_bits) & 31))
    return fp


FAMILIES = {"symmetric": symmetric_family, "fragments": fragment_family, "values": value_edge_family,
            "random": lambda: [random_graph(n, n + k, np.random.default_rng(n)) for n in (9, 33, 64) for k in (-1, 0, 2)]}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_oracle_equals_the_restatement(family):
    mols = FAMILIES[family]()
    g = batch(mols)
    for radius in (0, 1, 2, 3, 5, 16):
        folded = {bits: want(g, radius, bits) for bits in (128, 2048)}
        for i, m in enumerate(mols):
            ref = morgan_codes_py(m, radius)
            got = oracle.morgan_codes(*m.arrays(), radius)
            assert got.tolist() == ref, (family, i, radius)
            for bits, fp in folded.items():
                assert (fp[i] == _fold(ref, bits)).all(), (family, i, radius, bits)


def test_families_reach_the_tie_break_and_both_duplicate_paths():
    """The symmetric family must produce, in one round, two live atoms with equal bitsets and equal invariants (the
    index decides), equal bitsets with different invariants, and a bitset emitted in an earlier round."""
    seen = {"index": 0, "invariant": 0, "earlier": 0}
    for m in symmetric_family():
        adj = [[] for _ in range(m.n)]
        for b, (u, v) in enumerate(m.edges):
            adj[u].append((b, v))
            adj[v].append((b, u))
        inv, nbhd, dead, emitted = [int(x) for x in m.inv], [0] * m.n, [False] * m.n, set()
        for layer in range(m.diameter() + 1):
            nxt, new, tuples = [0] * m.n, list(nbhd), []
            for a in range(m.n):
                if dead[a] or not adj[a]:
                    dead[a] = True
                    continue
                env = nbhd[a]
                for b, o in adj[a]:
                    env |= (1 << b) | nbhd[o]
                invar = _hc(layer, inv[a])
                for t, s in sorted((int(m.btype[b]), inv[o]) for b, o in adj[a]):
                    invar = _hc(invar, _hc(_hc(0, t), s))
                nxt[a], new[a] = invar, env
                tuples.append((env, invar, a))
            tuples.sort()
            for k in range(1, len(tuples)):
                if tuples[k][0] == tuples[k - 1][0]:
                    seen["index" if tuples[k][1] == tuples[k - 1][1] else "invariant"] += 1
            earlier = set(emitted)
            for env, _, a in tuples:
                seen["earlier"] += env in earlier
                dead[a] = env in emitted
                emitted.add(env)
            inv, nbhd = nxt, new
    assert all(v > 0 for v in seen.values()), seen


# ------------------------------------------------------------------ the layout mirror
@pytest.mark.parametrize("radius,largest", [(0, 704), (1, 704), (2, 608), (3, 544), (5, 462), (16, 288)])
def test_layout_mirror_pins_the_shared_memory_limits(radius, largest):
    assert largest_square(radius, 2048, SHARED_BUDGET) == largest
    assert shared_warps(largest, largest, radius, 2048) == 1
    assert shared_warps(largest + 1, largest + 1, radius, 2048) is None


def test_layout_mirror_keeps_the_documented_size_at_every_radius():
    for radius in range(17):
        for bits in (32, 2048, 65536):
            assert shared_warps(1024, 1024, radius, bits) is None  # global memory, not refused
    assert largest_square(16, 2048, GLOBAL_SLAB_CAP) == 10912
    assert shared_warps(10912, 10912, 16, 2048) is None and shared_warps(10913, 10913, 16, 2048) == 0
    assert slab_bytes(0, 0, 0, 32) == slab_bytes(1, 1, 1, 32) == 11 * 16  # every one of the 11 arrays rounds up to 16 B


def test_every_warp_count_has_a_size():
    sizes = [size_for_warps(w) for w in range(1, 9)]
    assert sizes == sorted(sizes, reverse=True) and all(shared_warps(n, n, 2, 2048) == w
                                                        for w, n in zip(range(1, 9), sizes))
    for w, n in zip(range(1, 9), sizes):  # n is the boundary: one more atom and bond takes the next launch
        assert shared_warps(n + 1, n + 1, 2, 2048) == (w - 1 or None)
    assert sizes[0] == largest_square(2, 2048, SHARED_BUDGET)


# ------------------------------------------------------------------ MolGraphBatch refuses what the kernel cannot take
def _two_mols(**over):
    a = dict(atom_starts=[0, 3, 5], bond_starts=[0, 2, 3], atom_inv=[1, 2, 3, 4, 5], bond_inv=[1, 1, 2],
             bond_a=[0, 1, 0], bond_b=[1, 2, 1])
    a.update(over)
    return MolGraphBatch(**a)


def test_molgraph_accepts_valid_batches():
    assert len(_two_mols()) == 2
    assert len(MolGraphBatch([0], [0], [], [], [], [])) == 0
    assert len(MolGraphBatch([0, 0, 1, 1], [0, 0, 0, 0], [9], [], [], [])) == 3  # 0-, 1- and 0-atom molecules
    assert len(batch(fragment_family() + symmetric_family())) > 0


@pytest.mark.parametrize("over,msg", [
    (dict(bond_b=[1, 3, 1]), "not an atom"),  # endpoint == its molecule's atom count (an atom of the next one)
    (dict(bond_a=[0, 1, 2]), "not an atom"),  # in the second molecule, local index 2 of 2 atoms
    (dict(bond_a=[0, 1, 65535]), "not an atom"),
    (dict(bond_a=[0, 2, 0], bond_b=[1, 2, 1]), "itself"),
    (dict(bond_a=[0, 1, 1]), "itself"),
    (dict(atom_starts=[0, 6, 5]), "atom_starts"),
    (dict(atom_starts=[1, 3, 5]), "atom_starts"),
    (dict(atom_starts=[0, 3, 4]), "atom_starts"),
    (dict(bond_starts=[0, 3, 2]), "bond_starts"),
    (dict(bond_starts=[0, 2, 4]), "bond_starts"),
    (dict(bond_a=[0, 1]), "one entry per bond"),
    (dict(bond_b=[1, 2, 1, 0]), "one entry per bond"),
    (dict(bond_starts=[0, 3]), "nMols\\+1"),
])
def test_molgraph_refuses_what_the_kernel_cannot_take(over, msg):
    with pytest.raises(ValueError, match=msg):
        _two_mols(**over)


def test_generator_refuses_widths_and_radius_before_device_work():
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    for bits in (0, 32, 64, 96, 384, 4096, -128):
        with pytest.raises(ValueError, match="fpSize"):
            MorganFingerprintGenerator(2, bits)
    with pytest.raises(ValueError, match="radius"):
        MorganFingerprintGenerator(-1, 2048)
