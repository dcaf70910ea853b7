"""Morgan fingerprints on the GPU, bit for bit against the oracle: symmetric, fragmented and high-degree graphs, value
and count edges, every width, every launch shape of the shared-memory kernel, both slab locations, and every refusal.
Graph families, the slab-layout mirror and the restatement the oracle is checked against are in test_morgan.py."""

import ctypes as C

import numpy as np
import pytest
import torch

import test_morgan as M
from nvmolkit_b200 import _lib

pytestmark = pytest.mark.gpu


def _gen(radius, bits):
    from nvmolkit_b200.fingerprints import MorganFingerprintGenerator

    return MorganFingerprintGenerator(radius, bits)


def python_fp(g, radius, bits, stream=None):
    return _gen(radius, bits).GetFingerprints(g, stream=stream).numpy().view(np.uint32)


def _dev(a, cuda):
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16}.get(a.dtype, a.dtype)
    return torch.from_numpy(a.view(view)).to(cuda)


def abi_fp(g, radius, bits, cuda, max_atoms=None, max_bonds=None, stream=None):
    """One b200mol_morgan call with the stated maxima (default: the batch's own), rows filled with a pattern first."""
    t = [_dev(a, cuda) for a in (g.atom_starts, g.bond_starts, g.atom_inv, g.bond_inv, g.bond_a, g.bond_b)]
    out = torch.full((len(g), max(bits, 32) // 32), 0x5A5A5A5A, dtype=torch.int32, device=cuda)
    ma = int(g.atoms_per_mol.max(initial=0)) if max_atoms is None else max_atoms
    mb = int(g.bonds_per_mol.max(initial=0)) if max_bonds is None else max_bonds
    sptr = 0 if stream is None else stream.cuda_stream
    torch.cuda.synchronize()
    _lib.call("b200mol_morgan", *[x.data_ptr() for x in t], len(g), ma, mb, radius, bits, out.data_ptr(), C.c_void_p(sptr))
    return out.cpu().numpy().view(np.uint32)


def global_slab_last():
    return _lib.get_option("morgan_global_slab_last")


def check(got, g, radius, bits):
    want = M.want(g, radius, bits)
    assert got.shape == want.shape
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert len(bad) == 0, f"rows {bad[:10].tolist()} differ (radius {radius}, {bits} bits)"


# ------------------------------------------------------------------ symmetry
@pytest.mark.parametrize("bits", [128, 2048])
def test_symmetric_graphs_every_radius(cuda, bits):
    """K_2..K_17 (degree 16), stars of 15 and 16, C_3..C_70, prisms, the cube and Q4, the two-atom molecule, benzene,
    cubane, neopentane and adamantane, with equal invariants: every radius 0..16 covers diameter - 1, diameter and
    diameter + 1 of each molecule up to C_30, and 16 for the rest."""
    mols = M.symmetric_family()
    g = M.batch(mols)
    for radius in range(17):
        check(python_fp(g, radius, bits), g, radius, bits)
    assert max(m.diameter() for m in mols) == 35


# ------------------------------------------------------------------ fragments and values
@pytest.mark.parametrize("radius", [0, 1, 2, 3, 16])
def test_fragments_isolated_atoms_and_empty_molecules(cuda, radius):
    mols = M.fragment_family()
    g = M.batch(mols)
    for bits in (128, 2048):
        check(python_fp(g, radius, bits), g, radius, bits)
    # the same molecules in another order, empty and one-atom molecules first and last
    g2 = M.batch([M.Mol(0, []), M.Mol(1, [])] + mols[::-1] + [M.Mol(1, []), M.Mol(0, [])])
    got = abi_fp(g2, radius, 2048, cuda)
    check(got, g2, radius, 2048)
    assert (got[[0, -1]] == 0).all() and (got[[1, -2]] != 0).any(axis=1).all()


@pytest.mark.parametrize("radius", [0, 1, 2, 4, 16])
def test_value_edges(cuda, radius):
    """Bond invariants >= 2^31 next to small ones at one atom (sorted as int32), atom invariants 0 and 0xFFFFFFFF, and
    invariants congruent modulo the width."""
    g = M.batch(M.value_edge_family())
    for bits in (32, 128, 2048, 65536):
        check(abi_fp(g, radius, bits, cuda), g, radius, bits)


# ------------------------------------------------------------------ counts and widths
COUNTS = [31, 32, 33, 63, 64, 65, 95, 96, 97, 255, 256, 257]


@pytest.mark.parametrize("n", COUNTS)
def test_atom_and_bond_counts_at_word_and_lane_boundaries(cuda, n):
    rng = np.random.default_rng(n)
    mols = [M.random_graph(n, n, rng), M.random_graph(n, n - 1, rng), M.random_graph(n + 1, n, rng),
            M.random_graph(n, n + 1, rng)]
    for k in range(4):  # stated maxima equal to each molecule's own counts: bw = ceil(bonds / 32) exactly
        g = M.batch([mols[k]])
        for radius in (1, 2, 5):
            check(abi_fp(g, radius, 2048, cuda), g, radius, 2048)
    g = M.batch(mols)
    check(python_fp(g, 3, 1024), g, 3, 1024)


def test_every_python_width_and_the_abi_widths(cuda):
    g = M.batch(M.fragment_family()[:6] + [M.random_graph(40, 42, np.random.default_rng(3))])
    for bits in (128, 256, 512, 1024, 2048):
        check(python_fp(g, 2, bits), g, 2, bits)
    for bits in (32, 96, 160, 992, 4096, 65536):  # not powers of two: inv % bits is no mask
        check(abi_fp(g, 2, bits, cuda), g, 2, bits)
    for bits in (0, 31, -32, 48):
        with pytest.raises(ValueError, match="fpBits"):
            abi_fp(g, 2, bits, cuda)
    check(abi_fp(g, 2, 96, cuda), g, 2, 96)


# ------------------------------------------------------------------ launch shapes
@pytest.mark.parametrize("w", range(1, 9))
def test_every_warps_per_cta(cuda, w):
    """A stated size that gives w warps per CTA, with 1, w - 1, w + 1 and 3w + 2 molecules (partial last CTA)."""
    n = M.size_for_warps(w)
    assert M.shared_warps(n, n, 2, 2048) == w
    rng = np.random.default_rng(w)
    pool = [M.random_graph(n, n, rng)] + [M.random_graph(int(k), int(k) + 1, rng)
                                          for k in rng.integers(5, max(6, n), size=3 * w + 1)]
    for count in sorted({1, max(w - 1, 1), w + 1, 3 * w + 2}):
        g = M.batch(pool[:count])
        check(abi_fp(g, 2, 2048, cuda, max_atoms=n, max_bonds=n), g, 2, 2048)
        assert global_slab_last() == 0


def test_a_hundred_thousand_small_molecules(cuda):
    rng = np.random.default_rng(5)
    shapes = [M.random_graph(int(k), int(k) - 1 + int(r), rng) for k, r in zip(rng.integers(5, 13, size=64),
                                                                              rng.integers(0, 2, size=64))]
    mols = [shapes[i] for i in rng.integers(0, len(shapes), size=100_000)]
    g = M.batch(mols)
    check(python_fp(g, 2, 2048), g, 2, 2048)


def test_interleaved_size_classes_come_back_in_input_order(cuda):
    rng = np.random.default_rng(6)
    sizes = [10, 300, 40, 100, 700, 20, 200, 64, 65, 256, 257, 1, 0, 33, 128, 129]
    mols = [M.random_graph(n, max(n - 1 + (n > 4), 0), rng) if n else M.Mol(0, []) for n in sizes]
    g = M.batch(mols)
    got = python_fp(g, 2, 1024)
    check(got, g, 2, 1024)
    for i in (1, 4, 7):
        assert (got[i] == python_fp(M.batch([mols[i]]), 2, 1024)[0]).all()


# ------------------------------------------------------------------ size limits and the slab location
@pytest.mark.parametrize("radius", [0, 2, 3, 16])
def test_largest_shared_slab_and_one_past_it(cuda, radius):
    n = M.largest_square(radius, 2048, M.SHARED_BUDGET)
    rng = np.random.default_rng(radius)
    for size, location in ((n, 0), (n + 1, 1)):
        g = M.batch([M.random_graph(size, size, rng)])
        check(python_fp(g, radius, 2048), g, radius, 2048)
        assert global_slab_last() == location


@pytest.mark.parametrize("radius", [0, 2, 16])
def test_documented_size_1024_atoms_1024_bonds(cuda, radius):
    rng = np.random.default_rng(1024 + radius)
    big = M.random_graph(1024, 1024, rng)
    g = M.batch([big])
    check(python_fp(g, radius, 2048), g, radius, 2048)
    assert global_slab_last() == 1
    # mixed with small molecules in one call: more molecules than warps, so warps reuse their slabs
    small = [M.random_graph(int(k), int(k), rng) for k in rng.integers(5, 40, size=299)]
    mols = small[:150] + [big] + small[150:]
    g = M.batch(mols)
    got = abi_fp(g, radius, 2048, cuda, max_atoms=1024, max_bonds=1024)
    check(got, g, radius, 2048)
    assert global_slab_last() == 1


def test_first_size_past_the_stated_limit_is_refused_before_launch(cuda):
    g = M.batch([M.random_graph(20, 20, np.random.default_rng(9))])
    n = M.largest_square(16, 2048, M.GLOBAL_SLAB_CAP)
    before = _lib.launch_count()
    with pytest.raises(ValueError, match="too large"):
        abi_fp(g, 16, 2048, cuda, max_atoms=n + 1, max_bonds=n + 1)
    with pytest.raises(ValueError, match="too large"):
        abi_fp(g, 16, 2048, cuda, max_atoms=65535, max_bonds=65535)  # a slab of more than 2^32 bytes
    assert _lib.launch_count() == before
    check(abi_fp(g, 16, 2048, cuda), g, 16, 2048)


# ------------------------------------------------------------------ refusals
def test_refusals_and_the_next_call_on_the_stream(cuda):
    good = M.batch(M.fragment_family()[:4])
    side = torch.cuda.Stream()
    hub = M.star(17)
    with pytest.raises(ValueError, match="more than 16 bonds"):
        python_fp(M.batch([M.Mol(3, [(0, 1)]), hub]), 1, 2048)
    check(abi_fp(good, 2, 2048, cuda, stream=side), good, 2, 2048)
    check(python_fp(M.batch([hub]), 0, 2048), M.batch([hub]), 0, 2048)  # radius 0 reads no neighbours
    g = M.batch([M.random_graph(40, 41, np.random.default_rng(2)), M.random_graph(70, 70, np.random.default_rng(3))])
    with pytest.raises(ValueError, match="exceeds maxAtomsPerMol"):
        abi_fp(g, 2, 2048, cuda, max_atoms=69, max_bonds=70, stream=side)
    with pytest.raises(ValueError, match="exceeds maxAtomsPerMol"):
        abi_fp(g, 2, 2048, cuda, max_atoms=70, max_bonds=69)
    check(abi_fp(g, 2, 2048, cuda, stream=side), g, 2, 2048)
    with pytest.raises(ValueError, match="radius"):
        python_fp(good, 17, 2048)
    check(python_fp(good, 16, 2048), good, 16, 2048)


# ------------------------------------------------------------------ streams and repeatability
def test_side_stream_repeat_and_alone_equal_batched(cuda):
    mols = M.symmetric_family()[::3] + M.fragment_family()
    g = M.batch(mols)
    default = python_fp(g, 3, 2048)
    side = torch.cuda.Stream()
    assert (python_fp(g, 3, 2048, stream=side) == default).all()
    assert (python_fp(g, 3, 2048) == default).all()
    check(default, g, 3, 2048)
    for i in (0, len(mols) // 2, len(mols) - 3):
        assert (python_fp(M.batch([mols[i]]), 3, 2048)[0] == default[i]).all()
