"""Morgan count fingerprints on the GPU, compared with == against the count oracle (oracle.morgan_codes folded with
bincount): every graph family of test_morgan.py, radii 0 to 4, all five widths, both slab locations, and the invariant
that the non-zero bins are GetFingerprints' bits."""

import ctypes as C

import numpy as np
import pytest
import torch

import test_morgan as M
from nvmolkit_b200 import _lib
from nvmolkit_b200.fingerprints import MorganFingerprintGenerator, pack_fingerprint
from oracle import count as oracle_count

pytestmark = pytest.mark.gpu
WIDTHS = (128, 256, 512, 1024, 2048)


def want(g, radius, bits):
    return oracle_count.morgan_counts(g.atom_starts, g.bond_starts, g.atom_inv, g.bond_inv, g.bond_a, g.bond_b, radius,
                                      bits)


def gpu_counts(g, radius, bits, stream=None):
    return MorganFingerprintGenerator(radius, bits).GetCountFingerprints(g, stream=stream).numpy()


def check(got, g, radius, bits):
    w = want(g, radius, bits)
    assert got.dtype == np.int32 and got.shape == w.shape
    bad = np.nonzero((got != w).any(axis=1))[0]
    assert len(bad) == 0, f"rows {bad[:10].tolist()} differ (radius {radius}, {bits} bins)"


@pytest.mark.parametrize("family", sorted(M.FAMILIES))
def test_every_family_radius_and_width(cuda, family):
    g = M.batch(M.FAMILIES[family]())
    for radius in range(5):
        for bits in WIDTHS:
            got = gpu_counts(g, radius, bits)
            check(got, g, radius, bits)
            bits_gpu = MorganFingerprintGenerator(radius, bits).GetFingerprints(g).torch()
            assert torch.equal(pack_fingerprint(torch.from_numpy(got).cuda() > 0), bits_gpu)


@pytest.mark.parametrize("radius", [0, 2, 3])
def test_shared_and_global_slab(cuda, radius):
    n = M.largest_square(radius, 2048, M.SHARED_BUDGET)
    rng = np.random.default_rng(40 + radius)
    for size, location in ((n, 0), (n + 1, 1)):
        mols = [M.random_graph(size, size, rng)] + [M.random_graph(int(k), int(k), rng) for k in rng.integers(5, 30, size=40)]
        g = M.batch(mols)
        check(gpu_counts(g, radius, 2048), g, radius, 2048)
        assert _lib.get_option("morgan_global_slab_last") == location


def test_abi_global_slab_with_more_molecules_than_warps_and_a_zeroed_refused_row(cuda):
    rng = np.random.default_rng(7)
    big = M.random_graph(1024, 1024, rng)
    small = [M.random_graph(int(k), int(k), rng) for k in rng.integers(5, 40, size=299)]
    g = M.batch(small[:150] + [big] + small[150:])
    t = [torch.from_numpy(np.ascontiguousarray(a).view({np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16}.get(
        a.dtype, a.dtype))).cuda() for a in (g.atom_starts, g.bond_starts, g.atom_inv, g.bond_inv, g.bond_a, g.bond_b)]
    out = torch.full((len(g), 2048), 7, dtype=torch.int32, device="cuda")
    _lib.call("b200mol_morgan_counts", *[x.data_ptr() for x in t], len(g), 1024, 1024, 2, 2048, out.data_ptr(), None)
    check(out.cpu().numpy(), g, 2, 2048)
    assert _lib.get_option("morgan_global_slab_last") == 1
    out.fill_(7)
    with pytest.raises(ValueError, match="exceeds maxAtomsPerMol"):
        _lib.call("b200mol_morgan_counts", *[x.data_ptr() for x in t], len(g), 1023, 1024, 2, 2048, out.data_ptr(), None)
    got = out.cpu().numpy()
    assert (got[150] == 0).all()  # the refused molecule's row is zero, the others are counted
    rest = np.r_[0:150, 151:len(g)]
    assert np.array_equal(got[rest], want(g, 2, 2048)[rest])


def test_refusals_streams_and_repeats(cuda):
    with pytest.raises(ValueError, match="more than 16 bonds"):
        gpu_counts(M.batch([M.star(17)]), 1, 2048)
    g = M.batch(M.symmetric_family()[::3] + M.fragment_family())
    default = gpu_counts(g, 3, 2048)
    side = torch.cuda.Stream()
    assert np.array_equal(gpu_counts(g, 3, 2048, stream=side), default)
    assert np.array_equal(gpu_counts(g, 3, 2048), default)
    check(default, g, 3, 2048)


def test_synthetic_molecules_at_size(cuda):
    from nvmolkit_b200 import synthetic

    g = synthetic.random_molgraphs(20000, seed=3)
    got = gpu_counts(g, 2, 2048)
    check(got, g, 2, 2048)
    bits = MorganFingerprintGenerator(2, 2048).GetFingerprints(g).torch()
    assert torch.equal(pack_fingerprint(torch.from_numpy(got).cuda() > 0), bits)
