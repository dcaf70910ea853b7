"""TFD matrices on the GPU (b200mol_tfd_matrices) against the fp64 oracle (oracle_tfd.c), to 1e-5 absolute: conformer
counts around the pair-pass tiles, every torsion type, rows too large for full-height tiles, degenerate and wrapping
dihedrals, bitwise repeatability, the return types and streams, and the Device3DResult path."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle import tfd as oracle_tfd
from nvmolkit_b200 import synthetic as S
from nvmolkit_b200 import tfd

pytestmark = pytest.mark.gpu

TOL = 1e-5
FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")


def random_torsions(rng, n_atoms, n_single=3, sym_q=(2, 4, 9), rings=(3, 6), weights=True, spec=False):
    """One molecule's torsion list over random atoms: singles, symmetric torsions of the given Q, ring torsions of the
    given sizes (consecutive quartets of a random atom cycle)."""
    pick = lambda k: [int(x) for x in rng.choice(n_atoms, size=k, replace=False)]  # noqa: E731
    w = (lambda: float(rng.uniform(0.01, 2.0))) if weights else (lambda: 1.0)  # noqa: E731
    out = []
    for _ in range(n_single):
        out.append(([tuple(pick(4))], tfd.SINGLE, w(), 180.0))
    for q in sym_q:
        base = pick(2)
        quartets = [(int(rng.integers(n_atoms)), base[0], base[1], int(rng.integers(n_atoms))) for _ in range(q)]
        out.append((quartets, tfd.SYMMETRIC, w(), float(rng.choice([30.0, 60.0, 90.0])) if spec else 180.0))
    for n in rings:
        ring = pick(n)
        quartets = [(ring[i], ring[(i + 1) % n], ring[(i + 2) % n], ring[(i + 3) % n]) for i in range(n)]
        out.append((quartets, tfd.RING, w(), tfd._ring_maxdev(n)))
    return out


def check(flat, **kw):
    """GPU matrices of a FlatTFDMolecules against the oracle; returns the GPU result (list of numpy arrays)."""
    got = tfd.GetTFDMatrices(flat, return_type="numpy", **kw)
    t = flat.torsions
    want = oracle_tfd.matrices(flat.mol_conf_start, flat.conf_atom_start, np.asarray(flat.xyz), t.tors_start,
                               t.quartet_start, t.quartets, t.type, t.weight, t.maxdev)
    assert len(got) == len(want)
    for m, (g, w) in enumerate(zip(got, want)):
        assert g.dtype == np.float32 and g.shape == w.shape, m
        if len(w):
            assert np.abs(g - w).max() <= TOL, (m, float(np.abs(g - w).max()))
    return got


def batch(rng, conf_counts, n_atoms=16, **kw):
    per_mol = [random_torsions(rng, n_atoms, **kw) for _ in conf_counts]
    coords = [rng.normal(0.0, 1.5, (c, n_atoms, 3)) for c in conf_counts]
    return tfd.FlatTFDMolecules.from_coordinates(tfd.TFDTorsions.from_lists(per_mol), coords)


def test_conformer_counts_at_the_tile_edges(cuda):
    rng = np.random.default_rng(1)
    check(batch(rng, [0, 1, 2, 63, 64, 65, 127, 128, 129, 3]))
    check(batch(rng, [2048], n_single=2, sym_q=(3,), rings=(5,)))


@pytest.mark.parametrize("weights", [True, False])
@pytest.mark.parametrize("spec", [False, True])
def test_every_torsion_type(cuda, weights, spec):
    """Symmetric Q 2...9 and ring sizes 3...16 in one batch, weights on and off, equal and spec maxDevs."""
    rng = np.random.default_rng(2 + weights + 2 * spec)
    per_mol = [random_torsions(rng, 20, n_single=k % 3, sym_q=(q,), rings=(n,), weights=weights, spec=spec)
               for k, (q, n) in enumerate(zip(list(range(2, 10)) * 2, range(3, 17)))]
    coords = [rng.normal(0.0, 1.5, (30 + 7 * k, 20, 3)) for k in range(len(per_mol))]
    check(tfd.FlatTFDMolecules.from_coordinates(tfd.TFDTorsions.from_lists(per_mol), coords))


def test_no_torsions_empty_batch_and_many_tiny_molecules(cuda):
    rng = np.random.default_rng(3)
    none = tfd.FlatTFDMolecules.from_coordinates(tfd.TFDTorsions.from_lists([[], []]),
                                                 [rng.normal(size=(5, 4, 3)), rng.normal(size=(70, 4, 3))])
    got = check(none)
    assert all((g == 0.0).all() for g in got) and [len(g) for g in got] == [10, 2415]
    empty = tfd.FlatTFDMolecules.from_coordinates(tfd.TFDTorsions.from_lists([]), [])
    assert tfd.GetTFDMatrices(empty) == []
    counts = rng.integers(0, 6, size=3000)
    check(batch(rng, counts, n_atoms=8, n_single=1, sym_q=(2,), rings=(3,)))


def test_feature_rows_too_large_for_full_height_tiles(cuda):
    """60 symmetric torsions of 9 quartets: 544-float rows, 16 x 16 tiles; 100 of them: 900 floats, 8 x 8 tiles."""
    rng = np.random.default_rng(4)
    per_mol = [random_torsions(rng, 24, n_single=2, sym_q=(9,) * 60, rings=(7,)),
               random_torsions(rng, 24, n_single=1, sym_q=(3,), rings=()),
               random_torsions(rng, 24, n_single=0, sym_q=(9,) * 100, rings=())]  # 900 floats: 8 x 8 tiles
    coords = [rng.normal(0.0, 1.5, (150, 24, 3)), rng.normal(0.0, 1.5, (90, 24, 3)), rng.normal(0.0, 1.5, (41, 24, 3))]
    check(tfd.FlatTFDMolecules.from_coordinates(tfd.TFDTorsions.from_lists(per_mol), coords))


def butane(phi_deg, r=1.5):
    p = math.radians(phi_deg)
    return np.array([[1.0, 0, 0], [0, 0, 0], [0, r, 0], [math.cos(p), r, -math.sin(p)]])


def test_degenerate_quartets_and_the_wrap(cuda):
    """Collinear atoms (exactly zero cross products: phi = 0 on both sides) and angles at 0 / 180 / 360."""
    collinear = np.array([[0.0, 0, 0], [1.0, 0, 0], [2.0, 0, 0], [2.0, 1.0, 0]])
    confs = [butane(a) for a in (0.0, 180.0, -180.0, 179.9999, -179.9999, 360.0, 1e-7, -1e-7, 90.0)] + [collinear]
    t = tfd.TFDTorsions.from_lists([[([(0, 1, 2, 3)], tfd.SINGLE, 1.0, 180.0),
                                     ([(0, 1, 2, 3), (3, 2, 1, 0)], tfd.RING, 0.5, tfd._ring_maxdev(4)),
                                     ([(0, 1, 2, 3), (1, 2, 3, 0)], tfd.SYMMETRIC, 2.0, 60.0)]])
    got = check(tfd.FlatTFDMolecules.from_coordinates(t, [confs]))[0]
    assert got[9 * 8 // 2 + 0] == 0.0  # collinear against the planar phi = 0 conformer: every quartet at phi = 0
    assert abs(got[5 * 4 // 2 + 0]) <= TOL  # 360 against 0
    assert abs(got[4 * 3 // 2 + 3]) <= 1e-3  # 179.9999 against -179.9999 across the wrap


def test_bitwise_repeatable_and_return_types_agree_on_any_stream(cuda):
    rng = np.random.default_rng(5)
    flat = batch(rng, [40, 200, 3, 65])
    a = tfd.GetTFDMatrices(flat, return_type="tensor")
    b = tfd.GetTFDMatrices(flat, return_type="tensor")
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    s = torch.cuda.Stream()
    c = tfd.GetTFDMatrices(flat, return_type="tensor", stream=s)
    s.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, c))
    n = tfd.GetTFDMatrices(flat, return_type="numpy")
    lst = tfd.GetTFDMatrices(flat, return_type="list", stream=s)
    for x, y, z in zip(a, n, lst):
        assert isinstance(z, list) and all(isinstance(v, float) for v in z)
        assert np.array_equal(x.cpu().numpy(), y) and np.array_equal(np.array(z, np.float32), y)


@pytest.fixture
def Chem(monkeypatch):
    monkeypatch.syspath_prepend(FAKE)
    for name in [m for m in sys.modules if m in ("rdkit", "tfd_molecules") or m.startswith("rdkit.")]:
        monkeypatch.delitem(sys.modules, name)
    import tfd_molecules

    yield tfd_molecules
    for name in [m for m in sys.modules if m in ("rdkit", "tfd_molecules") or m.startswith("rdkit.")]:
        sys.modules.pop(name, None)


def test_device_result_equals_host_conformers(cuda, Chem):
    """EmbedMolecules(FlatEmbedMolecules, output=DEVICE) -> GetTFDMatrices(coordinates=result) is torch.equal to the
    same coordinates passed as RDKit conformers, and matches the oracle."""
    from nvmolkit_b200.embedMolecules import EmbedMolecules, EmbedParameters
    from nvmolkit_b200.types import CoordinateOutput

    flat, raw = S.random_embed_molecules(5, 6, 14, seed=6)
    mols = [Chem.Mol(d) for d in raw]
    tors = tfd.tfd_torsions(mols)
    assert len(tors.type) > 0
    res = EmbedMolecules(flat, EmbedParameters(randomSeed=11), confsPerMolecule=6, output=CoordinateOutput.DEVICE)
    dev = tfd.GetTFDMatrices(mols, coordinates=res, torsions=tors, return_type="tensor")
    per_mol = res.per_molecule()
    host_mols = [Chem.Mol(d, conformers=[c.cpu().numpy() for c in confs]) for d, confs in zip(raw, per_mol)]
    host = tfd.GetTFDMatrices(host_mols, return_type="tensor")
    assert all(torch.equal(x, y) for x, y in zip(dev, host))
    coords = [[c.cpu().numpy() for c in confs] for confs in per_mol]
    check(tfd.FlatTFDMolecules.from_coordinates(tors, coords))


def test_device_result_with_a_molecule_without_conformers(cuda, Chem):
    """A molecule absent from the Device3DResult (every embedding failed) gets an empty matrix; conformers are taken in
    conf_indices order whatever their order in the result."""
    from nvmolkit_b200.types import AsyncGpuResult, Device3DResult

    _flat, raw = S.random_embed_molecules(3, 6, 10, seed=7)
    mols = [Chem.Mol(d) for d in raw]
    rng = np.random.default_rng(7)
    n0, n2 = len(raw[0]["z"]), len(raw[2]["z"])
    c0 = [rng.normal(size=(n0, 3)) for _ in range(4)]
    c2 = [rng.normal(size=(n2, 3)) for _ in range(3)]
    entries = [(0, 2, c0[2]), (2, 1, c2[1]), (0, 0, c0[0]), (2, 0, c2[0]), (0, 3, c0[3]), (2, 2, c2[2]), (0, 1, c0[1])]
    values = np.concatenate([e[2] for e in entries])
    starts = np.concatenate([[0], np.cumsum([len(e[2]) for e in entries])]).astype(np.int32)
    t = lambda a: AsyncGpuResult(torch.as_tensor(a).cuda())  # noqa: E731
    res = Device3DResult(t(values), t(starts), t(np.array([e[0] for e in entries], np.int32)),
                         t(np.array([e[1] for e in entries], np.int32)), 0, 3)
    got = tfd.GetTFDMatrices(mols, coordinates=res, return_type="numpy")
    assert [len(g) for g in got] == [6, 0, 3]
    want = tfd.GetTFDMatrices([Chem.Mol(raw[0], conformers=c0), Chem.Mol(raw[2], conformers=c2)], return_type="numpy")
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[1])
