"""Conformer RMSD matrices on the GPU (b200mol_conformer_rmsd) against the fp64 oracle (oracle_rmsd.c): at most 1e-5 A
for every pair and 1e-8 A for pairs whose oracle RMSD is at least 0.05 A. Conformer counts around the 32-conformer
tiles, atom counts around the 16-atom MMA chunks, degenerate geometries (collinear, planar, mirror images, rigid
motions, identical conformers) near the origin and 1e3 A away, both modes, repeatability and batching, the RDKit and
Device3DResult inputs, and Butina on the matrix."""
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from oracle import rmsd as oracle_rmsd
from nvmolkit_b200 import conformerRmsd as cr
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult

pytestmark = pytest.mark.gpu

FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")
R = 32  # pair-pass tile side (csrc/conformer_rmsd.cu)


@pytest.fixture
def Chem(monkeypatch):
    monkeypatch.syspath_prepend(FAKE)
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        monkeypatch.delitem(sys.modules, name)
    from rdkit import Chem as chem

    yield chem
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        sys.modules.pop(name, None)


def make_mol(Chem, n, confs=()):
    return Chem.Mol({"z": [6] * n, "bonds": [], "nbrs": [[] for _ in range(n)]}, conformers=list(confs))


def assert_close(got, want, what=""):
    assert got.dtype == np.float64 and got.shape == want.shape, what
    if len(want):
        err = np.abs(got - want)
        assert err.max() <= 1e-5, (what, float(err.max()))
        far = want >= 0.05
        if far.any():
            assert err[far].max() <= 1e-8, (what, float(err[far].max()))


def run(Chem, coords, prealigned=False):
    """coords[m]: list of [n, 3] conformers; GPU against the oracle; returns the GPU matrices (numpy)."""
    mols = [make_mol(Chem, len(c[0]) if len(c) else 3, c) for c in coords]
    res = cr.GetConformerRMSMatrixBatch(mols, prealigned=prealigned)
    torch.cuda.synchronize()
    got = [r.torch().cpu().numpy() for r in res]
    want = oracle_rmsd.molecules(coords, prealigned)
    for m, (g, w) in enumerate(zip(got, want)):
        assert_close(g, w, (m, prealigned))
    return got


def rotation(rng):
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1.0
    return q


def conformers(rng, c, n, spread=0.6):
    base = rng.normal(size=(n, 3)) * 1.5
    return [base @ rotation(rng) + rng.normal(size=3) * 3.0 + rng.normal(size=(n, 3)) * spread for _ in range(c)]


@pytest.mark.parametrize("prealigned", [False, True])
def test_conformer_counts_around_the_tile(cuda, Chem, prealigned):
    rng = np.random.default_rng(1)
    counts = [0, 1, 2, R - 1, R, R + 1, 2 * R - 1, 2 * R + 1, 5]
    run(Chem, [conformers(rng, c, 12) for c in counts], prealigned)


def test_one_molecule_of_2048_conformers(cuda, Chem):
    rng = np.random.default_rng(2)
    got = run(Chem, [conformers(rng, 2048, 10)])
    assert len(got[0]) == 2048 * 2047 // 2


@pytest.mark.parametrize("prealigned", [False, True])
def test_atom_counts_around_the_mma_depth_and_chunks(cuda, Chem, prealigned):
    rng = np.random.default_rng(3)
    sizes = [1, 2, 3, 15, 16, 17, 31, 32, 33, 47, 48, 49, 1000]
    run(Chem, [conformers(rng, 37, n) for n in sizes], prealigned)


def degenerate_sets(rng):
    """Per molecule a conformer list: collinear (two atoms, a line), planar, rigid motions, mirror images, identical."""
    line = np.outer(rng.normal(size=9), [0.3, -0.8, 0.5])
    plane = np.c_[rng.normal(size=(8, 2)) * 1.5, np.zeros(8)] @ rotation(rng)
    chiral = rng.normal(size=(7, 3)) * 1.5
    ring = np.c_[np.cos(np.arange(6) * np.pi / 3), np.sin(np.arange(6) * np.pi / 3), np.zeros(6)] * 1.4
    moves = lambda a, k: [a @ rotation(rng) + rng.normal(size=3) * 4.0 for _ in range(k)]  # noqa: E731
    return [
        [a for a in moves(np.array([[0.0, 0, 0], [1.5, 0, 0]]), 5)] + [np.array([[0.0, 0, 0], [0, 2.0, 0]])],
        moves(line, 6) + [line * 1.3, np.outer(rng.normal(size=9), [1.0, 0, 0])],
        moves(plane, 6) + [plane + np.c_[np.zeros((8, 2)), rng.normal(size=8) * 0.2]],
        moves(ring, 5) + [ring * [1.0, 1.0, -1.0]],
        moves(chiral, 4) + [c * [1.0, 1.0, -1.0] for c in moves(chiral, 4)],
        [chiral.copy() for _ in range(5)],
        moves(rng.normal(size=(3, 3)), 6),
    ]


@pytest.mark.parametrize("shift", [0.0, 1e3])
@pytest.mark.parametrize("prealigned", [False, True])
def test_degenerate_geometries(cuda, Chem, shift, prealigned):
    rng = np.random.default_rng(4)
    sets = [[c + shift * np.array([1.0, -0.6, 0.8]) for c in confs] for confs in degenerate_sets(rng)]
    got = run(Chem, sets, prealigned)
    if not prealigned:
        for m, k in enumerate([5, 6, 6, 5, 4, 5, 6]):  # the first k conformers are rigid motions of one another
            assert max(got[m][i * (i - 1) // 2 + j] for i in range(k) for j in range(i)) <= 1e-5, m
        mirrors = [got[4][i * (i - 1) // 2 + j] for i in range(4, 8) for j in range(4)]
        assert min(mirrors) > 0.1  # a chiral set does not superpose onto its mirror image


def test_repeatable_batch_independent_and_on_any_stream(cuda, Chem):
    rng = np.random.default_rng(5)
    coords = [conformers(rng, c, n) for c, n in [(40, 20), (70, 33), (3, 5), (65, 100)]]
    mols = [make_mol(Chem, len(c[0]), c) for c in coords]
    a = cr.GetConformerRMSMatrixBatch(mols)
    b = cr.GetConformerRMSMatrixBatch(mols)
    assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(a, b))
    for m, mol in enumerate(mols):
        assert torch.equal(cr.GetConformerRMSMatrix(mol).torch(), a[m].torch())
    s = torch.cuda.Stream()
    c = cr.GetConformerRMSMatrixBatch(mols, stream=s)
    s.synchronize()
    assert all(isinstance(x, AsyncGpuResult) for x in c)
    assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(a, c))
    single = cr.GetConformerRMSMatrix(mols[1], stream=s)
    s.synchronize()
    assert torch.equal(single.torch(), a[1].torch())
    assert cr.GetConformerRMSMatrixBatch([]) == []
    assert cr.GetConformerRMSMatrix(make_mol(Chem, 4, [np.zeros((4, 3))])).torch().numel() == 0


def test_errors_before_device_work(cuda, Chem):
    with pytest.raises(ValueError):
        cr.GetConformerRMSMatrix(None)
    with pytest.raises(ValueError):
        cr.GetConformerRMSMatrix(make_mol(Chem, 0, [np.zeros((0, 3))] * 3))
    with pytest.raises(TypeError):
        cr.GetConformerRMSMatrix(make_mol(Chem, 2, [np.zeros((2, 3))] * 2), stream=0)


@pytest.mark.parametrize("prealigned", [False, True])
def test_rdkit_molecules_equal_the_device_result(cuda, Chem, prealigned):
    """The same coordinates through RDKit conformers and through a Device3DResult whose molecule and conformer tables
    are shuffled: bitwise equal matrices."""
    rng = np.random.default_rng(6)
    coords = [conformers(rng, c, n) for c, n in [(5, 14), (0, 6), (40, 9), (1, 3), (33, 17)]]
    mols = [make_mol(Chem, len(c[0]) if c else 6, c) for c in coords]
    host = cr.GetConformerRMSMatrixBatch(mols, prealigned=prealigned)
    entries = [(m, k, c) for m, confs in enumerate(coords) for k, c in enumerate(confs)]
    entries = [entries[i] for i in rng.permutation(len(entries))]
    t = lambda a: AsyncGpuResult(torch.as_tensor(np.asarray(a)).cuda())  # noqa: E731
    starts = np.concatenate([[0], np.cumsum([len(e[2]) for e in entries])]).astype(np.int32)
    res = Device3DResult(t(np.concatenate([e[2] for e in entries])), t(starts),
                         t(np.array([e[0] for e in entries], np.int32)), t(np.array([e[1] for e in entries], np.int32)),
                         0, len(mols))
    dev = cr.GetConformerRMSMatrixBatch(mols, prealigned=prealigned, coordinates=res)
    assert [x.torch().numel() for x in dev] == [10, 0, 780, 0, 528]
    assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(host, dev))


def test_butina_on_the_matrix_matches_the_oracle(cuda, Chem):
    """Well-separated clusters of conformers: the condensed matrix squared with torch and clustered by
    clustering.butina gives the oracle Butina's ids and centroids on the oracle matrix."""
    from nvmolkit_b200.clustering import butina

    rng = np.random.default_rng(7)
    n = 15
    centres = [rng.normal(size=(n, 3)) * 2.0 for _ in range(6)]
    sizes = [9, 7, 5, 4, 2, 1]
    confs = []
    for c, k in zip(centres, sizes):
        confs += [c @ rotation(rng) + rng.normal(size=3) * 5.0 + rng.normal(size=(n, 3)) * 0.05 for _ in range(k)]
    order = rng.permutation(len(confs))
    confs = [confs[i] for i in order]
    cond = cr.GetConformerRMSMatrix(make_mol(Chem, n, confs)).torch()
    c = len(confs)
    square = torch.zeros(c, c, dtype=torch.float64, device=cond.device)
    idx = torch.tril_indices(c, c, offset=-1, device=cond.device)
    square[idx[0], idx[1]] = cond
    square = square + square.T
    ids, cen = butina(square, 0.5, return_centroids=True)
    want = oracle_rmsd.molecules([confs])[0]
    assert (want[want < 0.5].max() < 0.4) and (want[want >= 0.5].min() > 0.6)  # no pair near the cutoff
    sq = np.zeros((c, c))
    sq[np.tril_indices(c, -1)] = want
    ids_o, cen_o = oracle.butina_dense(sq + sq.T, 0.5)
    assert np.array_equal(ids.torch().cpu().numpy(), ids_o)
    assert np.array_equal(cen.torch().cpu().numpy(), cen_o)
