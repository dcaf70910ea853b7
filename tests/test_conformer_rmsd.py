"""Conformer RMSD matrices on the CPU: the fp64 oracle (oracle_rmsd.c) on known answers and against an SVD Kabsch,
the argument checks of nvmolkit_b200.conformerRmsd (fake RDKit), which all run before any device work, and the host
planning tables (int64 pair offsets, the Device3DResult conformer order, the C-ABI's checks)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import rmsd as oracle_rmsd
from nvmolkit_b200 import conformerRmsd as cr
from nvmolkit_b200._hostutil import device_conformer_order
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult

FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")


def kabsch_rmsd(p, q):
    """Independent best-superposition RMSD by numpy SVD (proper rotations only)."""
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


def test_oracle_known_answers():
    rng = np.random.default_rng(0)
    a = rng.normal(size=(9, 3))
    moved = a @ rotation(rng) + np.array([3.0, -2.0, 7.0])
    assert oracle_rmsd.molecules([[a, moved]])[0][0] <= 1e-6  # rigid motion: sqrt of an fp64 rounding residue
    # stretched collinear triple: centred, no rotation helps; SSD = 1 + 1 + 0
    line = np.array([[-1.0, 0, 0], [1.0, 0, 0], [0.0, 0, 0]])
    assert oracle_rmsd.molecules([[line, 2.0 * line]])[0][0] == pytest.approx(np.sqrt(2.0 / 3.0), abs=1e-12)
    # prealigned: a rigid shift by (1, 2, 2) is an RMSD of 3
    assert oracle_rmsd.molecules([[a, a + [1.0, 2.0, 2.0]]], prealigned=True)[0][0] == pytest.approx(3.0, abs=1e-12)
    # a chiral tetrahedron and its mirror image do not superpose by a rotation
    tet = np.array([[0.0, 0, 0], [1.5, 0, 0], [0.0, 1.0, 0], [0.0, 0, 0.7]])
    mirror = tet * [1.0, 1.0, -1.0]
    got = oracle_rmsd.molecules([[tet, mirror]])[0][0]
    assert got > 0.1 and got == pytest.approx(kabsch_rmsd(tet, mirror), abs=1e-10)


@pytest.mark.parametrize("n", [3, 6, 30, 100])
def test_oracle_matches_svd_kabsch(n):
    rng = np.random.default_rng(n)
    confs = [rng.normal(size=(n, 3)) * 2.0 + rng.normal(size=3) * 20.0 for _ in range(12)]
    got = oracle_rmsd.molecules([confs])[0]
    want = np.array([kabsch_rmsd(confs[i], confs[j]) for i in range(12) for j in range(i)])
    assert np.abs(got - want).max() <= 1e-10
    pre = oracle_rmsd.molecules([confs], prealigned=True)[0]
    want_pre = np.array([np.sqrt(((confs[i] - confs[j]) ** 2).sum() / n) for i in range(12) for j in range(i)])
    assert np.abs(pre - want_pre).max() <= 1e-10


def test_oracle_conformer_order_and_empty_molecules():
    rng = np.random.default_rng(1)
    confs = [rng.normal(size=(5, 3)) for _ in range(4)]
    xyz = np.concatenate(confs)
    cas = np.arange(0, 25, 5)
    order = np.array([2, 0, 3, 1])
    got = oracle_rmsd.matrices([0, 0, 1, 5], [5, 5, 5], cas, xyz, conf_order=np.r_[0, order])
    assert [len(g) for g in got] == [0, 0, 6]
    want = oracle_rmsd.molecules([[confs[k] for k in order]])[0]
    assert np.array_equal(got[2], want)


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


def test_argument_checks_run_before_device_work(Chem):
    good = make_mol(Chem, 3, [np.zeros((3, 3))] * 2)
    with pytest.raises(ValueError, match="must not be None"):
        cr.GetConformerRMSMatrix(None)
    with pytest.raises(ValueError, match="index 1 must not be None"):
        cr.GetConformerRMSMatrixBatch([good, None])
    with pytest.raises(TypeError, match="torch.cuda.Stream"):
        cr.GetConformerRMSMatrix(good, stream=1)
    with pytest.raises(TypeError, match="torch.cuda.Stream"):
        cr.GetConformerRMSMatrixBatch([good], stream="s")
    empty = make_mol(Chem, 0, [np.zeros((0, 3))] * 2)
    with pytest.raises(ValueError, match="conformers but no atoms"):
        cr.GetConformerRMSMatrix(empty)
    with pytest.raises(ValueError, match="index 1 has conformers but no atoms"):
        cr.GetConformerRMSMatrixBatch([good, make_mol(Chem, 0, [np.zeros((0, 3))])])
    with pytest.raises(ValueError, match="conformer of 2 atoms"):
        cr.GetConformerRMSMatrixBatch([make_mol(Chem, 3, [np.zeros((3, 3)), np.zeros((2, 3))])])
    assert cr.GetConformerRMSMatrixBatch([]) == []
    with pytest.raises(TypeError, match="Device3DResult"):
        cr.GetConformerRMSMatrixBatch([good], coordinates=object())


def device_result(entries, n_mols):
    """(mol, conf index, [n, 3] coordinates) entries -> a Device3DResult on host tensors."""
    t = lambda a: AsyncGpuResult(torch.as_tensor(np.asarray(a)))  # noqa: E731
    values = np.concatenate([e[2] for e in entries]) if entries else np.zeros((0, 3))
    starts = np.concatenate([[0], np.cumsum([len(e[2]) for e in entries])]).astype(np.int32)
    return Device3DResult(t(values), t(starts), t(np.array([e[0] for e in entries], np.int32)),
                          t(np.array([e[1] for e in entries], np.int32)), 0, n_mols)


def test_device_result_plan_and_checks(Chem):
    z = lambda n: np.zeros((n, 3))  # noqa: E731
    res = device_result([(2, 1, z(4)), (0, 1, z(3)), (2, 0, z(4)), (0, 0, z(3)), (0, 2, z(3))], 3)
    order, counts, _ = device_conformer_order(res, [3, 5, 4])
    assert order.tolist() == [3, 1, 4, 2, 0] and counts.tolist() == [3, 0, 2]
    with pytest.raises(ValueError, match="molecule index out of range"):
        device_conformer_order(res, [3, 5])
    with pytest.raises(ValueError, match="conformer 1 has 3 atoms, molecule 0 has 2"):
        device_conformer_order(res, [2, 5, 4])
    mols = [make_mol(Chem, 3), make_mol(Chem, 5), make_mol(Chem, 4)]
    with pytest.raises(ValueError, match="coordinates hold 3 molecules, mols has 2"):
        cr.GetConformerRMSMatrixBatch(mols[:2], coordinates=res)
    zero = device_result([(0, 0, z(0)), (0, 1, z(0))], 1)
    with pytest.raises(ValueError, match="conformers but no atoms"):
        cr.GetConformerRMSMatrixBatch([make_mol(Chem, 0)], coordinates=zero)


def test_pair_offsets_are_int64_past_int_max():
    off = cr.pair_offsets([0, 1, 2, 70000, 3])
    assert off.dtype == np.int64
    assert off.tolist() == [0, 0, 0, 1, 1 + 70000 * 69999 // 2, 1 + 70000 * 69999 // 2 + 3]
    assert off[-1] > 2**31


def test_c_abi_checks_without_a_device(built_lib):
    """The planning checks and the nothing-to-do cases return before any CUDA call."""
    from nvmolkit_b200 import _lib

    def call(mcs, atoms):
        mcs = np.asarray(mcs, np.int32)
        atoms = np.asarray(atoms, np.int32)
        return built_lib.b200mol_conformer_rmsd(len(atoms), mcs.ctypes.data, atoms.ctypes.data, None, None, None, 0,
                                                None, None)

    assert call([0, 1, 1, 2], [4, 0, 7]) == _lib.B200MOL_OK  # no molecule has a pair: nothing to do
    assert built_lib.b200mol_conformer_rmsd(0, None, None, None, None, None, 0, None, None) == _lib.B200MOL_OK
    assert call([0, 2], [0]) == _lib.ERR_INVALID
    assert b"conformers but no atoms" in built_lib.b200mol_last_error()
    assert call([0, 3, 2], [3, 3]) == _lib.ERR_INVALID
    assert call([0, 2], [-1]) == _lib.ERR_INVALID
    assert call([0, 2, 4], [3, 3]) == _lib.ERR_INVALID  # pairs to compute, but no coordinates or output
