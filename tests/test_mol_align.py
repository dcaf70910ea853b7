"""Conformer alignment on the CPU: the fp64 oracle (oracle_align.c, RDKit's AlignPoints restated) against a NumPy SVD
Kabsch and known answers, every argument refusal of ``nvmolkit_b200.molAlign`` before device work, and the C-ABI's host
checks of ``b200mol_align`` without a device."""
import os
import re
import sys

import numpy as np
import pytest

from nvmolkit_b200 import _lib
from nvmolkit_b200 import molAlign as ma
from oracle import align as oa

FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")
Chem = None


@pytest.fixture(autouse=True)
def fake_rdkit(monkeypatch):
    """The stand-in RDKit of tests/fake_rdkit for the duration of one test."""
    global Chem
    monkeypatch.syspath_prepend(FAKE)
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        monkeypatch.delitem(sys.modules, name)
    from rdkit import Chem as chem

    Chem = chem
    yield
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        sys.modules.pop(name, None)


def kabsch(p, q, w=None, reflect=False):
    """(RMSD over L pairs, R, t) of the weighted best superposition of p (negated when reflect) onto q, by SVD."""
    w = np.ones(len(p)) if w is None else np.asarray(w, np.float64)
    p = -p if reflect else p
    pb, qb = (w[:, None] * p).sum(0) / w.sum(), (w[:, None] * q).sum(0) / w.sum()
    P, Q = p - pb, q - qb
    u, _, vt = np.linalg.svd((w[:, None] * P).T @ Q)
    R = vt.T @ np.diag([1.0, 1.0, np.sign(np.linalg.det(vt.T @ u.T))]) @ u.T
    return np.sqrt((w * ((P @ R.T - Q) ** 2).sum(1)).sum() / len(p)), R, qb - R @ pb


def rotation(rng):
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1.0
    return q


# ------------------------------------------------------------------ oracle
@pytest.mark.parametrize("L", [3, 4, 10, 50])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("reflect", [False, True])
def test_oracle_is_the_svd_kabsch(L, weighted, reflect):
    rng = np.random.default_rng(L + 7 * weighted + 13 * reflect)
    for _ in range(5):
        p, q = rng.normal(size=(L, 3)) * 2.0 + 5.0, rng.normal(size=(L, 3)) * 2.0 - 3.0
        w = rng.uniform(0.1, 2.0, L) if weighted else None
        got, T = oa.align(p, q, weights=w, reflect=reflect)
        want, R, t = kabsch(p, q, w, reflect)
        assert abs(got - want) <= 1e-12 * (1 + want)
        assert np.abs(T[:3, :3] - (-R if reflect else R)).max() <= 1e-12
        assert np.abs(T[:3, 3] - t).max() <= 1e-10
        assert T[3].tolist() == [0.0, 0.0, 0.0, 1.0]


def test_rigid_copy_recovers_the_motion():
    rng = np.random.default_rng(1)
    ref = rng.normal(size=(12, 3)) * 2.0
    R, t = rotation(rng), rng.normal(size=3) * 10.0
    prb = (ref - t) @ R  # ref = R prb + t
    rmsd, T = oa.align(prb, ref)
    assert rmsd <= 1e-7
    assert np.abs(T[:3, :3] - R).max() <= 1e-12 and np.abs(T[:3, 3] - t).max() <= 1e-10
    assert np.abs(oa.apply(T, prb) - ref).max() <= 1e-10


def test_mirror_image_needs_reflect():
    rng = np.random.default_rng(2)
    ref = rng.normal(size=(10, 3)) * 2.0
    prb = (-ref) @ rotation(rng).T + 3.0
    assert oa.align(prb, ref, reflect=True)[0] <= 1e-7
    assert oa.align(prb, ref)[0] > 0.1
    _, T = oa.align(prb, ref, reflect=True)
    assert np.linalg.det(T[:3, :3]) < 0 and np.abs(oa.apply(T, prb) - ref).max() <= 1e-10


def test_zero_weights_drop_atoms_and_scale_by_the_pair_count():
    rng = np.random.default_rng(3)
    p, q = rng.normal(size=(20, 3)), rng.normal(size=(20, 3))
    w = np.ones(20)
    w[[1, 4, 5, 11, 19]] = 0.0
    keep = w > 0
    full, T = oa.align(p, q, weights=w)
    part, T2 = oa.align(p[keep], q[keep])
    assert abs(full - part * np.sqrt(keep.sum() / 20)) <= 1e-12
    assert np.abs(T - T2).max() <= 1e-12


def test_far_from_the_origin_changes_nothing():
    rng = np.random.default_rng(4)
    p, q = rng.normal(size=(30, 3)) * 2.0, rng.normal(size=(30, 3)) * 2.0
    w = rng.uniform(0.5, 1.5, 30)
    near, T = oa.align(p, q, weights=w)
    shift = np.array([1e4, -1e4, 1e4])
    far, Tf = oa.align(p + shift, q + shift, weights=w)
    assert abs(near - far) <= 1e-10
    assert np.abs(T[:3, :3] - Tf[:3, :3]).max() <= 1e-10


def test_one_pair_is_the_identity_rotation():
    rmsd, T = oa.align(np.array([[1.0, 2.0, 3.0], [9.0, 9.0, 9.0]]), np.array([[-4.0, 0.5, 7.0]]), pairs=[[0, 0]])
    assert rmsd == 0.0 and np.array_equal(T[:3, :3], np.eye(3))
    assert np.allclose(T[:3, 3], [-5.0, -1.5, 4.0])


def test_max_iters_caps_the_sweeps():
    rng = np.random.default_rng(5)
    p, q = rng.normal(size=(15, 3)), rng.normal(size=(15, 3))
    conv = oa.align(p, q, maxIters=50)[0]
    assert oa.align(p, q, maxIters=1)[0] != conv
    assert oa.align(p, q, maxIters=1000)[0] == conv


def test_pair_lists_are_shared_by_key():
    lists = ma.PairLists()
    a = lists.add([[0, 1], [2, 3]], None, key="a")
    b = lists.add([[1, 1]], np.array([2.0]))
    assert lists.add([[5, 5]], None, key="a") == a and lists.find("a") == a and lists.find("x") is None
    start, pairs, w = lists.tables()
    assert start.tolist() == [0, 2, 3] and pairs.tolist() == [[0, 1], [2, 3], [1, 1]] and w.tolist() == [1, 1, 2]
    assert b == 1 and lists.max_atoms(a) == (2, 3)


# ------------------------------------------------------------------ refusals before device work
def mol(n=4, confs=2, seed=0):
    rng = np.random.default_rng(seed)
    d = {"z": [6] * n, "bonds": [(i, i + 1) for i in range(n - 1)], "nbrs": [[] for _ in range(n)]}
    return Chem.Mol(d, conformers=[rng.normal(size=(n, 3)) for _ in range(confs)])


@pytest.mark.parametrize("kw,msg", [
    ({"maxIters": 0}, "maxIters must be >= 1"),
    ({"atomIds": []}, "non-empty"),
    ({"atomIds": [0, 0]}, "twice"),
    ({"atomIds": [4]}, "outside"),
    ({"atomIds": [-1]}, "outside"),
    ({"weights": [1.0] * 3}, "holds 3 weights, 4 expected"),
    ({"atomIds": [0, 1], "weights": [1.0] * 4}, "holds 4 weights, 2 expected"),
    ({"weights": [1.0, -1.0, 1.0, 1.0]}, "finite and >= 0"),
    ({"weights": [1.0, np.nan, 1.0, 1.0]}, "finite and >= 0"),
    ({"weights": [0.0] * 4}, "sum to 0"),
    ({"confIds": [0, 7]}, "no conformer with id 7"),
    ({"confIds": [1, 1]}, "twice"),
])
def test_align_mol_conformers_refusals(kw, msg):
    m = mol()
    before = [c.GetPositions().copy() for c in m.GetConformers()]
    with pytest.raises(ValueError, match=msg):
        ma.AlignMolConformers(m, **kw)
    assert all(np.array_equal(b, c.GetPositions()) for b, c in zip(before, m.GetConformers()))


def test_batch_refusals():
    m = mol()
    with pytest.raises(ValueError, match="must not be None"):
        ma.AlignMolConformers(None)
    with pytest.raises(ValueError, match="must not be None"):
        ma.AlignMolConformersBatch([m, None])
    with pytest.raises(ValueError, match="atomIds holds 1 entries"):
        ma.AlignMolConformersBatch([m, m], atomIds=[[0]])
    with pytest.raises(TypeError):
        ma.AlignMolConformers(m, stream=0)
    with pytest.raises(TypeError):
        ma.AlignMolConformersBatch([m], coordinates=np.zeros((8, 3)))
    # fewer than two conformers is a no-op, without a device
    one = mol(confs=1)
    rms = []
    ma.AlignMolConformers(one, RMSlist=rms)
    assert rms == []
    assert ma.AlignMolConformersBatch([one, mol(confs=3)], confIds=[None, [2]])[1].torch().numel() == 0


@pytest.mark.parametrize("kw,msg", [
    ({"maxIters": 0}, "maxIters must be >= 1"),
    ({"prbCid": 5}, "no conformer with id 5"),
    ({"refCid": 5}, "no conformer with id 5"),
    ({"atomMap": [(0, 0), (0, 1)]}, "twice"),
    ({"atomMap": [(0, 0), (1, 9)]}, "outside"),
    ({"atomMap": [(0, 0, 0)]}, "pairs"),
    ({"atomMap": [(0, 0), (1, 1)], "weights": [1.0]}, "holds 1 weights, 2 expected"),
    ({"weights": [-1.0, 1.0, 1.0, 1.0]}, "finite and >= 0"),
])
def test_align_mol_refusals(kw, msg):
    prb, ref = mol(seed=1), mol(seed=2)
    for fn in (ma.AlignMol, ma.GetAlignmentTransform):
        with pytest.raises(ValueError, match=msg):
            fn(prb, ref, **kw)


def test_align_mol_batch_refusals():
    prb, ref = mol(seed=1), mol(seed=2)
    with pytest.raises(ValueError, match="identity needs equal atom counts"):
        ma.AlignMol(mol(n=5), ref)
    with pytest.raises(ValueError, match="has no conformers"):
        ma.AlignMol(mol(confs=0), ref)
    with pytest.raises(ValueError, match="must not be None"):
        ma.AlignMolBatch([prb, None], [ref, ref])
    with pytest.raises(ValueError, match="refMols holds 1"):
        ma.AlignMolBatch([prb, prb], [ref])
    with pytest.raises(ValueError, match="moved twice or is also a reference"):
        ma.AlignMolBatch([prb, prb], [ref, ref])
    with pytest.raises(ValueError, match="moved twice or is also a reference"):
        ma.AlignMolBatch([prb, ref], [ref, prb], prbCids=[0, 0], refCids=[0, 0])
    with pytest.raises(TypeError):
        ma.GetAlignmentTransformBatch([prb], [ref], stream=0)
    amap = [(0, 0), (3, 3)]  # one map object on molecules too small for it
    with pytest.raises(ValueError, match="outside its molecules"):
        ma.GetAlignmentTransformBatch([prb, mol(n=2)], [ref, mol(n=2)], atomMaps=[amap, amap])


def test_rdkit_positional_order_is_kept():
    import inspect

    names = lambda f: [p.name for p in inspect.signature(f).parameters.values()]  # noqa: E731
    assert names(ma.AlignMolConformers)[:7] == ["mol", "atomIds", "confIds", "weights", "reflect", "maxIters", "RMSlist"]
    assert names(ma.AlignMol)[:8] == ["prbMol", "refMol", "prbCid", "refCid", "atomMap", "weights", "reflect", "maxIters"]
    assert names(ma.GetAlignmentTransform)[:8] == names(ma.AlignMol)[:8]


# ------------------------------------------------------------------ C-ABI checks without a device
def call_align(probe, ref, lst, conf_atoms, start, pairs, weights=None, maxIters=50, move=1):
    probe, ref, lst, conf_atoms = (np.asarray(x, np.int32) for x in (probe, ref, lst, conf_atoms))
    start, pairs = np.asarray(start, np.int64), np.asarray(pairs, np.int32).reshape(-1)
    w = None if weights is None else np.asarray(weights, np.float64)
    return _lib.call("b200mol_align", len(probe), probe.ctypes.data, ref.ctypes.data, lst.ctypes.data, len(conf_atoms),
                     conf_atoms.ctypes.data, None, None, len(start) - 1, start.ctypes.data, pairs.ctypes.data,
                     None if w is None else w.ctypes.data, 0, maxIters, move, None, None, None)


GOOD = dict(probe=[1, 2], ref=[0, 0], lst=[0, 0], conf_atoms=[3, 3, 3], start=[0, 2], pairs=[0, 0, 2, 2])


@pytest.mark.parametrize("change,msg", [
    ({"maxIters": 0}, "maxIters must be >= 1"),
    ({"start": [0, 0], "pairs": []}, "pair list 0 is empty"),
    ({"start": [1, 2]}, "must start at 0"),
    ({"pairs": [0, 0, 3, 2]}, "holds probe atom 3, conformer 1 has 3 atoms"),
    ({"pairs": [0, 0, 2, 3]}, "holds reference atom 3, conformer 0 has 3 atoms"),
    ({"pairs": [0, -1, 2, 2]}, "negative atom index"),
    ({"weights": [1.0, -0.5]}, "weight -0.5 must be finite and >= 0"),
    ({"weights": [1.0, np.inf]}, "must be finite and >= 0"),
    ({"weights": [0.0, 0.0]}, "its weights sum to 0"),
    ({"probe": [1, 3]}, "job 1: conformer outside [0, 3)"),
    ({"lst": [0, 1]}, "job 1: pair list 1 outside [0, 1)"),
    ({"conf_atoms": [3, 3, -1]}, "conformer 2: negative atom count"),
    ({"probe": [1, 1]}, "job 1: probe conformer 1 is moved by an earlier job too"),
    ({"probe": [1, 0], "ref": [0, 2]}, "job 1: probe conformer 0 is also a reference"),
    ({"probe": [0, 1], "ref": [1, 2]}, "job 1: probe conformer 1 is also a reference"),
])
def test_c_abi_refuses_bad_tables(built_lib, change, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        call_align(**{**GOOD, **change})


def test_c_abi_checks_pass_before_device_pointers(built_lib):
    # valid tables reach the device-pointer check; overlap is allowed when nothing moves
    with pytest.raises(ValueError, match="null device pointer"):
        call_align(**GOOD)
    with pytest.raises(ValueError, match="null device pointer"):
        call_align(**{**GOOD, "probe": [1, 1], "ref": [1, 0]}, move=0)
    call_align([], [], [], [], [0], [])  # no jobs: nothing to do
