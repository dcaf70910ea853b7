"""Replays tests/golden/rdkit_align.npz (written by tools/export_rdkit_fixtures.py where RDKit exists) against the oracle
on the CPU and against nvmolkit_b200.molAlign on the GPU. This pins the points the alignment restates from RDKit's
source: the RMSD divided by the pair count when weights are given, and the reflect convention. Skipped while the file
is absent."""
import os
import sys

import numpy as np
import pytest

from oracle import align as oa

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rdkit_align.npz")
FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")
pytestmark = pytest.mark.skipif(not os.path.exists(PATH), reason="tests/golden/rdkit_align.npz has not been exported")


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(PATH))


def amc_cases(fx):
    for k in range(int(fx["n_amc"])):
        before = fx[f"amc{k}_before"]
        ids = fx[f"amc{k}_atomids"]
        ids = np.arange(before.shape[1]) if len(ids) == 0 else ids
        w = fx[f"amc{k}_weights"]
        yield k, before, ids, (w if len(w) else None), bool(fx[f"amc{k}_reflect"])


def am_cases(fx):
    for j in range(int(fx["n_am"])):
        w = fx[f"am{j}_weights"]
        yield j, fx[f"am{j}_prb"], fx[f"am{j}_ref"], fx[f"am{j}_map"], (w if len(w) else None), bool(fx[f"am{j}_reflect"])


def test_oracle_replays_align_mol_conformers(fx):
    for k, before, ids, w, reflect in amc_cases(fx):
        pairs = np.stack([ids, ids], 1)
        for c in range(1, len(before)):
            rmsd, T = oa.align(before[c], before[0], pairs, w, reflect)
            assert abs(rmsd - fx[f"amc{k}_rms"][c - 1]) <= 1e-8, (k, c)
            assert np.abs(oa.apply(T, before[c]) - fx[f"amc{k}_after"][c]).max() <= 1e-6, (k, c)


def test_oracle_replays_align_mol(fx):
    for j, prb, ref, amap, w, reflect in am_cases(fx):
        rmsd, T = oa.align(prb, ref, amap, w, reflect)
        assert abs(rmsd - float(fx[f"am{j}_rmsd"])) <= 1e-8, j
        assert np.abs(T - fx[f"am{j}_transform"]).max() <= 1e-6, j
        assert np.abs(oa.apply(T, prb) - fx[f"am{j}_moved"]).max() <= 1e-6, j


@pytest.mark.gpu
def test_library_replays_rdkit(fx, cuda, monkeypatch):
    monkeypatch.syspath_prepend(FAKE)
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        monkeypatch.delitem(sys.modules, name)
    from rdkit import Chem

    from nvmolkit_b200 import molAlign as ma

    mk = lambda confs: Chem.Mol({"z": [6] * len(confs[0]), "bonds": [], "nbrs": [[] for _ in confs[0]]},  # noqa: E731
                                conformers=list(confs))
    for k, before, ids, w, reflect in amc_cases(fx):
        mol, rms = mk(before), []
        ma.AlignMolConformers(mol, atomIds=ids.tolist(), weights=w, reflect=reflect, RMSlist=rms)
        assert np.abs(np.array(rms) - fx[f"amc{k}_rms"]).max() <= 1e-8, k
        after = np.array([c.GetPositions() for c in mol.GetConformers()])
        assert np.abs(after - fx[f"amc{k}_after"]).max() <= 1e-6, k
    for j, prb, ref, amap, w, reflect in am_cases(fx):
        rmsd, T = ma.GetAlignmentTransform(mk([prb]), mk([ref]), atomMap=amap.tolist(), weights=w, reflect=reflect)
        assert abs(rmsd - float(fx[f"am{j}_rmsd"])) <= 1e-8 and np.abs(T - fx[f"am{j}_transform"]).max() <= 1e-6, j
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        sys.modules.pop(name, None)
