#!/usr/bin/env python
"""Export RDKit-pinned fixtures for the "parity unpinned" rows of DESIGN.md 2 / SURVEY.md 8c.

Run this WHERE RDKIT EXISTS (any RDKit 2025.03 .. 2026.03; no GPU needed):

    python tools/export_rdkit_fixtures.py [--smiles FILE] [--n 64] [--out tests/golden/rdkit_fixtures.npz]

and commit the resulting .npz. `tests/test_rdkit_fixtures.py` then replays it (skipped while the file is absent):
  * Morgan: the flattened molecular graphs + RDKit's own ECFP bits (radius 0..3, 2048 bits)   -> oracle / GPU bit-exact
  * Tanimoto: RDKit BulkTanimotoSimilarity matrix of those bit vectors                         -> bit-exact (fp64)
  * Butina: RDKit ML.Cluster.Butina.ClusterData(reordering=True) on the distance matrix        -> identical clusters
  * Morgan counts: GetCountFingerprintAsNumPy (radius 0..3, 2048 bins), and BulkTanimotoSimilarity /
    BulkDiceSimilarity of the radius-2 count fingerprints (tests/test_count_*.py)              -> bit-exact
  * MMFF / UFF: the flattened term tables (nvmolkit_b200.rdkit_adapter) + RDKit's energies, gradients and 200-iteration
    minimised energies on the same conformers (tests/test_mmff.cu:1521-1608 style)              -> <= 1e-4 relative
  * ETKDG: raw + smoothed bounds matrices, flattened DG / ETK / check tables, RDKit's EmbedMultipleConfs coordinates
    (per-molecule RMSD / bounds-violation statistics are compared, not coordinates)
  * TFD (to tests/golden/rdkit_tfd.npz, replayed by tests/test_tfd.py): RDKit's torsion lists and weights
    (TorsionFingerprints.CalculateTorsionLists / CalculateTorsionWeights) in the flat layout of b200mol_tfd_matrices,
    the tables nvmolkit_b200.tfd.tfd_torsions builds for the same molecules, ETKDG conformers and
    TorsionFingerprints.GetTFDMatrix on them
  * alignment (to tests/golden/rdkit_align.npz, replayed by tests/test_mol_align_rdkit.py): rdMolAlign.AlignMolConformers
    RMS lists and aligned coordinates over all atoms, heavy-atom atomIds, weights and reflect; rdMolAlign.AlignMol RMSDs
    and moved coordinates and GetAlignmentTransform matrices with atom maps, weights and reflect
  * best alignment (to tests/golden/rdkit_best_align.npz, replayed by tests/test_mol_align_best_rdkit.py):
    rdMolAlign.GetBestRMS (RMSD and moved coordinates), CalcRMS and GetBestAlignmentTransform (RMSD, transform, match)
    of every conformer against conformer 0 of a second copy of the molecule, on heavy-atom molecules with ring flips,
    carboxylates and a nitro group, with and without weights and symmetrizeConjugatedTerminalGroups; with each
    molecule's atoms, bonds (conjugation included) and raw GetSubstructMatches, so that the matching restatement
    (nvmolkit_b200.rdkit_adapter.probe_ref_matches) can be replayed without RDKit

The default molecule set is a small drug-like SMILES list embedded below (aspirin, ibuprofen, caffeine, ...); pass
--smiles benchmarks/data/chembl_10k.smi of the reference checkout for the BASELINE configs' real input.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT_SMILES = [
    "CC(=O)OC1=CC=CC=C1C(=O)O", "CC(C)CC1=CC=C(C=C1)C(C)C(=O)O", "CN1C=NC2=C1C(=O)N(C(=O)N2C)C", "CCCCC",
    "O=C(O)CC1CC1", "OCCCCO", "C[C@H](N)C(=O)O", "C1CCC2CCCCC2C1", "CC(=O)NC1=CC=C(O)C=C1", "C/C=C/C(=O)O",
    "CC#CCO", "c1ccc2[nH]ccc2c1", "CN(C)C(=O)c1ccccc1", "OC(=O)[C@@H]1CCCN1", "CCOC(=O)C1=CC=CN=C1", "CS(=O)(=O)Nc1ccccc1",
    "FC(F)(F)c1ccccc1", "CC(C)(C)OC(=O)N1CCNCC1", "O=C1CCCCC1", "NC(=O)c1cccnc1", "CCN(CC)CCOC(=O)c1ccc(N)cc1",
    "Clc1ccc(cc1)C(c1ccccc1)N1CCNCC1", "CC1(C)SC2C(NC(=O)Cc3ccccc3)C(=O)N2C1C(=O)O", "OP(=O)(O)OCC",
]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--smiles", default=None, help="SMILES file (one per line, first column)")
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--confs", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "rdkit_fixtures.npz"))
    args = ap.parse_args()

    import rdkit
    from rdkit import Chem, DataStructs
    from rdkit.Chem import AllChem, rdDistGeom, rdFingerprintGenerator
    from rdkit.Chem import rdForceFieldHelpers as FFH
    from rdkit.ML.Cluster import Butina

    from nvmolkit_b200 import rdkit_adapter as A
    from nvmolkit_b200.embedMolecules import EmbedParameters
    from nvmolkit_b200.molgraph import from_rdkit

    smiles = DEFAULT_SMILES
    if args.smiles:
        smiles = [line.split()[0] for line in open(args.smiles) if line.strip()][: args.n]
    mols = [m for m in (Chem.MolFromSmiles(s) for s in smiles[: args.n]) if m is not None]
    out = {"rdkit_version": np.array(rdkit.__version__), "smiles": np.array([Chem.MolToSmiles(m) for m in mols])}

    # ---- Morgan / Tanimoto / Butina
    g = from_rdkit(mols)
    for k in ("atom_starts", "bond_starts", "atom_inv", "bond_inv", "bond_a", "bond_b"):
        out[f"graph_{k}"] = getattr(g, k)
    fps = None
    for radius in range(4):
        gen = rdFingerprintGenerator.GetMorganGenerator(radius=radius, fpSize=2048)
        bvs = [gen.GetFingerprint(m) for m in mols]
        bits = np.zeros((len(mols), 2048), dtype=bool)
        for i, bv in enumerate(bvs):
            bits[i, list(bv.GetOnBits())] = True
        out[f"morgan_bits_r{radius}"] = np.packbits(bits, axis=1, bitorder="little").view(np.uint32)
        if radius == 2:
            fps = bvs
    n = len(mols)
    sim = np.array([DataStructs.BulkTanimotoSimilarity(fps[i], fps) for i in range(n)])
    out["tanimoto_r2"] = sim
    dists = [1.0 - sim[i, j] for i in range(1, n) for j in range(i)]  # RDKit's lower-triangle order
    for cutoff in (0.3, 0.6):
        clusters = Butina.ClusterData(dists, n, cutoff, isDistData=True, reordering=True)
        ids = np.full(n, -1, dtype=np.int32)
        for c, members in enumerate(clusters):
            ids[list(members)] = c
        key = str(cutoff).replace(".", "p")
        out[f"butina_ids_{key}"] = ids
        out[f"butina_centroids_{key}"] = np.array([c[0] for c in clusters], dtype=np.int32)

    # ---- Morgan counts, and Tanimoto / Dice on count vectors (tests/test_count_fingerprints.py, _similarity.py)
    for radius in range(4):
        gen = rdFingerprintGenerator.GetMorganGenerator(radius=radius, fpSize=2048)
        out[f"morgan_counts_r{radius}"] = np.stack([gen.GetCountFingerprintAsNumPy(m) for m in mols]).astype(np.int32)
    cfps = [rdFingerprintGenerator.GetMorganGenerator(radius=2, fpSize=2048).GetCountFingerprint(m) for m in mols]
    out["count_tanimoto_r2"] = np.array([DataStructs.BulkTanimotoSimilarity(cfps[i], cfps) for i in range(n)])
    out["count_dice_r2"] = np.array([DataStructs.BulkDiceSimilarity(cfps[i], cfps) for i in range(n)])

    # ---- conformers, MMFF / UFF
    hmols = []
    for m in mols:
        mh = Chem.AddHs(m)
        p = rdDistGeom.ETKDGv3()
        p.randomSeed = 42
        p.useRandomCoords = True
        if (len(rdDistGeom.EmbedMultipleConfs(mh, args.confs, p)) == args.confs and FFH.MMFFHasAllMoleculeParams(mh)
                and FFH.UFFHasAllMoleculeParams(mh)):
            hmols.append(mh)
    out["ff_smiles"] = np.array([Chem.MolToSmiles(m) for m in hmols])
    for kind, flatten in (("mmff", A.mmff_from_rdkit), ("uff", A.uff_from_rdkit)):
        flat = flatten(hmols)
        out[f"{kind}_atom_counts"] = flat.system.atom_counts
        for name, (st, ix, pr) in flat.system.tables.items():
            out[f"{kind}_{name}_starts"], out[f"{kind}_{name}_idx"], out[f"{kind}_{name}_par"] = st, ix, pr
        out[f"{kind}_conf_mol"], out[f"{kind}_atom_starts"], out[f"{kind}_positions"] = flat.batch.conf_mol, flat.batch.atom_starts, flat.batch.positions
        e0, grads, e_min = [], [], []
        for m in hmols:
            props = FFH.MMFFGetMoleculeProperties(m) if kind == "mmff" else None
            for conf in m.GetConformers():
                ff = (FFH.MMFFGetMoleculeForceField(m, props, confId=conf.GetId()) if kind == "mmff"
                      else FFH.UFFGetMoleculeForceField(m, confId=conf.GetId()))
                e0.append(ff.CalcEnergy())
                grads.append(np.array(ff.CalcGrad()).reshape(-1, 3))
            work = Chem.Mol(m)
            res = (FFH.MMFFOptimizeMoleculeConfs(work, maxIters=200) if kind == "mmff"
                   else FFH.UFFOptimizeMoleculeConfs(work, maxIters=1000))
            e_min += [[conv, e] for conv, e in res]
        out[f"{kind}_rdkit_energy"] = np.array(e0)
        out[f"{kind}_rdkit_grad"] = np.concatenate(grads)
        out[f"{kind}_rdkit_minimised"] = np.array(e_min)  # [not-converged flag, energy] per conformer

    # ---- ETKDG inputs and RDKit's own embedding of the same molecules
    params = EmbedParameters()
    raw, smooth = [], []
    for m in hmols:
        raw.append(np.asarray(rdDistGeom.GetMoleculeBoundsMatrix(m, doTriangleSmoothing=False), dtype=np.float64).ravel())
        smooth.append(np.asarray(rdDistGeom.GetMoleculeBoundsMatrix(m, doTriangleSmoothing=True), dtype=np.float64).ravel())
    out["bounds_raw"], out["bounds_smoothed"] = np.concatenate(raw), np.concatenate(smooth)
    out["bounds_starts"] = np.concatenate([[0], np.cumsum([len(b) for b in raw])])
    try:  # the adapter smooths on the GPU; substitute RDKit's own smoothing so the export needs no GPU
        import nvmolkit_b200.dgprep as dgprep

        def rdkit_smooth(mats, tol=0.0):
            done = [np.asarray(rdDistGeom.GetMoleculeBoundsMatrix(m, doTriangleSmoothing=True)) for m in hmols]
            return done, [True] * len(done)

        dgprep.triangle_smooth = rdkit_smooth
        flat = A.embed_molecules_from_rdkit(hmols, params)
        for sysname, system in (("dg", flat.dg), ("etk", flat.etk)):
            for name, (st, ix, pr) in system.tables.items():
                out[f"{sysname}_{name}_starts"], out[f"{sysname}_{name}_idx"], out[f"{sysname}_{name}_par"] = st, ix, pr
        for name, (st, ix, pr) in flat.checks.tables.items():
            out[f"check_{name}_starts"], out[f"check_{name}_idx"], out[f"check_{name}_par"] = st, ix, pr
        out["check_num_impropers"] = flat.checks.num_impropers
    except Exception as e:  # keep the rest of the export usable
        out["etkdg_export_error"] = np.array(repr(e))
    out["rdkit_embedded_positions"] = np.concatenate([c.GetPositions() for m in hmols for c in m.GetConformers()])
    np.savez_compressed(args.out, **out)
    print(f"wrote {args.out}: {len(mols)} molecules, {len(hmols)} with conformers, RDKit {rdkit.__version__}")
    export_tfd(hmols, os.path.join(os.path.dirname(os.path.abspath(args.out)), "rdkit_tfd.npz"))
    export_align(hmols, os.path.join(os.path.dirname(os.path.abspath(args.out)), "rdkit_align.npz"))
    export_best_align(os.path.join(os.path.dirname(os.path.abspath(args.out)), "rdkit_best_align.npz"))


def export_tfd(hmols, path: str, n_confs: int = 6) -> None:
    """RDKit's TFD inputs and matrices (weights on, maxDev 'equal', symmRadius 2, colinear bonds ignored)."""
    import rdkit
    from rdkit import Chem
    from rdkit.Chem import TorsionFingerprints as TF
    from rdkit.Chem import rdDistGeom

    from nvmolkit_b200 import tfd

    mols, per_mol, coords, matrices = [], [], [], []
    for m in hmols:
        mh = Chem.Mol(m)
        mh.RemoveAllConformers()
        p = rdDistGeom.ETKDGv3()
        p.randomSeed = 7
        if len(rdDistGeom.EmbedMultipleConfs(mh, n_confs, p)) < 2:
            continue
        tl, tlr = TF.CalculateTorsionLists(mh, maxDev="equal", symmRadius=2, ignoreColinearBonds=True)
        weights = TF.CalculateTorsionWeights(mh, ignoreColinearBonds=True) if (tl or tlr) else []
        tors = [([tuple(q) for q in quartets], tfd.SYMMETRIC if len(quartets) > 1 else tfd.SINGLE, 1.0, float(md))
                for quartets, md in tl]
        tors += [([tuple(q) for q in quartets], tfd.RING, 1.0, float(md)) for quartets, md in tlr]
        tors = [(q, t, float(w), md) for (q, t, _w, md), w in zip(tors, weights)] if len(weights) == len(tors) else tors
        mols.append(mh)
        per_mol.append(tors)
        coords.append([c.GetPositions() for c in mh.GetConformers()])
        matrices.append(np.asarray(TF.GetTFDMatrix(mh, useWeights=True, maxDev="equal"), np.float64))
    ref = tfd.TFDTorsions.from_lists(per_mol)
    flat = tfd.FlatTFDMolecules.from_coordinates(ref, coords)
    ours = tfd.tfd_torsions(mols)
    out = {"rdkit_version": np.array(rdkit.__version__), "smiles": np.array([Chem.MolToSmiles(m) for m in mols]),
           "mol_conf_start": flat.mol_conf_start, "conf_atom_start": flat.conf_atom_start, "xyz": flat.xyz,
           "tfd": np.concatenate(matrices) if matrices else np.zeros(0), "tfd_sizes": np.array([len(x) for x in matrices])}
    for k in ("tors_start", "quartet_start", "quartets", "type", "weight", "maxdev"):
        out[k] = getattr(ref, k)
        out[f"adapter_{k}"] = getattr(ours, k)
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(mols)} molecules")


def export_align(hmols, path: str, n_confs: int = 5) -> None:
    """RDKit's alignment on ETKDG conformers. AlignMolConformers case k: ``amc{k}_before`` / ``_after`` [C, n, 3],
    ``_rms`` [C - 1], ``_atomids`` (empty: all atoms), ``_weights`` (empty: none), ``_reflect``. AlignMol /
    GetAlignmentTransform case k: ``am{k}_prb``, ``_ref``, ``_map`` [L, 2], ``_weights``, ``_reflect``, ``_rmsd``,
    ``_transform`` [4, 4] and ``_moved`` (the probe after AlignMol)."""
    import rdkit
    from rdkit import Chem
    from rdkit.Chem import rdDistGeom, rdMolAlign

    out = {"rdkit_version": np.array(rdkit.__version__)}
    rng = np.random.default_rng(5)
    k = j = 0
    confmols = []
    for m in hmols:
        mh = Chem.Mol(m)
        mh.RemoveAllConformers()
        p = rdDistGeom.ETKDGv3()
        p.randomSeed = 11
        if len(rdDistGeom.EmbedMultipleConfs(mh, n_confs, p)) < 2:
            continue
        confmols.append(mh)
        n = mh.GetNumAtoms()
        heavy = [a.GetIdx() for a in mh.GetAtoms() if a.GetAtomicNum() > 1]
        for ids, weighted, reflect in ((None, False, False), (heavy, False, False), (None, True, False),
                                       (heavy, True, True)):
            work = Chem.Mol(mh)
            L = n if ids is None else len(ids)
            w = rng.uniform(0.5, 2.0, L).tolist() if weighted else []
            out[f"amc{k}_before"] = np.array([c.GetPositions() for c in work.GetConformers()])
            rms = []
            rdMolAlign.AlignMolConformers(work, atomIds=ids or [], weights=w, reflect=reflect, RMSlist=rms)
            out[f"amc{k}_after"] = np.array([c.GetPositions() for c in work.GetConformers()])
            out[f"amc{k}_rms"], out[f"amc{k}_atomids"] = np.array(rms), np.array(ids or [], np.int64)
            out[f"amc{k}_weights"], out[f"amc{k}_reflect"] = np.array(w, np.float64), np.array(reflect)
            k += 1
    for a, b in zip(confmols, confmols[1:] + confmols[:1]):  # a probe onto another molecule through a heavy-atom map
        L = min(a.GetNumHeavyAtoms(), b.GetNumHeavyAtoms(), 8)
        amap = list(zip(rng.permutation([x.GetIdx() for x in a.GetAtoms() if x.GetAtomicNum() > 1])[:L].tolist(),
                        rng.permutation([x.GetIdx() for x in b.GetAtoms() if x.GetAtomicNum() > 1])[:L].tolist()))
        for weighted, reflect in ((False, False), (True, False), (True, True)):
            w = rng.uniform(0.5, 2.0, L).tolist() if weighted else []
            prb = Chem.Mol(a)
            rmsd, T = rdMolAlign.GetAlignmentTransform(prb, b, atomMap=amap, weights=w, reflect=reflect)
            out[f"am{j}_prb"], out[f"am{j}_ref"] = prb.GetConformer().GetPositions(), b.GetConformer().GetPositions()
            out[f"am{j}_map"], out[f"am{j}_weights"] = np.array(amap, np.int64), np.array(w, np.float64)
            out[f"am{j}_reflect"], out[f"am{j}_transform"] = np.array(reflect), np.asarray(T, np.float64)
            out[f"am{j}_rmsd"] = np.array(rdMolAlign.AlignMol(prb, b, atomMap=amap, weights=w, reflect=reflect))
            out[f"am{j}_moved"] = prb.GetConformer().GetPositions()
            if abs(float(out[f"am{j}_rmsd"]) - rmsd) > 1e-12:
                raise RuntimeError("AlignMol and GetAlignmentTransform disagree")
            j += 1
    out["n_amc"], out["n_am"] = np.array(k), np.array(j)
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {k} AlignMolConformers and {j} AlignMol cases")


BEST_ALIGN_SMILES = ["[O-]C(=O)c1ccccc1", "CC(C)(C)c1ccc(cc1)C(=O)[O-]", "Cc1ccc(cc1)[N+](=O)[O-]", "OC(=O)CC1CC1",
                     "c1ccc(cc1)-c1ccccc1", "CC(=O)Oc1ccccc1C(=O)O", "OC(=O)[C@@H]1CCCN1"]


def export_best_align(path: str, n_confs: int = 4, max_matches: int = 1000000) -> None:
    """RDKit's GetBestRMS / CalcRMS / GetBestAlignmentTransform on heavy-atom ETKDG conformers. Molecule i:
    ``bam{i}_z`` [n], ``_bonds`` [B, 3] (begin, end, conjugated), ``_raw`` [M, n] (``GetSubstructMatches(mol,
    uniquify=False, maxMatches, useChirality=False)``), ``_xyz`` [C, n, 3]. Case j: ``ba{j}_mol``, ``_conf`` (the probe
    conformer; the reference is conformer 0 of a second copy), ``_sym``, ``_weights`` (empty: none), ``_calc``
    (CalcRMS), ``_trmsd`` / ``_transform`` / ``_match`` [L, 2] (GetBestAlignmentTransform), ``_rmsd`` / ``_moved``
    (GetBestRMS and the probe conformer after it)."""
    import rdkit
    from rdkit import Chem
    from rdkit.Chem import rdDistGeom, rdMolAlign

    out = {"rdkit_version": np.array(rdkit.__version__), "max_matches": np.array(max_matches)}
    rng = np.random.default_rng(7)
    i = j = 0
    for smi in BEST_ALIGN_SMILES:
        mh = Chem.AddHs(Chem.MolFromSmiles(smi))
        p = rdDistGeom.ETKDGv3()
        p.randomSeed = 13
        if len(rdDistGeom.EmbedMultipleConfs(mh, n_confs, p)) < 2:
            continue
        m = Chem.RemoveHs(mh)
        n = m.GetNumAtoms()
        ids = [c.GetId() for c in m.GetConformers()]
        out[f"bam{i}_z"] = np.array([a.GetAtomicNum() for a in m.GetAtoms()], np.int64)
        out[f"bam{i}_bonds"] = np.array([(b.GetBeginAtomIdx(), b.GetEndAtomIdx(), int(b.GetIsConjugated()))
                                         for b in m.GetBonds()], np.int64).reshape(-1, 3)
        out[f"bam{i}_raw"] = np.array(m.GetSubstructMatches(m, uniquify=False, maxMatches=max_matches,
                                                            useChirality=False), np.int64).reshape(-1, n)
        out[f"bam{i}_xyz"] = np.array([m.GetConformer(c).GetPositions() for c in ids])
        for sym, weighted in ((True, False), (False, False), (True, True), (False, True)):
            w = rng.uniform(0.5, 2.0, n).tolist() if weighted else []
            kw = dict(maxMatches=max_matches, symmetrizeConjugatedTerminalGroups=sym, weights=w)
            for c in range(1, len(ids)):
                prb, ref = Chem.Mol(m), Chem.Mol(m)  # conformers of one molecule read as two objects
                out[f"ba{j}_mol"], out[f"ba{j}_conf"] = np.array(i), np.array(c)
                out[f"ba{j}_sym"], out[f"ba{j}_weights"] = np.array(sym), np.array(w, np.float64)
                out[f"ba{j}_calc"] = np.array(rdMolAlign.CalcRMS(prb, ref, ids[c], ids[0], **kw))
                rmsd, T, match = rdMolAlign.GetBestAlignmentTransform(prb, ref, ids[c], ids[0], **kw)
                out[f"ba{j}_trmsd"], out[f"ba{j}_transform"] = np.array(rmsd), np.asarray(T, np.float64)
                out[f"ba{j}_match"] = np.array(match, np.int64).reshape(-1, 2)
                out[f"ba{j}_rmsd"] = np.array(rdMolAlign.GetBestRMS(prb, ref, ids[c], ids[0], **kw))
                out[f"ba{j}_moved"] = prb.GetConformer(ids[c]).GetPositions()
                j += 1
        i += 1
    out["n_bam"], out["n_ba"] = np.array(i), np.array(j)
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {i} molecules, {j} best-alignment cases")


if __name__ == "__main__":
    main()
