"""RDKit -> flat-table adapters (the CPU seam above the C-ABI; SURVEY.md 8 rows a1 / a8 / a13 / a17).

Imported only when RDKit molecules are handed to the public API; RDKit itself is imported lazily, so the package works
without it on pre-flattened inputs. RDKit is absent from the container this repository was built in. The module is
written against RDKit's documented Python API (2025.03 .. 2026.03) and is EXECUTED in tests/test_rdkit_adapter.py
against a small stand-in package that implements exactly the calls used here on the synthetic pseudo-molecules
(tests/fake_rdkit) - that pins the plumbing (index conventions, table layouts, error contracts), not RDKit's chemistry:
parity against a live RDKit stays unpinned until tools/export_rdkit_fixtures.py has been run where RDKit exists.

What it mirrors:
 * MMFF - ``MMFF::constructForcefieldContribs`` (rdkit_extensions/mmff_flattened_builder.cpp:453-556): bond, angle,
   stretch-bend, out-of-plane, torsion terms by topology; van der Waals and electrostatic pairs for every atom pair three
   or more bonds apart (1-4 pairs flagged) within ``nonBondedThreshold`` of the conformer geometry. One term block per
   molecule is shared by all its conformers (include/b200mol.h), so the pair list is the UNION over the molecule's
   conformers (the reference builds one list per conformer; at the default threshold of 100 A the two coincide).
 * UFF - ``UFF::constructForcefieldContribs`` (rdkit_extensions/uff_flattened_builder.cpp:142-560) through
   ``rdForceFieldHelpers.GetUFF*Params``: angle orders and C0..C2 by the centre's hybridisation (3- / 4-ring special
   angles included, force constant rescaled to the special theta0), torsion order / cosine term by the central bond's
   hybridisations (``calcTorsionParams``, :88-140), inversion coefficients by element, van der Waals threshold
   ``vdwThresh * x_ij``.
 * ETKDG - ``prepareEmbedderArgs`` (src/embedder_utils.cpp:671-708): RDKit's topological bounds
   (``rdDistGeom.GetMoleculeBoundsMatrix``; the triangle smoothing runs on the GPU, b200mol_triangle_smooth, with the
   reference's fallback ladder :289-345), experimental torsions (``rdDistGeom.GetExperimentalTorsions``), and Python ports
   of ``findChiralSets`` (:117-206) and ``findDoubleBonds`` (:617-664); bonds / angles / improper centres of
   ``CrystalFFDetails`` are not exposed by RDKit's Python API and are re-derived from the graph (RDKit
   TorsionPreferences.cpp: sp2 C / N / O centres with three neighbours; ``isCBoundToO`` = a carbon centre with an sp2
   oxygen neighbour).
"""

from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

from nvmolkit_b200.forcefield import ConformerBatch, FlatSystem

_LINEAR_MMFF_TYPES = frozenset({4, 53, 61})  # MMFFPROP.PAR `linh` = 1: =C=/-C#, =N=, isonitrile N
_TORSION_BOND_SMARTS = "[!$([D1]);!$(*#*)]~[!$([D1]);!$(*#*)]"  # RDKit DefaultTorsionBondSmarts


def _rdkit():
    try:
        from rdkit import Chem
        from rdkit.Chem import rdForceFieldHelpers as FFH
    except ImportError as e:  # pragma: no cover - RDKit is optional
        raise ImportError("RDKit molecules were passed but RDKit is not importable; pass pre-flattened "
                          "Flat*Molecules instead") from e
    return Chem, FFH


def _conformer_coords(mol) -> List[np.ndarray]:
    return [np.asarray(c.GetPositions(), dtype=np.float64) for c in mol.GetConformers()]


def _mmff_terms(Chem, FFH, mol, props, coords: Sequence[np.ndarray], non_bonded_thresh: float, ignore_interfrag: bool
                ) -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
    n = mol.GetNumAtoms()
    nbrs = [[a.GetIdx() for a in atom.GetNeighbors()] for atom in mol.GetAtoms()]
    types = [props.GetMMFFAtomType(i) for i in range(n)]
    t: Dict[str, Tuple[list, list]] = {k: ([], []) for k in ("bond", "angle", "strbend", "oop", "torsion", "vdw", "ele")}

    bond_r0: Dict[Tuple[int, int], float] = {}
    for b in mol.GetBonds():
        i, j = b.GetBeginAtomIdx(), b.GetEndAtomIdx()
        p = FFH.GetMMFFBondStretchParams(mol, i, j)  # (bondType, kb, r0)
        if p:
            t["bond"][0].append((i, j))
            t["bond"][1].append((p[2], p[1]))
            bond_r0[(i, j)] = bond_r0[(j, i)] = p[2]

    for j in range(n):
        if len(nbrs[j]) < 2:
            continue
        linear = types[j] in _LINEAR_MMFF_TYPES
        for a, i in enumerate(nbrs[j]):
            for k in nbrs[j][a + 1:]:
                pa = FFH.GetMMFFAngleBendParams(mol, i, j, k)  # (angleType, ka, theta0)
                if pa:
                    t["angle"][0].append((i, j, k))
                    t["angle"][1].append((pa[2], pa[1], 1.0 if linear else 0.0))
                if linear or not pa:
                    continue
                ps = FFH.GetMMFFStretchBendParams(mol, i, j, k)  # (stretchBendType, kbaIJK, kbaKJI)
                if ps and (i, j) in bond_r0 and (k, j) in bond_r0:
                    t["strbend"][0].append((i, j, k))
                    t["strbend"][1].append((pa[2], bond_r0[(i, j)], bond_r0[(k, j)], ps[1], ps[2]))

    for j in range(n):
        if len(nbrs[j]) != 3:
            continue
        i, k, l = nbrs[j]
        koop = FFH.GetMMFFOopBendParams(mol, i, j, k, l)
        if koop is None:
            continue
        for quad in ((i, j, k, l), (i, j, l, k), (k, j, l, i)):  # the three Wilson angles around the centre j
            t["oop"][0].append(quad)
            t["oop"][1].append((float(koop),))

    sp23 = (Chem.HybridizationType.SP2, Chem.HybridizationType.SP3)
    query = Chem.MolFromSmarts(_TORSION_BOND_SMARTS)
    for j, k in mol.GetSubstructMatches(query):
        if mol.GetAtomWithIdx(j).GetHybridization() not in sp23 or mol.GetAtomWithIdx(k).GetHybridization() not in sp23:
            continue
        for i in nbrs[j]:
            if i == k:
                continue
            for l in nbrs[k]:
                if l == j or l == i:
                    continue
                p = FFH.GetMMFFTorsionParams(mol, i, j, k, l)  # (torsionType, V1, V2, V3)
                if p:
                    t["torsion"][0].append((i, j, k, l))
                    t["torsion"][1].append((p[1], p[2], p[3]))

    topo = Chem.GetDistanceMatrix(mol)
    frags = None
    if ignore_interfrag:
        frags = np.zeros(n, dtype=np.int64)
        for f, atoms in enumerate(Chem.GetMolFrags(mol)):
            frags[list(atoms)] = f
    within = np.zeros((n, n), dtype=bool)
    for xyz in coords:
        d = np.sqrt(((xyz[:, None, :] - xyz[None, :, :]) ** 2).sum(-1))
        within |= d <= non_bonded_thresh
    charges = [props.GetMMFFPartialCharge(i) for i in range(n)]
    for i in range(n):
        for j in range(i + 1, n):
            if topo[i, j] < 3 or not within[i, j] or (frags is not None and frags[i] != frags[j]):
                continue
            pv = FFH.GetMMFFVdWParams(mol, i, j)  # (R_ij_starUnscaled, epsilonUnscaled, R_ij_star, epsilon)
            if pv:
                t["vdw"][0].append((i, j))
                t["vdw"][1].append((pv[2], pv[3]))
            qq = charges[i] * charges[j]  # constant dielectric, D = 1 (RDKit defaults; MMFFMolProperties has no getters)
            if abs(qq) > 1.0e-10:
                t["ele"][0].append((i, j))
                t["ele"][1].append((qq, 1.0, 1.0 if topo[i, j] == 3 else 0.0))
    return _as_tables("mmff", t)


def _as_tables(kind: str, t) -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
    """Lists of (indices, parameters) -> arrays with the widths of forcefield.LAYOUT (empty term types included)."""
    from nvmolkit_b200.forcefield import LAYOUT

    return {name: (np.array(t[name][0], dtype=np.int16).reshape(-1, k), np.array(t[name][1], dtype=np.float64).reshape(-1, p))
            for name, k, p in LAYOUT[kind] if name in t}  # (the restraint tables are added by BatchedForcefield only)


class _FlatWithMap:
    """FlatSystem + ConformerBatch + the (molecule, conformer id) each batch entry came from."""

    def __init__(self, system: FlatSystem, batch: ConformerBatch, conf_ids: List[List[int]]):
        self.system, self.batch, self.conf_ids = system, batch, conf_ids


def mmff_from_rdkit(molecules, properties=None, nonBondedThreshold: float = 100.0, ignoreInterfragInteractions: bool = True):
    """Flatten RDKit molecules (all conformers) into MMFF term tables. Error contract of the reference
    (nvmolkit/mmffOptimization.py:145-162): ValueError(message, {"none": [...], "no_params": [...]})."""
    Chem, FFH = _rdkit()
    molecules = list(molecules)
    none = [i for i, m in enumerate(molecules) if m is None]
    props_list = []
    if properties is not None and not isinstance(properties, (list, tuple)):
        properties = [properties] * len(molecules)
    no_params = []
    for i, m in enumerate(molecules):
        if m is None:
            props_list.append(None)
            continue
        p = properties[i] if properties is not None and properties[i] is not None else FFH.MMFFGetMoleculeProperties(m)
        if p is None:
            no_params.append(i)
        props_list.append(p)
    if none or no_params:
        raise ValueError("MMFF cannot be set up for some molecules (None entries or missing MMFF parameters)",
                         {"none": none, "no_params": no_params})
    per_mol, counts, coords_per_mol, conf_ids = [], [], [], []
    for m, p in zip(molecules, props_list):
        coords = _conformer_coords(m)
        per_mol.append(_mmff_terms(Chem, FFH, m, p, coords, float(nonBondedThreshold), bool(ignoreInterfragInteractions)))
        counts.append(m.GetNumAtoms())
        coords_per_mol.append(coords)
        conf_ids.append([c.GetId() for c in m.GetConformers()])
    system = FlatSystem.from_molecules("mmff", counts, per_mol)
    return _FlatWithMap(system, ConformerBatch.from_coords(system, coords_per_mol), conf_ids)


def write_back_conformers(molecules, coords_per_mol) -> None:
    """Overwrite the conformers of each RDKit molecule, in conformer order, with the optimised coordinates."""
    from rdkit.Geometry import Point3D

    for mol, confs in zip(molecules, coords_per_mol):
        for conf, xyz in zip(mol.GetConformers(), confs):
            for a, (x, y, z) in enumerate(np.asarray(xyz, dtype=np.float64)):
                conf.SetAtomPosition(a, Point3D(float(x), float(y), float(z)))


def add_conformers(molecules, coords_per_mol, prune_rms_thresh: float = -1.0) -> None:
    """Append embedded conformers to the RDKit molecules (reference: addConformersToMoleculeWithPruning,
    src/etkdg.cpp:430-484). With prune_rms_thresh > 0 a conformer is kept only if its heavy-atom RMSD (after alignment)
    to every conformer kept before it exceeds the threshold."""
    from rdkit import Chem
    from rdkit.Chem import rdMolAlign
    from rdkit.Geometry import Point3D

    for mol, confs in zip(molecules, coords_per_mol):
        heavy = [a.GetIdx() for a in mol.GetAtoms() if a.GetAtomicNum() > 1]
        amap = list(zip(heavy, heavy))
        for xyz in confs:
            conf = Chem.Conformer(mol.GetNumAtoms())
            for a, (x, y, z) in enumerate(np.asarray(xyz, dtype=np.float64)):
                conf.SetAtomPosition(a, Point3D(float(x), float(y), float(z)))
            cid = mol.AddConformer(conf, assignId=True)
            if prune_rms_thresh > 0.0:
                for other in [c.GetId() for c in mol.GetConformers() if c.GetId() != cid]:
                    if rdMolAlign.GetBestRMS(mol, mol, other, cid, map=[amap]) < prune_rms_thresh:
                        mol.RemoveConformer(cid)
                        break


# ------------------------------------------------------------------------------------------------------------ UFF
_GROUP6 = frozenset({8, 16, 34, 52, 84})


def _uff_angle_k(ka0: float, theta_a: float, theta_b: float, r12: float, r23: float) -> float:
    """Angle force constant at theta_b from the one RDKit reports at the atom-type angle theta_a. UFF eq. 13:
    K = 664.12 Z1 Z3 / r13^5 * r12 r23 (3 r12 r23 (1 - cos^2) - r13^2 cos); Z1 Z3 cancels in the ratio."""
    def shape(th):
        c = np.cos(th)
        r13sq = r12 * r12 + r23 * r23 - 2.0 * r12 * r23 * c
        return r12 * r23 * (3.0 * r12 * r23 * (1.0 - c * c) - r13sq * c) / r13sq ** 2.5

    return ka0 * shape(theta_b) / shape(theta_a)


def _uff_terms(Chem, FFH, mol, coords, vdw_thresh: float, ignore_interfrag: bool):
    from nvmolkit_b200.builders import inversion_coefficients

    n = mol.GetNumAtoms()
    H = Chem.HybridizationType
    atoms = list(mol.GetAtoms())
    nbrs = [[a.GetIdx() for a in atom.GetNeighbors()] for atom in atoms]
    hyb = [a.GetHybridization() for a in atoms]
    z = [a.GetAtomicNum() for a in atoms]
    ring = mol.GetRingInfo()
    t = {k: ([], []) for k in ("bond", "angle", "torsion", "inversion", "vdw")}
    r0 = {}
    for b in mol.GetBonds():
        i, j = b.GetBeginAtomIdx(), b.GetEndAtomIdx()
        p = FFH.GetUFFBondStretchParams(mol, i, j)  # (kb, r0)
        if p:
            t["bond"][0].append((i, j))
            t["bond"][1].append((p[1], p[0]))
            r0[(i, j)] = r0[(j, i)] = p[1]
    for j in range(n):  # uff_flattened_builder.cpp:142-229
        if hyb[j] == H.SP3D and len(nbrs[j]) == 5:
            continue  # trigonal bipyramid: the special case needs a conformer to pick the axis (:236-318); not flattened here
        for a, i in enumerate(nbrs[j]):
            for k in nbrs[j][a + 1:]:
                p = FFH.GetUFFAngleBendParams(mol, i, j, k)  # (ka, theta0 in degrees)
                if not p:
                    continue
                ka, theta0 = p[0], np.deg2rad(p[1])
                order, special = 0, None
                if hyb[j] == H.SP:
                    order = 1
                elif hyb[j] == H.SP2:
                    order = 3
                    for size, lone, both in ((3, 150.0, 60.0), (4, 135.0, 90.0)):
                        if ring.IsAtomInRingOfSize(j, size):
                            ri, rk = ring.IsAtomInRingOfSize(i, size), ring.IsAtomInRingOfSize(k, size)
                            if ri != rk:
                                special = lone
                            elif ri and rk:
                                special = both
                            break
                elif hyb[j] == H.SP3D2:
                    order = 4
                if special is not None and (i, j) in r0 and (k, j) in r0:
                    th = np.deg2rad(special)
                    ka, theta0, order = _uff_angle_k(ka, theta0, th, r0[(i, j)], r0[(k, j)]), th, 0
                c0 = c1 = c2 = 0.0
                if order == 0:
                    sn, cs = np.sin(theta0), np.cos(theta0)
                    c2 = 1.0 / (4.0 * max(sn * sn, 1.0e-8))
                    c1 = -4.0 * c2 * cs
                    c0 = c2 * (2.0 * cs * cs + 1.0)
                t["angle"][0].append((i, j, k))
                t["angle"][1].append((theta0, ka, float(order), c0, c1, c2))
    sp23 = (H.SP2, H.SP3)
    for b in mol.GetBonds():  # torsions around every sp2/sp3 - sp2/sp3 bond (:372-452)
        j, k = b.GetBeginAtomIdx(), b.GetEndAtomIdx()
        if hyb[j] not in sp23 or hyb[k] not in sp23:
            continue
        bo = b.GetBondTypeAsDouble()
        quads = [(i, l) for i in nbrs[j] if i != k for l in nbrs[k] if l != j and l != i]
        for i, l in quads:
            v = FFH.GetUFFTorsionParams(mol, i, j, k, l)
            if v is None:
                continue
            if hyb[j] == H.SP3 and hyb[k] == H.SP3:
                order, cos_term = (2, -1.0) if (bo == 1.0 and z[j] in _GROUP6 and z[k] in _GROUP6) else (3, -1.0)
            elif hyb[j] == H.SP2 and hyb[k] == H.SP2:
                order, cos_term = 2, 1.0
            else:
                order, cos_term = 6, 1.0
                if bo == 1.0:
                    sp3, other = (j, k) if hyb[j] == H.SP3 else (k, j)
                    if z[sp3] in _GROUP6 and z[other] not in _GROUP6:
                        order, cos_term = 2, -1.0
                    elif hyb[i] == H.SP2 or hyb[l] == H.SP2:  # "hasSP2": either end atom (:424-428)
                        order, cos_term = 3, -1.0
            t["torsion"][0].append((i, j, k, l))
            t["torsion"][1].append((float(v) / len(quads), float(order), cos_term))  # RDKit scales by the torsion count of the bond
    for j in range(n):  # inversions at three-coordinate sp2 C / N / O and group-15 centres (:454-530)
        if len(nbrs[j]) != 3:
            continue
        i, k, l = nbrs[j]
        kinv = FFH.GetUFFInversionParams(mol, i, j, k, l)
        if kinv is None:
            continue
        c_o = z[j] == 6 and any(z[q] == 8 and hyb[q] == H.SP2 for q in nbrs[j])
        _k3, c0, c1, c2 = inversion_coefficients(z[j], c_o)
        for quad in ((i, j, k, l), (i, j, l, k), (k, j, l, i)):
            t["inversion"][0].append(quad)
            t["inversion"][1].append((float(kinv), c0, c1, c2))
    topo = Chem.GetDistanceMatrix(mol)
    frags = None
    if ignore_interfrag:
        frags = np.zeros(n, dtype=np.int64)
        for f, members in enumerate(Chem.GetMolFrags(mol)):
            frags[list(members)] = f
    dmin = np.full((n, n), np.inf)
    for xyz in coords:
        dmin = np.minimum(dmin, np.sqrt(((xyz[:, None, :] - xyz[None, :, :]) ** 2).sum(-1)))
    for i in range(n):
        for j in range(i + 1, n):
            if topo[i, j] < 3 or (frags is not None and frags[i] != frags[j]):
                continue
            p = FFH.GetUFFVdWParams(mol, i, j)  # (x_ij, D_ij)
            if not p:
                continue
            thresh = vdw_thresh * p[0]
            if dmin[i, j] < thresh:  # :340-370 (per conformer there; the union over the conformers here)
                t["vdw"][0].append((i, j))
                t["vdw"][1].append((p[0], p[1], thresh))
    return _as_tables("uff", t)


def uff_from_rdkit(molecules, vdwThreshold: float = 10.0, ignoreInterfragInteractions: bool = True):
    """Flatten RDKit molecules (all conformers) into UFF term tables. Molecules without UFF parameters raise the
    reference's ValueError contract (nvmolkit/uffOptimization.py)."""
    Chem, FFH = _rdkit()
    molecules = list(molecules)
    none = [i for i, m in enumerate(molecules) if m is None]
    no_params = [i for i, m in enumerate(molecules) if m is not None and not FFH.UFFHasAllMoleculeParams(m)]
    if none or no_params:
        raise ValueError("UFF cannot be set up for some molecules (None entries or missing UFF parameters)",
                         {"none": none, "no_params": no_params})
    per_mol, counts, coords_per_mol, conf_ids = [], [], [], []
    for m in molecules:
        coords = _conformer_coords(m)
        per_mol.append(_uff_terms(Chem, FFH, m, coords, float(vdwThreshold), bool(ignoreInterfragInteractions)))
        counts.append(m.GetNumAtoms())
        coords_per_mol.append(coords)
        conf_ids.append([c.GetId() for c in m.GetConformers()])
    system = FlatSystem.from_molecules("uff", counts, per_mol)
    return _FlatWithMap(system, ConformerBatch.from_coords(system, coords_per_mol), conf_ids)


# ---------------------------------------------------------------------------------------------------------- ETKDG
def find_chiral_sets(Chem, mol):
    """Python port of findChiralSets (src/embedder_utils.cpp:117-206; coordMap not supported). Returns
    (chiral centres [n,5], volume bounds [n,2], tetrahedral centres [m,5], fused-small-ring flags [m])."""
    CT = Chem.ChiralType
    ring = mol.GetRingInfo()
    chiral, cbounds, tet, fused = [], [], [], []
    for atom in mol.GetAtoms():
        if atom.GetAtomicNum() == 1:
            continue
        tag = atom.GetChiralTag()
        stereo = tag in (CT.CHI_TETRAHEDRAL_CW, CT.CHI_TETRAHEDRAL_CCW)
        if not (stereo or (atom.GetAtomicNum() in (6, 7) and atom.GetDegree() == 4)):
            continue
        idx = atom.GetIdx()
        nbrs = [b.GetOtherAtomIdx(idx) for b in atom.GetBonds()]
        if len(nbrs) < 3:
            raise ValueError(f"atom {idx} cannot be a chiral centre")
        lower = 5.0
        if len(nbrs) < 4:
            lower = 2.0  # three neighbours give smaller volumes (RDKit github #5883)
            nbrs.append(idx)
        if tag == CT.CHI_TETRAHEDRAL_CCW:
            chiral.append([idx] + nbrs[:4])
            cbounds.append([lower, 100.0])
        elif tag == CT.CHI_TETRAHEDRAL_CW:
            chiral.append([idx] + nbrs[:4])
            cbounds.append([-100.0, -lower])
        elif not (ring.NumAtomRings(idx) < 2 or ring.IsAtomInRingOfSize(idx, 3)):
            tet.append([idx] + nbrs[:4])
            fused.append(1.0 if sum(1 for sz in ring.AtomRingSizes(idx) if sz < 5) > 1 else 0.0)
    return chiral, cbounds, tet, fused


def find_double_bonds(Chem, mol):
    """Python port of findDoubleBonds (src/embedder_utils.cpp:617-664): (ends [n,3], stereo quadruples [m,4], signs [m])."""
    BT, BS = Chem.BondType, Chem.BondStereo
    ends, quads, signs = [], [], []
    for bnd in mol.GetBonds():
        if bnd.GetBondType() != BT.DOUBLE:
            continue
        for a, o in ((bnd.GetBeginAtomIdx(), bnd.GetEndAtomIdx()), (bnd.GetEndAtomIdx(), bnd.GetBeginAtomIdx())):
            atom = mol.GetAtomWithIdx(a)
            if atom.GetDegree() < 2:
                continue
            for nbr in atom.GetNeighbors():
                if nbr.GetIdx() == o:
                    continue
                ob = mol.GetBondBetweenAtoms(a, nbr.GetIdx())
                if ob is None or (ob.GetBondType() != BT.SINGLE and atom.GetDegree() == 2):
                    continue
                ends.append([nbr.GetIdx(), a, o])
        if bnd.GetStereo() > BS.STEREOANY:
            sa = list(bnd.GetStereoAtoms())
            sign = -1.0 if bnd.GetStereo() in (BS.STEREOCIS, BS.STEREOZ) else 1.0
            quads.append([sa[0], bnd.GetBeginAtomIdx(), bnd.GetEndAtomIdx(), sa[1]])
            signs.append(sign)
    return ends, quads, signs


def crystalff_details(Chem, DG, mol, params):
    """CrystalFFDetails of one molecule: RDKit's experimental torsions + the bonds / angles / improper centres its Python
    API does not return (re-derived from the graph, see the module docstring)."""
    from nvmolkit_b200.builders import CrystalFFDetails

    use_et = bool(getattr(params, "useExpTorsionAnglePrefs", True))
    use_bk = bool(getattr(params, "useBasicKnowledge", True))
    tors, v, sg = [], [], []
    if use_et or use_bk:
        for d in DG.GetExperimentalTorsions(mol, useExpTorsionAnglePrefs=use_et,
                                            useSmallRingTorsions=bool(getattr(params, "useSmallRingTorsions", False)),
                                            useMacrocycleTorsions=bool(getattr(params, "useMacrocycleTorsions", True)),
                                            useBasicKnowledge=use_bk, ETversion=int(getattr(params, "ETversion", 2))):
            tors.append(list(d["atomIndices"]))
            vv, ss = list(d["V"])[:6], list(d["signs"])[:6]
            v.append(vv + [0.0] * (6 - len(vv)))
            sg.append(ss + [0] * (6 - len(ss)))
    H = Chem.HybridizationType
    bonds = [[b.GetBeginAtomIdx(), b.GetEndAtomIdx()] for b in mol.GetBonds()]
    angles, impropers = [], []
    for atom in mol.GetAtoms():
        j = atom.GetIdx()
        nb = [a.GetIdx() for a in atom.GetNeighbors()]
        linear = 1 if atom.GetHybridization() == H.SP else 0
        for x in range(len(nb)):
            for y in range(x + 1, len(nb)):
                angles.append([nb[x], j, nb[y], linear])
        if use_bk and len(nb) == 3 and atom.GetHybridization() == H.SP2 and atom.GetAtomicNum() in (6, 7, 8):
            c_o = atom.GetAtomicNum() == 6 and any(
                a.GetAtomicNum() == 8 and a.GetHybridization() == H.SP2 for a in atom.GetNeighbors())
            impropers.append([nb[0], j, nb[1], nb[2], atom.GetAtomicNum(), int(c_o)])
    return CrystalFFDetails(np.array(tors).reshape(-1, 4), np.array(v).reshape(-1, 6), np.array(sg).reshape(-1, 6),
                            np.array(impropers).reshape(-1, 6), np.array(bonds).reshape(-1, 2), np.array(angles).reshape(-1, 4),
                            float(getattr(params, "boundsMatForceScaling", 1.0)))


def embed_molecules_from_rdkit(molecules, params):
    """prepareEmbedderArgs for a list of RDKit molecules (src/embedder_utils.cpp:671-708), then the term construction of
    nvmolkit_b200.builders. The bounds matrices are smoothed on the GPU in one batch; a matrix that does not smooth is
    rebuilt without 1-5 bounds and with scaled van der Waals radii and smoothed again (the reference's ladder, :313-343);
    if that fails too the molecule raises unless params.ignoreSmoothingFailures."""
    Chem, _FFH = _rdkit()
    from rdkit.Chem import rdDistGeom as DG

    from nvmolkit_b200.builders import StereoInfo, flat_embed_from_parts
    from nvmolkit_b200.dgprep import triangle_smooth

    molecules = list(molecules)
    macro14 = bool(getattr(params, "useMacrocycle14config", True))
    raw = [np.asarray(DG.GetMoleculeBoundsMatrix(m, set15bounds=True, scaleVDW=False, doTriangleSmoothing=False,
                                                 useMacrocycle14config=macro14), dtype=np.float64) for m in molecules]
    smoothed, ok = triangle_smooth(raw)
    bad = [i for i, good in enumerate(ok) if not good]
    if bad:
        relaxed = [np.asarray(DG.GetMoleculeBoundsMatrix(molecules[i], set15bounds=False, scaleVDW=True,
                                                         doTriangleSmoothing=False, useMacrocycle14config=macro14),
                              dtype=np.float64) for i in bad]
        again, ok2 = triangle_smooth(relaxed)
        for k, i in enumerate(bad):
            if ok2[k]:
                smoothed[i] = again[k]
            elif bool(getattr(params, "ignoreSmoothingFailures", False)):
                smoothed[i] = relaxed[k]
            else:
                raise ValueError(f"Could not triangle bounds smooth molecule {i}")
    details, stereo = [], []
    for m in molecules:
        Chem.AssignStereochemistry(m)
        details.append(crystalff_details(Chem, DG, m, params))
        chiral, cbounds, tet, fused = find_chiral_sets(Chem, m)
        ends, quads, signs = find_double_bonds(Chem, m)
        stereo.append(StereoInfo(chiral, cbounds, tet, fused, ends, quads, signs))
    return flat_embed_from_parts(smoothed, details, stereo, bool(getattr(params, "useBasicKnowledge", True)))


def _terminal_groups(mol) -> List[List[int]]:
    """Groups of conjugated terminal atoms that ``symmetrizeConjugatedTerminalGroups`` makes equivalent: per atom, its
    neighbours of degree 1 that are N or O, joined to it by a conjugated bond, and of one element, when there are at
    least two (the two oxygens of a carboxylate or of a nitro group)."""
    groups = []
    for atom in mol.GetAtoms():
        by_element: Dict[int, List[int]] = {}
        for bond in atom.GetBonds():
            t = bond.GetOtherAtomIdx(atom.GetIdx())
            other = mol.GetAtomWithIdx(t)
            if other.GetDegree() == 1 and other.GetAtomicNum() in (7, 8) and bond.GetIsConjugated():
                by_element.setdefault(other.GetAtomicNum(), []).append(t)
        groups += [sorted(g) for g in by_element.values() if len(g) >= 2]
    return groups


def probe_ref_matches(prb, ref, maxMatches: int = 1000000, symmetrizeConjugatedTerminalGroups: bool = True
                      ) -> List[Tuple[int, ...]]:
    """The matches of a probe molecule inside a reference molecule that RDKit's ``GetBestRMS`` /
    ``GetBestAlignmentTransform`` / ``CalcRMS`` enumerate: ``ref.GetSubstructMatches(prb, uniquify=False,
    maxMatches=maxMatches, useChirality=False)``; ``match[q]`` is the reference atom that probe atom q lands on.

    With ``symmetrizeConjugatedTerminalGroups`` this restates RDKit's symmetrised query on the matches instead of on a
    query copy: every match m is followed by m composed with every permutation that reorders the atoms within each
    group of :func:`_terminal_groups` of the probe (``m'[q] = m[s[q]]``), in lexicographic order of the permutations,
    duplicates dropped, and the list cut at ``maxMatches``. The restatement is what the tests pin, not RDKit itself.
    An empty list means no match."""
    import itertools

    matches = [tuple(int(a) for a in m) for m in
               ref.GetSubstructMatches(prb, uniquify=False, maxMatches=maxMatches, useChirality=False)]
    groups = _terminal_groups(prb) if symmetrizeConjugatedTerminalGroups else []
    if not groups:
        return matches[:maxMatches]
    n = prb.GetNumAtoms()
    perms = []
    for choice in itertools.product(*[list(itertools.permutations(g)) for g in groups]):
        s = list(range(n))
        for g, p in zip(groups, choice):
            for a, b in zip(g, p):
                s[a] = b
        perms.append(s)
    out, seen = [], set()
    for m in matches:
        for s in perms:
            t = tuple(m[s[q]] for q in range(n))
            if t not in seen:
                seen.add(t)
                out.append(t)
                if len(out) == maxMatches:
                    return out
    return out


def self_matches(mol, maxMatches: int = 1000000, symmetrizeConjugatedTerminalGroups: bool = True) -> List[Tuple[int, ...]]:
    """The matches of a molecule onto itself that RDKit's ``GetBestRMS`` / ``GetAllConformerBestRMS`` enumerate:
    :func:`probe_ref_matches` ``(mol, mol, maxMatches, symmetrizeConjugatedTerminalGroups)``."""
    return probe_ref_matches(mol, mol, maxMatches, symmetrizeConjugatedTerminalGroups)
