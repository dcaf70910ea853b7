"""Symmetry-aware alignment on the CPU: the probe / reference matching (``rdkit_adapter.probe_ref_matches``) against
stand-in molecules, the fp64 oracle (oracle_best_align.c) against a brute-force SVD minimum over the mappings, every
argument refusal of ``molAlign.GetBestRMS`` / ``CalcRMS`` / ``GetBestAlignmentTransform`` and their batch forms before
device work, and the C-ABI's host checks of ``b200mol_best_align`` without a device."""
import re

import numpy as np
import pytest

from nvmolkit_b200 import _lib
from nvmolkit_b200 import conformerRmsd as cr
from nvmolkit_b200 import molAlign as ma
from nvmolkit_b200.rdkit_adapter import probe_ref_matches, self_matches
from oracle import best_align as ob


def kabsch(p, q, w=None, reflect=False):
    """RMSD over L pairs of the weighted best superposition of p (negated when reflect) onto q, by SVD."""
    w = np.ones(len(p)) if w is None else np.asarray(w, np.float64)
    p = -p if reflect else p
    P = p - (w[:, None] * p).sum(0) / w.sum()
    Q = q - (w[:, None] * q).sum(0) / w.sum()
    u, _, vt = np.linalg.svd((w[:, None] * P).T @ Q)
    R = vt.T @ np.diag([1.0, 1.0, np.sign(np.linalg.det(vt.T @ u.T))]) @ u.T
    return np.sqrt((w * ((P @ R.T - Q) ** 2).sum(1)).sum() / len(p))


# ------------------------------------------------------------------ stand-in molecules
class Atom:
    def __init__(self, mol, i):
        self.mol, self.i = mol, i

    def GetIdx(self):
        return self.i

    def GetAtomicNum(self):
        return self.mol.z[self.i]

    def GetDegree(self):
        return sum(self.i in b[:2] for b in self.mol.bonds)

    def GetBonds(self):
        return [Bond(b) for b in self.mol.bonds if self.i in b[:2]]


class Bond:
    def __init__(self, b):
        self.b = b

    def GetOtherAtomIdx(self, i):
        return self.b[1] if self.b[0] == i else self.b[0]

    def GetIsConjugated(self):
        return self.b[2]


class Conf:
    def __init__(self, cid, xyz):
        self.cid, self.xyz = cid, np.asarray(xyz, np.float64)

    def GetId(self):
        return self.cid

    def GetPositions(self):
        return self.xyz


class StandIn:
    """Atoms, bonds (a, b, conjugated), conformers, and the matches its GetSubstructMatches returns for any query."""

    def __init__(self, z, bonds, matches, confs=1, seed=0):
        rng = np.random.default_rng(seed)
        self.z, self.bonds, self.matches = list(z), list(bonds), list(matches)
        self.confs = [Conf(c, rng.normal(size=(len(z), 3))) for c in range(confs)]
        self.calls = []

    def GetNumAtoms(self):
        return len(self.z)

    def GetAtoms(self):
        return [Atom(self, i) for i in range(len(self.z))]

    def GetAtomWithIdx(self, i):
        return Atom(self, i)

    def GetConformers(self):
        return self.confs

    def GetSubstructMatches(self, query, uniquify=True, maxMatches=1000, useChirality=True):
        self.calls.append((query, uniquify, maxMatches, useChirality))
        return self.matches[:maxMatches]


def acetate(matches=((0, 1, 2, 3),), **kw):
    """CH3-C(=O)O-: C0 (methyl), C1, O2, O3; the two C-O bonds conjugated."""
    return StandIn([6, 6, 8, 8], [(0, 1, False), (1, 2, True), (1, 3, True)], matches, **kw)


# ------------------------------------------------------------------ matching
def test_probe_ref_matches_asks_the_reference_for_the_probe():
    prb, ref = acetate(), acetate([(0, 1, 3, 2)])
    assert probe_ref_matches(prb, ref, 7, False) == [(0, 1, 3, 2)]
    assert ref.calls == [(prb, False, 7, False)] and prb.calls == []


def test_terminal_groups_come_from_the_probe():
    # the reference draws no conjugated bonds: the probe's carboxylate oxygens still swap
    ref = StandIn([6, 6, 8, 8], [(0, 1, False), (1, 2, False), (1, 3, False)], [(0, 1, 2, 3)])
    assert probe_ref_matches(acetate(), ref, 100, True) == [(0, 1, 2, 3), (0, 1, 3, 2)]
    # and a probe without conjugated bonds gets no swap from a reference that has them
    prb = StandIn([6, 6, 8, 8], [(0, 1, False), (1, 2, False), (1, 3, False)], [])
    assert probe_ref_matches(prb, acetate(), 100, True) == [(0, 1, 2, 3)]


def test_the_cut_comes_after_the_expansion():
    ref = acetate([(0, 1, 2, 3), (1, 0, 2, 3)])
    assert probe_ref_matches(acetate(), ref, 3, True) == [(0, 1, 2, 3), (0, 1, 3, 2), (1, 0, 2, 3)]
    assert ref.calls[-1] == (ref.calls[-1][0], False, 3, False)  # RDKit is asked for maxMatches before the expansion
    assert probe_ref_matches(acetate(), acetate([(0, 1, 2, 3), (0, 1, 3, 2)]), 100, True) == \
        [(0, 1, 2, 3), (0, 1, 3, 2)]  # duplicates dropped


def test_self_matches_is_probe_ref_matches_of_the_molecule_with_itself():
    for sym in (False, True):
        for cut in (1, 2, 100):
            mol = acetate([(0, 1, 2, 3), (1, 0, 3, 2)])
            assert self_matches(mol, cut, sym) == probe_ref_matches(mol, mol, cut, sym)
            assert mol.calls[0][0] is mol


def test_no_match_is_refused_before_device_work():
    for fn in (ma.GetBestRMS, ma.CalcRMS, ma.GetBestAlignmentTransform):
        with pytest.raises(ValueError, match="No sub-structure match found between the reference and probe mol"):
            fn(acetate(), acetate([]))


def test_map_lists_take_two_atom_counts():
    p, q = cr._map_lists([[(0, 5), (2, 4)], [(2, 5), (0, 4)]], 3, "map", 6)
    assert p.tolist() == [0, 2] and q.tolist() == [[5, 4], [4, 5]]
    with pytest.raises(ValueError, match="outside"):
        cr._map_lists([[(0, 5)]], 3, "map")
    p, q, perm = cr._map_lists([[(2, 5), (0, 4)], [(2, 4), (0, 5)]], 3, "map", 6, order=True)
    assert perm.tolist() == [1, 0] and q.tolist() == [[4, 5], [5, 4]]
    with pytest.raises(ValueError, match="another order"):
        cr._map_lists([[(2, 5), (0, 4)], [(0, 4), (2, 5)]], 3, "map", 6, order=True)


# ------------------------------------------------------------------ oracle
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("reflect", [False, True])
@pytest.mark.parametrize("L,K", [(3, 1), (4, 6), (12, 9), (40, 3)])
def test_oracle_is_the_brute_force_minimum(L, K, weighted, reflect):
    rng = np.random.default_rng(L * 100 + K + 7 * weighted + 13 * reflect)
    A, B = L + 3, L + 5
    prb, ref = rng.normal(size=(A, 3)) * 2.0 + 4.0, rng.normal(size=(B, 3)) * 2.0 - 1.0
    P = rng.choice(A, L, replace=False)
    Q = np.stack([rng.choice(B, L, replace=False) for _ in range(K)])
    w = rng.uniform(0.2, 2.0, L) if weighted else None
    v, k, T, per = ob.best_align(prb, ref, P, Q, w, 0, reflect)
    want = np.array([kabsch(prb[P], ref[q], w, reflect) for q in Q])
    assert np.abs(per - want).max() <= 1e-10 * (1 + want.max())
    assert k == int(np.argmin(per)) and v == per[k]
    c, kc, _, perc = ob.best_align(prb, ref, P, Q, w, 1)
    ww = np.ones(L) if w is None else w
    wantc = np.array([np.sqrt((ww * ((prb[P] - ref[q]) ** 2).sum(1)).sum() / L) for q in Q])
    assert np.abs(perc - wantc).max() <= 1e-12 * (1 + wantc.max()) and kc == int(np.argmin(perc)) and c == perc[kc]


def test_oracle_takes_the_first_of_equal_minima():
    rng = np.random.default_rng(3)
    prb, ref = rng.normal(size=(8, 3)), rng.normal(size=(8, 3))
    Q = np.stack([rng.permutation(8) for _ in range(4)])
    v, k, T, per = ob.best_align(prb, ref, np.arange(8), Q)
    dup = np.concatenate([Q[:k + 1], Q[k:k + 1], Q[k + 1:]])  # the winner listed twice, the copy right after it
    v2, k2, T2, _ = ob.best_align(prb, ref, np.arange(8), dup)
    assert (v2, k2) == (v, k) and np.array_equal(T, T2)
    dup = np.concatenate([Q[k:k + 1], Q])  # and the copy first
    assert ob.best_align(prb, ref, np.arange(8), dup)[1] == 0
    kc = ob.best_align(prb, ref, np.arange(8), Q, mode=1)[1]
    assert ob.best_align(prb, ref, np.arange(8), np.concatenate([Q, Q[kc:kc + 1]]), mode=1)[1] == kc


# ------------------------------------------------------------------ refusals before device work
@pytest.mark.parametrize("kw,err,msg", [
    ({"maxMatches": 0}, ValueError, "maxMatches must be >= 1"),
    ({"weights": [1.0] * 3}, ValueError, "holds 3 weights, 4 expected"),
    ({"weights": [1.0, -1.0, 1.0, 1.0]}, ValueError, "finite and >= 0"),
    ({"weights": [1.0, np.inf, 1.0, 1.0]}, ValueError, "finite and >= 0"),
    ({"weights": [0.0] * 4}, ValueError, "sum to 0"),
    ({"map": [[(0, 9)]]}, ValueError, "outside"),
    ({"map": [[(0, 1), (0, 2)]]}, ValueError, "twice"),
    ({"map": [[(0, 1)], [(1, 0)]]}, ValueError, "other probe atoms"),
    ({"map": [[(0, 1, 2)]]}, ValueError, "pairs"),
    ({"map": [[(0, 1), (1, 0)], [(1, 1), (0, 0)]], "weights": [1.0, 2.0]}, ValueError, "another order"),
    ({"map": [[(0, 1), (1, 0)]], "weights": [1.0]}, ValueError, "holds 1 weights, 2 expected"),
    ({"stream": 0}, TypeError, "stream"),
])
def test_single_refusals(kw, err, msg):
    for fn in (ma.GetBestRMS, ma.CalcRMS, ma.GetBestAlignmentTransform):
        prb, ref = acetate(), acetate(seed=1)
        with pytest.raises(err, match=msg):
            fn(prb, ref, **kw)


def test_alignment_refusals():
    prb, ref = acetate(), acetate(seed=1)
    with pytest.raises(ValueError, match="maxIters must be >= 1"):
        ma.GetBestAlignmentTransform(prb, ref, maxIters=0)
    with pytest.raises(ValueError, match="must not be None"):
        ma.GetBestRMS(None, ref)
    with pytest.raises(ValueError, match="no conformer with id 5"):
        ma.GetBestRMS(prb, ref, prbId=5)
    with pytest.raises(ValueError, match="no conformer with id 5"):
        ma.CalcRMS(prb, ref, refId=5)
    with pytest.raises(ValueError, match="has no conformers"):
        ma.GetBestRMS(acetate(confs=0), ref)


def test_batch_refusals():
    prb, ref = acetate(confs=3), acetate(seed=1)
    with pytest.raises(ValueError, match="refMols holds 1"):
        ma.GetBestRMSBatch([prb, prb], [ref])
    with pytest.raises(ValueError, match="prbIds holds 1 entries"):
        ma.CalcRMSBatch([prb, prb], [ref, ref], prbIds=[[0]])
    with pytest.raises(ValueError, match="maps holds 1 entries"):
        ma.GetBestAlignmentTransformBatch([prb, prb], [ref, ref], maps=[None])
    with pytest.raises(ValueError, match="moved twice or is also a reference"):
        ma.GetBestRMSBatch([prb], [ref], prbIds=[[0, 1, 0]])
    with pytest.raises(ValueError, match="moved twice or is also a reference"):
        ma.GetBestRMSBatch([prb, ref], [ref, prb], prbIds=[[0], [0]], refIds=[0, 0])
    with pytest.raises(TypeError):
        ma.GetBestRMSBatch([prb], [ref], coordinates=np.zeros((4, 3)))
    with pytest.raises(TypeError):
        ma.CalcRMSBatch([prb], [ref], stream=0)
    # None: every conformer but the reference itself; one conformer against itself leaves nothing to do, without a device
    one = acetate()
    assert [r.torch().numel() for r in ma.GetBestRMSBatch([one], [one])] == [0]
    assert [r.torch().numel() for r in ma.CalcRMSBatch([prb], [ref], prbIds=[[]])] == [0]


def test_rdkit_positional_order_is_kept():
    import inspect

    names = lambda f: [p.name for p in inspect.signature(f).parameters.values()]  # noqa: E731
    common = ["prbMol", "refMol", "prbId", "refId", "map", "maxMatches", "symmetrizeConjugatedTerminalGroups", "weights"]
    assert names(ma.GetBestRMS)[:9] == common + ["numThreads"]
    assert names(ma.CalcRMS)[:8] == common
    assert names(ma.GetBestAlignmentTransform)[:11] == common + ["reflect", "maxIters", "numThreads"]
    assert inspect.signature(ma.GetBestRMS).parameters["maxMatches"].default == 1000000


# ------------------------------------------------------------------ C-ABI checks without a device
def call(probe, ref, sets, conf_atoms, start, count, length, atoms, weights=None, mode=0, reflect=0, maxIters=50,
         move=1, transform=False):
    probe, ref, sets, conf_atoms, count, length = (np.asarray(x, np.int32) for x in
                                                   (probe, ref, sets, conf_atoms, count, length))
    start, atoms = np.asarray(start, np.int64), np.asarray(atoms, np.int16)
    w = None if weights is None else np.asarray(weights, np.float64)
    fake = np.zeros(16)  # a non-null transform pointer for the in-place refusal; never written
    return _lib.call("b200mol_best_align", len(probe), probe.ctypes.data, ref.ctypes.data, sets.ctypes.data,
                     len(conf_atoms), conf_atoms.ctypes.data, None, None, len(count), start.ctypes.data,
                     count.ctypes.data, length.ctypes.data, atoms.ctypes.data, None if w is None else w.ctypes.data,
                     mode, reflect, maxIters, move, None, None, fake.ctypes.data if transform else None, None)


# two sets: K = 2, L = 2 (P = 0 2; Q = 0 2 / 2 0), and K = 1, L = 1
GOOD = dict(probe=[1, 2], ref=[0, 0], sets=[0, 1], conf_atoms=[3, 3, 3], start=[0, 6, 8], count=[2, 1],
            length=[2, 1], atoms=[0, 2, 0, 2, 2, 0, 1, 1])


@pytest.mark.parametrize("change,msg", [
    ({"maxIters": 0}, "maxIters must be >= 1"),
    ({"mode": 2}, "mode must be 0 (align) or 1 (in place)"),
    ({"mode": 1}, "in-place mode takes no move, reflect or transform"),
    ({"mode": 1, "move": 0, "reflect": 1}, "in-place mode takes no move, reflect or transform"),
    ({"mode": 1, "move": 0, "transform": True}, "in-place mode takes no move, reflect or transform"),
    ({"count": [0, 1], "start": [0, 2, 4]}, "mapping set 0: K = 0 and L = 2 must be >= 1"),
    ({"length": [2, 0], "start": [0, 6, 6]}, "mapping set 1: K = 1 and L = 0 must be >= 1"),
    ({"start": [0, 5, 8]}, "mapping set 0 holds 5 atoms, (K + 1) L = 6"),
    ({"start": [1, 6, 8]}, "must start at 0"),
    ({"atoms": [0, 2, 0, 2, 2, -1, 1, 1]}, "negative atom index"),
    ({"atoms": [0, 0, 0, 2, 2, 0, 1, 1]}, "mapping set 0: list 0 holds atom 0 twice"),
    ({"atoms": [0, 2, 0, 2, 2, 2, 1, 1]}, "mapping set 0: list 2 holds atom 2 twice"),
    ({"atoms": [0, 3, 0, 2, 2, 0, 1, 1]}, "holds probe atom 3, conformer 1 has 3 atoms"),
    ({"atoms": [0, 2, 0, 3, 2, 0, 1, 1]}, "holds reference atom 3, conformer 0 has 3 atoms"),
    ({"weights": [1.0, -0.5, 1.0]}, "mapping set 0: weight -0.5 must be finite and >= 0"),
    ({"weights": [1.0, 1.0, np.nan]}, "mapping set 1: weight nan must be finite and >= 0"),
    ({"weights": [0.0, 0.0, 1.0]}, "mapping set 0: its weights sum to 0"),
    ({"probe": [1, 3]}, "job 1: conformer outside [0, 3)"),
    ({"sets": [0, 2]}, "job 1: mapping set 2 outside [0, 2)"),
    ({"conf_atoms": [3, 3, -1]}, "conformer 2: negative atom count"),
    ({"probe": [1, 1]}, "job 1: probe conformer 1 is moved by an earlier job too"),
    ({"probe": [1, 0], "ref": [0, 2]}, "job 1: probe conformer 0 is also a reference"),
])
def test_c_abi_refuses_bad_tables(built_lib, change, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        call(**{**GOOD, **change})


def test_c_abi_checks_pass_before_device_pointers(built_lib):
    with pytest.raises(ValueError, match="null device pointer"):
        call(**GOOD)
    with pytest.raises(ValueError, match="null device pointer"):  # overlap is allowed when nothing moves
        call(**{**GOOD, "probe": [1, 1], "ref": [1, 0]}, move=0)
    with pytest.raises(ValueError, match="null device pointer"):
        call(**GOOD, mode=1, move=0, weights=[1.0, 0.0, 2.0])
    call([], [], [], [], [0], [], [], [])  # no jobs: nothing to do
