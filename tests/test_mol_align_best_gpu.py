"""Symmetry-aware alignment on the GPU (b200mol_best_align, molAlign.GetBestRMS / CalcRMS / GetBestAlignmentTransform)
against the fp64 oracle (oracle_best_align.c): mapping counts around the warp width and up to 1e5, pair counts from 1 to
1000, weights, mirror images and capped Jacobi sweeps; the first of exact ties; K = 1 against b200mol_align; a molecule
against itself against GetAllConformerBestRMS; what moves and what does not; the RDKit and Device3DResult paths;
repeatability, batch independence and streams; 1e6 jobs in one call. Every error is a host-side check: no test here
provokes a device fault."""
import os
import sys

import numpy as np
import pytest
import torch

from nvmolkit_b200 import conformerRmsd as cr
from nvmolkit_b200 import molAlign as ma
from nvmolkit_b200.types import AsyncGpuResult, Device3DResult
from oracle import align as oa
from oracle import best_align as ob

pytestmark = pytest.mark.gpu

FAKE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_rdkit")


@pytest.fixture
def Chem(monkeypatch):
    monkeypatch.syspath_prepend(FAKE)
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        monkeypatch.delitem(sys.modules, name)
    from rdkit import Chem as chem

    yield chem
    for name in [m for m in sys.modules if m == "rdkit" or m.startswith("rdkit.")]:
        sys.modules.pop(name, None)


def make_mol(Chem, n, confs=(), matches=None):
    """A fake-RDKit molecule of n atoms whose GetSubstructMatches returns ``matches`` (default: the identity)."""
    mol = Chem.Mol({"z": [6] * n, "bonds": [], "nbrs": [[] for _ in range(n)]}, conformers=list(confs))
    found = [tuple(range(n))] if matches is None else [tuple(int(a) for a in t) for t in matches]
    mol.GetSubstructMatches = lambda query, uniquify=True, maxMatches=1000, useChirality=False: found[:maxMatches]
    return mol


def rotation(rng):
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1.0
    return q


def horn_gap(p, q, w, reflect):
    """(G, relative gap of the two largest eigenvalues of Horn's N(S)) by NumPy."""
    w = np.ones(len(p)) if w is None else w
    p = -p if reflect else p
    P = p - (w[:, None] * p).sum(0) / w.sum()
    Q = q - (w[:, None] * q).sum(0) / w.sum()
    S = (w[:, None] * P).T @ Q
    N = np.array([[S[0, 0] + S[1, 1] + S[2, 2], S[1, 2] - S[2, 1], S[2, 0] - S[0, 2], S[0, 1] - S[1, 0]],
                  [S[1, 2] - S[2, 1], S[0, 0] - S[1, 1] - S[2, 2], S[0, 1] + S[1, 0], S[2, 0] + S[0, 2]],
                  [S[2, 0] - S[0, 2], S[0, 1] + S[1, 0], -S[0, 0] + S[1, 1] - S[2, 2], S[1, 2] + S[2, 1]],
                  [S[0, 1] - S[1, 0], S[2, 0] + S[0, 2], S[1, 2] + S[2, 1], -S[0, 0] - S[1, 1] + S[2, 2]]])
    ev = np.linalg.eigvalsh(N)
    G = float((w * (P * P).sum(1)).sum() + (w * (Q * Q).sum(1)).sum())
    return G, (ev[-1] - ev[-2]) / max(abs(ev[-1]), 1e-300)


class Batch:
    """Conformers in one space, mapping sets and jobs: the direct form of b200mol_best_align."""

    def __init__(self):
        self.blocks, self.sets, self.jobs = [], [], []

    def conf(self, xyz) -> int:
        self.blocks.append(np.asarray(xyz, np.float64))
        return len(self.blocks) - 1

    def set(self, P, Q, w=None) -> int:
        self.sets.append((np.asarray(P, np.int64), np.asarray(Q, np.int64).reshape(-1, len(P)), w))
        return len(self.sets) - 1

    def job(self, prb, ref, s):
        self.jobs.append((prb, ref, s))

    def run(self, mode=0, reflect=False, maxIters=50, move=True, transform=True, stream=None):
        atoms = np.array([len(b) for b in self.blocks], np.int64)
        xyz = torch.from_numpy(np.concatenate(self.blocks)).cuda()
        cas = torch.from_numpy(np.concatenate([[0], np.cumsum(atoms)]).astype(np.int32)).cuda()
        p, r, s = (np.array(x) for x in zip(*self.jobs))
        rmsd, best, T = ma._run_best(p, r, s, atoms, cas, xyz, self.sets, mode, reflect, maxIters, move, transform,
                                     stream)
        torch.cuda.synchronize()
        out = np.split(xyz.cpu().numpy(), np.cumsum(atoms)[:-1])
        return rmsd.cpu().numpy(), best.cpu().numpy(), None if T is None else T.cpu().numpy(), out


def posed(rng, L, K, weighted, offset=0.0):
    """A reference of A = L + 5 atoms, a probe that is a noisy rigid motion of it with its atoms shuffled, P = L probe
    atoms, K reference lists of which one (at a random position) is the true correspondence, weights or None."""
    A = L + 5
    ref = rng.normal(size=(A, 3)) * 2.0 + offset
    perm = rng.permutation(A)  # probe atom a is reference atom perm[a]
    prb = (ref[perm] - ref.mean(0)) @ rotation(rng) + rng.normal(size=3) * 5.0 + rng.normal(size=(A, 3)) * 0.3 + offset
    P = rng.choice(A, L, replace=False)
    Q = np.stack([rng.choice(A, L, replace=False) for _ in range(K)])
    Q[rng.integers(K)] = perm[P]
    w = None
    if weighted:
        w = rng.uniform(0.0, 2.0, L)
        w[0] = max(w[0], 0.5)
    return prb, ref, P, Q, w


SHAPES = [(K, L) for K in (1, 2, 31, 32, 33, 1000) for L in (1, 2, 3, 50)] + [(2, 1000), (33, 1000)]


def check(prb, ref, P, Q, w, reflect, maxIters, got, k, T, moved):
    L = len(P)
    want, kw, Tw, per = ob.best_align(prb, ref, P, Q, w, 0, reflect, maxIters)
    G, gap = horn_gap(prb[P], ref[Q[k]], w, reflect)
    Gw, _ = horn_gap(prb[P], ref[Q[kw]], w, reflect)
    tol = 1e-12 * max(G, Gw) / L + 1e-26
    assert abs(got ** 2 - want ** 2) <= tol, (L, len(Q), got, want)
    assert per[k] ** 2 - want ** 2 <= tol, (L, len(Q), k, kw)  # another index only within the tolerance of the best
    assert abs(per[k] ** 2 - got ** 2) <= tol
    assert np.abs(moved - oa.apply(T, prb)).max() <= 1e-9  # the kernel moves by the transform it reports
    if maxIters == 50 and L > 2 and gap >= 1e-3:  # ... and the transform is that of the reported index
        _, Tk = oa.align(prb, ref, np.stack([P, Q[k]], 1), w, reflect, maxIters)
        assert np.abs(T - Tk).max() <= 1e-9, (L, len(Q), k)


@pytest.mark.parametrize("maxIters", [1, 50])
@pytest.mark.parametrize("reflect", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_kernel_matches_the_oracle(cuda, weighted, reflect, maxIters):
    rng = np.random.default_rng(20 + 4 * weighted + 2 * reflect + (maxIters == 1))
    b, inputs = Batch(), []
    for K, L in SHAPES:
        prb, ref, P, Q, w = posed(rng, L, K, weighted)
        b.job(b.conf(prb), b.conf(ref), b.set(P, Q, w))
        inputs.append((prb, ref, P, Q, w))
    rmsd, best, T, out = b.run(0, reflect, maxIters)
    for j, (prb, ref, P, Q, w) in enumerate(inputs):
        assert 0 <= best[j] < len(Q)
        check(prb, ref, P, Q, w, reflect, maxIters, rmsd[j], best[j], T[j], out[b.jobs[j][0]])
        assert np.array_equal(out[b.jobs[j][1]], ref)
    # CalcRMS on the same jobs: nothing moves
    c, cb, cT, cout = b.run(1, move=False, transform=False)
    assert cT is None and all(np.array_equal(o, x) for o, x in zip(cout, b.blocks))
    for j, (prb, ref, P, Q, w) in enumerate(inputs):
        want, kw, _, per = ob.best_align(prb, ref, P, Q, w, 1)
        assert abs(c[j] - want) <= 1e-12 * (1 + want) and abs(per[cb[j]] - want) <= 1e-12 * (1 + want)


def test_a_hundred_thousand_mappings(cuda):
    rng = np.random.default_rng(30)
    b, inputs = Batch(), []
    for L in (3, 50):
        prb, ref, P, Q, w = posed(rng, L, 100000, L == 3)
        b.job(b.conf(prb), b.conf(ref), b.set(P, Q, w))
        inputs.append((prb, ref, P, Q, w))
    rmsd, best, T, out = b.run()
    for j, x in enumerate(inputs):
        check(*x, False, 50, rmsd[j], best[j], T[j], out[b.jobs[j][0]])


def test_an_exact_tie_picks_the_lower_index(cuda):
    """The best mapping listed twice among others, within one group of 32 lanes, across groups, and packed beside other
    jobs: the lower of the two indices wins, aligned and in place."""
    rng = np.random.default_rng(31)
    for mode in (0, 1):
        b, expect = Batch(), []
        for K, first, second in ((2, 1, 0), (5, 1, 4), (33, 3, 32), (100, 40, 70), (100, 20, 5)):
            prb, ref, P, Q, _ = posed(rng, 12, K + 1, False)
            kb = ob.best_align(prb, ref, P, Q, None, mode)[1]
            others = np.delete(Q, kb, 0)
            Q2 = others[:K].copy()
            Q2[first] = Q2[second] = Q[kb]
            b.job(b.conf(prb), b.conf(ref), b.set(P, Q2))
            expect.append(min(first, second))
        _, best, _, _ = b.run(mode, move=False, transform=False)
        assert best.tolist() == expect


@pytest.mark.parametrize("reflect", [False, True])
def test_one_mapping_is_b200mol_align(cuda, reflect):
    rng = np.random.default_rng(32 + reflect)
    b, lists, jobs = Batch(), ma.PairLists(), []
    for L in (1, 2, 3, 31, 32, 33, 64, 1000):
        for weighted in (False, True):
            prb, ref, P, Q, w = posed(rng, L, 1, weighted, offset=100.0)
            p, r = b.conf(prb), b.conf(ref)
            b.job(p, r, b.set(P, Q, w))
            jobs.append((p, r, lists.add(np.stack([P, Q[0]], 1), w)))
    rmsd, best, T, out = b.run(0, reflect)
    atoms = np.array([len(x) for x in b.blocks], np.int64)
    xyz = torch.from_numpy(np.concatenate(b.blocks)).cuda()
    cas = torch.from_numpy(np.concatenate([[0], np.cumsum(atoms)]).astype(np.int32)).cuda()
    p, r, l = (np.array(x) for x in zip(*jobs))
    want, Tw = ma._run(p, r, l, atoms, cas, xyz, lists, reflect, 50, True, True, None)
    assert np.array_equal(rmsd, want.cpu().numpy()) and np.array_equal(T, Tw.cpu().numpy())
    assert np.array_equal(np.concatenate(out), xyz.cpu().numpy()) and not best.any()


def conformer_set(rng, c, n, spread=0.5):
    base = rng.normal(size=(n, 3)) * 1.5
    return [(base + rng.normal(size=(n, 3)) * spread) @ rotation(rng).T + rng.normal(size=3) * 3.0 for _ in range(c)]


def test_a_molecule_against_itself_is_get_all_conformer_best_rms(cuda, Chem):
    rng = np.random.default_rng(33)
    n, C = 9, 12
    confs = conformer_set(rng, C, n)
    matches = [tuple(range(n))] + [tuple(rng.permutation(n)) for _ in range(6)]
    mol = make_mol(Chem, n, confs, matches)
    maps = [[(q, t[q]) for q in range(n)] for t in matches]
    for prealigned in (False, True):
        want = cr.GetAllConformerBestRMS(mol, map=maps, prealigned=prealigned).numpy()
        b = Batch()
        xs = [b.conf(c) for c in confs]
        s = b.set(np.arange(n), np.array(matches))
        for i in range(1, C):
            for j in range(i):
                b.job(xs[i], xs[j], s)
        got, _, _, _ = b.run(1 if prealigned else 0, move=False, transform=False)
        assert np.abs(got - want).max() <= (1e-12 if prealigned else 1e-7)


def test_what_moves(cuda, Chem):
    rng = np.random.default_rng(34)
    n = 10
    confs = conformer_set(rng, 5, n)
    ref_xyz = confs[0] + 1.0
    matches = [tuple(range(n)), tuple(rng.permutation(n))]
    w = rng.uniform(0.5, 1.5, n)
    make = lambda: (make_mol(Chem, n, confs, matches), make_mol(Chem, n, [ref_xyz], matches))  # noqa: E731
    prb, ref = make()
    before = [c.GetPositions().copy() for c in prb.GetConformers()]
    c = ma.CalcRMSBatch([prb], [ref], weights=[w])[0].numpy()
    r, T, k = (x[0].numpy() for x in ma.GetBestAlignmentTransformBatch([prb], [ref], weights=[w]))
    assert all(np.array_equal(a, x.GetPositions()) for a, x in zip(before, prb.GetConformers()))
    assert np.array_equal(ref.GetConformers()[0].GetPositions(), ref_xyz)
    P, Q = np.arange(n), np.array(matches)
    for i in range(5):
        want_c = ob.best_align(before[i], ref_xyz, P, Q, w, 1)[0]
        want, kw, _, _ = ob.best_align(before[i], ref_xyz, P, Q, w)
        assert abs(c[i] - want_c) <= 1e-12 and abs(r[i] - want) <= 1e-10 and k[i] == kw
    # GetBestRMS moves the listed probes only, by the transform of the transform form
    moved = ma.GetBestRMSBatch([prb], [ref], prbIds=[[1, 3]], weights=[w])[0].numpy()
    assert np.array_equal(moved, r[[1, 3]])
    for i, x in enumerate(prb.GetConformers()):
        if i in (1, 3):
            assert np.abs(x.GetPositions() - oa.apply(T[i], before[i])).max() <= 1e-9
        else:
            assert np.array_equal(x.GetPositions(), before[i])
    # the single forms, the same numbers
    prb, ref = make()
    one, T1, match = ma.GetBestAlignmentTransform(prb, ref, prbId=2, weights=w)
    assert one == r[2] and np.array_equal(T1, T[2]) and match == tuple((q, matches[k[2]][q]) for q in range(n))
    assert ma.CalcRMS(prb, ref, 2, weights=w) == c[2]
    assert ma.GetBestRMS(prb, ref, 2, weights=w) == r[2]
    # a reference conformer among the probes' molecule: None lists every other conformer
    mol = make_mol(Chem, n, confs, matches)
    got = ma.GetBestRMSBatch([mol], [mol], refIds=[2])[0].numpy()
    assert len(got) == 4 and np.array_equal(mol.GetConformers()[2].GetPositions(), confs[2])
    # a conformer against itself is compared with a copy of itself: ~0, and it moves by ~the identity
    mol = make_mol(Chem, n, confs, matches)
    assert ma.GetBestRMS(mol, mol, 3, 3) <= 1e-7
    assert np.abs(mol.GetConformers()[3].GetPositions() - confs[3]).max() <= 1e-7


def device_result(coords, rng):
    entries = [(m, k, c) for m, confs in enumerate(coords) for k, c in enumerate(confs)]
    entries = [entries[i] for i in rng.permutation(len(entries))]
    t = lambda a: AsyncGpuResult(torch.as_tensor(np.asarray(a)).cuda())  # noqa: E731
    starts = np.concatenate([[0], np.cumsum([len(e[2]) for e in entries])]).astype(np.int32)
    return Device3DResult(t(np.concatenate([e[2] for e in entries])), t(starts),
                          t(np.array([e[0] for e in entries], np.int32)), t(np.array([e[1] for e in entries], np.int32)),
                          0, len(coords)), entries


def test_rdkit_path_equals_the_device_result(cuda, Chem):
    rng = np.random.default_rng(35)
    sizes = [(6, 14, 3), (0, 6, 1), (40, 9, 40), (3, 17, 2)]  # (conformers, atoms, mappings)
    coords = [conformer_set(rng, c, n) for c, n, _ in sizes]
    matches = [[tuple(range(n))] + [tuple(rng.permutation(n)) for _ in range(K - 1)] for _, n, K in sizes]
    refs = [make_mol(Chem, n, conformer_set(rng, 2, n), m) for (_, n, _), m in zip(sizes, matches)]
    weights = [rng.uniform(0.1, 1.0, 14), None, None, rng.uniform(0.1, 1.0, 17)]
    prbIds = [[5, 0, 2], None, None, [1]]
    mols = [make_mol(Chem, n, c, m) for (_, n, _), c, m in zip(sizes, coords, matches)]
    res, entries = device_result(coords, rng)
    for fn in (ma.CalcRMSBatch, lambda *a, **k: ma.GetBestAlignmentTransformBatch(*a, reflect=True, **k)[1]):
        host = fn(mols, refs, prbIds, [1, -1, 0, 1], weights=weights)
        dev = fn([make_mol(Chem, n, (), m) for (_, n, _), m in zip(sizes, matches)], refs, prbIds, [1, -1, 0, 1],
                 weights=weights, coordinates=res)
        assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(host, dev))
    host = ma.GetBestRMSBatch(mols, refs, prbIds, [1, -1, 0, 1], weights=weights)
    dev = ma.GetBestRMSBatch([make_mol(Chem, n, (), m) for (_, n, _), m in zip(sizes, matches)], refs, prbIds,
                             [1, -1, 0, 1], weights=weights, coordinates=res)
    assert [x.torch().numel() for x in dev] == [3, 0, 40, 1]
    assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(host, dev))
    vals = res.values.torch().cpu().numpy()
    starts = res.atom_starts.torch().cpu().numpy()
    for e, (m, k, _) in enumerate(entries):  # moved on both paths alike, unlisted probes untouched
        assert np.array_equal(vals[starts[e]:starts[e + 1]], mols[m].GetConformers()[k].GetPositions()), (m, k)


def test_repeatable_batch_independent_and_on_any_stream(cuda):
    rng = np.random.default_rng(36)
    b = Batch()
    for K, L in SHAPES:
        prb, ref, P, Q, w = posed(rng, L, K, True)
        b.job(b.conf(prb), b.conf(ref), b.set(P, Q, w))
    a = b.run()
    again = b.run(stream=torch.cuda.Stream())
    assert all(np.array_equal(x, y) for x, y in zip(a[:3], again[:3]))
    for j in (0, 5, len(SHAPES) - 1):
        one = Batch()
        blocks = [b.blocks[b.jobs[j][0]], b.blocks[b.jobs[j][1]]]
        one.job(one.conf(blocks[0]), one.conf(blocks[1]), one.set(*b.sets[b.jobs[j][2]]))
        r, k, T, _ = one.run()
        assert r[0] == a[0][j] and k[0] == a[1][j] and np.array_equal(T[0], a[2][j])


def test_a_million_jobs(cuda):
    """1e6 probes of 8 atoms onto 1e4 references through 100 shared sets of K = 3 mappings of 6 atoms, moved."""
    rng = np.random.default_rng(37)
    n_ref, per, A = 10000, 100, 8
    refs = rng.normal(size=(n_ref, A, 3)) * 2.0
    probes = np.repeat(refs, per, 0) + rng.normal(size=(n_ref * per, A, 3)) * 0.3
    sets = [(np.arange(6), np.stack([rng.permutation(A)[:6] for _ in range(3)]), None) for _ in range(100)]
    xyz_h = np.concatenate([refs.reshape(-1, 3), probes.reshape(-1, 3)])
    xyz = torch.from_numpy(xyz_h).cuda()
    n = n_ref * (per + 1)
    cas = torch.arange(0, n * A + 1, A, dtype=torch.int32).cuda()
    jp = np.arange(n_ref, n)
    jr = np.repeat(np.arange(n_ref), per)
    js = jr % 100
    rmsd, best, T = ma._run_best(jp, jr, js, np.full(n, A, np.int64), cas, xyz, sets, 0, False, 50, True, True, None)
    torch.cuda.synchronize()
    rmsd, best, T = rmsd.cpu().numpy(), best.cpu().numpy(), T.cpu().numpy()
    out = xyz.cpu().numpy().reshape(n, A, 3)
    for j in rng.choice(len(jp), 300, replace=False):
        P, Q, _ = sets[js[j]]
        want, kw, _, _ = ob.best_align(probes[j], refs[jr[j]], P, Q)
        assert abs(rmsd[j] - want) <= 1e-10 and best[j] == kw
        assert np.abs(out[jp[j]] - oa.apply(T[j], probes[j])).max() <= 1e-9
    assert np.array_equal(out[:n_ref], refs)
