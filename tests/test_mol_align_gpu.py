"""Conformer alignment on the GPU (b200mol_align, nvmolkit_b200.molAlign) against the fp64 oracle (oracle_align.c): pair
counts around the warp width, atom subsets, weights, mirror images and capped Jacobi sweeps in one mixed batch;
self-consistency on degenerate inputs; agreement with the conformer RMSD matrices; the RDKit and Device3DResult paths;
repeatability, batch independence and streams; a batch of 2e5 jobs. Every error is a host-side check: no test here
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


def make_mol(Chem, n, confs=()):
    return Chem.Mol({"z": [6] * n, "bonds": [], "nbrs": [[] for _ in range(n)]}, conformers=list(confs))


def rotation(rng):
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1.0
    return q


def horn(p, q, w, reflect):
    """(G = sum w |p - p_bar|^2 + sum w |r - r_bar|^2, eigenvalues of N(S) ascending) by NumPy."""
    w = np.ones(len(p)) if w is None else w
    p = -p if reflect else p
    P = p - (w[:, None] * p).sum(0) / w.sum()
    Q = q - (w[:, None] * q).sum(0) / w.sum()
    S = (w[:, None] * P).T @ Q
    N = np.array([[S[0, 0] + S[1, 1] + S[2, 2], S[1, 2] - S[2, 1], S[2, 0] - S[0, 2], S[0, 1] - S[1, 0]],
                  [S[1, 2] - S[2, 1], S[0, 0] - S[1, 1] - S[2, 2], S[0, 1] + S[1, 0], S[2, 0] + S[0, 2]],
                  [S[2, 0] - S[0, 2], S[0, 1] + S[1, 0], -S[0, 0] + S[1, 1] - S[2, 2], S[1, 2] + S[2, 1]],
                  [S[0, 1] - S[1, 0], S[2, 0] + S[0, 2], S[1, 2] + S[2, 1], -S[0, 0] - S[1, 1] + S[2, 2]]])
    return float((w * (P * P).sum(1)).sum() + (w * (Q * Q).sum(1)).sum()), np.linalg.eigvalsh(N)


class Batch:
    """Conformers in one space, pair lists and jobs: the direct form of b200mol_align."""

    def __init__(self):
        self.blocks, self.lists, self.jobs = [], ma.PairLists(), []

    def conf(self, xyz) -> int:
        self.blocks.append(np.asarray(xyz, np.float64))
        return len(self.blocks) - 1

    def job(self, prb, ref, pairs, w=None):
        self.jobs.append((self.conf(prb), self.conf(ref), self.lists.add(pairs, w)))

    def run(self, reflect=False, maxIters=50, move=True, stream=None):
        atoms = np.array([len(b) for b in self.blocks], np.int64)
        xyz = torch.from_numpy(np.concatenate(self.blocks)).cuda()
        cas = torch.from_numpy(np.concatenate([[0], np.cumsum(atoms)]).astype(np.int32)).cuda()
        p, r, l = (np.array(x) for x in zip(*self.jobs))
        rmsd, T = ma._run(p, r, l, atoms, cas, xyz, self.lists, reflect, maxIters, move, True, stream)
        torch.cuda.synchronize()
        out = np.split(xyz.cpu().numpy(), np.cumsum(atoms)[:-1])
        return rmsd.cpu().numpy(), T.cpu().numpy(), out


def mixed_batch(rng, weighted, offset=0.0):
    """Probe / reference pairs at L = 1, 2, 3, 31, 32, 33, 64, 255, 1000 pairs of A = L + 7 atoms, atoms chosen at
    random on both sides; the probe a noisy rigid motion of the reference."""
    b, inputs = Batch(), []
    for L in (1, 2, 3, 31, 32, 33, 64, 255, 1000):
        for _ in range(3):
            A = L + 7
            ref = rng.normal(size=(A, 3)) * 2.0 + offset
            prb = (ref - ref.mean(0)) @ rotation(rng) + rng.normal(size=3) * 5.0 + rng.normal(size=(A, 3)) * 0.4 + offset
            pairs = np.stack([rng.choice(A, L, replace=False), rng.choice(A, L, replace=False)], 1)
            w = rng.uniform(0.0, 2.0, L) if weighted else None
            if w is not None and w.sum() == 0:
                w[0] = 1.0
            b.job(prb, ref, pairs, w)
            inputs.append((prb, ref, pairs, w))
    return b, inputs


@pytest.mark.parametrize("maxIters", [1, 3, 50])
@pytest.mark.parametrize("reflect", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_kernel_matches_the_oracle(cuda, weighted, reflect, maxIters):
    rng = np.random.default_rng(10 + 2 * weighted + reflect)
    b, inputs = mixed_batch(rng, weighted)
    rmsd, T, out = b.run(reflect, maxIters)
    for j, (prb, ref, pairs, w) in enumerate(inputs):
        L = len(pairs)
        want, Tw = oa.align(prb, ref, pairs, w, reflect, maxIters)
        G, ev = horn(prb[pairs[:, 0]], ref[pairs[:, 1]], w, reflect)
        assert abs(rmsd[j] ** 2 - want ** 2) <= 1e-12 * G / L + 1e-26, (j, L, rmsd[j], want)  # + the rounding of L = 1
        moved = out[b.jobs[j][0]]
        assert np.abs(moved - oa.apply(T[j], prb)).max() <= 1e-9  # the kernel moves by the transform it reports
        gap = ev[-1] - ev[-2]
        if maxIters == 50 and L > 2 and gap >= 1e-3 * abs(ev[-1]):
            assert np.abs(T[j] - Tw).max() <= 1e-9, (j, L)
            assert np.abs(moved - oa.apply(Tw, prb)).max() <= 1e-9, (j, L)
        if maxIters == 50:  # self-consistency: the moved probe's plain RMSD against the reference
            ww = np.ones(L) if w is None else w
            pre = np.sqrt((ww * ((moved[pairs[:, 0]] - ref[pairs[:, 1]]) ** 2).sum(1)).sum() / L)
            assert abs(pre ** 2 - rmsd[j] ** 2) <= 1e-10 * G / L + 1e-20, (j, L, pre, rmsd[j])
        assert np.array_equal(out[b.jobs[j][1]], ref)
    one = [j for j, x in enumerate(inputs) if len(x[2]) == 1]
    assert all(rmsd[j] == 0.0 and np.array_equal(T[j][:3, :3], (-1 if reflect else 1) * np.eye(3)) for j in one)


def test_degenerate_inputs_are_self_consistent(cuda):
    """Collinear atoms (lambda not simple), coincident atoms (N = 0), a 10^4 A offset: the moved probe reproduces the
    RMSD, and the RMSD matches the oracle."""
    rng = np.random.default_rng(3)
    b, inputs = Batch(), []
    line = np.outer(np.linspace(-2, 2, 6), [0.3, -0.5, 0.8])
    cases = [(line, line @ rotation(rng).T + 1.0), (line[:2], line[:2] + 4.0), (np.ones((5, 3)), rng.normal(size=(5, 3))),
             (rng.normal(size=(5, 3)), np.zeros((5, 3))), (line + 1e4, line @ rotation(rng).T - 1e4)]
    for prb, ref in cases:
        pairs = np.stack([np.arange(len(prb))] * 2, 1)
        b.job(prb, ref, pairs)
        inputs.append((prb, ref, pairs))
    rmsd, T, out = b.run()
    for j, (prb, ref, pairs) in enumerate(inputs):
        G, _ = horn(prb, ref, None, False)
        want, _ = oa.align(prb, ref, pairs)
        assert abs(rmsd[j] ** 2 - want ** 2) <= 1e-12 * G / len(prb) + 1e-20
        pre = np.sqrt(((out[b.jobs[j][0]] - ref) ** 2).sum() / len(prb))
        assert abs(pre ** 2 - rmsd[j] ** 2) <= 1e-10 * max(G, 1.0) / len(prb), (j, pre, rmsd[j])
        assert abs(np.linalg.det(T[j][:3, :3]) - 1.0) <= 1e-12


def test_far_from_the_origin(cuda):
    rng = np.random.default_rng(4)
    near_b, inputs = mixed_batch(rng, True)
    rng = np.random.default_rng(4)
    far_b, _ = mixed_batch(rng, True, offset=1e4)
    near, Tn, _ = near_b.run()
    far, Tf, _ = far_b.run()
    # the coordinates themselves are rounded to ~2e-12 A at 1e4 A: the results may differ by that much, no more
    assert np.abs(near - far).max() <= 1e-9
    unique = np.array([len(x[2]) != 2 for x in inputs])  # two pairs are collinear: the rotation is not unique
    assert np.abs(Tn[unique, :3, :3] - Tf[unique, :3, :3]).max() <= 1e-9


def conformer_set(rng, c, n, spread=0.5):
    base = rng.normal(size=(n, 3)) * 1.5
    return [(base + rng.normal(size=(n, 3)) * spread) @ rotation(rng).T + rng.normal(size=3) * 3.0 for _ in range(c)]


def test_align_mol_conformers_agrees_with_the_rmsd_matrix(cuda, Chem):
    rng = np.random.default_rng(5)
    mol = make_mol(Chem, 23, conformer_set(rng, 40, 23))
    before = cr.GetConformerRMSMatrix(mol).numpy()
    rms = []
    ma.AlignMolConformers(mol, RMSlist=rms)
    assert len(rms) == 39
    idx = [i * (i - 1) // 2 for i in range(1, 40)]
    assert np.abs(np.array(rms) - before[idx]).max() <= 1e-8
    after = cr.GetConformerRMSMatrix(mol, prealigned=True).numpy()
    assert np.abs(np.array(rms) - after[idx]).max() <= 1e-8


def test_reference_and_unlisted_conformers_are_untouched(cuda, Chem):
    rng = np.random.default_rng(6)
    confs = conformer_set(rng, 8, 11)
    mol = make_mol(Chem, 11, confs)
    w = rng.uniform(0.5, 2.0, 5)
    rms = []
    ma.AlignMolConformers(mol, atomIds=[0, 2, 4, 6, 8], confIds=[5, 1, 6], weights=w, reflect=True, RMSlist=rms)
    pos = [c.GetPositions() for c in mol.GetConformers()]
    for k in (0, 2, 3, 4, 5, 7):
        assert np.array_equal(pos[k], confs[k])
    pairs = np.stack([[0, 2, 4, 6, 8]] * 2, 1)
    for k, probe in enumerate((1, 6)):
        want, T = oa.align(confs[probe], confs[5], pairs, w, True)
        assert abs(rms[k] - want) <= 1e-10
        assert np.abs(pos[probe] - oa.apply(T, confs[probe])).max() <= 1e-9


def device_result(coords, rng):
    entries = [(m, k, c) for m, confs in enumerate(coords) for k, c in enumerate(confs)]
    entries = [entries[i] for i in rng.permutation(len(entries))]
    t = lambda a: AsyncGpuResult(torch.as_tensor(np.asarray(a)).cuda())  # noqa: E731
    starts = np.concatenate([[0], np.cumsum([len(e[2]) for e in entries])]).astype(np.int32)
    return Device3DResult(t(np.concatenate([e[2] for e in entries])), t(starts),
                          t(np.array([e[0] for e in entries], np.int32)), t(np.array([e[1] for e in entries], np.int32)),
                          0, len(coords)), entries


def test_rdkit_path_equals_the_device_result(cuda, Chem):
    rng = np.random.default_rng(7)
    coords = [conformer_set(rng, c, n) for c, n in [(5, 14), (0, 6), (40, 9), (1, 3), (33, 17)]]
    atomIds = [None, None, [0, 3, 5, 8], None, list(range(0, 17, 2))]
    weights = [rng.uniform(0.1, 1.0, 14), None, None, None, rng.uniform(0.1, 1.0, 9)]
    confIds = [None, None, [7, 3, 12, 0, 39], None, None]
    mols = [make_mol(Chem, len(c[0]) if c else 6, c) for c in coords]
    host = ma.AlignMolConformersBatch(mols, atomIds, confIds, weights, maxIters=50)
    res, entries = device_result(coords, rng)
    energies = AsyncGpuResult(torch.arange(len(entries), dtype=torch.float64).cuda())
    res.energies = energies
    dev = ma.AlignMolConformersBatch([make_mol(Chem, len(c[0]) if c else 6) for c in coords], atomIds, confIds, weights,
                                     coordinates=res)
    assert [x.torch().numel() for x in dev] == [4, 0, 4, 0, 32]
    assert all(torch.equal(x.torch(), y.torch()) for x, y in zip(host, dev))
    vals = res.values.torch().cpu().numpy()
    starts = res.atom_starts.torch().cpu().numpy()
    for e, (m, k, _) in enumerate(entries):
        assert np.array_equal(vals[starts[e]:starts[e + 1]], mols[m].GetConformers()[k].GetPositions()), (m, k)
    assert torch.equal(res.energies.torch(), torch.arange(len(entries), dtype=torch.float64).cuda())
    with pytest.raises(ValueError, match="contiguous float64"):
        bad, _ = device_result([[c.astype(np.float32) for c in confs] for confs in coords], rng)
        ma.AlignMolConformersBatch([make_mol(Chem, len(c[0]) if c else 6) for c in coords], coordinates=bad)


def test_repeatable_batch_independent_and_on_any_stream(cuda, Chem):
    rng = np.random.default_rng(8)
    coords = [conformer_set(rng, c, n) for c, n in [(12, 30), (50, 7), (3, 64)]]
    run = lambda ms, **kw: [r.torch().clone() for r in ma.AlignMolConformersBatch(ms, **kw)]  # noqa: E731
    fresh = lambda: [make_mol(Chem, len(c[0]), c) for c in coords]  # noqa: E731
    a, b = run(fresh()), run(fresh())
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for m in range(3):
        assert torch.equal(run([make_mol(Chem, len(coords[m][0]), coords[m])])[0], a[m])
    s = torch.cuda.Stream()
    mols = fresh()
    c = run(mols, stream=s)
    assert all(torch.equal(x, y) for x, y in zip(a, c))
    ref = fresh()
    ma.AlignMolConformersBatch(ref)
    for m1, m2 in zip(mols, ref):
        assert all(np.array_equal(x.GetPositions(), y.GetPositions()) for x, y in zip(m1.GetConformers(), m2.GetConformers()))


def test_align_mol_and_transforms(cuda, Chem):
    rng = np.random.default_rng(9)
    ref_xyz = rng.normal(size=(12, 3)) * 2.0
    tmpl = make_mol(Chem, 12, [ref_xyz])
    probes = [make_mol(Chem, 15, [rng.normal(size=(15, 3)) * 2.0 + 3.0]) for _ in range(50)]
    amap = [(k + 2, k) for k in range(10)]
    w = rng.uniform(0.2, 1.0, 10)
    saved = [p.GetConformers()[0].GetPositions().copy() for p in probes]
    rmsd, T = ma.GetAlignmentTransformBatch(probes, [tmpl] * 50, atomMaps=[amap] * 50, weights=[w] * 50, reflect=True)
    rmsd, T = rmsd.numpy(), T.numpy()
    pairs = np.array(amap)
    for i, p in enumerate(probes):
        assert np.array_equal(p.GetConformers()[0].GetPositions(), saved[i])  # nothing moved
        want, Tw = oa.align(saved[i], ref_xyz, pairs, w, True)
        assert abs(rmsd[i] - want) <= 1e-10 and np.abs(T[i] - Tw).max() <= 1e-9
    assert np.array_equal(tmpl.GetConformers()[0].GetPositions(), ref_xyz)
    one, T1 = ma.GetAlignmentTransform(probes[3], tmpl, atomMap=amap, weights=w, reflect=True)
    assert one == rmsd[3] and np.array_equal(T1, T[3])
    got = ma.AlignMol(probes[3], tmpl, atomMap=amap, weights=w, reflect=True)
    assert got == rmsd[3]
    assert np.abs(probes[3].GetConformers()[0].GetPositions() - oa.apply(T[3], saved[3])).max() <= 1e-9
    moved = ma.AlignMolBatch(probes[4:9], [tmpl] * 5, atomMaps=[amap] * 5, weights=[w] * 5, reflect=True).numpy()
    assert np.array_equal(moved, rmsd[4:9])
    # identity map over equal atom counts, a non-default stream
    a = make_mol(Chem, 15, [rng.normal(size=(15, 3))])
    s = torch.cuda.Stream()
    r, _ = ma.GetAlignmentTransform(a, probes[0], stream=s)
    assert abs(r - oa.align(a.GetConformers()[0].GetPositions(), saved[0])[0]) <= 1e-10


def test_two_hundred_thousand_jobs(cuda):
    """2e5 probes of 20 atoms onto 2,000 references through 2,000 shared 12-pair weighted lists, moved in place."""
    rng = np.random.default_rng(11)
    n_ref, per, A = 2000, 100, 20
    refs = rng.normal(size=(n_ref, A, 3)) * 2.0
    probes = np.repeat(refs, per, 0) + rng.normal(size=(n_ref * per, A, 3)) * 0.3 + rng.normal(size=(n_ref * per, 1, 3))
    lists = ma.PairLists()
    for _ in range(n_ref):
        lists.add(np.stack([rng.choice(A, 12, replace=False)] * 2, 1), rng.uniform(0.5, 1.5, 12))
    xyz_h = np.concatenate([refs.reshape(-1, 3), probes.reshape(-1, 3)])
    xyz = torch.from_numpy(xyz_h).cuda()
    n = n_ref + n_ref * per
    atoms = np.full(n, A, np.int64)
    cas = torch.arange(0, n * A + 1, A, dtype=torch.int32).cuda()
    jp = np.arange(n_ref, n)
    jr = np.repeat(np.arange(n_ref), per)
    rmsd, T = ma._run(jp, jr, jr, atoms, cas, xyz, lists, False, 50, True, True, None)
    torch.cuda.synchronize()
    rmsd, T, out = rmsd.cpu().numpy(), T.cpu().numpy(), xyz.cpu().numpy().reshape(n, A, 3)
    assert np.array_equal(out[:n_ref], refs)
    start, pairs, wts = lists.tables()
    for j in rng.choice(len(jp), 300, replace=False):
        l = jr[j]
        pr = pairs[start[l]:start[l + 1]]
        want, Tw = oa.align(probes[j], refs[l], pr, wts[start[l]:start[l + 1]])
        assert abs(rmsd[j] - want) <= 1e-10 and np.abs(T[j] - Tw).max() <= 1e-9
        assert np.abs(out[n_ref + j] - oa.apply(Tw, probes[j])).max() <= 1e-9
