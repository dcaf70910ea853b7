"""GPU parity of path B (force fields, BFGS, DG preparation, ETKDG) against the CPU oracle, through the C-ABI."""

import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from nvmolkit_b200 import synthetic as S
from nvmolkit_b200.forcefield import ConformerBatch, FlatSystem

pytestmark = pytest.mark.gpu

E_RTOL = 1e-4  # north_star: minimised energies within 1e-4 relative


def _rel(a, b):
    return np.abs(a - b) / np.maximum(1.0, np.abs(b))


# ------------------------------------------------------------------ BFGS on analytic systems (reference known answers)
def test_bfgs_quartic_and_harmonic(cuda):
    from nvmolkit_b200.minimizer import poly_minimize

    sizes = [28, 12, 40, 4]
    starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    n = starts[-1]
    c = np.arange(n, dtype=np.float64)  # tests/test_bfgs_minimizer.cu:822-930: target = global position index
    x0 = c + np.random.default_rng(1).uniform(-2, 2, n)
    x, e, status, iters = poly_minimize(starts, 4, np.ones(n), c, x0, 400, 1e-5, False)
    x = x.cpu().numpy()
    assert np.abs(x - c).max() < 0.1
    for s in range(len(sizes)):
        xo, eo, so, io = oracle.poly_minimize(4, np.ones(sizes[s]), c[starts[s]:starts[s + 1]], x0[starts[s]:starts[s + 1]], 400, 1e-5)
        assert np.abs(x[starts[s]:starts[s + 1]] - xo).max() < 1e-4  # same minimum as the CPU transcription
        assert int(status[s]) == so and abs(int(iters[s]) - io) <= 3
    rng = np.random.default_rng(2)
    w, cc = rng.uniform(0.5, 3.0, n), rng.normal(0, 3, n)
    x, e, status, iters = poly_minimize(starts, 2, w, cc, np.zeros(n), 200, 1e-6, True)
    assert (status.cpu().numpy() == 0).all() and np.abs(x.cpu().numpy() - cc).max() < 1e-4
    x2, e2, status2, iters2 = poly_minimize(starts, 2, w, cc, x.cpu().numpy(), 200, 1e-6, True)  # two calls == one call
    assert (iters2.cpu().numpy() <= 1).all() and np.abs((x2 - x).cpu().numpy()).max() < 1e-6


# ------------------------------------------------------------------ force-field energies and gradients
def test_mmff_energy_and_gradient_parity(cuda):
    from nvmolkit_b200.minimizer import energy_and_grad

    system, xyz, mols = S.random_mmff_system(12, 4, 40, seed=21)
    rng = np.random.default_rng(0)
    coords = [[x + rng.normal(0, 0.05, x.shape), x + rng.normal(0, 0.2, x.shape)] for x in xyz]
    # the same batch again with one molecule near the energy kernel's 948-atom limit among the small ones
    _, xyz_l, mols_l = S.random_mmff_system(1, 440, 450, seed=42)
    assert len(mols_l[0]["z"]) == 895
    mols_b = mols[:6] + mols_l + mols[6:]
    system_b = FlatSystem.from_molecules("mmff", [len(m["z"]) for m in mols_b], [m["terms"] for m in mols_b])
    coords_b = coords[:6] + [[x + rng.normal(0, 0.05, x.shape), x + rng.normal(0, 0.2, x.shape)] for x in xyz_l] + coords[6:]
    for system, coords in ((system, coords), (system_b, coords_b)):
        batch = ConformerBatch.from_coords(system, coords)
        e, g = energy_and_grad(system, batch)
        e, g = e.cpu().numpy(), g.cpu().numpy()
        for c in range(batch.n_conf):
            a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
            eo, go, _ = oracle.ff_energy_grad("mmff", system.atom_counts, system.tables, batch.conf_mol[c], batch.positions[a0:a1])
            assert _rel(e[c], eo) < 1e-11, (len(system.atom_counts), c)
            assert np.abs(g[a0:a1] - go).max() < 1e-9 * max(1.0, np.abs(go).max())


def test_dg_and_etk_energy_and_gradient_parity(cuda):
    from nvmolkit_b200.minimizer import energy_and_grad

    flat, _ = S.random_embed_molecules(8, 4, 16, seed=22)
    rng = np.random.default_rng(1)
    coords = [[rng.normal(0, 2.0, (n, 4)), rng.normal(0, 1.0, (n, 4))] for n in flat.atom_counts]
    for kind, system, kw in (("dg", flat.dg, dict(chiral_weight=1.0, fourth_dim_weight=0.1)),
                             ("dg", flat.dg, dict(chiral_weight=0.2, fourth_dim_weight=1.0)), ("etk", flat.etk, {})):
        batch = ConformerBatch.from_coords(system, coords)
        e, g = energy_and_grad(system, batch, **kw)
        e, g = e.cpu().numpy(), g.cpu().numpy()
        for c in range(batch.n_conf):
            a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
            eo, go, _ = oracle.ff_energy_grad(kind, system.atom_counts, system.tables, batch.conf_mol[c],
                                              batch.positions[a0:a1], dim=4, **kw)
            assert _rel(e[c], eo) < 1e-11, (kind, c)
            assert np.abs(g[a0:a1] - go).max() < 1e-9 * max(1.0, np.abs(go).max())
    # window refresh: energies with the windows re-centred on the evaluated geometry itself
    batch = ConformerBatch.from_coords(flat.etk, coords)
    e, _ = energy_and_grad(flat.etk, batch, want_grad=False, recentre=True)
    for c in range(batch.n_conf):
        a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
        p = batch.positions[a0:a1]
        eo, _, _ = oracle.ff_energy_grad("etk", flat.etk.atom_counts, flat.etk.tables, batch.conf_mol[c], p, False, ref_pos=p)
        assert _rel(e.cpu().numpy()[c], eo) < 1e-11


# ------------------------------------------------------------------ minimisation
def _relaxed_start(system, xyz, iters=2000):
    """'Pre-embedded' coordinates: relax the generator's geometry on the CPU, then perturb (config 4 recipe)."""
    batch = ConformerBatch.from_coords(system, [[x] for x in xyz])
    pos, e, conv, it = oracle.ff_minimize("mmff", system.atom_counts, system.tables, batch.conf_mol, batch.atom_starts,
                                          batch.positions, iters, 1e-4)
    return [pos[batch.atom_starts[c]:batch.atom_starts[c + 1]] for c in range(batch.n_conf)]


def test_mmff_minimize_parity(cuda):
    from nvmolkit_b200.minimizer import minimize

    system, xyz, _ = S.random_mmff_system(10, 4, 30, seed=23)
    relaxed = _relaxed_start(system, xyz)
    rng = np.random.default_rng(3)
    coords = [[r + rng.normal(0, 0.1, r.shape) for _ in range(3)] for r in relaxed]
    batch = ConformerBatch.from_coords(system, coords)
    res = minimize(system, batch, 200, 1e-4)
    pos_o, e_o, conv_o, it_o = oracle.ff_minimize("mmff", system.atom_counts, system.tables, batch.conf_mol, batch.atom_starts,
                                                  batch.positions, 200, 1e-4)
    e, st = res.energies.cpu().numpy(), res.status.cpu().numpy()
    pos = res.positions.cpu().numpy()
    # reported energy == energy of the returned coordinates (src/minimizer/bfgs_minimize.cu:1050-1052)
    for c in range(batch.n_conf):
        a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
        ec = oracle.ff_energy_grad("mmff", system.atom_counts, system.tables, batch.conf_mol[c], pos[a0:a1], False)[0]
        assert _rel(e[c], ec) < 1e-10
    both = (st == 0) & (conv_o == 1)
    assert both.mean() > 0.8
    # gradients are summed in a fixed order (wave schedule, no atomics): EVERY conformer that converged on both sides
    # must sit in the same minimum, energy within north_star's 1e-4 relative
    rel = _rel(e[both], e_o[both])
    assert (rel < E_RTOL).all(), rel.max()
    assert ((st == 0) == (conv_o == 1)).mean() > 0.9
    for c in np.nonzero(both)[0]:  # positions agree too (RMSD < 0.05 A; north_star's bar is 0.5 A)
        a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
        assert np.sqrt(((pos[a0:a1] - pos_o[a0:a1]) ** 2).sum(1).mean()) < 0.05
    # same number of BFGS iterations as the CPU transcription on almost every conformer (the convergence-rate check)
    it_g = res.iters.cpu().numpy()
    assert (np.abs(it_g[both] - it_o[both]) <= 2).mean() > 0.8, (it_g, it_o)
    # and a second GPU run repeats the first bit for bit
    res2 = minimize(system, batch, 200, 1e-4)
    assert torch.equal(res2.energies, res.energies) and torch.equal(res2.positions, res.positions)
    assert torch.equal(res2.iters, res.iters) and torch.equal(res2.status, res.status)


def test_mmff_optimize_api_and_large_molecule(cuda):
    from nvmolkit_b200.mmffOptimization import FlatMMFFMolecules, MMFFOptimizeMoleculesConfs
    from nvmolkit_b200.types import CoordinateOutput

    system, xyz, _ = S.random_mmff_system(4, 30, 70, seed=24)  # up to ~150 atoms: beyond the reference's 64-atom shared-memory path
    batch = ConformerBatch.from_coords(system, [[x, x + 0.05] for x in xyz])
    energies, coords = MMFFOptimizeMoleculesConfs(FlatMMFFMolecules(system, batch), maxIters=50)
    assert [len(e) for e in energies] == [2, 2, 2, 2]
    for m in range(4):
        for k in range(2):
            e0 = oracle.ff_energy_grad("mmff", system.atom_counts, system.tables, m, batch.positions[batch.atom_starts[2 * m + k]:batch.atom_starts[2 * m + k + 1]], False)[0]
            e1 = oracle.ff_energy_grad("mmff", system.atom_counts, system.tables, m, coords[m][k], False)[0]
            assert e1 < e0 and abs(e1 - energies[m][k]) < 1e-8 * max(1, abs(e1))
    dev = MMFFOptimizeMoleculesConfs(FlatMMFFMolecules(system, batch), maxIters=50, output=CoordinateOutput.DEVICE)
    assert dev.num_conformers == 8 and dev.values.torch().shape == (int(batch.atom_starts[-1]), 3)
    # two GPU runs give the same bits (fixed-order gradient and Hessian-sweep sums)
    assert np.array_equal(dev.energies.numpy(), np.array(energies).ravel())
    assert len(dev.per_molecule()) == 4 and dev.dense().values.shape[:2] == (4, 2)


def test_dg_and_etk_minimize_parity(cuda):
    from nvmolkit_b200.minimizer import minimize

    flat, _ = S.random_embed_molecules(6, 4, 12, seed=25)
    rng = np.random.default_rng(4)
    start = [[(rng.random((n, 4)) - 0.5) * 10.0] for n in flat.atom_counts]
    batch = ConformerBatch.from_coords(flat.dg, start)
    res = minimize(flat.dg, batch, 400, 1e-3, chiral_weight=1.0, fourth_dim_weight=0.1)
    pos_o, e_o, conv_o, it_o = oracle.ff_minimize("dg", flat.dg.atom_counts, flat.dg.tables, batch.conf_mol, batch.atom_starts,
                                                  batch.positions, 400, 1e-3, dim=4, chiral_weight=1.0, fourth_dim_weight=0.1)
    e = res.energies.cpu().numpy()
    # chaotic from a random start: compare through the property both must satisfy — a low DG energy at the reported point
    pos = res.positions.cpu().numpy()
    for c in range(batch.n_conf):
        a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
        ec = oracle.ff_energy_grad("dg", flat.dg.atom_counts, flat.dg.tables, c, pos[a0:a1], False, dim=4)[0]
        assert _rel(e[c], ec) < 1e-10
    assert np.median(e) < 10 * max(1.0, np.median(e_o)) and np.median(e) < 5.0
    # ETK from the CPU result (a settled geometry): same trajectory, tight agreement
    batch2 = ConformerBatch(batch.conf_mol, batch.atom_starts, pos_o)
    res2 = minimize(flat.etk, batch2, 300, 1e-3, recentre=True)
    pos2_o, e2_o, conv2_o, _ = oracle.ff_minimize("etk", flat.etk.atom_counts, flat.etk.tables, batch2.conf_mol, batch2.atom_starts,
                                                  batch2.positions, 300, 1e-3, recentre=True)
    e2 = res2.energies.cpu().numpy()
    pos2 = res2.positions.cpu().numpy()
    for c in range(batch2.n_conf):  # reported energy = ETK energy at the returned point w.r.t. the refreshed windows
        a0, a1 = batch2.atom_starts[c], batch2.atom_starts[c + 1]
        ec = oracle.ff_energy_grad("etk", flat.etk.atom_counts, flat.etk.tables, c, pos2[a0:a1], False, ref_pos=pos_o[a0:a1])[0]
        assert _rel(e2[c], ec) < 1e-9
    close = _rel(e2, e2_o) < 1e-3
    assert close.mean() >= 0.5
    # bit-reproducible: DG from a random start and ETK, run twice
    res_b = minimize(flat.dg, batch, 400, 1e-3, chiral_weight=1.0, fourth_dim_weight=0.1)
    assert torch.equal(res_b.energies, res.energies) and torch.equal(res_b.positions, res.positions)
    res2_b = minimize(flat.etk, batch2, 300, 1e-3, recentre=True)
    assert torch.equal(res2_b.energies, res2.energies) and torch.equal(res2_b.positions, res2.positions)


# ------------------------------------------------------------------ DG preparation
def test_triangle_smoothing_equals_cpu(cuda):
    from nvmolkit_b200.dgprep import triangle_smooth

    flat, mols = S.random_embed_molecules(10, 3, 30, seed=26)
    raw = [m["bounds_raw"] for m in mols]
    bad = np.array([[0, 1.0, 1.0], [0.9, 0, 1.0], [5.0, 0.9, 0]])
    got, ok = triangle_smooth(raw + [bad])
    for i, m in enumerate(mols):
        want, okc = oracle.triangle_smooth(m["bounds_raw"])
        assert ok[i] and okc
        assert np.array_equal(got[i], want)  # min / add / subtract only: bit-identical
    assert not ok[-1]


def test_triangle_smoothing_large_matrix_in_global_memory(cuda):
    from nvmolkit_b200.dgprep import triangle_smooth

    rng = np.random.default_rng(5)
    n = 200  # 320 KB > shared memory: in-place global path
    xyz = rng.normal(0, 6.0, (n, 3))
    d = np.linalg.norm(xyz[:, None] - xyz[None], axis=2)
    b = np.triu(d + rng.uniform(0.1, 3.0, (n, n)), 1) + np.tril(np.maximum(d - rng.uniform(0.1, 3.0, (n, n)), 0.0), -1)
    got, ok = triangle_smooth([b])
    want, okc = oracle.triangle_smooth(b)
    assert ok[0] == okc and np.array_equal(got[0], want)


def test_eigen_known_answers_and_embedding(cuda):
    from nvmolkit_b200.dgprep import eig_topk, metric_embed

    m1 = np.array([0.0, 1.0, 1.732, 2.268, 3.268, 1.0, 0.0, 1.0, 1.732, 2.268, 1.732, 1.0, 0.0, 1.0, 1.732, 2.268, 1.732,
                   1.0, 0.0, 1.0, 3.268, 2.268, 1.732, 1.0, 0.0]).reshape(5, 5)
    m2 = np.ones((5, 5)) - np.eye(5)
    vals, vecs, conv = eig_topk([m1, m2], 5)  # internal start vectors
    assert np.allclose(vals[0], [6.981, -3.982, -1.395, -1.016, -0.586], atol=1e-2)  # tests/test_coordgen.cu:98-135
    assert np.allclose(vals[1], [4.0, -1.0, -1.0, -1.0, -1.0], atol=1e-2)
    rng = np.random.default_rng(6)
    mats, v0s = [], []
    for n in (6, 17, 40, 90):
        a = rng.normal(0, 1, (n, n))
        mats.append(a @ a.T + n * np.eye(n))
        v0s.append(rng.random((3, n)))
    vals, vecs, conv = eig_topk(mats, 3, v0=v0s)
    for i, m in enumerate(mats):
        vo, veco, k = oracle.power_eigen(m, 3, v0s[i])
        assert conv[i] == k == 3
        assert np.allclose(vals[i], vo, rtol=1e-9) and np.allclose(np.abs(vecs[i]), np.abs(veco), atol=1e-7)
    for dim in (3, 4):  # the reference's coordinate generator is 3-D only (src/forcefields/coord_gen.cu:64)
        pts = [rng.normal(0, 2.0, (n, dim)) for n in (8, 25, 60)]
        dists = [np.linalg.norm(p[:, None] - p[None], axis=2) for p in pts]
        v0 = [rng.random((dim, len(p))) for p in pts]
        coords, ok = metric_embed(dists, dim, v0=v0)
        for i, p in enumerate(pts):
            want = oracle.metric_embed(dists[i], dim, v0[i])
            assert ok[i] and want is not None
            assert np.allclose(np.abs(coords[i]), np.abs(want), atol=1e-6)
            d2 = np.linalg.norm(coords[i][:, None] - coords[i][None], axis=2)
            assert np.abs(d2 - dists[i]).max() < 0.1


# ------------------------------------------------------------------ ETKDG
PARAMS = dict(seed=1234, boxSize=10.0, optimizerForceTol=1e-3, enforceChirality=1, useExpTorsions=1, useBasicKnowledge=1,
              maxAttempts=30, dgIters=400, fourthIters=200, etkIters=300, maxRestarts=20)


def _check_masks_gpu(flat, slot_mol, pos4_list):
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.embedMolecules import EmbedParamsC

    dev = torch.device("cuda", 0)
    dg, _a = flat.dg.to_device(dev)
    etk, _b = flat.etk.to_device(dev)
    chk, _c = flat.checks.to_device(dev)
    pc = EmbedParamsC(**PARAMS)
    starts = np.concatenate([[0], np.cumsum([len(p) for p in pos4_list])]).astype(np.int32)
    d_pos = torch.from_numpy(np.concatenate(pos4_list)).to(dev)
    d_mol = torch.from_numpy(np.asarray(slot_mol, dtype=np.int32)).to(dev)
    d_st = torch.from_numpy(starts).to(dev)
    masks = torch.zeros(len(slot_mol), dtype=torch.int32, device=dev)
    _lib.call("b200mol_etkdg_check", C.byref(dg), C.byref(etk), C.byref(chk), C.byref(pc), len(slot_mol), d_mol.data_ptr(),
              d_st.data_ptr(), int(flat.atom_counts.max()), d_pos.data_ptr(), masks.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    return masks.cpu().numpy().astype(np.uint32)


def test_etkdg_acceptance_checks_equal_cpu(cuda):
    flat, mols = S.random_embed_molecules(12, 5, 16, seed=27)
    rng = np.random.default_rng(7)
    slot_mol, pos4 = [], []
    for m in range(len(flat)):
        n = flat.atom_counts[m]
        for scale in (0.3, 1.5, 4.0):  # collapsed, plausible, exploded geometries: every check fires somewhere
            slot_mol.append(m)
            pos4.append(rng.normal(0, scale, (n, 4)))
    got = _check_masks_gpu(flat, slot_mol, pos4)
    want = np.array([oracle.etkdg_check((flat.dg.atom_counts, flat.dg.tables), (flat.etk.atom_counts, flat.etk.tables),
                                        flat.checks.tables, flat.checks.num_impropers, PARAMS, m, p)
                     for m, p in zip(slot_mol, pos4)], dtype=np.uint32)
    assert (got == want).all()
    assert len(set(want.tolist())) > 2


@pytest.fixture(params=[0, 1], ids=["hessian_f32", "hessian_f64"])
def embedder_hessian(request):
    """The embedder's BFGS inverse Hessian in fp32 (default) and in fp64 (option etkdg_hessian_fp64, the reference's type)."""
    from nvmolkit_b200 import _lib

    _lib.set_option("etkdg_hessian_fp64", request.param)
    yield request.param
    _lib.set_option("etkdg_hessian_fp64", 0)


def test_etkdg_embed_produces_conformers_the_cpu_accepts(cuda, embedder_hessian):
    from nvmolkit_b200.embedMolecules import EmbedMolecules, EmbedParameters, embed_slots
    from nvmolkit_b200.types import CoordinateOutput

    flat, mols = S.random_embed_molecules(16, 5, 14, seed=28)
    params = EmbedParameters(randomSeed=1234)
    raw = embed_slots(flat, params, 3, max_iterations=30)
    ok = raw.ok.cpu().numpy().astype(bool)
    coords = raw.coords.cpu().numpy()
    assert ok.mean() > 0.5
    # every accepted conformer passes the CPU restatement of every acceptance check (4th coordinate dropped = 0)
    for s in np.nonzero(ok)[0]:
        m = raw.slot_mol[s]
        xyz = coords[raw.slot_atom_start[s]:raw.slot_atom_start[s + 1]]
        p4 = np.concatenate([xyz, np.zeros((len(xyz), 1))], axis=1)
        mask = oracle.etkdg_check((flat.dg.atom_counts, flat.dg.tables), (flat.etk.atom_counts, flat.etk.tables),
                                  flat.checks.tables, flat.checks.num_impropers, PARAMS, int(m), p4)
        # stages 1-3 are judged on the 4-D geometry BEFORE the collapse / ETK refinement; 5-10 must hold on the result
        assert mask & 0b11111100000 == 0, (s, bin(mask))
        b = mols[m]["bounds"]
        d = np.linalg.norm(xyz[:, None] - xyz[None], axis=2)
        one_two = [(i, j) for i, j in mols[m]["bonds"]]
        assert max(abs(d[i, j] - 0.5 * (b[min(i, j), max(i, j)] + b[max(i, j), min(i, j)])) for i, j in one_two) < 0.4
    # statistical agreement with the CPU pipeline driven by the same random stream (same slots, same attempts budget)
    cpu_out, cpu_att, cpu_en, cpu_fail = oracle.etkdg_embed((flat.dg.atom_counts, flat.dg.tables), (flat.etk.atom_counts, flat.etk.tables),
                                                            flat.checks.tables, flat.checks.num_impropers, PARAMS, raw.slot_mol.tolist())
    cpu_ok = np.array([o is not None for o in cpu_out])
    assert abs(cpu_ok.mean() - ok.mean()) < 0.25
    assert abs(np.median(cpu_att) - np.median(raw.attempts.cpu().numpy())) <= 3
    # same seed -> same random starts, same (atomic-free) arithmetic, and the accepted conformer of a slot is its lowest
    # successful attempt whatever the scheduling: the embedding repeats bit for bit
    raw2 = embed_slots(flat, params, 3, max_iterations=30)
    assert torch.equal(raw2.ok, raw.ok) and torch.equal(raw2.attempts, raw.attempts)
    assert torch.equal(raw2.coords, raw.coords)  # (rows of failed slots stay zero)
    # public API surface
    res = EmbedMolecules(flat, params, confsPerMolecule=3, maxIterations=30, output=CoordinateOutput.DEVICE)
    assert res.num_conformers == int(ok.sum()) and res.n_mols == 16
    per = EmbedMolecules(flat, params, confsPerMolecule=3, maxIterations=30)
    assert sum(len(c) for c in per) == int(ok.sum()) and len(per) == 16


def test_initial_coordinates_equal_cpu(cuda):
    """Stage 0 alone: the random 4-D box is bit-identical to the CPU stream; the metric-matrix start (random distance matrix
    inside the bounds -> metric matrix -> top-4 eigenpairs by power iteration, SURVEY.md 8f-1) agrees with the CPU
    restatement to the eigensolver's tolerance and fails on exactly the same attempts."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.embedMolecules import EmbedParamsC

    flat, mols = S.random_embed_molecules(10, 3, 20, seed=29)
    dev = torch.device("cuda", 0)
    dg, _a = flat.dg.to_device(dev)
    slot_mol = np.repeat(np.arange(len(flat), dtype=np.int32), 3)
    starts = np.concatenate([[0], np.cumsum(flat.atom_counts[slot_mol])]).astype(np.int32)
    d_mol, d_st = torch.from_numpy(slot_mol).to(dev), torch.from_numpy(starts).to(dev)
    for metric in (0, 1):
        n_ok = 0
        for attempt in (0, 5):
            p = dict(PARAMS, useMetricStart=metric)
            pc = EmbedParamsC(**p)
            pos = torch.full((int(starts[-1]), 4), 7.0, dtype=torch.float64, device=dev)
            ok = torch.zeros(len(slot_mol), dtype=torch.int8, device=dev)
            _lib.call("b200mol_etkdg_initial_coords", C.byref(dg), C.byref(pc), len(slot_mol), d_mol.data_ptr(), d_st.data_ptr(),
                      int(flat.atom_counts.max()), attempt, pos.data_ptr(), ok.data_ptr(), torch.cuda.current_stream().cuda_stream)
            pos, ok = pos.cpu().numpy(), ok.cpu().numpy().astype(bool)
            for s_, m in enumerate(slot_mol):
                want, ok_c = oracle.etkdg_initial_coords((flat.dg.atom_counts, flat.dg.tables), p, s_, int(m), attempt)
                got = pos[starts[s_]:starts[s_ + 1]]
                assert ok[s_] == ok_c, (metric, attempt, s_)
                if not ok_c:
                    continue
                n_ok += 1
                if metric == 0:
                    assert np.array_equal(got, want)
                else:
                    # (the power iteration stops when the eigenvalue estimate moves by < 1e-3, so the two sides agree to
                    # about that, not to rounding: the same iteration count gives 1e-9, one iteration apart ~1e-3)
                    assert np.allclose(got, want, atol=5e-3 * max(1.0, np.abs(want).max())), (s_, np.abs(got - want).max())
        assert n_ok > 0


def test_etkdg_embed_from_the_metric_matrix_start(cuda):
    """useRandomCoords=False (refused by the reference, src/etkdg.cpp:99-101): every attempt starts from the on-device
    eigen embedding of a random distance matrix; the accepted conformers pass the CPU's acceptance checks."""
    from nvmolkit_b200.embedMolecules import EmbedMolecules, EmbedParameters, embed_slots

    flat, mols = S.random_embed_molecules(12, 5, 14, seed=30)
    params = EmbedParameters(randomSeed=77, useRandomCoords=False)
    raw = embed_slots(flat, params, 2, max_iterations=40)
    ok = raw.ok.cpu().numpy().astype(bool)
    assert ok.mean() > 0.3
    fails = raw.stage_failures.cpu().numpy()
    coords = raw.coords.cpu().numpy()
    for s_ in np.nonzero(ok)[0]:
        xyz = coords[raw.slot_atom_start[s_]:raw.slot_atom_start[s_ + 1]]
        p4 = np.concatenate([xyz, np.zeros((len(xyz), 1))], axis=1)
        mask = oracle.etkdg_check((flat.dg.atom_counts, flat.dg.tables), (flat.etk.atom_counts, flat.etk.tables),
                                  flat.checks.tables, flat.checks.num_impropers, PARAMS, int(raw.slot_mol[s_]), p4)
        assert mask & 0b11111100000 == 0
    raw2 = embed_slots(flat, params, 2, max_iterations=40)  # bit-reproducible like the random-box start
    assert torch.equal(raw2.ok, raw.ok) and torch.equal(raw2.coords, raw.coords)
    # the CPU pipeline with the same streams: same statistics
    cpu_out, cpu_att, _e, cpu_fail = oracle.etkdg_embed((flat.dg.atom_counts, flat.dg.tables), (flat.etk.atom_counts, flat.etk.tables),
                                                        flat.checks.tables, flat.checks.num_impropers,
                                                        dict(PARAMS, seed=77, maxAttempts=40, useMetricStart=1), raw.slot_mol.tolist())
    cpu_ok = np.array([o is not None for o in cpu_out])
    assert abs(cpu_ok.mean() - ok.mean()) < 0.3
    assert (fails[0] > 0) == (cpu_fail[0] > 0)  # stage-0 failures (degenerate metric matrices) occur on both or neither
    per = EmbedMolecules(flat, params, confsPerMolecule=2, maxIterations=40)
    assert sum(len(c) for c in per) == int(ok.sum())


# ------------------------------------------------------------------ UFF
def test_uff_energy_gradient_and_minimize_parity(cuda):
    from nvmolkit_b200.minimizer import energy_and_grad, minimize
    from nvmolkit_b200.uffOptimization import FlatUFFMolecules, UFFOptimizeMoleculesConfs

    system, xyz, _ = S.random_uff_system(8, 4, 30, seed=31)
    rng = np.random.default_rng(2)
    batch = ConformerBatch.from_coords(system, [[x + rng.normal(0, 0.05, x.shape), x + rng.normal(0, 0.15, x.shape)] for x in xyz])
    e, g = energy_and_grad(system, batch)
    e, g = e.cpu().numpy(), g.cpu().numpy()
    for c in range(batch.n_conf):
        a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
        eo, go, _ = oracle.ff_energy_grad("uff", system.atom_counts, system.tables, batch.conf_mol[c], batch.positions[a0:a1])
        assert _rel(e[c], eo) < 1e-11
        assert np.abs(g[a0:a1] - go).max() < 1e-9 * max(1.0, np.abs(go).max())
    # minimise from a CPU-relaxed geometry + perturbation, compare minima
    pos0, _, _, _ = oracle.ff_minimize("uff", system.atom_counts, system.tables, np.arange(8, dtype=np.int32),
                                       np.concatenate([[0], np.cumsum(system.atom_counts)]).astype(np.int32),
                                       np.concatenate(xyz), 2000, 1e-4)
    st0 = np.concatenate([[0], np.cumsum(system.atom_counts)])
    relaxed = [pos0[st0[m]:st0[m + 1]] for m in range(8)]
    b2 = ConformerBatch.from_coords(system, [[r + rng.normal(0, 0.05, r.shape) for _ in range(2)] for r in relaxed])
    res = minimize(system, b2, 1000, 1e-4)
    pos_o, e_o, conv_o, _ = oracle.ff_minimize("uff", system.atom_counts, system.tables, b2.conf_mol, b2.atom_starts, b2.positions, 1000, 1e-4)
    eg, st = res.energies.cpu().numpy(), res.status.cpu().numpy()
    both = (st == 0) & (conv_o == 1)
    assert both.mean() > 0.7
    # this random UFF system is frustrated (random torsion orders / angle orders): GPU (FMA-contracted) and CPU
    # (uncontracted) trajectories differ in the last bits and a perturbed start may settle in a neighbouring minimum.
    # Most must agree to E_RTOL; the others are still converged minima (status 0 on both sides) of comparable energy.
    rel = _rel(eg[both], e_o[both])
    assert (rel < E_RTOL).mean() >= 0.75 and np.median(rel) < E_RTOL and (rel < 0.1).all(), rel
    energies, coords = UFFOptimizeMoleculesConfs(FlatUFFMolecules(system, b2), maxIters=1000)
    assert np.array_equal(np.array(energies).ravel(), eg)  # a second GPU run: the same bits


# ------------------------------------------------------------------ RMS pruning on the device
def test_rms_pruning_equals_cpu(cuda):
    """b200mol_rms_prune vs the CPU restatement (different alignment algorithm: Horn quaternion eigenproblem by Jacobi
    there, closed-form 3x3 singular values here): same keep flags; symmetric self matches and invalid slots honoured."""
    from nvmolkit_b200.pruning import rms_prune

    rng = np.random.default_rng(61)
    xyz, cas, mcs, matches, counts = [], [0], [0], [], []
    for m in range(12):
        n = int(rng.integers(4, 40))
        base = rng.normal(0, 2.0, (n, 3))
        n_conf = int(rng.integers(1, 9))
        for c in range(n_conf):
            kind = rng.integers(0, 3)
            if kind == 0 and c:  # rigid copy of an earlier conformer + small noise: must be pruned
                q, _r = np.linalg.qr(rng.normal(size=(3, 3)))
                q *= np.sign(np.linalg.det(q))
                x = base @ q.T + rng.normal(0, 3.0, 3) + rng.normal(0, 0.02, (n, 3))
            elif kind == 1:
                x = base + rng.normal(0, 0.6, (n, 3))  # around the threshold
            else:
                x = rng.normal(0, 2.0, (n, 3))
            xyz.append(x)
            cas.append(cas[-1] + n)
        mcs.append(mcs[-1] + n_conf)
        counts.append(n)
        heavy = np.sort(rng.permutation(n)[: max(3, n // 2)])
        swapped = heavy.copy()
        swapped[[0, 1]] = swapped[[1, 0]]  # a "symmetry-equivalent" second mapping
        matches.append(np.stack([heavy, swapped]) if m % 2 else None)
    xyz = np.concatenate(xyz)
    valid = (rng.random(len(cas) - 1) < 0.9).astype(np.uint8)
    for thresh in (0.3, 0.8):
        for mt in (None, matches):
            got = rms_prune(torch.from_numpy(xyz).to(cuda), np.array(cas), np.array(mcs), thresh, mt, counts,
                            valid=torch.from_numpy(valid).to(cuda)).cpu().numpy()
            want = oracle.rms_prune(xyz, cas, mcs, thresh, mt, valid)
            assert np.array_equal(got, want), (thresh, mt is None)
            assert not got[valid == 0].any() and 0 < got.sum() < len(got)


def test_embed_with_rms_pruning_on_device_output(cuda):
    from nvmolkit_b200.embedMolecules import EmbedMolecules, EmbedParameters
    from nvmolkit_b200.types import CoordinateOutput

    flat, _ = S.random_embed_molecules(6, 5, 10, seed=62)
    base = EmbedMolecules(flat, EmbedParameters(randomSeed=5), confsPerMolecule=6, maxIterations=30, output=CoordinateOutput.DEVICE)
    pruned = EmbedMolecules(flat, EmbedParameters(randomSeed=5, pruneRmsThresh=1.5), confsPerMolecule=6, maxIterations=30,
                            output=CoordinateOutput.DEVICE)  # the reference raises here (src/etkdg.cpp:106-110)
    assert 0 < pruned.num_conformers <= base.num_conformers
    for confs in pruned.per_molecule():  # every kept pair is at least 1.5 A apart after alignment
        pts = [c.cpu().numpy() for c in confs]
        for i in range(len(pts)):
            for j in range(i):
                assert np.sqrt(oracle.best_ssd(pts[i], pts[j]) / len(pts[i])) >= 1.5 - 1e-9
