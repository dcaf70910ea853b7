"""The BFGS minimiser step by step against the fp64 oracle.

Most of a BFGS iteration goes into one sweep over the upper triangle of the inverse Hessian (hessianSweepT in
bfgs_device.cuh). It applies the pending rank-2 update of the previous iteration and accumulates H*dGrad and H*grad
from the stored half. A wrong row sum, mask or chunk bound there does not move the minimum; it bends the path to it.
So these tests stop both minimisers after k iterations and compare the points they reached:
  * analytic systems (b200mol_poly_minimize) at every size class of the sweep: n mod 4, n mod 32, around the 64-column
    (fp64) and 128-column (fp32) chunks, n < 4 and the largest size the shared-memory check accepts, all in one batch,
    and with one CTA per SM so that one slab serves conformers of different n;
  * both slab types: fp64 (the force-field minimisers) and fp32 (the embedder's default);
  * a rejected update after accepted ones (the sweep with no pending update);
  * MMFF, UFF, DG and ETK systems at the sizes the benchmark runs.
Tight comparisons use p = 2, or p = 4 up to three iterations: further on, a different summation order of the energy
can flip a near-tie in the line search's acceptance test and send the two minimisers down different, equally valid paths.
"""

import contextlib

import numpy as np
import pytest
import torch

import oracle
from nvmolkit_b200 import synthetic as S
from nvmolkit_b200.forcefield import ConformerBatch

MAX_DIM = 1828  # (6 + 8 warps) vectors of max_dim doubles must fit the 200 KB of dynamic shared memory
SIZES = [1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 66, 67, 127, 128, 129, 255, 257, 1000, MAX_DIM]
SIZES_F32 = [1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 66, 67, 127, 128, 129, 255, 256, 257, 1000]
EPS = 3e-8  # the curvature test of the update: fac > sqrt(EPS |dGrad|^2 |xi|^2)


@pytest.fixture(params=[0, 1], ids=["default_ctas", "one_cta_per_sm"])
def ctas_per_sm(request, cuda):
    """Default CTA count, or one CTA per SM with more systems than CTAs: each slab then serves several systems."""
    from nvmolkit_b200 import _lib

    with _lib.options(bfgs_ctas_per_sm=1) if request.param else contextlib.nullcontext():
        yield request.param


def _batch_sizes(sizes, reuse, seed):
    """All sizes once in shuffled order (the smallest never last); with `reuse`, plus more systems up to three per SM."""
    rng = np.random.default_rng(seed)
    out = list(sizes)
    if reuse:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        out += rng.choice([s for s in sizes if s <= 257], 3 * sms - len(sizes)).tolist()
    out = [int(v) for v in rng.permutation(out)]
    if out[-1] == min(out):
        out[-1], out[0] = out[0], out[-1]
    return out


def _poly_systems(sizes, power, seed):
    rng = np.random.default_rng(seed)
    starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    n = int(starts[-1])
    w = rng.uniform(0.5, 3.0, n)
    c = rng.normal(0.0, 3.0, n)
    x0 = c + rng.uniform(-2.0, 2.0, n)
    return starts, w, c, x0


def _compare_poly(starts, power, w, c, x0, k, grad_tol, scale, fp32, x_tol, e_tol):
    from nvmolkit_b200.minimizer import poly_minimize

    x, e, status, iters = poly_minimize(starts, power, w, c, x0, k, grad_tol, scale, hessian_fp32=fp32)
    x, e, status, iters = x.cpu().numpy(), e.cpu().numpy(), status.cpu().numpy(), iters.cpu().numpy()
    for s in range(len(starts) - 1):
        a, b = starts[s], starts[s + 1]
        xo, eo, so, io = oracle.poly_minimize(power, w[a:b], c[a:b], x0[a:b], k, grad_tol, scale_grads=scale)
        step = np.abs(xo - x0[a:b]).max()
        where = (s, b - a, k)
        assert int(status[s]) == so and int(iters[s]) == io, (where, int(status[s]), so, int(iters[s]), io)
        assert np.abs(x[a:b] - xo).max() <= x_tol * step, (where, np.abs(x[a:b] - xo).max() / step)
        assert abs(e[s] - eo) <= e_tol * max(abs(eo), 1.0), (where, e[s], eo)


# ------------------------------------------------------------------ analytic systems, fp64 slab
@pytest.mark.gpu
@pytest.mark.parametrize("power,k", [(2, 1), (2, 2), (2, 3), (2, 5), (2, 12), (4, 1), (4, 2), (4, 3)])
def test_truncated_trajectories_fp64_slab(ctas_per_sm, power, k):
    sizes = _batch_sizes(SIZES, ctas_per_sm, seed=10 * k + power)
    starts, w, c, x0 = _poly_systems(sizes, power, seed=k + 100 * power)
    _compare_poly(starts, power, w, c, x0, k, 1e-8, True, False, 1e-10, 1e-12)


@pytest.mark.gpu
def test_zero_iterations_return_the_start(cuda):
    from nvmolkit_b200.minimizer import poly_minimize

    sizes = _batch_sizes(SIZES, False, seed=3)
    starts, w, c, x0 = _poly_systems(sizes, 2, seed=3)
    for fp32 in (False, True):
        x, e, status, iters = poly_minimize(starts, 2, w, c, x0, 0, 1e-8, True, hessian_fp32=fp32)
        assert np.array_equal(x.cpu().numpy(), x0)
        assert (status.cpu().numpy() == 1).all() and (iters.cpu().numpy() == 0).all()
        for s in range(len(sizes)):
            a, b = starts[s], starts[s + 1]
            e0 = float(np.sum(w[a:b] * (x0[a:b] - c[a:b]) ** 2))
            assert abs(e.cpu().numpy()[s] - e0) <= 1e-12 * max(abs(e0), 1.0)


# ------------------------------------------------------------------ analytic systems, fp32 slab
@pytest.mark.gpu
@pytest.mark.parametrize("k", [3, 5])
def test_truncated_trajectories_fp32_slab(ctas_per_sm, k):
    """The embedder's slab type. A correct fp32 sweep stays within about 4e-7 of the step size of the fp64 oracle here;
    a skipped update term, a diagonal counted twice or a dropped batch of row sums moves it by 4e-5 or more."""
    sizes = _batch_sizes(SIZES_F32, ctas_per_sm, seed=20 + k)
    starts, w, c, x0 = _poly_systems(sizes, 2, seed=200 + k)
    _compare_poly(starts, 2, w, c, x0, k, 1e-8, True, True, 1e-5, 1e-6)


# ------------------------------------------------------------------ a rejected update after accepted ones
# An indefinite quadratic: w > 0 everywhere except one coordinate with w < 0 that starts 1e-3 from its (unstable)
# stationary point. The positive coordinates dominate the first steps; then the negative one takes over, the curvature
# along the step turns negative and the update is skipped. The sweep of the next iteration has no pending update.
INDEF_N, INDEF_NEG, INDEF_SEED = 150, 140, 3
INDEF_REJECTED = (13, 14)  # iterations (0-based) whose update is skipped; 0..12 and 15 are accepted


def _indefinite_system():
    rng = np.random.default_rng(INDEF_SEED)
    w = rng.uniform(0.5, 3.0, INDEF_N)
    w[INDEF_NEG] = -rng.uniform(0.05, 0.3)
    c = rng.normal(0.0, 3.0, INDEF_N)
    x0 = c + rng.normal(0.0, 2.0, INDEF_N)
    x0[INDEF_NEG] = c[INDEF_NEG] + 1e-3
    return w, c, x0


def test_indefinite_system_skips_the_update_on_the_oracle():
    """CPU: on the chosen seed the oracle accepts the updates of iterations 0..12, skips those of 13 and 14 and accepts
    that of 15, each by a clear margin (curvature test evaluated on the analytic gradients of consecutive iterates)."""
    w, c, x0 = _indefinite_system()
    xs = [x0] + [oracle.poly_minimize(2, w, c, x0, k, 1e-12, scale_grads=False)[0] for k in range(1, 17)]
    for j in range(16):
        xi = xs[j + 1] - xs[j]
        dg = 2.0 * w * (xs[j + 1] - c) - 2.0 * w * (xs[j] - c)
        fac, bound = dg @ xi, np.sqrt(EPS * (dg @ dg) * (xi @ xi))
        if j in INDEF_REJECTED:
            assert fac < 0.0, (j, fac, bound)
        else:
            assert fac > 2.0 * bound, (j, fac, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("fp32", [False, True], ids=["fp64_slab", "fp32_slab"])
def test_trajectory_across_a_rejected_update(cuda, fp32):
    """Iterations 14 and 15 sweep a stored H with no pending update, 16 applies the update of 15 again. From iteration
    16 the negative coordinate runs away (from 0.14 to 84 off its stationary point), which amplifies the fp32 slab's
    rounding past its tolerance, so the fp32 comparison stops at 16 iterations."""
    w, c, x0 = _indefinite_system()
    starts = np.array([0, INDEF_N], dtype=np.int32)
    tol = 1e-5 if fp32 else 1e-10
    for k in (13, 14, 15, 16) if fp32 else (13, 14, 15, 16, 17):
        # after the runaway the energy is a difference of terms 40 times its size: 1e-9 relative there
        e_tol = 1e-6 if fp32 else 1e-12 if k < 17 else 1e-9
        _compare_poly(starts, 2, w, c, x0, k, 1e-12, False, fp32, tol, e_tol)


# ------------------------------------------------------------------ force fields, truncated
_FF_CASES = {}


def _ff_case(kind):
    """(system, batch, minimize kwargs, oracle kwargs), two conformers per molecule. MMFF: 164, 299, 487 and 525 atoms
    in one batch; UFF: 482-535 atoms; DG / ETK: 55-101 atoms, the size of the benchmark's molecules."""
    if kind in _FF_CASES:
        return _FF_CASES[kind]
    rng = np.random.default_rng(55)
    if kind in ("mmff", "uff"):
        system, xyz, _ = (S.random_mmff_system(4, 70, 250, seed=52) if kind == "mmff" else
                          S.random_uff_system(3, 240, 250, seed=52))
        coords = [[x + rng.normal(0.0, 0.1, x.shape) for _ in range(2)] for x in xyz]
        kw, okw = {}, {}
    else:
        flat, _ = S.random_embed_molecules(6, 22, 52, seed=54)
        coords = [[(rng.random((n, 4)) - 0.5) * 10.0 for _ in range(2)] for n in flat.atom_counts]
        if kind == "etk":
            system, kw, okw = flat.etk, dict(recentre=True), dict(recentre=True)
        else:
            cw, fw = (1.0, 0.1) if kind == "dg" else (0.2, 1.0)
            system, kw = flat.dg, dict(chiral_weight=cw, fourth_dim_weight=fw)
            okw = dict(kw, dim=4)
    _FF_CASES[kind] = (system, ConformerBatch.from_coords(system, coords), kw, okw)
    return _FF_CASES[kind]


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 3, 5])
@pytest.mark.parametrize("kind", ["mmff", "uff", "dg", "dg_weights", "etk"])
def test_force_field_trajectories_truncated(cuda, kind, k):
    """The same k iterations as the oracle on real force fields; this also runs the wave-scheduled gradients at sizes
    the parity tests do not reach."""
    from nvmolkit_b200.minimizer import minimize

    system, batch, kw, okw = _ff_case(kind)
    res = minimize(system, batch, k, 1e-4, **kw)
    pos_o, e_o, conv_o, it_o = oracle.ff_minimize(system.kind, system.atom_counts, system.tables, batch.conf_mol,
                                                  batch.atom_starts, batch.positions, k, 1e-4, **okw)
    pos, e = res.positions.cpu().numpy(), res.energies.cpu().numpy()
    st, it = res.status.cpu().numpy(), res.iters.cpu().numpy()
    for c in range(batch.n_conf):
        a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
        step = np.abs(pos_o[a0:a1] - batch.positions[a0:a1]).max()
        where = (kind, k, c, a1 - a0)
        assert st[c] == (0 if conv_o[c] else 1) and it[c] == it_o[c], (where, st[c], conv_o[c], it[c], it_o[c])
        assert np.abs(pos[a0:a1] - pos_o[a0:a1]).max() <= 1e-9 * step, (where, np.abs(pos[a0:a1] - pos_o[a0:a1]).max() / step)
        assert abs(e[c] - e_o[c]) <= 1e-9 * max(abs(e_o[c]), 1.0), (where, e[c], e_o[c])


# ------------------------------------------------------------------ size limits and the active mask
@pytest.mark.gpu
def test_size_limits_raise_before_any_launch(cuda):
    """One past the largest size the shared-memory minimiser takes is refused with an error, and nothing is launched."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.minimizer import minimize, poly_minimize

    mmff, xyz, _ = S.random_mmff_system(1, 300, 306, seed=80)
    assert mmff.atom_counts[0] == 610  # 14 vectors x 3 x 8 B x 610 > 200 KB
    flat, _ = S.random_embed_molecules(1, 218, 222, seed=1)
    assert flat.atom_counts[0] > 426  # ETK keeps a 15th vector (the window reference): 426 atoms at most
    mmff.to_device()
    flat.etk.to_device()
    before = _lib.launch_count()
    n = MAX_DIM + 1
    for fp32 in (False, True):
        with pytest.raises(ValueError, match="too large"):
            poly_minimize(np.array([0, 3, 3 + n], dtype=np.int32), 2, np.ones(n + 3), np.zeros(n + 3), np.ones(n + 3), 5,
                          1e-8, True, hessian_fp32=fp32)
    with pytest.raises(ValueError, match="too large"):
        minimize(mmff, ConformerBatch.from_coords(mmff, [[xyz[0]]]), 5)
    etk_start = [[np.zeros((int(flat.atom_counts[0]), 4))]]
    with pytest.raises(ValueError, match="too large"):
        minimize(flat.etk, ConformerBatch.from_coords(flat.etk, etk_start), 5, recentre=True)
    torch.cuda.synchronize()
    assert _lib.launch_count() == before


@pytest.mark.gpu
def test_active_mask_skips_conformers_bit_for_bit(cuda):
    from nvmolkit_b200.minimizer import minimize

    system, batch, _, _ = _ff_case("mmff")
    active = np.zeros(batch.n_conf, dtype=np.uint8)
    active[[0, 3, 4, 7]] = 1
    full = minimize(system, batch, 20, 1e-4)
    part = minimize(system, batch, 20, 1e-4, active=torch.from_numpy(active).cuda())
    p_full, p_part = full.positions.cpu().numpy(), part.positions.cpu().numpy()
    for c in range(batch.n_conf):
        a0, a1 = batch.atom_starts[c], batch.atom_starts[c + 1]
        if active[c]:
            assert np.array_equal(p_part[a0:a1], p_full[a0:a1])
            assert part.energies[c] == full.energies[c] and part.iters[c] == full.iters[c]
            assert part.status[c] == full.status[c]
        else:
            assert np.array_equal(p_part[a0:a1], batch.positions[a0:a1])
