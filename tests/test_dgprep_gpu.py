"""GPU tier of the distance-geometry preparation (triangle smoothing, power eigensolver, metric embedding) against the
numpy restatement and the fp64 oracle of tests/test_dgprep.py, at each shared-memory boundary, tie and failure exit.

Shared-memory limits of these kernels (220 KB = 28160 doubles): triangle smoothing keeps n^2 on chip up to n = 167;
eig_topk keeps n^2 + 2 n up to n = 166; metric_embed keeps n^2 + (3 + dim) n + dim up to n = 164. Larger matrices run in
place in global memory. Each CTA handles matrices blockIdx.x, blockIdx.x + grid, ...; the grid is 2 CTAs per SM.
"""

import numpy as np
import pytest
import torch

import oracle
import test_dgprep as D
from nvmolkit_b200 import _lib
from nvmolkit_b200.dgprep import _concat, eig_topk, metric_embed, triangle_smooth

pytestmark = pytest.mark.gpu

MARGIN = 1e-6  # stopping decisions closer than this to their threshold may go either way between GPU and oracle
NAN = float("nan")


def _grid():
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count


def _v0(v0, dev):
    if v0 is None:
        return None
    return torch.from_numpy(np.concatenate([np.ascontiguousarray(v, dtype=np.float64).ravel() for v in v0])).to(dev)


def eig_abi(mats, k, v0=None, seed=42):
    """b200mol_eig_topk with NaN-filled outputs, so that every slot the kernel leaves alone is visible."""
    dev = torch.device("cuda", 0)
    d, st, _ = _concat(mats, dev)
    ns = np.array([m.shape[0] for m in mats], np.int64)
    vstarts = np.concatenate([[0], np.cumsum(ns * k)]).astype(np.int64)
    vs = torch.from_numpy(vstarts).to(dev)
    vals = torch.full((len(mats), k), NAN, dtype=torch.float64, device=dev)
    vecs = torch.full((int(vstarts[-1]),), NAN, dtype=torch.float64, device=dev)
    conv = torch.full((len(mats),), -1, dtype=torch.int8, device=dev)
    dv0 = _v0(v0, dev)
    _lib.call("b200mol_eig_topk", d.data_ptr(), st.data_ptr(), len(mats), k, dv0.data_ptr() if dv0 is not None else None,
              vs.data_ptr() if dv0 is not None else None, seed, vals.data_ptr(), vecs.data_ptr(), vs.data_ptr(),
              conv.data_ptr(), torch.cuda.current_stream().cuda_stream)
    vh = vecs.cpu().numpy()
    vecs = [vh[vstarts[i]:vstarts[i + 1]].reshape(k, ns[i]) for i in range(len(mats))]
    vals, conv = vals.cpu().numpy(), conv.cpu().numpy().astype(int)
    for i in range(len(mats)):  # pairs past the converged count are never written
        c = conv[i]
        assert 0 <= c <= k
        assert np.isfinite(vals[i, :c]).all() and np.isnan(vals[i, c:]).all()
        assert np.isfinite(vecs[i][:c]).all() and np.isnan(vecs[i][c:]).all()
    return vals, vecs, conv


def embed_abi(dists, dim, v0=None, seed=42):
    """b200mol_metric_embed with NaN-filled coordinates: written exactly for the matrices with ok = 1."""
    dev = torch.device("cuda", 0)
    d, st, _ = _concat(dists, dev)
    ns = np.array([m.shape[0] for m in dists], np.int64)
    astarts = np.concatenate([[0], np.cumsum(ns)]).astype(np.int32)
    vstarts = torch.from_numpy(np.concatenate([[0], np.cumsum(ns * dim)]).astype(np.int64)).to(dev)
    a = torch.from_numpy(astarts).to(dev)
    coords = torch.full((int(astarts[-1]), dim), NAN, dtype=torch.float64, device=dev)
    ok = torch.full((len(dists),), -1, dtype=torch.int8, device=dev)
    dv0 = _v0(v0, dev)
    _lib.call("b200mol_metric_embed", d.data_ptr(), st.data_ptr(), a.data_ptr(), len(dists), dim,
              dv0.data_ptr() if dv0 is not None else None, vstarts.data_ptr() if dv0 is not None else None, seed,
              coords.data_ptr(), ok.data_ptr(), torch.cuda.current_stream().cuda_stream)
    ch, ok = coords.cpu().numpy(), ok.cpu().numpy().astype(int)
    out = [ch[astarts[i]:astarts[i + 1]] for i in range(len(dists))]
    for i, c in enumerate(out):
        assert ok[i] in (0, 1)
        assert np.isfinite(c).all() if ok[i] else np.isnan(c).all()
    return out, ok


def _safe(trace):
    """The oracle's stopping decisions are all at least MARGIN from their thresholds."""
    _, _, _, iters, conv, zero = trace
    tried = iters >= 0
    return bool(np.all(conv[tried] > MARGIN) and np.all(zero[tried] > 1e-12))


def _same_pairs(vals, vecs, c, n, want_vals, want_vecs):
    """Eigenvalues to 1e-9 of the matrix scale (rounding differs with the order of the sums); eigenvectors of the first
    min(n, c) pairs to 1e-8. Pairs past n are the deflation residual of an exhausted matrix: their vectors are not stable."""
    scale = np.abs(want_vals[:c]).max(initial=0.0)
    assert np.all(np.abs(vals[:c] - want_vals[:c]) <= 1e-9 * scale)
    c = min(c, n)
    sign = np.sign(np.sum(vecs[:c] * want_vecs[:c], axis=1))[:, None]
    assert np.abs(vecs[:c] * sign - want_vecs[:c]).max(initial=0.0) <= 1e-8


# ------------------------------------------------------------------------------------------------ triangle smoothing
SMOOTH_SIZES = [31, 32, 33, 166, 167, 168, 169, 600]


def _smoothing_cases(rng):
    mats = [c[1] for c in D.HAND_CASES]  # n = 0, 1, 2, 3, 4 and every tie
    for n in SMOOTH_SIZES:
        mats.append(D.chain_bounds(rng, n))
        mats.append(D.chain_bounds(rng, n, bad_pair=(1, 6)))  # fails after a few pivots
        if n < 100:
            mats.append(D.bounds_from_points(rng, n))
    return mats


@pytest.mark.parametrize("tol", [0.0, 0.05])
def test_smoothing_sizes_equal_restatement(cuda, tol):
    mats = _smoothing_cases(np.random.default_rng(1))
    got, ok = triangle_smooth(mats, tol)
    kinds = set()
    for b, g, o in zip(mats, got, ok):
        want, wok, _ = D.smooth_np(b, tol)
        assert o == wok and np.array_equal(g, want), b.shape
        kinds.add((b.shape[0] > 167, bool(o)))
    assert kinds == {(False, False), (False, True), (True, False), (True, True)}
    for case, g, o in zip(D.HAND_CASES, got, ok):  # the stated answers of the hand-built matrices
        name, b, ctol, want, wok, _ = case
        if ctol == tol and want is not None:
            assert o == wok and np.array_equal(g, want), name


def test_smoothing_hand_tolerances(cuda):
    # every hand-built matrix at its own tol (the exact-gap ones need tol = 0.125 and one ulp more); the 0-atom matrix
    # is in the batches above (a batch of only empty matrices has no bounds buffer at all)
    for name, b, ctol, want, wok, _ in [c for c in D.HAND_CASES if c[1].size]:
        got, ok = triangle_smooth([b, b], ctol)
        w, o, _ = D.smooth_np(b, ctol)
        assert ok[0] == ok[1] == o == wok and np.array_equal(got[0], w) and np.array_equal(got[1], w), name


def test_smoothing_batch_larger_than_grid(cuda):
    rng = np.random.default_rng(2)
    grid = _grid()
    mats = []
    for m in range(2 * grid + grid // 2 + 7):
        n = int(rng.choice([168, 180])) if m % 97 == 5 else int(rng.integers(3, 40))
        b = D.bounds_from_points(rng, n)
        if rng.random() < 0.5:
            i, j = sorted(rng.choice(n, 2, replace=False))
            b[j, i] = b[i, j] * 1.5
        mats.append(b)
    for tol in (0.0, 0.05):
        got, ok = triangle_smooth(mats, tol)
        want = [D.smooth_np(b, tol) for b in mats]
        for m, (g, o, w) in enumerate(zip(got, ok, want)):
            assert o == w[1] and np.array_equal(g, w[0]), m
        # some CTA handled a failing matrix and then a consistent one, and the other way round
        flags = np.array([w[1] for w in want])
        first, second = flags[:grid], flags[grid:2 * grid]
        assert (~first & second).any() and (first & ~second).any()


def test_smoothing_side_stream(cuda):
    mats = [b for b in _smoothing_cases(np.random.default_rng(3)) if 3 < b.shape[0] < 200]
    s = torch.cuda.Stream()
    got, ok = triangle_smooth(mats, 0.0, stream=s)
    for b, g, o in zip(mats, got, ok):
        want, wok, _ = D.smooth_np(b)
        assert o == wok and np.array_equal(g, want)


# ------------------------------------------------------------------------------------------------ power eigensolver
EIG_SIZES = [1, 31, 32, 33, 166, 167, 255, 256, 257, 300]


def _eig_cases(k, rng):
    mats, v0s = [], []
    for n in sorted(set(EIG_SIZES + ([k - 1] if k > 1 else []))):
        mats.append(D.rotated(D.separated_spectrum(n, min(n, k), rng), rng))
        v0s.append(rng.random((k, n)))
    return mats, v0s


@pytest.mark.parametrize("k", range(1, 9))
def test_eig_sizes_against_oracle(cuda, k):
    rng = np.random.default_rng(10 + k)
    mats, v0s = _eig_cases(k, rng)
    vals, vecs, conv = eig_abi(mats, k, v0s)
    wrapped = eig_topk(mats, k, v0=v0s)
    compared = 0
    for i, (a, v0) in enumerate(zip(mats, v0s)):
        n = a.shape[0]
        assert np.array_equal(wrapped[0][i, :conv[i]], vals[i, :conv[i]]) and wrapped[2][i] == conv[i]
        trace = oracle.power_eigen_trace(a, k, v0)
        if _safe(trace):
            compared += 1
            assert conv[i] == trace[2], n
            _same_pairs(vals[i], vecs[i], conv[i], n, trace[0], trace[1])
        else:  # pairs of an exhausted matrix (n < k) are noise; the first min(n, k) are eigenpairs
            c = min(n, k)
            assert conv[i] >= c
            D.assert_close_to_eigh(a, vals[i], vecs[i], c)
    assert compared >= len(mats) - 2


def test_eig_hashed_start(cuda):
    rng = np.random.default_rng(30)
    for k in (1, 4, 8):
        mats = [D.rotated(D.separated_spectrum(n, min(n, k), rng), rng) for n in (33, 167, 257)]
        vals, vecs, conv = eig_abi(mats, k, seed=7)
        vals2, vecs2, conv2 = eig_abi(mats, k, seed=7)
        assert np.array_equal(conv, conv2) and np.array_equal(vals, vals2, equal_nan=True)
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(vecs, vecs2))
        for i, a in enumerate(mats):
            assert conv[i] == k
            D.assert_close_to_eigh(a, vals[i], vecs[i], k)


def test_eig_ties_first_index_wins(cuda):
    mats, want = [], []
    for lo, hi in D.TIE_PAIRS:
        for sign in (-1.0, 1.0):
            for noise in (None, np.random.default_rng(lo)):
                mats.append(D.tie_matrix(320, lo, hi, sign, noise))
                want.append(3.0 * sign)
    vals, vecs, conv = eig_abi(mats, 1, [np.ones((1, 320))] * len(mats))
    for i, a in enumerate(mats):
        ov, _, ok_ = oracle.power_eigen(a, 1, np.ones((1, 320)))
        assert conv[i] == ok_ == 1 and vals[i, 0] == ov[0] == want[i]


def test_eig_failure_exits(cuda):
    rng = np.random.default_rng(40)
    mats, v0s, ks = [], [], []
    for rank in range(8):  # |eig| < 1e-10 after exactly `rank` pairs
        a, v0 = D.deflatable(300 if rank % 2 else 50, rank, rng)
        mats.append(a)
        v0s.append(v0)
        ks.append(rank)
    for n in (40, 300):  # 1000 iterations without convergence: no pair at all
        mats.append(D.pm_pair(n, np.random.default_rng(n)))
        v0s.append(np.random.default_rng(n).random((3, n)))
        ks.append(0)
    a = D.rotated(D.separated_spectrum(60, 4, rng, negative_first=True), rng)
    mats.append(a)
    v0s.append(rng.random((4, 60)))
    ks.append(4)
    for i, (a, v0, want) in enumerate(zip(mats, v0s, ks)):
        kk = v0.shape[0]
        vals, vecs, conv = eig_abi([a], kk, [v0])
        ov, ovec, ok_ = oracle.power_eigen(a, kk, v0)
        assert conv[0] == ok_ == want, i
        assert np.array_equal(np.sign(vals[0, :want]), np.sign(ov[:want])), i
        if i < 8:  # exact arithmetic
            assert np.array_equal(vals[0, :want], ov[:want])
    assert vals[0, 0] < 0.0  # the negative dominant eigenvalue comes first


def test_eig_refuses_oversized(cuda):
    with pytest.raises(ValueError):
        eig_topk([np.broadcast_to(np.float64(0.0), (14081, 14081))], 3)


# ------------------------------------------------------------------------------------------------ metric embedding
EMBED_SIZES = [5, 32, 33, 164, 165, 300]


@pytest.mark.parametrize("dim", [3, 4])
def test_embed_euclidean(cuda, dim):
    rng = np.random.default_rng(50 + dim)
    pts = [D.euclidean_points(n, dim, rng) for n in EMBED_SIZES]
    dists = [D.dist(p) for p in pts]
    v0 = [rng.random((dim, len(p))) for p in pts]
    coords, ok = embed_abi(dists, dim, v0)
    wrapped, wok = metric_embed(dists, dim, v0=v0)
    hashed, hok = embed_abi(dists, dim)
    compared = 0
    for i, d in enumerate(dists):
        assert ok[i] and wok[i] and hok[i]
        assert np.array_equal(wrapped[i], coords[i])
        for c in (coords[i], hashed[i]):
            assert np.abs(D.dist(c) - d).max() <= D.EIG_RTOL * d.max()
            mds, _ = D.classical_mds(d, dim)
            assert np.abs(np.abs(c) - np.abs(mds)).max() <= D.EIG_RTOL * np.abs(mds).max()
        if _safe(oracle.power_eigen_trace(oracle.metric_matrix(d), dim, v0[i])):
            compared += 1
            want = oracle.metric_embed(d, dim, v0[i])
            assert np.abs(coords[i] - want).max() <= 1e-9 * np.abs(want).max()
    assert compared >= len(dists) - 1


def _failures(rng):
    return [D.dist(rng.normal(size=(1, 3))), D.dist(rng.normal(size=(2, 3))), D.ring_distances(40)]


@pytest.mark.parametrize("dim", [3, 4])
def test_embed_failures_leave_coords_unwritten(cuda, dim):
    rng = np.random.default_rng(60 + dim)
    dists = _failures(rng)
    v0 = [rng.random((dim, len(d))) for d in dists]
    coords, ok = embed_abi(dists, dim, v0)
    assert not ok.any()
    for d, v in zip(dists, v0):
        assert oracle.metric_embed(d, dim, v) is None


def test_embed_batch_larger_than_grid(cuda):
    rng = np.random.default_rng(70)
    grid = _grid()
    dists = []
    for m in range(2 * grid + 11):
        r = rng.random()
        if r < 0.3:
            dists.append(_failures(rng)[int(rng.integers(0, 3))])
        else:
            n = 170 if m % 101 == 3 else int(rng.integers(5, 40))
            dists.append(D.dist(D.euclidean_points(n, 3, rng)))
    v0 = [rng.random((3, len(d))) for d in dists]
    coords, ok = embed_abi(dists, 3, v0)
    checked = 0
    for i, d in enumerate(dists):
        if _safe(oracle.power_eigen_trace(oracle.metric_matrix(d), 3, v0[i])):
            checked += 1
            want = oracle.metric_embed(d, 3, v0[i])
            assert ok[i] == (want is not None), i
            if ok[i]:
                assert np.abs(coords[i] - want).max() <= 1e-9 * np.abs(want).max()
    assert checked >= 0.95 * len(dists)
    assert ok[:grid].any() and not ok[:grid].all() and ok[grid:].any() and not ok[grid:].all()


def test_embed_refuses_oversized_head(cuda):
    # (3 + dim) n + dim doubles stay in shared memory: n = 4022 is the largest at dim 4
    d = D.dist(D.euclidean_points(4023, 4, np.random.default_rng(80)))
    with pytest.raises(ValueError):
        metric_embed([d], 4)
    coords, ok = embed_abi([d, D.dist(D.euclidean_points(20, 4, np.random.default_rng(81)))], 4)
    assert ok.tolist() == [0, 1]
    coords, ok = embed_abi([d[:-1, :-1]], 4)
    assert ok.tolist() == [1] and np.abs(D.dist(coords[0]) - d[:-1, :-1]).max() <= D.EIG_RTOL * d.max()
