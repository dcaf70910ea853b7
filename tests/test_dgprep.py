"""Distance-geometry preparation restated in numpy, and the fixtures of the GPU tier (tests/test_dgprep_gpu.py) with the
answers the fp64 oracle gives for them. CPU only.

smooth_np is RDKit's triangleSmoothBounds one pivot at a time with all pairs of a pivot at once. Within pivot k every pair
update reads only pairs that contain k, which pivot k never writes, so the vectorised pivot equals the sequential loop bit
for bit. It also defines the state of a failing matrix the way the GPU kernel leaves it: the pivot in which lb > ub first
appears is completed for every pair, later pivots are not run (the sequential oracle stops in the middle of that pivot).
"""

import numpy as np
import pytest
from scipy.spatial.distance import cdist

import oracle

# The power method stops when two successive estimates (the largest-|z| element of A v) differ by less than 1e-3. That
# bounds a step, not the error: with a ratio r <= 0.5 between consecutive |lambda| the geometric tail of the remaining
# steps is <= 1e-3 r / (1 - r), but an estimate can also stall for one step in the first few iterations and stop there.
# The eigh comparisons therefore use spectra with every requested |lambda| >= 20, ratios <= 0.5 and the rest of the
# spectrum at most half the last one asked for. Over 2400 seeded spectra of that family the oracle's eigenvalues stayed
# within 2.9 % of |lambda| (eigh) and its eigenvectors within 1 - |cos| < 3.6e-3; the bounds allow about twice that.
EIG_RTOL = 5e-2
VEC_TOL = 1e-2


# ------------------------------------------------------------------------------------------------ triangle smoothing
def smooth_np(b, tol=0.0, pivots=None):
    """Smooth a copy of the RDKit-layout bounds matrix b. Returns (matrix, ok, first failing pivot or -1)."""
    b = np.array(b, dtype=np.float64, copy=True)
    n = b.shape[0]
    idx = np.arange(n)
    upper = idx[:, None] < idx[None, :]
    for k in range(n if pivots is None else pivots):
        m = upper & (idx != k)[:, None] & (idx != k)[None, :]  # the pairs (i < j) that pivot k updates
        uk = np.where(idx < k, b[:, k], b[k, :])  # upper bound of the pair (x, k): b[min][max]
        lk = np.where(idx < k, b[k, :], b[:, k])  # lower bound: b[max][min]
        # entry [i][j] of each array below is the value for the pair i < j
        sum_u, d1, d2 = uk[:, None] + uk[None, :], lk[:, None] - uk[None, :], lk[None, :] - uk[:, None]
        u, l = b, b.T
        u = np.where(u > sum_u, sum_u, u)
        l = np.where(l < d1, d1, np.where(l < d2, d2, l))  # RDKit's else-if: d2 is not looked at once l < d1
        gap = l - u
        with np.errstate(divide="ignore", invalid="ignore"):
            rescue = (gap > 0.0) & (gap / l < tol) if tol > 0.0 else np.zeros_like(m)
        u = np.where(rescue, l, u)
        b = np.where(m, u, b)
        b = np.where(m.T, l.T, b)
        if (m & (gap > 0.0) & ~rescue).any():
            return b, False, k
    return b, True, -1


def floyd_warshall_upper(b):
    """All-pairs shortest paths over the upper bounds, same pivot order; returns the full symmetric matrix."""
    n = b.shape[0]
    d = np.triu(b, 1)
    d = d + d.T
    for k in range(n):
        d = np.minimum(d, d[:, k:k + 1] + d[k:k + 1, :])
    return d


def bounds_from_points(rng, n, slack=(0.05, 1.5), spread=4.0):
    """Consistent bounds: true distances widened by a random slack on each side."""
    x = rng.normal(0.0, spread, (n, 3))
    d = np.linalg.norm(x[:, None] - x[None], axis=2)
    up = d + rng.uniform(*slack, (n, n))
    lo = np.maximum(d - rng.uniform(*slack, (n, n)), 0.0)
    return np.triu(up, 1) + np.tril(lo.T, -1)


def chain_bounds(rng, n, tight=0.2, loose=1e3, bad_pair=None):
    """A chain whose neighbours are tightly bounded and all other pairs have loose upper bounds, so that every pivot
    lowers some upper bound. bad_pair (i, j) gets a lower bound above the chain's longest route, so smoothing fails."""
    step = rng.uniform(1.0, 1.5, n - 1)
    pos = np.concatenate([[0.0], np.cumsum(step)])
    b = np.zeros((n, n))
    iu, ju = np.triu_indices(n, 1)
    b[iu, ju] = loose + rng.uniform(0.0, 1.0, iu.size)
    b[ju, iu] = rng.uniform(0.0, 1.0, iu.size)
    r = np.arange(n - 1)
    b[r, r + 1] = step + tight
    b[r + 1, r] = step - tight
    if bad_pair is not None:
        i, j = bad_pair
        b[j, i] = pos[j] - pos[i] + (j - i) * tight + 5.0
    return b


def oracle_failed_state(b, tol):
    """Where the sequential oracle stops in a failing matrix: the pairs of the failing pivot up to and including the
    first failing one (row-major) are updated, the later ones not."""
    after, ok, k = smooth_np(b, tol)
    before, _, _ = smooth_np(b, tol, pivots=k)
    n = b.shape[0]
    iu, ju = np.triu_indices(n, 1)
    processed = (iu != k) & (ju != k)
    bad = processed & (after[ju, iu] - after[iu, ju] > 0.0)
    last = np.flatnonzero(bad)[0]
    take = processed & (np.arange(iu.size) <= last)
    want = before.copy()
    want[iu[take], ju[take]] = after[iu[take], ju[take]]
    want[ju[take], iu[take]] = after[ju[take], iu[take]]
    return want


def tri(u01, u02, u12, l01, l02, l12):
    return np.array([[0.0, u01, u02], [l01, 0.0, u12], [l02, l12, 0.0]])


ULP = np.nextafter
# Hand-built dyadic matrices (exact arithmetic) on each side of each comparison: (name, bounds, tol, want, ok, pivot).
# In a 3-atom matrix pivot 0 updates the pair (1, 2) from (0, 1) and (0, 2): sumU = U01 + U02, d1 = L01 - U02,
# d2 = L02 - U01.
_T_COLLINEAR = tri(1.0, 1.5, 2.5, 1.0, 1.5, 2.5)  # points at 0, -1, 1.5: every gap exactly 0
HAND_CASES = [
    # u == sumU at pivot 0 (kept), then every gap is exactly 0: consistent
    ("gap0", tri(1.0, 1.5, 2.5, 0.5, 1.0, 2.5), 0.0, _T_COLLINEAR, True, -1),
    # u one ulp above sumU: lowered to sumU, same result
    ("u_above_sum", tri(1.0, 1.5, ULP(2.5, 9.0), 0.5, 1.0, 2.5), 0.0, _T_COLLINEAR, True, -1),
    # l one ulp above the lowest consistent value: gap > 0 fails at tol 0 ...
    ("gap_ulp", tri(1.0, 1.5, 3.0, 0.5, 1.0, ULP(2.5, 9.0)), 0.0,
     tri(1.0, 1.5, 2.5, 0.5, 1.0, ULP(2.5, 9.0)), False, 0),
    # ... and is rescued (u = l) at tol 0.05; the later pivots then see a triangle one ulp off and rescue that too
    ("gap_ulp_tol", tri(1.0, 1.5, 3.0, 0.5, 1.0, ULP(2.5, 9.0)), 0.05, None, True, -1),
    # l < d1 < d2: RDKit's else-if keeps d1 = -3.5 and never looks at d2 = 2.5
    ("elseif_quirk", tri(1.0, 4.0, 5.0, 0.5, 3.5, -8.0), 0.0, tri(1.0, 4.0, 5.0, 0.5, 3.5, -3.5), True, -1),
    # l == d1 < d2: not below d1, so the else-if raises it to d2
    ("l_eq_d1", tri(1.0, 4.0, 5.0, 0.5, 3.5, -3.5), 0.0, tri(1.0, 4.0, 5.0, 0.5, 3.5, 2.5), True, -1),
    # l one ulp below d1: set to d1
    ("l_below_d1", tri(1.0, 4.0, 5.0, 0.5, 3.5, ULP(-3.5, -9.0)), 0.0, tri(1.0, 4.0, 5.0, 0.5, 3.5, -3.5), True, -1),
    # gap / l exactly tol (0.5 / 4 = 0.125): not below tol, fails at pivot 0 with u lowered to sumU = 3.5
    ("gap_eq_tol", tri(1.5, 2.0, 8.0, 1.0, 1.0, 4.0), 0.125, tri(1.5, 2.0, 3.5, 1.0, 1.0, 4.0), False, 0),
    # tol one ulp larger: rescued at pivot 0 (U12 = 4); pivot 1 then lifts L02 to 4 - 1.5 = 2.5 > U02 = 2, gap 0.2: fails
    ("gap_tol_ulp", tri(1.5, 2.0, 8.0, 1.0, 1.0, 4.0), ULP(0.125, 1.0), tri(1.5, 2.0, 4.0, 1.0, 2.5, 4.0), False, 1),
    # tol 0.25 rescues both, and pivot 2 lifts L01 to 4 - 2.5 = 1.5: collinear, consistent
    ("tol_rescues_all", tri(1.5, 2.0, 8.0, 1.0, 1.0, 4.0), 0.25, tri(1.5, 2.5, 4.0, 1.5, 2.5, 4.0), True, -1),
    # 4 atoms: pivot 0 fails at its first pair (1, 2) and still lowers (1, 3) and (2, 3) to U0i + U0j = 2
    ("fail_mid_pivot", np.array([[0.0, 1.0, 1.0, 1.0], [0.5, 0.0, 4.0, 9.0], [0.5, 3.0, 0.0, 9.0], [0.5, 0.5, 0.5, 0.0]]),
     0.0, np.array([[0.0, 1.0, 1.0, 1.0], [0.5, 0.0, 2.0, 2.0], [0.5, 3.0, 0.0, 2.0], [0.5, 0.5, 0.5, 0.0]]), False, 0),
    # n = 0, 1, 2: no pivot has a pair to update, so even lb > ub in a 2-atom matrix is reported consistent
    ("n0", np.zeros((0, 0)), 0.0, np.zeros((0, 0)), True, -1),
    ("n1", np.zeros((1, 1)), 0.0, np.zeros((1, 1)), True, -1),
    ("n2_inverted", np.array([[0.0, 1.0], [2.0, 0.0]]), 0.0, np.array([[0.0, 1.0], [2.0, 0.0]]), True, -1),
]


@pytest.mark.parametrize("case", HAND_CASES, ids=[c[0] for c in HAND_CASES])
def test_smoothing_hand_cases(case):
    name, b, tol, want, ok, pivot = case
    got, gok, gk = smooth_np(b, tol)
    assert (gok, gk) == (ok, pivot)
    if want is not None:
        assert np.array_equal(got, want)
    else:  # every pair rescued to a zero gap
        assert np.array_equal(np.triu(got, 1), np.tril(got, -1).T)
    ob, ook = oracle.triangle_smooth(b, tol)
    assert ook == ok
    if ok:
        assert np.array_equal(ob, got)
    elif b.shape[0] > 3:
        assert np.array_equal(ob, oracle_failed_state(b, tol))
        assert not np.array_equal(ob, got)  # the oracle stopped in the middle of the pivot
    else:  # one pair per pivot: the oracle stops where the pivot ends
        assert np.array_equal(ob, got)


def random_bounds(seed):
    """Random bounds of 3-20 atoms: consistent ones, and ones with a lower bound pushed up so that some fail."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(3, 21))
    b = bounds_from_points(rng, n)
    if rng.random() < 0.5:
        i, j = sorted(rng.choice(n, 2, replace=False))
        b[j, i] = b[i, j] * rng.uniform(0.9, 1.6)
    return b


@pytest.mark.parametrize("tol", [0.0, 0.05])
def test_smoothing_restatement_equals_oracle(tol):
    fails = 0
    for seed in range(200):
        b = random_bounds(seed)
        got, ok, k = smooth_np(b, tol)
        want, okc = oracle.triangle_smooth(b, tol)
        assert ok == okc, seed
        if ok:
            assert np.array_equal(got, want), seed
            if tol == 0.0:  # upper bounds are the shortest paths over upper bounds
                fw = floyd_warshall_upper(b)
                assert np.array_equal(np.triu(got, 1), np.triu(fw, 1)), seed
        else:
            fails += 1
            assert np.array_equal(want, oracle_failed_state(b, tol)), seed
    assert 30 <= fails <= 170  # both kinds are exercised


def test_smoothing_chain_changes_every_pivot():
    rng = np.random.default_rng(3)
    b = chain_bounds(rng, 40)
    changed = 0
    prev = b
    for k in range(1, 41):
        cur, ok, _ = smooth_np(b, 0.0, pivots=k)
        changed += not np.array_equal(cur, prev)
        prev = cur
    assert ok and changed >= 38  # every pivot but the first and the last lowers some upper bound
    want, okc = oracle.triangle_smooth(b)
    assert okc and np.array_equal(prev, want)
    got, ok, k = smooth_np(chain_bounds(np.random.default_rng(3), 40, bad_pair=(2, 30)))
    assert not ok and k > 0


# ------------------------------------------------------------------------------------------------ power eigensolver
def tie_matrix(n, lo, hi, sign_lo, rng=None):
    """diag with +-3 at two indices (opposite signs), smaller entries elsewhere: the largest |z| is an exact tie."""
    d = np.zeros(n) if rng is None else rng.uniform(-1.0, 1.0, n)
    d[lo], d[hi] = 3.0 * sign_lo, -3.0 * sign_lo
    return np.diag(d)


# (lo, hi): one thread (i, i + 256), lanes of one warp, two warps, a tie between the second stride and the first.
TIE_PAIRS = [(5, 37), (37, 300), (5, 261), (3, 9), (40, 290)]


def deflatable(n, rank, rng):
    """Diagonal of the given rank with entries of distinct magnitude; start vectors = unit vectors on those entries,
    then on a zero entry. Every step is exact: the solver returns exactly `rank` pairs when asked for more."""
    at = rng.choice(n, min(n, rank + 1), replace=False)
    d = np.zeros(n)
    d[at[:rank]] = rng.choice([-1.0, 1.0], rank) * 2.0 ** np.arange(rank, 0, -1)
    v0 = np.zeros((rank + 1, n))
    v0[np.arange(len(at)), at] = 1.0
    return np.diag(d), v0


def rotated(spec, rng):
    n = len(spec)
    q = np.linalg.qr(rng.normal(size=(n, n)))[0]
    a = (q * spec) @ q.T
    return 0.5 * (a + a.T)


def separated_spectrum(n, k, rng, negative_first=False):
    """k eigenvalues with |lambda| >= 20 and ratio <= 0.5 between consecutive ones, the rest at most half the k-th."""
    r = rng.uniform(0.15, 0.5, max(k - 1, 0))
    lam = rng.uniform(20.0, 80.0) / np.concatenate([np.cumprod(r[::-1])[::-1], [1.0]])
    lam *= rng.choice([-1.0, 1.0], k)
    if negative_first:
        lam[0] = -abs(lam[0])
    rest = rng.uniform(-0.5, 0.5, n - k) * abs(lam[-1])
    return np.concatenate([lam, rest])


def pm_pair(n, rng):
    """Eigenvalues 3 and -3 (then smaller ones) in a rotated basis: the estimate alternates and never settles."""
    spec = np.concatenate([[3.0, -3.0], rng.uniform(-1.0, 1.0, n - 2)])
    return rotated(spec, rng)


def eigh_by_magnitude(a):
    w, u = np.linalg.eigh(a)
    o = np.argsort(-np.abs(w), kind="stable")
    return w[o], u[:, o].T


def assert_close_to_eigh(a, vals, vecs, k):
    w, u = eigh_by_magnitude(a)
    assert np.all(np.abs(vals[:k] - w[:k]) <= EIG_RTOL * np.abs(w[:k]))
    assert np.all(1.0 - np.abs(np.sum(vecs[:k] * u[:k], axis=1)) <= VEC_TOL)


@pytest.mark.parametrize("lo,hi", TIE_PAIRS)
def test_power_tie_first_index_wins(lo, hi):
    for sign in (-1.0, 1.0):
        for rng in (None, np.random.default_rng(lo)):
            a = tie_matrix(320, lo, hi, sign, rng)
            vals, vecs, k = oracle.power_eigen(a, 1, np.ones((1, 320)))
            assert k == 1 and vals[0] == 3.0 * sign  # the sign of the entry at the lower index
            assert abs(vecs[0, lo]) == abs(vecs[0, hi])
            assert rng is not None or abs(vecs[0, lo]) == 1.0 / np.sqrt(2.0)


@pytest.mark.parametrize("rank", range(8))
def test_power_deflatable_returns_its_rank(rank):
    a, v0 = deflatable(50, rank, np.random.default_rng(rank))
    vals, vecs, k = oracle.power_eigen(a, rank + 1, v0)
    assert k == rank
    assert np.array_equal(np.sort(vals[:rank]), np.sort(np.diag(a)[np.diag(a) != 0.0]))


def test_power_pm_pair_never_converges():
    for n in (40, 300):
        rng = np.random.default_rng(n)
        vals, vecs, k, iters, conv, zero = oracle.power_eigen_trace(pm_pair(n, rng), 3, rng.random((3, n)))
        assert k == 0 and iters[0] == 1000 and conv[0] > 1e-6


def test_power_negative_dominant():
    rng = np.random.default_rng(11)
    a = rotated(separated_spectrum(60, 4, rng, negative_first=True), rng)
    vals, vecs, k = oracle.power_eigen(a, 4, rng.random((4, 60)))
    assert k == 4 and vals[0] < 0.0
    assert_close_to_eigh(a, vals, vecs, 4)


@pytest.mark.parametrize("k", range(1, 9))
def test_power_separated_spectra_match_eigh(k):
    for seed in range(25):
        rng = np.random.default_rng(100 * k + seed)
        n = int(rng.choice([k + 1, 17, 33, 90]))
        a = rotated(separated_spectrum(n, k, rng), rng)
        vals, vecs, got = oracle.power_eigen(a, k, rng.random((k, n)))
        assert got == k
        assert_close_to_eigh(a, vals, vecs, k)


def test_power_trace_matches_plain_oracle():
    rng = np.random.default_rng(7)
    a = rotated(separated_spectrum(30, 5, rng), rng)
    v0 = rng.random((5, 30))
    vals, vecs, k = oracle.power_eigen(a, 5, v0)
    tv, tvec, tk, iters, conv, zero = oracle.power_eigen_trace(a, 5, v0)
    assert k == tk == 5 and np.array_equal(vals, tv) and np.array_equal(vecs, tvec)
    assert np.all(iters >= 2) and np.all(conv > 0.0) and np.all(zero > 0.1)


# ------------------------------------------------------------------------------------------------ metric embedding
def euclidean_points(n, dim, rng):
    """n centred points whose metric matrix has eigenvalues n * (16, 6, 2, 0.6)[:dim]: consecutive ratios <= 0.5."""
    g = rng.normal(size=(n, dim))
    g -= g.mean(0)
    q = np.linalg.qr(g)[0]
    return q * np.sqrt(n * np.array([16.0, 6.0, 2.0, 0.6])[:dim])


def dist(x):
    return cdist(x, x)


def classical_mds(d, dim):
    w, u = eigh_by_magnitude(oracle.metric_matrix(d))
    return u[:dim].T * np.sqrt(w[:dim]), w


def ring_distances(n):
    """Shortest-path distances around a ring of n atoms: not Euclidean. Its metric matrix has eigenvalues
    (a, a, -b, -b, c, c, ...) with b about a / 4, so a negative one is among the top 3 and the top 4 by |lambda|."""
    i = np.arange(n)
    g = np.abs(i[:, None] - i[None])
    return np.minimum(g, n - g).astype(np.float64)


def test_metric_matrix_is_classical_mds():
    rng = np.random.default_rng(4)
    x = euclidean_points(30, 4, rng)
    t = oracle.metric_matrix(dist(x))
    assert np.abs(t - x @ x.T).max() <= 1e-9 * np.abs(t).max()


@pytest.mark.parametrize("dim", [3, 4])
def test_metric_embed_oracle_matches_mds(dim):
    for n in (5, 32, 33, 90):
        rng = np.random.default_rng(n + dim)
        x = euclidean_points(n, dim, rng)
        d = dist(x)
        got = oracle.metric_embed(d, dim, rng.random((dim, n)))
        want, w = classical_mds(d, dim)
        assert got is not None
        assert np.abs(dist(got) - d).max() <= EIG_RTOL * d.max()
        assert np.abs(np.abs(got) - np.abs(want)).max() <= EIG_RTOL * np.abs(want).max()


def test_metric_embed_failures():
    rng = np.random.default_rng(5)
    for dim in (3, 4):
        for n in (1, 2):
            assert oracle.metric_embed(dist(rng.normal(size=(n, 3))), dim, rng.random((dim, n))) is None
    d = ring_distances(40)
    w, _ = eigh_by_magnitude(oracle.metric_matrix(d))
    assert w[0] > 0.0 and w[1] > 0.0 and w[2] < 0.0 and w[3] < 0.0
    for dim in (3, 4):
        vals, _, k, _, conv, _ = oracle.power_eigen_trace(oracle.metric_matrix(d), dim, rng.random((dim, 40)))
        assert k == dim and vals[2] < 0.0 and conv.min() > 1e-6  # converged, and the third eigenvalue is negative
        assert oracle.metric_embed(d, dim, rng.random((dim, 40))) is None
